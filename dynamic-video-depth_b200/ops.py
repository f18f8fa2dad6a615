"""Python face of the C ABI: argument checks, output allocation, autograd wiring.

PyTorch is plumbing here (device memory, streams, autograd graph); all arithmetic of the hot path
happens inside libdvd_b200.so. Argument / shape / dtype / contiguity violations raise ValueError
before any launch; a non-zero return from the library raises RuntimeError (SURVEY.md §8(b)).
"""
import contextlib
import ctypes
import os

import torch

from . import _lib
from ._lib import LossCfg, MlpCfg


# number of dvd_b200 kernel launches issued through this module (bench.py reports it as gpu_launches)
LAUNCHES = {'n': 0}


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


# ---- ordered reductions -------------------------------------------------------------------------------------------------------
# Under torch.use_deterministic_algorithms(True) every backward launch that would add partial sums with fp32 atomics calls its
# *_ordered entry point instead (DESIGN.md 2.11): same split, partials through a workspace, added in a fixed order. A training
# step reads torch's switch once and runs inside `ordered_reductions(flag)`; a launch outside a step reads the switch itself.
_ORDERED = [None]


@contextlib.contextmanager
def ordered_reductions(flag):
    prev = _ORDERED[0]
    _ORDERED[0] = bool(flag)
    try:
        yield
    finally:
        _ORDERED[0] = prev


def ordered():
    """Whether the backward launches issued now take their ordered (run-to-run reproducible) variants."""
    return torch.are_deterministic_algorithms_enabled() if _ORDERED[0] is None else _ORDERED[0]


_ORD_WS = {}     # (device index, site) -> workspace of dvd_ordered_workspace_bytes(site) bytes


def ordered_workspace(device, site):
    """The workspace of one ordered-reduction site on this device (sites are separate so that launches on different streams
    never share one). Allocated once, outside graph capture: the eager steps before a capture allocate it."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    ws = _ORD_WS.get((idx, site))
    if ws is None:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError('ordered-reduction workspace %d is allocated by an eager launch before a graph capture' % site)
        n = _lib.load().dvd_ordered_workspace_bytes(site)
        ws = _ORD_WS[(idx, site)] = torch.empty((n + 15) // 16 * 4, dtype=torch.float32, device=torch.device('cuda', idx))
    return ws


def _ws(t):
    """(pointer, bytes) of a workspace tensor"""
    return _ptr(t), t.numel() * t.element_size()


def _chk(t, name, shape=None):
    if not isinstance(t, torch.Tensor):
        raise ValueError('%s must be a torch.Tensor' % name)
    if not t.is_cuda:
        raise ValueError('%s must live on a CUDA device (dvd_b200 has no CPU path)' % name)
    if t.dtype != torch.float32:
        raise ValueError('%s must be float32, got %s' % (name, t.dtype))
    if not t.is_contiguous():
        raise ValueError('%s must be contiguous' % name)
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError('%s has shape %s, expected %s' % (name, tuple(t.shape), tuple(shape)))
    return t


def make_loss_cfg(midas=True, warm=False, use_disp=True, use_disp_ratio=False, flow_mul=1.0, disp_mul=1.0):
    """Flags → struct dvd_loss_cfg (models/scene_flow_motion_field.py:140-150,285-319)."""
    mode = 0 if use_disp else (1 if use_disp_ratio else 2)
    return LossCfg(int(bool(midas)), int(bool(warm)), mode, int(bool(use_disp)), float(flow_mul), float(disp_mul))


def pack_poses(K, K_inv, R_1_T, R_2_T, t_1, t_2):
    """Reference-format pose tensors → [B,48] pose blocks of the C ABI.

    The reference stores transposes for row-vector algebra: K = K^T, K_inv = (K^-1)^T,
    R_i_T = R_c2w_i (scripts/preprocess/davis/generate_sequence_midas.py:61-76). Accepts the
    [B,1,1,3,3] / [B,1,1,1,3] shapes of the batch dict (or anything reshapeable to [B,3,3] / [B,3])."""
    B = K.reshape(-1, 3, 3).shape[0]
    Kc = K.reshape(B, 3, 3).transpose(1, 2)
    Ki = K_inv.reshape(B, 3, 3).transpose(1, 2)
    out = torch.zeros(B, 48, dtype=torch.float32, device=K.device)
    out[:, 0:9] = Ki.reshape(B, 9)
    out[:, 9:18] = Kc.reshape(B, 9)
    out[:, 18:27] = R_1_T.reshape(B, 9)
    out[:, 27:36] = R_2_T.reshape(B, 9)
    out[:, 36:39] = t_1.reshape(B, 3)
    out[:, 39:42] = t_2.reshape(B, 3)
    return out


def pack_poses_from_batch(batch):
    return pack_poses(batch['K'], batch['K_inv'], batch['R_1_T'], batch['R_2_T'], batch['t_1'], batch['t_2'])


# ------------------------------------------------------------------------------------------------
# raw calls (no autograd)

def unproject_fwd(depth, poses, which=1):
    B, C, H, W = depth.shape
    _chk(depth, 'depth', (B, 1, H, W)), _chk(poses, 'poses', (B, 48))
    P = torch.empty(B, 3, H, W, dtype=torch.float32, device=depth.device)
    lib = _lib.load()
    LAUNCHES['n'] += 1
    _lib.check(lib.dvd_unproject_fwd(_ptr(depth), _ptr(poses), _ptr(P), B, H, W, int(which), _stream()),
               'dvd_unproject_fwd')
    return P


def unproject_bwd(gP, poses, which=1):
    B, C, H, W = gP.shape
    _chk(gP, 'gP', (B, 3, H, W)), _chk(poses, 'poses', (B, 48))
    gd = torch.empty(B, 1, H, W, dtype=torch.float32, device=gP.device)
    lib = _lib.load()
    LAUNCHES['n'] += 1
    _lib.check(lib.dvd_unproject_bwd(_ptr(gP), _ptr(poses), _ptr(gd), B, H, W, int(which), _stream()),
               'dvd_unproject_bwd')
    return gd


def _chk_reproject(depth_1, depth_2, flow, mask, sf, poses):
    if depth_1.dim() != 4:
        raise ValueError('depth_1 must be [B,1,H,W]')
    B, _, H, W = depth_1.shape
    _chk(depth_1, 'depth_1', (B, 1, H, W)), _chk(depth_2, 'depth_2', (B, 1, H, W))
    _chk(flow, 'flow_1_2', (B, H, W, 2)), _chk(poses, 'poses', (B, 48))
    if mask is not None:
        _chk(mask, 'mask_2')
        if mask.numel() != B * H * W:
            raise ValueError('mask_2 must have B*H*W elements')
    if sf is not None:
        _chk(sf, 'sf', (B, 3, H, W))
    return B, H, W


def reproject_loss_fwd(depth_1, depth_2, flow, mask, sf, poses, cfg):
    """→ scalars [8] (see enum in include/dvd_b200.h): flow, disp, sf, loss, mask-sum, cf, cd, 0."""
    B, H, W = _chk_reproject(depth_1, depth_2, flow, mask, sf, poses)
    lib = _lib.load()
    n = lib.dvd_reproject_partials_size(B, H, W)
    partials = torch.empty(n, dtype=torch.float32, device=depth_1.device)
    scalars = torch.empty(8, dtype=torch.float32, device=depth_1.device)
    LAUNCHES['n'] += 2
    _lib.check(lib.dvd_reproject_loss_fwd(_ptr(depth_1), _ptr(depth_2), _ptr(flow), _ptr(mask), _ptr(sf), _ptr(poses),
                                          ctypes.byref(cfg), _ptr(partials), _ptr(scalars), B, H, W, _stream()),
               'dvd_reproject_loss_fwd')
    return scalars


def reproject_loss_bwd(depth_1, depth_2, flow, mask, sf, poses, cfg, scalars, gscale=1.0, gscale_dev=None,
                       need_depth_grad=True):
    B, H, W = _chk_reproject(depth_1, depth_2, flow, mask, sf, poses)
    _chk(scalars, 'scalars', (8,))
    g_sf = torch.empty_like(sf)
    g_d2 = torch.empty_like(depth_2) if need_depth_grad else None
    lib = _lib.load()
    if g_d2 is not None and ordered():
        # the sort buffers of the ordered scatter are per call, like the step's other intermediates
        ws = torch.empty(lib.dvd_reproject_ordered_bytes(B, H, W), dtype=torch.uint8, device=depth_1.device)
        LAUNCHES['n'] += 3
        _lib.check(lib.dvd_reproject_loss_bwd_ordered(_ptr(depth_1), _ptr(depth_2), _ptr(flow), _ptr(mask), _ptr(sf), _ptr(poses),
                                                      ctypes.byref(cfg), _ptr(scalars), float(gscale), _ptr(gscale_dev),
                                                      _ptr(g_sf), _ptr(g_d2), B, H, W, *_ws(ws), _stream()),
                   'dvd_reproject_loss_bwd_ordered')
        return g_sf, g_d2
    LAUNCHES['n'] += 1
    _lib.check(lib.dvd_reproject_loss_bwd(_ptr(depth_1), _ptr(depth_2), _ptr(flow), _ptr(mask), _ptr(sf), _ptr(poses),
                                          ctypes.byref(cfg), _ptr(scalars), float(gscale), _ptr(gscale_dev),
                                          _ptr(g_sf), _ptr(g_d2), B, H, W, _stream()),
               'dvd_reproject_loss_bwd')
    return g_sf, g_d2


_MAT_KEYS3 = ('global_p1', 'sf_by_depth', 'warped_global_p2', 'warped_p2_camera_2', 'p1_camera_2')
_MAT_KEYS2 = ('dflow_1_2', 'staticflow_1_2')
_MAT_KEYS1 = ('depth_image_1_2', 'depth_warp_1_2')


def reproject_materialize(depth_1, depth_2, flow, sf, poses, keys=None):
    """Per-pixel tensors of flow_by_depth / scene_flow_projection_slack, channel-planar."""
    B, H, W = _chk_reproject(depth_1, depth_2, flow, None, sf, poses)
    allk = _MAT_KEYS3 + _MAT_KEYS2 + _MAT_KEYS1
    keys = allk if keys is None else keys
    out = {}
    for k in allk:
        if k in keys:
            c = 3 if k in _MAT_KEYS3 else (2 if k in _MAT_KEYS2 else 1)
            out[k] = torch.empty(B, c, H, W, dtype=torch.float32, device=depth_1.device)
    lib = _lib.load()
    LAUNCHES['n'] += 1
    _lib.check(lib.dvd_reproject_materialize(_ptr(depth_1), _ptr(depth_2), _ptr(flow), _ptr(sf), _ptr(poses),
                                             *[_ptr(out.get(k)) for k in allk], B, H, W, _stream()),
               'dvd_reproject_materialize')
    return out


# ------------------------------------------------------------------------------------------------
# autograd wiring

class Unproject(torch.autograd.Function):
    """unproject_ptcld.forward (losses/scene_flow_projection.py:48-67) → [B,3,H,W]."""

    @staticmethod
    def forward(ctx, depth, poses, which):
        ctx.save_for_backward(poses)
        ctx.which = which
        return unproject_fwd(depth.contiguous(), poses, which)

    @staticmethod
    def backward(ctx, gP):
        (poses,) = ctx.saved_tensors
        return unproject_bwd(gP.contiguous(), poses, ctx.which), None, None


def unproject(depth, poses, which=1):
    return Unproject.apply(depth, poses, which)


class ReprojectLoss(torch.autograd.Function):
    """Fused W1+W2+L1. Returns (loss, scalars[8]); only `loss` is differentiable."""

    @staticmethod
    def forward(ctx, depth_1, depth_2, sf, flow, mask, poses, cfg, gscale):
        depth_1, depth_2, sf = depth_1.contiguous(), depth_2.contiguous(), sf.contiguous()
        scalars = reproject_loss_fwd(depth_1, depth_2, flow, mask, sf, poses, cfg)
        ctx.save_for_backward(depth_1, depth_2, sf, flow, mask, poses, scalars)
        ctx.cfg, ctx.gscale = cfg, gscale
        ctx.need_depth = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        loss = scalars[3] * gscale if gscale != 1.0 else scalars[3].clone()
        ctx.mark_non_differentiable(scalars)
        return loss, scalars

    @staticmethod
    def backward(ctx, g_loss, _g_scalars):
        depth_1, depth_2, sf, flow, mask, poses, scalars = ctx.saved_tensors
        g = g_loss.contiguous().to(torch.float32)
        g_sf, g_d2 = reproject_loss_bwd(depth_1, depth_2, flow, mask, sf, poses, ctx.cfg, scalars,
                                        gscale=ctx.gscale, gscale_dev=g, need_depth_grad=ctx.need_depth)
        g_d1 = None
        if ctx.needs_input_grad[0]:
            # global_p1 and sf enter the chain only as P1 + sf  =>  dL/dP1 == dL/dsf
            g_d1 = unproject_bwd(g_sf, poses, 1)
        return g_d1, (g_d2 if ctx.needs_input_grad[1] else None), g_sf, None, None, None, None, None


def reproject_loss(depth_1, depth_2, sf, flow, mask, poses, cfg, gscale=1.0):
    return ReprojectLoss.apply(depth_1, depth_2, sf, flow, mask, poses, cfg, float(gscale))


# ================================================================================================
# scene-flow MLP (wgmma kernels)

def mlp_n_in(n_freq_xyz, n_freq_t, time_dependent):
    """Input width of the scene-flow MLP's first layer (networks/sceneflow_field.py:22-24)."""
    return (1 + 2 * n_freq_t if time_dependent else 0) + 3 + 6 * n_freq_xyz


def check_mlp_counts(n_freq_xyz, n_freq_t, time_dependent):
    """Raise ValueError unless the kernels run this positional encoding: non-negative counts and at most
    DVD_MLP_MAX_NIN (256) input features (n_freq_t is ignored when the field is not time-dependent)."""
    if int(n_freq_xyz) != n_freq_xyz or int(n_freq_t) != n_freq_t or n_freq_xyz < 0 or (time_dependent and n_freq_t < 0):
        raise ValueError('n_freq_xyz / n_freq_t must be non-negative integers (got %r, %r)' % (n_freq_xyz, n_freq_t))
    nin = mlp_n_in(n_freq_xyz, n_freq_t, time_dependent)
    if nin > _lib.DVD_MLP_MAX_NIN:
        raise ValueError('scene-flow MLP input width (time_dependent ? 1 + 2 n_freq_t : 0) + 3 + 6 n_freq_xyz = %d for '
                         'n_freq_xyz=%d n_freq_t=%d time_dependent=%s exceeds the supported %d'
                         % (nin, n_freq_xyz, n_freq_t, bool(time_dependent), _lib.DVD_MLP_MAX_NIN))


def make_mlp_cfg(n_freq_xyz=16, n_freq_t=16, time_dependent=True, sf_mag_div=100.0):
    """struct dvd_mlp_cfg; frequencies = torch.linspace(1, N+1, N) in fp32 exactly as
    PeriodicEmbed builds them (networks/blocks.py:23-24). Any encoding with at most 256 input features
    (check_mlp_counts)."""
    check_mlp_counts(n_freq_xyz, n_freq_t, time_dependent)
    c = MlpCfg()
    c.n_freq_xyz, c.n_freq_t, c.time_dependent, c.sf_mag_div = int(n_freq_xyz), int(n_freq_t), int(bool(time_dependent)), float(sf_mag_div)
    n_t = int(n_freq_t) if time_dependent else 0
    fx = torch.linspace(1, n_freq_xyz + 1, steps=n_freq_xyz, dtype=torch.float32).tolist() if n_freq_xyz > 0 else []
    ft = torch.linspace(1, n_t + 1, steps=n_t, dtype=torch.float32).tolist() if n_t > 0 else []
    for i, f in enumerate(fx):
        c.freq_xyz[i] = f
    for i, f in enumerate(ft):
        c.freq_t[i] = f
    return c


def _ptr_array(tensors):
    arr = (ctypes.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr() if t is not None else None
    return arr


class PackedMlp:
    """Device-side bf16 (hi,lo) wgmma images of the six weight matrices + the fp32 bias vector.
    Re-pack after every optimiser step (`refresh`)."""

    def __init__(self, cfg, device):
        lib = _lib.load()
        self.cfg = cfg
        n = lib.dvd_mlp_packed_weights_bytes(ctypes.byref(cfg))
        self.fwd = torch.empty(n, dtype=torch.uint8, device=device)
        self.bwd = torch.empty(n, dtype=torch.uint8, device=device)
        self.bias = torch.zeros(5 * 256 + 16, dtype=torch.float32, device=device)

    def refresh(self, weights, biases):
        """weights[l]: [out,in(,1,1)] fp32 contiguous cuda tensors, biases[l]: [out]."""
        if len(weights) != 6 or len(biases) != 6:
            raise ValueError('the scene-flow MLP has 6 layers')
        ws = [_chk(w.detach(), 'weight[%d]' % i) for i, w in enumerate(weights)]
        lib = _lib.load()
        LAUNCHES['n'] += 1
        _lib.check(lib.dvd_mlp_pack_weights(ctypes.byref(self.cfg), _ptr_array(ws), _ptr(self.fwd), _ptr(self.bwd),
                                            _stream()), 'dvd_mlp_pack_weights')
        with torch.no_grad():
            for l in range(5):
                self.bias[l * 256:(l + 1) * 256].copy_(biases[l].detach())
            self.bias[1280:1283].copy_(biases[5].detach())
        return self


def mlp_chain_fwd(packed, p0, t0, dt, n_eval, n_acc, save=False, want_steps=True):
    """Raw forward. Returns dict(acc, s_steps, p_steps, save) (tensors or None)."""
    cfg = packed.cfg
    B, C, H, W = p0.shape
    _chk(p0, 'p0', (B, 3, H, W))
    if cfg.time_dependent:
        _chk(t0, 't0', (B, 1, H, W))
    npx, hw = B * H * W, H * W
    dev = p0.device
    lib = _lib.load()
    acc = torch.empty_like(p0)
    s_steps = torch.empty(n_eval, B, 3, H, W, dtype=torch.float32, device=dev) if (want_steps or save) else None
    p_steps = sv = None
    if save:
        p_steps = torch.empty(n_eval, B, 3, H, W, dtype=torch.float32, device=dev)
        per = lib.dvd_mlp_save_bytes_per_eval(ctypes.byref(cfg), npx)
        sv = torch.empty(n_eval * per, dtype=torch.uint8, device=dev)
    LAUNCHES['n'] += 1
    _lib.check(lib.dvd_mlp_chain_fwd(ctypes.byref(cfg), _ptr(packed.fwd), _ptr(packed.bias), _ptr(p0),
                                     _ptr(t0) if cfg.time_dependent else ctypes.c_void_p(0), float(dt), int(n_eval),
                                     int(n_acc), _ptr(acc), _ptr(s_steps), _ptr(p_steps), _ptr(sv), npx, hw, _stream()),
               'dvd_mlp_chain_fwd')
    return {'acc': acc, 's_steps': s_steps, 'p_steps': p_steps, 'save': sv}


_SIDE_STREAMS = {}


def _side_stream(dev):
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    st = _SIDE_STREAMS.get(idx)
    if st is None:
        st = _SIDE_STREAMS[idx] = torch.cuda.Stream(device=idx)
    return st


def mlp_chain_bwd(packed, fwd, t0, dt, n_acc, g_acc, g_steps, grad_w, grad_b):
    """Raw backward over all evals: dgrad chain + wgrad per eval (descending).
    g_acc [B,3,H,W] or None; g_steps: list (len n_eval) of [B,3,H,W] or None entries.
    grad_w / grad_b: lists of 6 fp32 tensors ACCUMULATED into. Returns dL/dp0."""
    cfg = packed.cfg
    p_steps, sv = fwd['p_steps'], fwd['save']
    n_eval, B, _, H, W = p_steps.shape
    npx, hw = B * H * W, H * W
    dev = p_steps.device
    lib = _lib.load()
    per = lib.dvd_mlp_save_bytes_per_eval(ctypes.byref(cfg), npx)
    # Two streams: the weight gradient of evaluation e (HBM-bound: it streams the saved activations) runs on a side stream while the
    # main stream continues with the data gradient of evaluation e - 1 (tensor-bound). dY is double-buffered; the data gradient that
    # re-uses a dY buffer waits for the weight gradient that read it two evaluations earlier.
    overlap = os.environ.get('DVD_BWD_OVERLAP', '1') != '0' and n_eval > 1
    nbuf = 2 if overlap else 1
    dys = [torch.empty(lib.dvd_mlp_dy_bytes(ctypes.byref(cfg), npx), dtype=torch.uint8, device=dev) for _ in range(nbuf)]
    side = _side_stream(dev) if overlap else None
    main = torch.cuda.current_stream()
    wdone = [None] * nbuf
    a = None
    gb5 = grad_b[5]
    if gb5.numel() != 3:
        raise ValueError('grad of the output bias must have 3 elements')
    gw_arr, gb_arr = _ptr_array(grad_w), _ptr_array(grad_b)
    if ordered():
        ws_d, ws_w = _ws(ordered_workspace(dev, _lib.DVD_ORD_MLP_DGRAD)), _ws(ordered_workspace(dev, _lib.DVD_ORD_MLP_WGRAD))

        def dgrad(*a):
            LAUNCHES['n'] += 1
            return lib.dvd_mlp_dgrad_ordered(*a[:-1], *ws_d, a[-1])

        def wgrad(*a):
            LAUNCHES['n'] += 1
            return lib.dvd_mlp_wgrad_ordered(*a[:-1], *ws_w, a[-1])
    else:
        dgrad, wgrad = lib.dvd_mlp_dgrad, lib.dvd_mlp_wgrad
    for i, e in enumerate(range(n_eval - 1, -1, -1)):
        dy = dys[i % nbuf]
        if wdone[i % nbuf] is not None:
            main.wait_event(wdone[i % nbuf])
        a_out = torch.empty(B, 3, H, W, dtype=torch.float32, device=dev)
        gs = g_steps[e] if g_steps is not None else None
        save_e = ctypes.c_void_p(sv.data_ptr() + e * per)
        LAUNCHES['n'] += 1
        _lib.check(dgrad(ctypes.byref(cfg), _ptr(packed.bwd), _ptr(p_steps[e]),
                                     _ptr(t0) if cfg.time_dependent else ctypes.c_void_p(0), float(dt), e,
                                     int(e < n_acc and g_acc is not None), _ptr(g_acc), _ptr(gs), _ptr(a), _ptr(a_out),
                                     save_e, _ptr(dy), _ptr(gb5), npx, hw, _stream()), 'dvd_mlp_dgrad')
        a = a_out
        LAUNCHES['n'] += 1
        if side is not None:
            ev = torch.cuda.Event()
            ev.record(main)
            side.wait_event(ev)
            with torch.cuda.stream(side):
                _lib.check(wgrad(ctypes.byref(cfg), save_e, _ptr(dy), gw_arr, gb_arr, npx, _stream()), 'dvd_mlp_wgrad')
                wdone[i % nbuf] = torch.cuda.Event()
                wdone[i % nbuf].record(side)
        else:
            _lib.check(wgrad(ctypes.byref(cfg), save_e, _ptr(dy), gw_arr, gb_arr, npx, _stream()), 'dvd_mlp_wgrad')
    if side is not None:       # join: the weight gradients are final (and dY / the saved activations may be freed) after this
        for ev in wdone:
            if ev is not None:
                main.wait_event(ev)
    return a_out


def acc_reg(s0, s1, acc_mul, gscale=1.0, want_grad=True):
    """Model._opt_reg value + gradients w.r.t. (s0, s1) (smf.py:326-344)."""
    _chk(s0, 's0'), _chk(s1, 's1', s0.shape)
    lib = _lib.load()
    g0 = torch.empty_like(s0) if want_grad else None
    g1 = torch.empty_like(s1) if want_grad else None
    partials = torch.empty(1024, dtype=torch.float32, device=s0.device)
    out = torch.empty(1, dtype=torch.float32, device=s0.device)
    LAUNCHES['n'] += 2
    _lib.check(lib.dvd_acc_reg(_ptr(s0), _ptr(s1), float(acc_mul), float(gscale), _ptr(g0), _ptr(g1), _ptr(partials),
                               _ptr(out), s0.numel(), _stream()), 'dvd_acc_reg')
    return out, g0, g1


class SceneFlowChain(torch.autograd.Function):
    """Euler chain of the scene-flow field as one autograd node.

    forward(p0, t0, w0..w5, b0..b5 | packed, dt, n_eval, n_acc) -> (acc, s_steps)
    acc = sum_{i<n_acc} s_i   (Model.forward_sf_net_multi_step, smf.py:360-367);
    s_steps [n_eval,B,3,H,W] exposes the individual steps (the acceleration regulariser reuses s_0, s_1)."""

    @staticmethod
    def forward(ctx, p0, t0, packed, dt, n_eval, n_acc, *params):
        need = any(ctx.needs_input_grad)
        p0c = p0.contiguous()
        f = mlp_chain_fwd(packed, p0c, t0, dt, n_eval, n_acc, save=need, want_steps=True)
        ctx.packed, ctx.dt, ctx.n_acc, ctx.t0 = packed, dt, n_acc, t0
        ctx.fwd = f
        ctx.param_shapes = [p.shape for p in params]
        return f['acc'], f['s_steps']

    @staticmethod
    def backward(ctx, g_acc, g_steps):
        f = ctx.fwd
        n_eval = f['p_steps'].shape[0]
        dev = f['p_steps'].device
        shapes = ctx.param_shapes
        gw = [torch.zeros(shapes[l], dtype=torch.float32, device=dev) for l in range(6)]
        gb = [torch.zeros(shapes[6 + l], dtype=torch.float32, device=dev) for l in range(6)]
        g_acc = g_acc.contiguous() if g_acc is not None else None
        gsl = None
        if g_steps is not None:
            g_steps = g_steps.contiguous()
            gsl = [g_steps[e] for e in range(n_eval)]
        gp = mlp_chain_bwd(ctx.packed, f, ctx.t0, ctx.dt, ctx.n_acc, g_acc, gsl, gw, gb)
        ctx.fwd = None
        return (gp, None, None, None, None, None, *gw, *gb)


def scene_flow_chain(p0, t0, packed, dt, n_eval, n_acc, weights, biases):
    return SceneFlowChain.apply(p0, t0, packed, float(dt), int(n_eval), int(n_acc), *weights, *biases)


# ================================================================================================
# channels-last glue of the depth nets (csrc/nhwc_ops.cu)

def _is_cl(t):
    return t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last)


def _as_cl(t):
    return t if _is_cl(t) else t.contiguous(memory_format=torch.channels_last)


class BnAct(torch.autograd.Function):
    """Eval-mode BatchNorm (+ residual) (+ ReLU) on channels-last tensors, one pass forward and one backward.
    forward(x, res|None, gamma, beta, running_mean, running_var, eps, relu) -> y"""

    @staticmethod
    def forward(ctx, x, res, gamma, beta, mean, var, eps, relu):
        x = _as_cl(x)
        if x.dtype != torch.float32 or not x.is_cuda:
            raise ValueError('BnAct needs float32 CUDA tensors')
        N, C, H, W = x.shape
        if C % 4:
            raise ValueError('channel count must be a multiple of 4')
        r = _as_cl(res) if res is not None else None
        y = torch.empty_like(x)   # preserves channels_last
        lib = _lib.load()
        LAUNCHES['n'] += 1
        _lib.check(lib.dvd_bn_act_fwd(_ptr(x), _ptr(r), _ptr(gamma), _ptr(beta), _ptr(mean), _ptr(var), float(eps), _ptr(y),
                                      N * H * W, C, int(relu), _stream()), 'dvd_bn_act_fwd')
        ctx.save_for_backward(x, y, gamma, mean, var)
        ctx.beta = beta
        ctx.eps, ctx.relu, ctx.has_res = float(eps), bool(relu), res is not None
        return y

    @staticmethod
    def backward(ctx, g):
        x, y, gamma, mean, var = ctx.saved_tensors
        g = _as_cl(g)
        N, C, H, W = x.shape
        gx = torch.empty_like(x)
        gres = torch.empty_like(x) if ctx.has_res else None
        beta = ctx.beta
        # The per-channel sums are atomically ACCUMULATED by the kernel. When gamma/beta live in the flat gradient buffer of
        # dvd_b200.flat.FlatParams (zeroed once per step) they are accumulated there directly and autograd gets None (= zero)
        # for them: no fill, no extra add kernels.
        # Explicit opt-in: only parameters that dvd_b200.flat.FlatParams has re-homed carry `_dvd_flat_grad` (set there, cleared
        # nowhere else); any other parameter gets its gradient through autograd like every other tensor, so torch.autograd.grad,
        # hooks and foreign optimisers keep working.
        direct = (getattr(gamma, '_dvd_flat_grad', False) and getattr(beta, '_dvd_flat_grad', False)
                  and gamma.requires_grad and beta.requires_grad and gamma.grad is not None and beta.grad is not None
                  and gamma.grad.is_contiguous() and beta.grad.is_contiguous() and gamma.grad.dtype == torch.float32)
        if direct:
            gg, gb = gamma.grad, beta.grad
        else:
            ggb = torch.zeros(2, C, dtype=torch.float32, device=x.device)   # one fill for both per-channel sums
            gg, gb = ggb[0], ggb[1]
        lib = _lib.load()
        if ordered():
            LAUNCHES['n'] += 2
            ws = _ws(ordered_workspace(x.device, _lib.DVD_ORD_CHANNEL_SUMS))
            _lib.check(lib.dvd_bn_act_bwd_ordered(_ptr(g), _ptr(x), _ptr(y), _ptr(gamma), _ptr(mean), _ptr(var), ctx.eps, _ptr(gx),
                                                  _ptr(gres), _ptr(gg), _ptr(gb), N * H * W, C, int(ctx.relu), *ws, _stream()),
                       'dvd_bn_act_bwd_ordered')
        else:
            LAUNCHES['n'] += 1
            _lib.check(lib.dvd_bn_act_bwd(_ptr(g), _ptr(x), _ptr(y), _ptr(gamma), _ptr(mean), _ptr(var), ctx.eps, _ptr(gx),
                                          _ptr(gres), _ptr(gg), _ptr(gb), N * H * W, C, int(ctx.relu), _stream()), 'dvd_bn_act_bwd')
        if direct:
            return gx, gres, None, None, None, None, None, None
        return gx, gres, gg, gb, None, None, None, None


def bn_act(x, bn, res=None, relu=True):
    """`relu(bn(x) + res)` for an nn.BatchNorm2d in eval mode (affine)."""
    return BnAct.apply(x, res, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, relu)


class Upsample2x(torch.autograd.Function):
    """F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=...) on channels-last tensors."""

    @staticmethod
    def forward(ctx, x, align_corners):
        x = _as_cl(x)
        if x.dtype != torch.float32 or not x.is_cuda:
            raise ValueError('Upsample2x needs float32 CUDA tensors')
        N, C, H, W = x.shape
        if C % 4:
            raise ValueError('channel count must be a multiple of 4')
        y = torch.empty((N, C, 2 * H, 2 * W), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        lib = _lib.load()
        LAUNCHES['n'] += 1
        _lib.check(lib.dvd_upsample2x_fwd(_ptr(x), _ptr(y), N, H, W, C, int(align_corners), 0, _stream()), 'dvd_upsample2x_fwd')
        ctx.shape, ctx.align = (N, C, H, W), bool(align_corners)
        return y

    @staticmethod
    def backward(ctx, g):
        g = _as_cl(g)
        N, C, H, W = ctx.shape
        gx = torch.empty((N, C, H, W), dtype=g.dtype, device=g.device, memory_format=torch.channels_last)
        lib = _lib.load()
        LAUNCHES['n'] += 1
        _lib.check(lib.dvd_upsample2x_bwd(_ptr(g), _ptr(gx), N, H, W, C, int(ctx.align), 0, _stream()), 'dvd_upsample2x_bwd')
        return gx, None


def upsample2x(x, align_corners):
    return Upsample2x.apply(x, bool(align_corners))


# ================================================================================================
# differentiable materialisation (operator-level drop-in of the two projection modules)

_MAT_ALL = _MAT_KEYS3 + _MAT_KEYS2 + _MAT_KEYS1


class ReprojectMaterialize(torch.autograd.Function):
    """All nine per-pixel tensors of flow_by_depth / scene_flow_projection_slack (channel-planar), differentiable
    w.r.t. depth_1, depth_2 and sf for arbitrary cotangents (dvd_reproject_materialize_bwd)."""

    @staticmethod
    def forward(ctx, depth_1, depth_2, sf, flow, poses):
        depth_1, depth_2 = depth_1.contiguous(), depth_2.contiguous()
        sf = sf.contiguous() if sf is not None else None
        out = reproject_materialize(depth_1, depth_2, flow, sf, poses)
        ctx.save_for_backward(depth_1, depth_2, sf if sf is not None else depth_1.new_empty(0), flow, poses)
        ctx.has_sf = sf is not None
        return tuple(out[k] for k in _MAT_ALL)

    @staticmethod
    def backward(ctx, *grads):
        depth_1, depth_2, sf, flow, poses = ctx.saved_tensors
        sf = sf if ctx.has_sf else None
        B, _, H, W = depth_1.shape
        gs = [g.contiguous() if g is not None else None for g in grads]
        g_d1 = torch.empty_like(depth_1) if ctx.needs_input_grad[0] else None
        g_d2 = torch.empty_like(depth_2) if ctx.needs_input_grad[1] else None
        g_sf = torch.empty(B, 3, H, W, dtype=torch.float32, device=depth_1.device) if (ctx.has_sf and ctx.needs_input_grad[2]) else None
        lib = _lib.load()
        LAUNCHES['n'] += 1
        _lib.check(lib.dvd_reproject_materialize_bwd(_ptr(depth_1), _ptr(depth_2), _ptr(flow), _ptr(sf), _ptr(poses),
                                                     *[_ptr(g) for g in gs], _ptr(g_d1), _ptr(g_d2), _ptr(g_sf), B, H, W,
                                                     _stream()), 'dvd_reproject_materialize_bwd')
        return g_d1, g_d2, g_sf, None, None


def reproject_tensors(depth_1, depth_2, sf, flow, poses):
    """dict of the nine differentiable per-pixel tensors."""
    _chk_reproject(depth_1.contiguous(), depth_2.contiguous(), flow, None, sf.contiguous() if sf is not None else None, poses)
    return dict(zip(_MAT_ALL, ReprojectMaterialize.apply(depth_1, depth_2, sf, flow, poses)))


# ---- flow-pair preprocessing (csrc/flow_pairs.cu) ---------------------------------------------------------------------------
MASK_CONVENTIONS = {'flowpair': _lib.DVD_MASKS_FLOWPAIR_U8, 'pair_file': _lib.DVD_MASKS_PAIRFILE_F32}


def _chk_flows(flow, name):
    _chk(flow, name)
    if flow.dim() != 4 or flow.shape[-1] != 2:
        raise ValueError('%s must be [B,H,W,2] (NHWC flow), got %s' % (name, tuple(flow.shape)))
    if flow.data_ptr() % 8:
        raise ValueError('%s must be 8-byte aligned' % name)
    return flow


def flow_resize_cubic(flow, H, W):
    """The reference's `resize_flow` (generate_flows.py:44-54) on the GPU: cv2 INTER_CUBIC resize of [B,h,w,2] fp32 flows to
    [B,H,W,2], then x *= W / w and y *= H / h."""
    _chk_flows(flow, 'flow')
    H, W = int(H), int(W)
    if H < 1 or W < 1:
        raise ValueError('output size must be positive, got %dx%d' % (H, W))
    B, h, w, _ = flow.shape
    out = torch.empty(B, H, W, 2, dtype=torch.float32, device=flow.device)
    lib = _lib.load()
    LAUNCHES['n'] += 1
    _lib.check(lib.dvd_flow_resize_cubic(_ptr(flow), flow.numel() * 4, _ptr(out), out.numel() * 4, B, h, w, H, W, _stream()),
               'dvd_flow_resize_cubic')
    return out


def flow_pair_masks(flow_1_2, flow_2_1, convention='pair_file'):
    """Forward / backward consistency masks of two [B,H,W,2] fp32 flows (generate_flows.py:57-82,139-148) -> (mask_1, mask_2).
    convention 'flowpair': uint8 [B,H,W], 1 = inconsistent or out of bounds (flowpair_*.npz);
               'pair_file': fp32 [B,H,W,1,1], 1 - ceil(mask), 1 = valid (the sequence .pt files, the Model's mask_1 / mask_2)."""
    if convention not in MASK_CONVENTIONS:
        raise ValueError('convention must be one of %s, got %r' % (sorted(MASK_CONVENTIONS), convention))
    _chk_flows(flow_1_2, 'flow_1_2')
    _chk_flows(flow_2_1, 'flow_2_1')
    if flow_1_2.shape != flow_2_1.shape or flow_1_2.device != flow_2_1.device:
        raise ValueError('flow_1_2 %s and flow_2_1 %s must match' % (tuple(flow_1_2.shape), tuple(flow_2_1.shape)))
    B, H, W, _ = flow_1_2.shape
    if H < 2 or W < 2:
        raise ValueError('flows must be at least 2x2, got %dx%d' % (H, W))
    u8 = convention == 'flowpair'
    shape, dtype = ((B, H, W), torch.uint8) if u8 else ((B, H, W, 1, 1), torch.float32)
    m1 = torch.empty(shape, dtype=dtype, device=flow_1_2.device)
    m2 = torch.empty_like(m1)
    lib = _lib.load()
    LAUNCHES['n'] += 1
    _lib.check(lib.dvd_flow_pair_masks(_ptr(flow_1_2), _ptr(flow_2_1), flow_1_2.numel() * 4, _ptr(m1), _ptr(m2),
                                       m1.numel() * m1.element_size(), B, H, W, MASK_CONVENTIONS[convention], _stream()),
               'dvd_flow_pair_masks')
    return m1, m2


# ---- validation metric (csrc/eval_ops.cu) -----------------------------------------------------------------------------------
def disp_vali(depth, depth_gt, want_terms=False, out=None):
    """The reference's `disp_vali` (models/video_base.py:66-74) per frame: depth, depth_gt [N,1,H,W] fp32 -> frame_sse [N], the
    sum over each frame of (disp(depth)·v - disp(gt)·v)² with v = [gt > 1e-2] (bitwise torch's fp32 terms, fixed-order sums).
    A frame's MSE is frame_sse / (H·W). `out` may be a caller-owned contiguous [N] fp32 buffer (e.g. a slice of a longer one).
    With want_terms, returns (frame_sse, terms [N,1,H,W])."""
    _chk(depth, 'depth')
    _chk(depth_gt, 'depth_gt')
    if depth.dim() != 4 or depth.shape[1] != 1:
        raise ValueError('depth must be [N,1,H,W], got %s' % (tuple(depth.shape),))
    if depth_gt.shape != depth.shape or depth_gt.device != depth.device:
        raise ValueError('depth_gt %s must match depth %s' % (tuple(depth_gt.shape), tuple(depth.shape)))
    N, _, H, W = depth.shape
    if out is None:
        out = torch.empty(N, dtype=torch.float32, device=depth.device)
    else:
        _chk(out, 'out', (N,))
    terms = torch.empty_like(depth) if want_terms else None
    lib = _lib.load()
    n_part = lib.dvd_disp_vali_partials_size(N, H, W)
    if n_part < 1:
        raise ValueError('bad shape for dvd_disp_vali: %s' % (tuple(depth.shape),))
    partials = torch.empty(n_part, dtype=torch.float32, device=depth.device)
    LAUNCHES['n'] += 2
    _lib.check(lib.dvd_disp_vali(_ptr(depth), _ptr(depth_gt), _ptr(out), _ptr(terms), _ptr(partials), N, H, W, _stream()),
               'dvd_disp_vali')
    return (out, terms) if want_terms else out


# ---- frame preparation (csrc/frame_prep.cu) ---------------------------------------------------------------------------------
def _chk_dtype(t, name, dtype, dim):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError('%s must be a CUDA tensor (dvd_b200 has no CPU path)' % name)
    if t.dtype != dtype or not t.is_contiguous() or t.dim() != dim:
        raise ValueError('%s must be a contiguous %d-d %s tensor, got %s %s' % (name, dim, dtype, t.dtype, tuple(t.shape)))
    return t


def resize_bicubic_ac(x, H, W):
    """F.interpolate(x, (H, W), mode='bicubic', align_corners=True) of a [N,C,h,w] fp32 tensor, any sizes."""
    _chk(x, 'x')
    if x.dim() != 4:
        raise ValueError('x must be [N,C,h,w], got %s' % (tuple(x.shape),))
    H, W = int(H), int(W)
    if H < 1 or W < 1:
        raise ValueError('output size must be positive, got %dx%d' % (H, W))
    N, C, h, w = x.shape
    out = torch.empty(N, C, H, W, dtype=torch.float32, device=x.device)
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_resize_bicubic_ac(_ptr(x), x.numel() * 4, _ptr(out), out.numel() * 4, N * C, h, w, H, W, _stream()),
               'dvd_resize_bicubic_ac')
    return out


def spline_prefilter(maps, out=None):
    """scipy.ndimage.spline_filter(m, 3, output=float64, mode='constant') of each [H,W] map of [N,H,W] fp32 -> fp64 [N,H,W]."""
    _chk(maps, 'maps')
    if maps.dim() != 3:
        raise ValueError('maps must be [N,H,W], got %s' % (tuple(maps.shape),))
    if out is None:
        out = torch.empty(maps.shape, dtype=torch.float64, device=maps.device)
    elif _chk_dtype(out, 'out', torch.float64, 3).shape != maps.shape:
        raise ValueError('out %s must match maps %s' % (tuple(out.shape), tuple(maps.shape)))
    N, H, W = maps.shape
    LAUNCHES['n'] += 2
    _lib.check(_lib.load().dvd_spline_prefilter(_ptr(maps), maps.numel() * 4, _ptr(out), out.numel() * 8, N, H, W, _stream()),
               'dvd_spline_prefilter')
    return out


def spline_sample(coef, vu):
    """map_coordinates(map[n], [v, u], order=3, mode='constant') from spline_prefilter's coef [N,H,W] at vu [N,P,2] fp64 (v, u)
    -> [N,P] fp32; coordinates outside the map, NaN or inf give 0."""
    _chk_dtype(coef, 'coef', torch.float64, 3)
    _chk_dtype(vu, 'vu', torch.float64, 3)
    N, H, W = coef.shape
    if vu.shape[0] != N or vu.shape[2] != 2 or vu.shape[1] < 1 or vu.device != coef.device:
        raise ValueError('vu must be [%d,P,2] on %s, got %s' % (N, coef.device, tuple(vu.shape)))
    P = vu.shape[1]
    out = torch.empty(N, P, dtype=torch.float32, device=coef.device)
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_spline_sample(_ptr(coef), coef.numel() * 8, N, H, W, _ptr(vu), _ptr(out), P, _stream()),
               'dvd_spline_sample')
    return out


def calib_ratios(depth_coef, mask_coef, w2c, points, fx, fy, cx, cy, out=None):
    """The reference's per-frame point selection and nn / depth ratios (generate_frame_midas.py:81-101): depth_coef, mask_coef
    [N,H,W] fp64 (spline_prefilter of the full-resolution depth and mask), w2c [N,4,4] fp64, points [V,3] fp64 -> ratio [N,V]
    fp64, NaN for a rejected point. `out` may be a caller-owned [N,V] fp64 buffer (e.g. rows of a longer one)."""
    _chk_dtype(depth_coef, 'depth_coef', torch.float64, 3)
    _chk_dtype(mask_coef, 'mask_coef', torch.float64, 3)
    _chk_dtype(w2c, 'w2c', torch.float64, 3)
    _chk_dtype(points, 'points', torch.float64, 2)
    N, H, W = depth_coef.shape
    dev = depth_coef.device
    if mask_coef.shape != depth_coef.shape or tuple(w2c.shape) != (N, 4, 4) or points.shape[1] != 3 or points.shape[0] < 1:
        raise ValueError('bad shapes: depth_coef %s, mask_coef %s, w2c %s, points %s' % (
            tuple(depth_coef.shape), tuple(mask_coef.shape), tuple(w2c.shape), tuple(points.shape)))
    if any(t.device != dev for t in (mask_coef, w2c, points)):
        raise ValueError('all tensors must be on %s' % dev)
    V = points.shape[0]
    if out is None:
        out = torch.empty(N, V, dtype=torch.float64, device=dev)
    elif tuple(_chk_dtype(out, 'out', torch.float64, 2).shape) != (N, V):
        raise ValueError('out must be [%d,%d], got %s' % (N, V, tuple(out.shape)))
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_calib_ratios(_ptr(depth_coef), _ptr(mask_coef), depth_coef.numel() * 8, _ptr(w2c), _ptr(points), V,
                                            float(fx), float(fy), float(cx), float(cy), _ptr(out), out.numel() * 8, N, H, W,
                                            _stream()), 'dvd_calib_ratios')
    return out


def row_medians(ratio):
    """np.median of the non-NaN entries of each row of [N,V] fp64 or fp32 -> (median [N] of the same dtype, count [N] int32).
    The rows are sorted on the device first (NaN last). For fp32 rows the median is numpy's fp32 one: the middle element, or
    the fp32 (a + b) / 2 of the two middle ones."""
    if isinstance(ratio, torch.Tensor) and ratio.dtype == torch.float32:
        _chk_dtype(ratio, 'ratio', torch.float32, 2)
    else:
        _chk_dtype(ratio, 'ratio', torch.float64, 2)
    N, V = ratio.shape
    if V < 1 or V > 2 ** 31 - 1:
        raise ValueError('ratio rows must hold 1 .. 2^31 - 1 entries, got %d' % V)
    srt = torch.sort(ratio, dim=1)[0].contiguous()
    med = torch.empty(N, dtype=ratio.dtype, device=ratio.device)
    cnt = torch.empty(N, dtype=torch.int32, device=ratio.device)
    LAUNCHES['n'] += 1
    if ratio.dtype == torch.float32:
        _lib.check(_lib.load().dvd_sorted_median_f32(_ptr(srt), srt.numel() * 4, N, V, _ptr(med), _ptr(cnt), _stream()),
                   'dvd_sorted_median_f32')
    else:
        _lib.check(_lib.load().dvd_sorted_median(_ptr(srt), srt.numel() * 8, N, V, _ptr(med), _ptr(cnt), _stream()),
                   'dvd_sorted_median')
    return med, cnt


def dense_ratios(nn, mvs):
    """The ShutterStock calibration's ratios (shutterstock/generate_frame_midas.py:167-172): nn [N,H,W] fp32 (MiDaS depth at the
    stored size) and mvs [N,H,W] fp32 or fp64 -> [N,H*W] of mvs's dtype, nn / mvs where mvs > 1e-3 and a positive NaN
    elsewhere, in numpy's arithmetic (fp32 threshold and quotient for fp32 maps). row_medians of the result gives the
    per-frame medians of the script."""
    _chk_dtype(nn, 'nn', torch.float32, 3)
    if not isinstance(mvs, torch.Tensor) or mvs.dtype not in (torch.float32, torch.float64):
        raise ValueError('mvs must be a float32 or float64 tensor, got %s' % getattr(mvs, 'dtype', type(mvs)))
    _chk_dtype(mvs, 'mvs', mvs.dtype, 3)
    if mvs.shape != nn.shape or mvs.device != nn.device or nn.numel() == 0:
        raise ValueError('nn %s and mvs %s must be non-empty, of one shape, on one device' % (tuple(nn.shape), tuple(mvs.shape)))
    N, H, W = nn.shape
    out = torch.empty(N, H * W, dtype=mvs.dtype, device=nn.device)
    es = mvs.element_size()
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_dense_ratios(_ptr(nn), nn.numel() * 4, _ptr(mvs), mvs.numel() * es, int(es == 8), _ptr(out),
                                            out.numel() * es, N, H * W, _stream()), 'dvd_dense_ratios')
    return out


def gaussian_weights(n_in, n_out):
    """skimage's anti-aliasing kernel along an axis shrunk from n_in to n_out: sigma = max(0, (n_in / n_out - 1) / 2), then
    scipy.ndimage's gaussian_filter1d weights (truncate 4: radius int(4 sigma + 0.5), exp(-x² / (2 sigma²)) normalised by its sum).
    An axis with sigma <= 1e-15 is not filtered by scipy: the single weight 1 leaves it unchanged. Returns (radius, fp64 weights)."""
    import numpy as np
    sigma = max(0.0, (float(np.divide(n_in, n_out)) - 1.0) / 2.0)
    if sigma <= 1e-15:
        return 0, np.ones(1)
    radius = int(4.0 * sigma + 0.5)
    x = np.arange(-radius, radius + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    return radius, phi / phi.sum()


def aa_resize(src, OH, OW, weights=None):
    """skimage.transform.resize(img, (OH, OW), preserve_range=True) (skimage >= 0.19: Gaussian anti-aliasing when shrinking, order 1,
    mode 'reflect', clip) of each frame of a [N,H,W,C] fp32 tensor -> [N,OH,OW,C] fp32. `weights` = the two fp64 device weight
    tensors of gaussian_weights (built here when None)."""
    _chk(src, 'src')
    if src.dim() != 4:
        raise ValueError('src must be [N,H,W,C], got %s' % (tuple(src.shape),))
    OH, OW = int(OH), int(OW)
    if OH < 1 or OW < 1:
        raise ValueError('output size must be positive, got %dx%d' % (OH, OW))
    N, H, W, C = src.shape
    if weights is None:
        weights = [torch.from_numpy(gaussian_weights(n, o)[1]).to(src.device) for n, o in ((H, OH), (W, OW))]
    wy, wx = weights
    for name, t in (('wy', wy), ('wx', wx)):
        if _chk_dtype(t, name, torch.float64, 1).numel() % 2 == 0:
            raise ValueError('%s must have an odd length 2 r + 1' % name)
    lib = _lib.load()
    nb = lib.dvd_aa_resize_scratch_bytes(N, H, W, C)
    scratch = torch.empty(nb // 4, dtype=torch.float32, device=src.device)
    out = torch.empty(N, OH, OW, C, dtype=torch.float32, device=src.device)
    LAUNCHES['n'] += 4
    _lib.check(lib.dvd_aa_resize(_ptr(src), src.numel() * 4, _ptr(out), out.numel() * 4, _ptr(scratch), nb, _ptr(wy),
                                 wy.numel() // 2, _ptr(wx), wx.numel() // 2, N, H, W, C, OH, OW, _stream()), 'dvd_aa_resize')
    return out


# ---- point-cloud export (csrc/points.cu) -------------------------------------------------------------------------------------
class KeyRangeError(ValueError):
    """A voxel key left the 2^21-voxel range of an axis."""


def points_select(depth, img, P, edge_tol, voxel=None, origin=(0, 0, 0), base=0):
    """dvd_points_select: depth [N,H,W], img [N,3,H,W], P [N,3,H,W] fp32 -> dict of the kept pixels in pixel order: mask [N,H,W]
    uint8 (all pixels), index [M] int64 (base + flat pixel index), xyz [M,3] fp32, rgb [M,3] uint8 and, with a voxel size,
    key [M] int64 relative to the voxel `origin`. Waits for the stream (M sizes the outputs). Raises KeyRangeError when a key
    is out of range."""
    _chk(depth, 'depth')
    if depth.dim() != 3:
        raise ValueError('depth must be [N,H,W], got %s' % (tuple(depth.shape),))
    N, H, W = depth.shape
    _chk(img, 'img', (N, 3, H, W)), _chk(P, 'P', (N, 3, H, W))
    if img.device != depth.device or P.device != depth.device:
        raise ValueError('depth, img and P must be on one device')
    dev, n = depth.device, N * H * W
    lib = _lib.load()
    scratch = torch.empty(lib.dvd_points_select_scratch_bytes(N, H, W), dtype=torch.uint8, device=dev)
    mask = torch.empty(N, H, W, dtype=torch.uint8, device=dev)
    key = torch.empty(n, dtype=torch.int64, device=dev) if voxel is not None else None
    index = torch.empty(n, dtype=torch.int64, device=dev)
    xyz = torch.empty(n, 3, dtype=torch.float32, device=dev)
    rgb = torch.empty(n, 3, dtype=torch.uint8, device=dev)
    m = ctypes.c_longlong(0)
    LAUNCHES['n'] += 3
    ox, oy, oz = (int(o) for o in origin)
    rc = lib.dvd_points_select(_ptr(depth), _ptr(img), _ptr(P), N, H, W, float(edge_tol), float(voxel or 0.0), ox, oy, oz, int(base),
                               _ptr(mask), _ptr(key), _ptr(index), _ptr(xyz), _ptr(rgb), _ptr(scratch), scratch.numel(),
                               ctypes.byref(m), _stream())
    if rc == -3:
        raise KeyRangeError(lib.dvd_last_error().decode())
    _lib.check(rc, 'dvd_points_select')
    M = m.value
    out = {'mask': mask, 'index': index[:M], 'xyz': xyz[:M], 'rgb': rgb[:M]}
    if key is not None:
        out['key'] = key[:M]
    return out


def voxel_reduce(skey, order, index, xyz, rgb, hw, min_views):
    """dvd_voxel_reduce: skey [M] sorted int64 keys, order [M] int64 the stable sort's permutation of the items index [M] int64,
    xyz [M,3] fp32, rgb [M,3] uint8 (frame = index // hw) -> dict of the runs seen in >= min_views frames, in key order: xyz,
    rgb [R,3] fp64 means, count, views [R] int32. Waits for the stream (R sizes the outputs)."""
    M = skey.numel()
    for name, t, dt in (('skey', skey, torch.int64), ('order', order, torch.int64), ('index', index, torch.int64),
                        ('xyz', xyz, torch.float32), ('rgb', rgb, torch.uint8)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != dt or not t.is_contiguous() or t.shape[0] != M:
            raise ValueError('%s must be a contiguous CUDA %s tensor with %d rows' % (name, dt, M))
    if tuple(xyz.shape) != (M, 3) or tuple(rgb.shape) != (M, 3):
        raise ValueError('xyz and rgb must be [%d,3]' % M)
    dev = skey.device
    if M == 0:
        z = torch.empty(0, 3, dtype=torch.float64, device=dev)
        return {'xyz': z, 'rgb': z.clone(), 'count': torch.empty(0, dtype=torch.int32, device=dev),
                'views': torch.empty(0, dtype=torch.int32, device=dev)}
    lib = _lib.load()
    scratch = torch.empty(lib.dvd_voxel_reduce_scratch_bytes(M), dtype=torch.uint8, device=dev)
    mx = torch.empty(M, 3, dtype=torch.float64, device=dev)
    mc = torch.empty(M, 3, dtype=torch.float64, device=dev)
    cnt = torch.empty(M, dtype=torch.int32, device=dev)
    views = torch.empty(M, dtype=torch.int32, device=dev)
    r = ctypes.c_longlong(0)
    LAUNCHES['n'] += 6
    _lib.check(lib.dvd_voxel_reduce(_ptr(skey), _ptr(order), _ptr(index), _ptr(xyz), _ptr(rgb), M, int(hw), int(min_views), _ptr(mx),
                                    _ptr(mc), _ptr(cnt), _ptr(views), _ptr(scratch), scratch.numel(), ctypes.byref(r), _stream()),
               'dvd_voxel_reduce')
    R = r.value
    return {'xyz': mx[:R], 'rgb': mc[:R], 'count': cnt[:R], 'views': views[:R]}


# ---- test-end visualisation (csrc/test_videos.cu) -----------------------------------------------------------------------------
VIS_TRANSFORMS = {'disp': _lib.DVD_VIS_DISP, 'gt_disp': _lib.DVD_VIS_GT_DISP, 'rgb': _lib.DVD_VIS_RGB}


def vis_panel(src, transform, rows, cols, y0, x0, strides, offset=0, vmin=None, vmax=None):
    """One panel of `vis_panels`: pixel (y0 + y, x0 + x) of canvas c reads element offset + c·s_canvas + y·s_row + x·s_col
    (+ k·s_chan for channel k of 'rgb') of the contiguous fp32 CUDA tensor `src`; strides = (s_canvas, s_row, s_col, s_chan) in
    elements. 'disp' and 'gt_disp' are colour-mapped through vmin[c], vmax[c] (contiguous fp64 CUDA tensors)."""
    if transform not in VIS_TRANSFORMS:
        raise ValueError('transform must be one of %s, got %r' % (sorted(VIS_TRANSFORMS), transform))
    return dict(src=src, transform=transform, rows=int(rows), cols=int(cols), y0=int(y0), x0=int(x0),
                strides=tuple(int(s) for s in strides), offset=int(offset), vmin=vmin, vmax=vmax)


def vis_panels(tmpl, panels, lut, out, tmpl_stride=0):
    """dvd_vis_panels: writes out [n,CH,CW,3] uint8 (BGR): canvas c = the template tmpl[c·tmpl_stride bytes …] ([CH,CW,3] uint8;
    tmpl_stride = 0 shares one template) with the pixels of each `vis_panel` replaced. lut: [256,3] uint8 BGR colour table.
    Every read a panel makes is checked against its source tensor before the launch."""
    _chk_dtype(out, 'out', torch.uint8, 4)
    n, CH, CW, C = out.shape
    if C != 3:
        raise ValueError('out must be [n,CH,CW,3], got %s' % (tuple(out.shape),))
    if not isinstance(tmpl, torch.Tensor) or not tmpl.is_cuda or tmpl.dtype != torch.uint8 or not tmpl.is_contiguous():
        raise ValueError('tmpl must be a contiguous uint8 CUDA tensor')
    tmpl_stride = int(tmpl_stride)
    if tmpl_stride < 0 or tmpl.numel() < (n - 1) * tmpl_stride + CH * CW * 3:
        raise ValueError('tmpl holds %d bytes, %d canvases of %dx%d at stride %d need more' % (tmpl.numel(), n, CH, CW, tmpl_stride))
    if len(panels) > _lib.DVD_VIS_MAX_PANELS:
        raise ValueError('at most %d panels per call, got %d' % (_lib.DVD_VIS_MAX_PANELS, len(panels)))
    arr = (_lib.VisPanel * max(len(panels), 1))()
    mapped = False
    for q, p in enumerate(panels):
        src = _chk(p['src'], 'panels[%d].src' % q)
        if src.device != out.device or tmpl.device != out.device:
            raise ValueError('panels[%d]: the sources, the template and out must be on one device' % q)
        s = p['strides']
        if len(s) != 4 or min(s) < 0 or p['offset'] < 0:
            raise ValueError('panels[%d]: strides %s and offset %d must be 4 non-negative integers' % (q, s, p['offset']))
        last = p['offset'] + (n - 1) * s[0] + (p['rows'] - 1) * s[1] + (p['cols'] - 1) * s[2] + (2 * s[3] if p['transform'] == 'rgb' else 0)
        if p['rows'] < 1 or p['cols'] < 1 or last >= src.numel():
            raise ValueError('panels[%d]: %dx%d panel reads element %d of a %d-element source' % (q, p['rows'], p['cols'], last, src.numel()))
        rng = (0, 0)
        if p['transform'] != 'rgb':
            mapped = True
            for name in ('vmin', 'vmax'):
                t = p[name]
                if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float64 or not t.is_contiguous() or t.numel() < n:
                    raise ValueError('panels[%d].%s must be a contiguous fp64 CUDA tensor of at least %d values' % (q, name, n))
            rng = (p['vmin'].data_ptr(), p['vmax'].data_ptr())
        arr[q] = _lib.VisPanel(src.data_ptr() + 4 * p['offset'], rng[0], rng[1], *s, p['rows'], p['cols'], p['y0'], p['x0'],
                               VIS_TRANSFORMS[p['transform']], 0)
    if mapped and (not isinstance(lut, torch.Tensor) or not lut.is_cuda or lut.dtype != torch.uint8 or not lut.is_contiguous()
                   or tuple(lut.shape) != (256, 3)):
        raise ValueError('lut must be a contiguous [256,3] uint8 CUDA tensor')
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_vis_panels(_ptr(tmpl), tmpl_stride, n, CH, CW, arr, len(panels), _ptr(lut if mapped else None),
                                          _ptr(out), _stream()), 'dvd_vis_panels')
    return out


# ---- training / validation page images (csrc/train_vis.cu) ----------------------------------------------------------------------
VIS_MAP_KINDS = {'depth': (_lib.DVD_VIS_MAP_DEPTH, 1), 'flow': (_lib.DVD_VIS_MAP_FLOW, 2), 'img': (_lib.DVD_VIS_MAP_IMG, 3)}


def vis_map_array(maps, turbo, wheel):
    """The checked host array of struct dvd_vis_map for `vis_tiles`: (array, H, W, number of tiles)."""
    if not 1 <= len(maps) <= _lib.DVD_VIS_MAX_MAPS:
        raise ValueError('1 to %d maps per call, got %d' % (_lib.DVD_VIS_MAX_MAPS, len(maps)))
    for name, t, shape in (('turbo', turbo, (256, 3)), ('wheel', wheel, (55, 3))):
        _chk_dtype(t, name, torch.float64, 2)
        if tuple(t.shape) != shape:
            raise ValueError('%s must be %s, got %s' % (name, shape, tuple(t.shape)))
    H = W = None
    arr = (_lib.VisMap * len(maps))()
    n_tiles = 0
    for q, (kind, src) in enumerate(maps):
        if kind not in VIS_MAP_KINDS:
            raise ValueError('maps[%d]: kind must be one of %s, got %r' % (q, sorted(VIS_MAP_KINDS), kind))
        code, chans = VIS_MAP_KINDS[kind]
        if not isinstance(src, torch.Tensor) or not src.is_cuda or src.dtype != torch.float32:
            raise ValueError('maps[%d] must be a float32 CUDA tensor' % q)
        if src.dim() != 4 or src.shape[1] != chans or min(src.stride()) < 0 or src.numel() == 0:
            raise ValueError('maps[%d]: a %s map must be a non-empty [n,%d,H,W] view, got %s' % (q, kind, chans, tuple(src.shape)))
        if H is None:
            H, W = int(src.shape[2]), int(src.shape[3])
        if (src.shape[2], src.shape[3]) != (H, W) or src.device != turbo.device or wheel.device != turbo.device:
            raise ValueError('maps[%d]: every map of a call has the same H x W (%dx%d) and device, got %s' % (q, H, W, tuple(src.shape)))
        n = int(src.shape[0])
        arr[q] = _lib.VisMap(src.data_ptr(), *src.stride(), code, n, 2 * n_tiles, n_tiles)
        n_tiles += n
    return arr, H, W, n_tiles


def vis_tiles(maps, turbo, wheel):
    """dvd_vis_ranges + dvd_vis_tiles: the uint8 RGB tiles [T,H,W,3] of `maps`, a list of (kind, src) with kind 'depth', 'flow'
    or 'img' and src an fp32 CUDA tensor indexed (image, channel, y, x) - any strides, so `flow.permute(0, 3, 1, 2)` of a
    [B,H,W,2] flow is read in place. The tiles of map q follow those of maps 0..q-1, one per image. turbo: [256,3] fp64 RGB
    colour table, wheel: [55,3] fp64 flow colour wheel over 255, both contiguous on the maps' device."""
    arr, H, W, n_tiles = vis_map_array(maps, turbo, wheel)
    dev = turbo.device
    ranges = torch.empty(2 * n_tiles, dtype=torch.float32, device=dev)
    tiles = torch.empty(n_tiles, H, W, 3, dtype=torch.uint8, device=dev)
    lib = _lib.load()
    LAUNCHES['n'] += 2
    _lib.check(lib.dvd_vis_ranges(arr, len(maps), H, W, _ptr(ranges), _stream()), 'dvd_vis_ranges')
    _lib.check(lib.dvd_vis_tiles(arr, len(maps), H, W, _ptr(ranges), _ptr(turbo), _ptr(wheel), _ptr(tiles), _stream()),
               'dvd_vis_tiles')
    return tiles


# ---- novel views (csrc/render_views.cu) ---------------------------------------------------------------------------------------
def view_keys(n, H, W, device):
    """A key buffer for splat_views: [n,H,W] int64 (read as uint64 by the kernels), all ones, i.e. no point yet."""
    return torch.full((n, H, W), -1, dtype=torch.int64, device=device)


def splat_views(keys, xyz, cams, splat=1, index=None):
    """dvd_splat_views: splats the points xyz [M,3] fp32 into the key buffer keys [F,H,W] int64 (view_keys) seen through cams
    [F,21] fp32 (w2c 3x4 | K 3x3, row-major). With index [M] int64 (dvd_points_select's, chunk-relative: frame * H * W + pixel),
    point p goes into view index[p] // (H W) only and carries its pixel index; without, every point goes into every view and
    point r carries H W + r. Each pixel keeps the minimum key (bits(q2) << 32) | index, so repeated calls accumulate."""
    _chk_dtype(keys, 'keys', torch.int64, 3)
    F, H, W = keys.shape
    _chk(cams, 'cams', (F, _lib.DVD_VIEW_CAM_FLOATS))
    _chk(xyz, 'xyz')
    if xyz.dim() != 2 or xyz.shape[1] != 3:
        raise ValueError('xyz must be [M,3], got %s' % (tuple(xyz.shape),))
    if not 1 <= int(splat) <= _lib.DVD_SPLAT_MAX:
        raise ValueError('splat must be in [1, %d], got %r' % (_lib.DVD_SPLAT_MAX, splat))
    if xyz.device != keys.device or cams.device != keys.device:
        raise ValueError('keys, xyz and cams must be on one device')
    M, HW = xyz.shape[0], H * W
    if index is not None:
        _chk_dtype(index, 'index', torch.int64, 1)
        if index.shape[0] != M or index.device != keys.device:
            raise ValueError('index must hold one entry per point (%d) on the points\' device' % M)
        if M:
            lo, hi = (int(v) for v in index.aminmax())
            if lo < 0 or hi >= F * HW:
                raise ValueError('index spans [%d, %d], outside the %d views of %dx%d pixels' % (lo, hi, F, H, W))
    elif HW + M >= 2 ** 32:
        raise ValueError('H W + %d static points = %d reach 2^32, beyond the 32-bit index of a key' % (M, HW + M))
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_splat_views(_ptr(xyz), _ptr(index), M, _ptr(cams), F, H, W, int(splat), _ptr(keys), _stream()),
               'dvd_splat_views')
    return keys


def resolve_views(keys, img, static_rgb=None, out=None, coverage=None):
    """dvd_resolve_views: keys [F,H,W] of splat_views, img [F,3,H,W] fp32 of the views' own frames, static_rgb [R,3] uint8 RGB of
    the static cloud splatted into them (None when there was none) -> (out [F,H,W,3] uint8 BGR, coverage [F] int32: the pixels
    that received a point). Empty pixels are black. `out` and `coverage` may be given (e.g. views of one staging buffer)."""
    _chk_dtype(keys, 'keys', torch.int64, 3)
    F, H, W = keys.shape
    _chk(img, 'img', (F, 3, H, W))
    if static_rgb is not None:
        _chk_dtype(static_rgb, 'static_rgb', torch.uint8, 2)
        if static_rgb.shape[1] != 3 or static_rgb.device != keys.device:
            raise ValueError('static_rgb must be [R,3] on the keys\' device, got %s' % (tuple(static_rgb.shape),))
    if out is None:
        out = torch.empty(F, H, W, 3, dtype=torch.uint8, device=keys.device)
    _chk_dtype(out, 'out', torch.uint8, 4)
    if tuple(out.shape) != (F, H, W, 3) or out.device != keys.device or img.device != keys.device:
        raise ValueError('out must be [%d,%d,%d,3] and img on the keys\' device' % (F, H, W))
    if coverage is None:
        coverage = torch.empty(F, dtype=torch.int32, device=keys.device)
    _chk_dtype(coverage, 'coverage', torch.int32, 1)
    if coverage.shape[0] != F or coverage.device != keys.device:
        raise ValueError('coverage must be [%d] on the keys\' device' % F)
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_resolve_views(_ptr(keys), _ptr(img), _ptr(static_rgb), F, H, W, _ptr(out), _ptr(coverage), _stream()),
               'dvd_resolve_views')
    return out, coverage


# ---- synthetic depth of field (csrc/refocus.cu) -------------------------------------------------------------------------------
def refocus(depth, img, focus_disp, scale, max_radius, out=None):
    """dvd_refocus: frames depth [N,H,W] fp32 and img [N,3,H,W] fp32 RGB, blurred by each pixel's blur radius
    c = min(max_radius, scale |disp - focus_disp[n]|) with the exact gather rule of include/dvd_b200.h -> out [N,H,W,3] uint8
    BGR (which may be given, e.g. a view of a staging buffer). focus_disp [N] fp32 is the frames' focal disparities; scale is
    a finite fp32 >= 0 and 0 <= max_radius <= 32. With scale 0 or max_radius 0 the frames come out as floor(255 clip(img))."""
    _chk(depth, 'depth')
    if depth.dim() != 3:
        raise ValueError('depth must be [N,H,W], got %s' % (tuple(depth.shape),))
    N, H, W = depth.shape
    _chk(img, 'img', (N, 3, H, W))
    _chk(focus_disp, 'focus_disp', (N,))
    if not 0 <= int(max_radius) <= _lib.DVD_REFOCUS_MAX_RADIUS or int(max_radius) != max_radius:
        raise ValueError('max_radius must be an integer in [0, %d], got %r' % (_lib.DVD_REFOCUS_MAX_RADIUS, max_radius))
    scale = float(scale)
    if not (scale >= 0 and scale < float('inf')):
        raise ValueError('scale must be finite and >= 0, got %r' % scale)
    if not 1 <= N <= 65535:
        raise ValueError('refocus takes 1 to 65535 frames per call, got %d' % N)
    if out is None:
        out = torch.empty(N, H, W, 3, dtype=torch.uint8, device=depth.device)
    _chk_dtype(out, 'out', torch.uint8, 4)
    if tuple(out.shape) != (N, H, W, 3) or not (out.device == img.device == focus_disp.device == depth.device):
        raise ValueError('out must be [%d,%d,%d,3], and every tensor on one device' % (N, H, W))
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_refocus(_ptr(depth), _ptr(img), _ptr(focus_disp), scale, int(max_radius), _ptr(out), N, H, W,
                                       _stream()), 'dvd_refocus')
    return out
