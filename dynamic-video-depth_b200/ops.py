"""Python face of the C ABI: argument checks, output allocation, autograd wiring.

PyTorch is plumbing here (device memory, streams, autograd graph); all arithmetic of the hot path
happens inside libdvd_b200.so. Argument / shape / dtype / contiguity violations raise ValueError
before any launch; a non-zero return from the library raises RuntimeError (SURVEY.md §8(b)).
"""
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
    for i, e in enumerate(range(n_eval - 1, -1, -1)):
        dy = dys[i % nbuf]
        if wdone[i % nbuf] is not None:
            main.wait_event(wdone[i % nbuf])
        a_out = torch.empty(B, 3, H, W, dtype=torch.float32, device=dev)
        gs = g_steps[e] if g_steps is not None else None
        save_e = ctypes.c_void_p(sv.data_ptr() + e * per)
        LAUNCHES['n'] += 1
        _lib.check(lib.dvd_mlp_dgrad(ctypes.byref(cfg), _ptr(packed.bwd), _ptr(p_steps[e]),
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
                _lib.check(lib.dvd_mlp_wgrad(ctypes.byref(cfg), save_e, _ptr(dy), gw_arr, gb_arr, npx, _stream()), 'dvd_mlp_wgrad')
                wdone[i % nbuf] = torch.cuda.Event()
                wdone[i % nbuf].record(side)
        else:
            _lib.check(lib.dvd_mlp_wgrad(ctypes.byref(cfg), save_e, _ptr(dy), gw_arr, gb_arr, npx, _stream()), 'dvd_mlp_wgrad')
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
        LAUNCHES['n'] += 1
        _lib.check(lib.dvd_bn_act_bwd(_ptr(g), _ptr(x), _ptr(y), _ptr(gamma), _ptr(mean), _ptr(var), ctx.eps, _ptr(gx), _ptr(gres),
                                      _ptr(gg), _ptr(gb), N * H * W, C, int(ctx.relu), _stream()), 'dvd_bn_act_bwd')
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
