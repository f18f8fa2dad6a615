"""The re-projection kernels (csrc/reproject.cu) against the bit-faithful fp32 emulation of their own arithmetic
(oracle/reproject_fp32.py), pixel by pixel.

Every per-pixel value is compared bit for bit (int32 views): g_sf of the loss backward, the nine materialised tensors and
unproject_fwd / unproject_bwd at VEC = 4, 2 and 1. The emulation's rcp.approx.ftz.f32 is the hardware instruction itself,
compiled at test time by NVRTC through torch's jiterator. Reductions are checked against bounds computed from the launch
geometry, not from observed errors:

* the mask count N (scalars[4]) is exact: fp32 sums of 0 / 1 below 2^24 do not round;
* scalars[0..2]·N lies within γ_n·Σ|terms| of the fp64 sum of the emulated fp32 terms, n = grid-stride iterations per
  thread + pixel slots + 5 shuffle levels + 8 warp partials + 1, + 2 for the finalising division;
* cf, cd are exact given N; the loss is within 1.5 ulp of flow_mul·fl + disp_mul·second (two rounded products and a
  rounded sum, or one of them contracted);
* g_depth_2 is exactly zero where no pixel contributes, and within k·2^-24·Σ|contributions| of the fp64 sum of the
  emulated contributions elsewhere (k = the element's contribution count);
* single-pixel probes (a one-pixel mask, N = 1) make every sum one term: the scalars equal the emulated terms and g_depth_2
  equals the four emulated tap gradients bit for bit, at the first and last pixel, every i00 % 4 residue, a right-clamped
  column, a bottom-clamped row, the ragged last tile and pairs 63 / 64 / 65 across pose chunks, on both paths.

The materialise adjoint is written with plain * and + that nvcc may contract, so it is held to MAT_BWD_ULPS · 2^-24 of
each tensor's maximum instead (observed at most 21 on an NVIDIA H100 80GB HBM3 with a 700 W power limit, for g_depth_1 at
4x224x384). Which kernel ran is asserted from torch.profiler kernel names; the staged / VEC-4 size threshold is
num_sms·2048 pixels. The module runs in about two minutes on that H100, most of it in the numpy emulation.
"""
import math
import warnings

import numpy as np
import pytest
import torch

from oracle import reproject_fp32 as R

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
# materialise adjoint (plain * and + that nvcc may contract) against the emulation, in units of 2^-24 of each tensor's maximum
MAT_BWD_ULPS = 64
GSCALE, GSCALE_DEV = 0.75, 1.25
# cfg subsets: all 24 raw configurations at the generic shapes and at the bench resolution; at the other staged shapes the
# scene-flow term (the only one that gives the ne tap a gradient of its own), both disparity terms of the reference, and
# the three ABI-only combinations
SUBSET = [R.cfg_dict(1, 0, 2, 0), R.cfg_dict(1, 0, 0, 1), R.cfg_dict(0, 1, 1, 0), R.cfg_dict(1, 1, 1, 1),
          R.cfg_dict(0, 0, 2, 1), R.cfg_dict(0, 1, 0, 0)]


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.fixture(scope='module')
def emu():
    """Fp32 emulation whose rcp is the hardware rcp.approx.ftz.f32 (NVRTC-compiled inline PTX)."""
    code = ('template <typename T> T dvd_rcp_approx_ftz(T x) { float r; '
            'asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"((float)x)); return r; }')
    fn = torch.cuda.jiterator._create_jit_fn(code)

    def rcp(x):
        x = np.ascontiguousarray(x, dtype=np.float32)
        return fn(torch.from_numpy(x).cuda()).cpu().numpy().astype(np.float32)
    v = np.array([3.0, 1e-3, 7.25, 1e8], np.float32)
    assert np.all(np.abs(rcp(v).astype(np.float64) * v - 1) <= 2.0 ** -22)
    return R.Fp32(rcp=rcp)


def _bits_equal(gpu, ref):
    a = np.ascontiguousarray(gpu.detach().cpu().numpy(), dtype=np.float32).view(np.int32)
    b = np.ascontiguousarray(np.broadcast_to(ref, a.shape), dtype=np.float32).view(np.int32)
    return int((a != b).sum())


def _misaligned(t):
    """contiguous copy whose data pointer sits 4 bytes past a 16-byte boundary"""
    buf = torch.empty(t.numel() + 4, dtype=t.dtype, device=t.device)
    out = buf[1:1 + t.numel()].view(t.shape)
    out.copy_(t)
    return out


def _kernels(fn, *expected):
    """fn() under torch.profiler → (result, the names of every event), asserting that kernels whose names contain each
    of `expected` ran. The profiler's device records are not always delivered: the first kernels of a session can be
    missing, and now and then a whole session has none. So fn runs twice between runs of small padding kernels, and a
    session without the expected records is repeated (up to five times). A session that recorded device kernels (the
    padding) but not the expected ones is a failure only once every retry agrees; a different kernel can never produce
    the expected names. If no session delivered any device record, the kernel identity is unobservable in this process
    and a warning says so (the numerical checks of the caller still run)."""
    pad = torch.zeros(1, device='cuda')
    seen_device = False
    for _ in range(5):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                                torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _i in range(32):
                pad.add_(1)
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
            out = fn()
            torch.cuda.synchronize()
            for _i in range(128):
                pad.add_(1)
            torch.cuda.synchronize()
        device = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        names = ' | '.join(device)
        seen_device = seen_device or bool(device)
        if all(e in names for e in expected):
            return out, names
    if seen_device:
        raise AssertionError(('kernels not seen', expected, names))
    warnings.warn('torch.profiler delivered no device records in 5 sessions: kernel identity %s not checked' % (expected,))
    return out, names


def _loss_cfg(cfg):
    from dvd_b200 import _lib
    return _lib.LossCfg(cfg['midas'], cfg['warm'], cfg['disp_mode'], cfg['second_is_disp'], cfg['flow_mul'], cfg['disp_mul'])


def _staged(B, H, W):
    return W % 4 == 0 and B * H * W >= 2048 * _sms()


def _reduction_depth(B, H, W, staged):
    """rounded additions on the way of one term into scalars[0..2] (see the module docstring)"""
    HW, sms = H * W, _sms()
    if staged:
        tpp, iters = math.ceil(HW / 512), 0
        for b0 in range(0, B, 64):
            nb = min(B - b0, 64)
            iters = max(iters, math.ceil(nb * tpp / min(nb * tpp, 3 * sms)))
        slots = 2
    else:
        slots = 2 if W % 2 == 0 else 1
        items = HW // slots
        per_pair = max(1, min(math.ceil(items / 256), math.ceil(sms * 8 / B)))
        iters = math.ceil(items / (per_pair * 256))
    return iters + slots + 5 + 8 + 1 + 2


def _gamma(n):
    return n * U / (1 - n * U)


class Case:
    """Inputs of one shape on the CPU and the GPU, and the emulated forward chain (mask- and cfg-independent)."""

    def __init__(self, A, B, H, W, seed, sigma):
        self.A, self.B, self.H, self.W = A, B, H, W
        self.inp = R.edge_inputs(B, H, W, seed=seed, sigma=sigma)
        self.np = {k: self.inp[k][:, 0].numpy() if k in ('d1', 'd2') else self.inp[k].numpy()
                   for k in ('d1', 'd2', 'flow', 'mask', 'sf', 'poses')}
        self.refresh()

    def refresh(self):
        """re-run the emulated forward after the CPU inputs changed"""
        A = self.A
        self.ps = R.derive_pose(A, self.np['poses'])
        self.o = R.pixel_forward(A, self.ps, self.np['d2'], self.np['flow'], self.np['d1'], self.np['sf'])
        c = lambda t: t.cuda().contiguous()  # noqa: E731
        self.g = [c(self.inp['d1']), c(self.inp['d2']), c(self.inp['flow']), c(self.inp['mask']), c(self.inp['sf']),
                  c(self.inp['poses'])]

    def misaligned(self):
        return [_misaligned(t) for t in self.g[:5]] + [self.g[5]]


def _check_loss(case, cfg, ins, staged):
    """One full-mask forward + backward through the raw ABI against the emulation."""
    from dvd_b200 import ops
    A, o, B, H, W = case.A, case.o, case.B, case.H, case.W
    lc = _loss_cfg(cfg)
    s_t = ops.reproject_loss_fwd(*ins, lc)
    gdev = torch.tensor([GSCALE_DEV], device='cuda')
    g_sf, g_d2 = ops.reproject_loss_bwd(*ins, lc, s_t, gscale=GSCALE, gscale_dev=gdev)
    s = s_t.cpu().numpy()
    f = R.loss_forward(A, cfg, case.ps, None, None, None, case.np['mask'], None, o=o)
    N = f['scalars']['masksum']
    assert float(s[4]) == N, ('mask count', float(s[4]), N)
    nf = np.float32(np.float32(N) + np.float32(1e-8))
    n = _reduction_depth(B, H, W, staged)
    for k in range(3):
        t = f['terms'][k].astype(np.float64)
        assert abs(float(s[k]) * float(nf) - t.sum()) <= _gamma(n) * np.abs(t).sum(), ('sum', k, cfg)
    assert s[5] == np.float32(np.float32(cfg['flow_mul']) / nf) and s[6] == np.float32(np.float32(cfg['disp_mul']) / nf)
    second = s[1] if cfg['second_is_disp'] else s[2]
    exact = float(np.float32(cfg['flow_mul'])) * float(s[0]) + float(np.float32(cfg['disp_mul'])) * float(second)
    assert abs(float(s[3]) - exact) <= 1.5 * float(np.spacing(np.float32(exact))), ('loss', float(s[3]), exact)
    # backward, teacher-forced with the kernel's own cf / cd and the kernel's gscale product
    gs = np.float32(np.float32(GSCALE) * np.float32(GSCALE_DEV))
    cf, cd = np.float32(s[5] * gs), np.float32(s[6] * gs)
    gv, h = R.pixel_backward(A, cfg, case.ps, o, f['m'], cf, cd)
    want = np.stack(gv, 1)
    got = g_sf.detach().cpu().numpy()
    bad = np.argwhere(got.view(np.int32) != want.view(np.int32))
    if len(bad):
        info = [(tuple(int(v) for v in i), float(got[tuple(i)]), float(want[tuple(i)]),
                 {k: float(o[k][i[0], i[2], i[3]]) for k in ('rz', 'ex', 'ey', 'x0f', 'y0f')},
                 float(o['p12'][2][i[0], i[2], i[3]]), float(o['wpc'][2][i[0], i[2], i[3]]),
                 float(f['m'][i[0], i[2], i[3]])) for i in bad[:6]]
        raise AssertionError(('g_sf bits', len(bad), cfg, info))
    tot, ab, cnt = R.scatter(o, R.tap_grads(A, o, *h), B, H * W)
    gd = g_d2.detach().cpu().numpy().reshape(B, H * W).astype(np.float64)
    assert (gd[cnt == 0] == 0).all(), ('g_d2 non-zero pattern', cfg)
    excess = np.abs(gd - tot) - cnt * U * ab
    assert (excess <= 0).all(), ('g_d2 bound', float(excess.max()), cfg)


# ---------------------------------------------------------------------------------------------------------------------
# full masks

FULL = [((1, 17, 23), 3.0, 'all'), ((3, 30, 50), 14.0, 'all'), ((4, 224, 384), 3.0, 'all'), ((5, 203, 384), 60.0, 'subset'),
        ((65, 96, 128), 14.0, 'subset'), ((200, 48, 64), 3.0, 'subset')]


@pytest.mark.parametrize('shape,sigma,cfgs', FULL, ids=lambda v: 'x'.join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_loss_full_mask_against_emulation(emu, shape, sigma, cfgs):
    """(1,17,23): generic, one pixel per thread; (3,30,50): generic, a pixel pair; (4,224,384) and (5,203,384): staged,
    the latter with a ragged last tile; (65,96,128) and (200,48,64): two and four 64-pair pose chunks, so a constant-bank
    slot is reused within one call. The staged inputs also run through 4-byte-misaligned copies (generic path)."""
    from dvd_b200 import ops
    B, H, W = shape
    case = Case(emu, B, H, W, seed=B + H, sigma=sigma)
    staged = _staged(B, H, W)
    cfg_list = R.all_cfgs(flow_mul=1.0, disp_mul=0.7) if cfgs == 'all' else SUBSET
    paths = [(case.g, staged)] + ([(case.misaligned(), False)] if staged else [])
    for ins, st in paths:
        expected = (('reproject_loss_fwd_staged_kernel', 'reproject_loss_bwd_staged_kernel') if st else
                    ('reproject_loss_fwd_kernel<%d>' % (2 if W % 2 == 0 else 1), 'reproject_loss_bwd_kernel'))
        _, names = _kernels(lambda: ops.reproject_loss_bwd(*ins, _loss_cfg(cfg_list[0]),
                                                           ops.reproject_loss_fwd(*ins, _loss_cfg(cfg_list[0]))), *expected)
        assert st or 'staged' not in names
        for cfg in cfg_list:
            _check_loss(case, cfg, ins, st)


# ---------------------------------------------------------------------------------------------------------------------
# single-pixel probes

PROBE_SHAPES = [(4, 224, 384), (5, 203, 384), (65, 96, 128), (200, 48, 64)]
PROBE_CFGS = [R.cfg_dict(0, 0, 2, 0, 1.0, 0.7), R.cfg_dict(0, 1, 1, 1, 1.0, 0.7)]


def _probes(B, H, W):
    """(b, y, x, target qx, target qy): the flow of pixel (b, y, x) is set so that it samples at (qx, qy)"""
    HW = H * W
    last = HW - 1
    out = [(0, 0, 0, 3.5, 2.25), (B - 1, last // W, last % W, W - 7.75, H - 3.5)]
    out += [(min(1, B - 1), H // 2, 3 + r, 8 + r + 0.375, H // 2 + 0.625) for r in range(4)]   # i00 % 4 = 0..3
    out += [(0, 5, 9, W + 5.0, 7.25), (B - 1, 7, 11, 13.75, H + 5.0)]                          # right / bottom clamp
    p = (HW // 512) * 512 + 37 if HW % 512 else HW - 300                                      # ragged (or last) tile
    out.append((B - 1, p // W, p % W, 21.25, 4.5))
    out += [(b, 3, 5 + 2 * (b % 3), 30.125, 6.875) for b in (63, 64, 65) if b < B]
    return out


@pytest.mark.parametrize('shape', PROBE_SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_single_pixel_probes(emu, shape):
    from dvd_b200 import ops
    B, H, W = shape
    assert _staged(B, H, W)
    case = Case(emu, B, H, W, seed=7 + B, sigma=3.0)
    probes = _probes(B, H, W)
    for (b, y, x, qx, qy) in probes:
        case.inp['flow'][b, y, x, 0] = qx - x
        case.inp['flow'][b, y, x, 1] = qy - y
        case.inp['sf'][b, :, y, x] = 0.01
    case.np['flow'], case.np['sf'] = case.inp['flow'].numpy(), case.inp['sf'].numpy()
    case.refresh()
    A, o = emu, case.o
    assert (o['i00'][[p[0] for p in probes[2:6]], [p[1] for p in probes[2:6]], [p[2] for p in probes[2:6]]] % 4 ==
            np.arange(4)).all()
    assert o['sx1'][probes[6][0], probes[6][1], probes[6][2]] == 0 and o['sy1'][probes[7][0], probes[7][1], probes[7][2]] == 0
    idx = R.tap_index(o)
    for cfg in PROBE_CFGS:
        lc = _loss_cfg(cfg)
        fl, dl, sl = R.loss_terms(A, cfg, o)
        ones = A.f(np.ones_like(o['d1']))
        nf = np.float32(np.float32(1.0) + np.float32(1e-8))
        gv, h = R.pixel_backward(A, cfg, case.ps, o, ones, np.float32(cfg['flow_mul']) / nf,
                                 np.float32(cfg['disp_mul']) / nf)
        taps = R.tap_grads(A, o, *h)
        for path in ('staged', 'generic'):
            for i, (b, y, x, _, _) in enumerate(probes):
                mask = torch.zeros(B, H, W, device='cuda')
                mask[b, y, x] = 1.0
                ins = case.g[:3] + [mask] + case.g[4:]
                if path == 'generic':
                    ins = [_misaligned(t) for t in ins[:5]] + [ins[5]]

                def run():
                    s = ops.reproject_loss_fwd(*ins, lc)
                    return s, ops.reproject_loss_bwd(*ins, lc, s)[1]
                if i == 0:
                    (s, g_d2), names = _kernels(run, 'reproject_loss_fwd_staged_kernel' if path == 'staged' else
                                                'reproject_loss_fwd_kernel<2>')
                    assert path == 'staged' or 'staged' not in names
                else:
                    s, g_d2 = run()
                s = s.cpu().numpy()
                where = (path, cfg['disp_mode'], (b, y, x))
                assert s[4] == 1.0, where
                for k, t in enumerate((fl, dl, sl)):
                    assert s[k].view(np.int32) == np.float32(t[b, y, x]).view(np.int32), (where, k, s[k], t[b, y, x])
                want = torch.zeros(B, H * W, dtype=torch.float32)
                for k in range(4):
                    g = np.float32(taps[k][b, y, x])
                    if g != 0:
                        want[b, int(idx[k][b, y, x])] += float(g)
                got = g_d2.reshape(B, H * W).cpu()
                assert torch.equal(got, want), (where, (got != want).nonzero()[:8].tolist())
                nz = want != 0
                assert torch.equal(got[nz].view(torch.int32), want[nz].view(torch.int32)), where


# ---------------------------------------------------------------------------------------------------------------------
# materialise and un-project

@pytest.mark.parametrize('shape', [(1, 17, 23), (3, 30, 50), (4, 224, 384)], ids=lambda s: 'x'.join(map(str, s)))
def test_materialize_bitwise_and_adjoint(emu, shape):
    from dvd_b200 import ops
    B, H, W = shape
    case = Case(emu, B, H, W, seed=3 + H, sigma=14.0)
    d1, d2, flow, _, sf, poses = case.g
    out, _ = _kernels(lambda: ops.reproject_materialize(d1, d2, flow, sf, poses), 'reproject_materialize_kernel')
    ref = R.materialize(emu, case.ps, case.np['d1'], case.np['d2'], case.np['flow'], case.np['sf'])
    for k, v in ref.items():
        assert _bits_equal(out[k], v) == 0, k
    gen = torch.Generator().manual_seed(11)
    G = {k: torch.randn(v.shape, generator=gen) for k, v in ref.items()}
    d1g, d2g, sfg = (t.clone().requires_grad_() for t in (d1, d2, sf))
    mine = ops.reproject_tensors(d1g, d2g, sfg, flow, poses)
    total = sum((mine[k] * G[k].cuda()).sum() for k in ref)
    grads, _ = _kernels(lambda: torch.autograd.grad(total, [d1g, d2g, sfg], retain_graph=True),
                        'reproject_materialize_bwd_kernel')
    g_d1, g_d2, g_sf = R.materialize_bwd(emu, case.ps, case.np['d1'], case.np['d2'], case.np['flow'], case.np['sf'],
                                         {k: v.numpy() for k, v in G.items()})
    for got, want, name in ((grads[0][:, 0], g_d1, 'g_d1'), (grads[1][:, 0], g_d2, 'g_d2'), (grads[2], g_sf, 'g_sf')):
        got = got.detach().cpu().numpy().astype(np.float64)
        want = np.asarray(want, np.float64)
        # in ulps of the tensor's maximum: g_d1 = -<gP, ray> cancels, so per-element ulps are not a usable scale
        worst = float(np.abs(got - want).max() / np.abs(want).max()) / U
        print('materialize_bwd %s %s: %.2f ulp of max' % (shape, name, worst))
        assert worst <= MAT_BWD_ULPS, (name, worst)


def _unproject_shapes():
    sms = _sms()
    return {4: (4, 224, 384), 2: (3, math.ceil(512 * sms / (3 * 202)) + 1, 202), 1: (1, 17, 23)}


@pytest.mark.parametrize('vec', [4, 2, 1])
def test_unproject_bitwise(emu, vec):
    from dvd_b200 import ops
    B, H, W = _unproject_shapes()[vec]
    case = Case(emu, B, H, W, seed=vec, sigma=3.0)
    d1, poses = case.g[0], case.g[5]
    gP = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(vec))
    for which in (1, 2):
        P, _ = _kernels(lambda: ops.unproject_fwd(d1, poses, which), 'unproject_fwd_kernel<%d>' % vec)
        assert _bits_equal(P, R.unproject_fwd(emu, case.np['d1'], case.np['poses'], which)) == 0
        gd, _ = _kernels(lambda: ops.unproject_bwd(gP.cuda(), poses, which), 'unproject_bwd_kernel<%d>' % vec)
        assert _bits_equal(gd[:, 0], R.unproject_bwd(emu, gP.numpy(), case.np['poses'], which)) == 0


# ---------------------------------------------------------------------------------------------------------------------
# constant-bank pose slots

def _fwd_bwd(ins, lc):
    from dvd_b200 import ops
    s = ops.reproject_loss_fwd(*ins, lc)
    g_sf, g_d2 = ops.reproject_loss_bwd(*ins, lc, s)
    return s, g_sf, g_d2


def test_pose_slots_with_calls_in_flight_on_four_streams(emu):
    """Four streams, each with its own staged batch of 130 pairs (three pose chunks), enqueued back to back without a host
    synchronisation: each stream's scalars and g_sf are bitwise those of the same call run alone."""
    B, H, W = 130, 48, 64
    assert _staged(B, H, W)
    lc = _loss_cfg(R.cfg_dict(1, 0, 2, 0))
    cases = [Case(emu, B, H, W, seed=100 + i, sigma=3.0 + 4 * i) for i in range(4)]
    alone = []
    for c in cases:
        s, g_sf, _ = _fwd_bwd(c.g, lc)
        torch.cuda.synchronize()
        alone.append((s.clone(), g_sf.clone()))
    streams = [torch.cuda.Stream() for _ in cases]
    torch.cuda.synchronize()
    outs = []
    for c, st in zip(cases, streams):
        with torch.cuda.stream(st):
            outs.append(_fwd_bwd(c.g, lc))
    torch.cuda.synchronize()
    for (s, g_sf, _), (s0, g0) in zip(outs, alone):
        assert torch.equal(s.view(torch.int32), s0.view(torch.int32))
        assert torch.equal(g_sf.view(torch.int32), g0.view(torch.int32))


def test_pose_slots_under_graph_replay(emu):
    """One CUDA graph of forward + backward at B = 70 (two pose chunks). Replay it, overwrite the poses in place, run one
    eager call on the same stream, and replay again: each replay is bitwise equal to eager calls with the poses current at
    that replay."""
    B, H = 70, 64
    W = 4 * math.ceil(2048 * _sms() / (B * H * 4))
    assert _staged(B, H, W)
    lc = _loss_cfg(R.cfg_dict(1, 1, 0, 1))
    case = Case(emu, B, H, W, seed=70, sigma=5.0)
    poses0 = case.g[5].clone()
    poses1 = torch.roll(poses0, 1, 0)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for _ in range(2):
            _fwd_bwd(case.g, lc)
    torch.cuda.current_stream().wait_stream(st)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode='thread_local'):
        static = _fwd_bwd(case.g, lc)
    replays = []
    g.replay()
    replays.append([t.clone() for t in static])
    case.g[5].copy_(poses1)
    eager_mid = [t.clone() for t in _fwd_bwd(case.g, lc)]
    g.replay()
    replays.append([t.clone() for t in static])
    torch.cuda.synchronize()
    for rep, poses in zip(replays, (poses0, poses1)):
        ins = case.g[:5] + [poses]
        want = _fwd_bwd(ins, lc)
        torch.cuda.synchronize()
        for a, b in zip(rep[:2], want[:2]):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        assert torch.equal(rep[2], want[2]) or float((rep[2] - want[2]).abs().max()) <= 1e-6 * float(want[2].abs().max())
    assert torch.equal(eager_mid[1].view(torch.int32), replays[1][1].view(torch.int32))
    assert not torch.equal(replays[0][1], replays[1][1])
