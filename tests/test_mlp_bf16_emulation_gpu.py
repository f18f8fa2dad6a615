"""The scene-flow MLP kernels (csrc/sf_mlp_tc.cu) against an fp64 emulation of their own arithmetic (oracle/sf_mlp_bf16.py):
the reference's structure with the kernels' bf16 (hi, lo) split, rounding points and packed weight images. What is left between
the two is fp32 accumulation order, the fast_sincos residual of the embedding and the occasional one-step bf16 flip, so the
bounds below sit at least 30 times under what a dropped split product (bf16x2 instead of bf16x3) or a dropped
64-pixel chunk of the weight gradient changes. Each case asserts that margin (10x) at its own shape; the one-chunk margin
holds at the three smaller shapes, not at the bench resolution (see that test).

Driven through the raw ABI: ops.mlp_chain_fwd(save=True), then per eval dvd_mlp_dgrad / dvd_mlp_wgrad with this test's own dY
buffer, zeroed gradients and the kernel's own a_in, p_steps and mask bits (teacher forcing). Then the autograd path
(ops.scene_flow_chain) with the two-stream backward and with DVD_BWD_OVERLAP=0 against the sum of the per-eval results.

Shapes: 1x17x23 (ragged last tile), 1x27x33 (7 tiles: the weight gradient's split-K has empty ranges on an H100's 132 SMs),
1x128x192 (192 tiles: the chain kernels' persistent tile loop) and 2x224x384 (the bench resolution) for the default encoding.

Bounds: set at about 3x the largest value observed over all cases below, measured on an NVIDIA H100 80GB HBM3 with a 700 W
power limit; observed maxima in the comments. The whole module runs in about 15 s there."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

# forward, saved X_l hi planes against the emulation (each eval from the kernel's p_steps[e]): share of elements that differ,
# share more than one bf16 step off, and the error of those relative to the plane's maximum; observed 6.4e-3, 5.9e-4, 9.4e-6
X_DIFF, X_FAR, X_FAR_REL = 2e-2, 2e-3, 3e-5
# LeakyReLU mask bits: share that differ from the emulation's, and the largest |pre-activation| at a flip relative to the
# layer's maximum; observed 2.0e-5, 3.5e-6
MASK_FLIPS, MASK_BAND = 6e-5, 1e-5
# s_steps against the emulation (max-norm relative to the tensor's maximum); observed 2.2e-5
S_REL = 6e-5
# data gradient: dY_l hi planes (as X; observed 5.4e-3, 5.5e-4, 7.0e-6), a_out and g_bias5 (observed 1.4e-5, 1.3e-6)
DY_DIFF, DY_FAR, DY_FAR_REL = 1.6e-2, 1.6e-3, 2e-5
A_OUT_REL, GB5_REL = 4e-5, 4e-6
# weight gradient on the kernel's own operands: g_w[l], g_b[l] against fp64 sums of the same bf16 products (relative max-norm).
# What is left is the tensor cores' fp32 accumulation, which grows with the pixels one CTA sums: observed 6.5e-6 / 7.8e-7 at up
# to 24,576 pixels (at most 35 chunks of 64 pixels per CTA), 7.3e-5 / 1.3e-5 at 2 x 224 x 384 (245 chunks per CTA)
WGRAD_REL, GB_REL = 2e-5, 2.5e-6
WGRAD_REL_BENCH, GB_REL_BENCH = 2.2e-4, 4e-5
# the autograd path's weight gradients: two-stream vs one-stream vs the sum of the per-eval raw-ABI results (atomic order);
# observed 1.2e-6
ATOMIC_REL = 3.5e-6
# every bound is at least this far below what the defects change (bf16x2: 1.6e-3 of a_out, 2.6e-3 of s, 61 % of the saved
# planes; one chunk of dW / db: 1.4e-3 / 1.8e-3 at 1 x 128 x 192)
MARGIN = 10.0

N_EVAL, N_ACC, DT = 3, 2, 1.0 / 80
CONFIGS = {'16-16-T': (16, 16, True), '16-0-F': (16, 0, False), '8-4-T': (8, 4, True), '20-0-F': (20, 0, False),
           '30-0-F': (30, 0, False), '36-16-T': (36, 16, True), '0-0-T': (0, 0, True)}
KPAD0 = {'16-16-T': 144, '16-0-F': 112, '8-4-T': 64, '20-0-F': 128, '30-0-F': 192, '36-16-T': 256, '0-0-T': 64}
SHAPES = [(1, 17, 23), (1, 27, 33), (1, 128, 192)]


def make_case(name, B, H, W, seed=0):
    """CPU inputs: layers (kaiming weights, small random biases), p0 uniform in [-50, 50]^3, t0 uniform in [0, 1], a coherent
    cotangent of acc and white-noise cotangents of the steps"""
    from oracle import sf_mlp
    from oracle.sf_mlp_bf16 import n_in
    fx, ft, td = CONFIGS[name]
    g = torch.Generator().manual_seed(1000 * seed + H)
    layers = sf_mlp.init_layers(n_in=n_in(fx, ft, td), seed=seed)
    layers = [(w, torch.randn(b.shape, generator=g) * 0.05) for w, b in layers]
    p0 = (torch.rand(B, 3, H, W, generator=g) * 2 - 1) * 50
    t0 = torch.rand(B, 1, H, W, generator=g)
    g_acc = 1.0 + 0.3 * torch.nn.functional.interpolate(torch.randn(B, 3, 5, 7, generator=g), size=(H, W), mode='bilinear')
    g_steps = torch.randn(N_EVAL, B, 3, H, W, generator=g) * 0.3
    return layers, p0, t0, g_acc, g_steps


def _kw(name):
    fx, ft, td = CONFIGS[name]
    return dict(n_freq_xyz=fx, n_freq_t=ft, time_dependent=td)


class Worst:
    def __init__(self):
        self.v = {}

    def __call__(self, key, val):
        self.v[key] = max(self.v.get(key, 0.0), val)

    def low(self, key, val):
        self.v[key] = min(self.v.get(key, float('inf')), val)


def _check_pack(pk, ws, L):
    """decoded images == split2 of the zero-padded weights, bit for bit (so the padding is exactly zero)"""
    from oracle.sf_mlp_bf16 import LAYERS, bf16_bits, decode_image
    for l in range(LAYERS):
        for fwd in (True, False):
            hi, lo = decode_image(pk.fwd if fwd else pk.bwd, L, l, fwd)
            w = ws[l] if fwd else ws[l].t()
            full = torch.zeros(hi.shape, dtype=torch.float32, device=hi.device)
            full[:w.shape[0], :w.shape[1]] = w
            h32 = full.to(torch.bfloat16).float()
            assert torch.equal(hi, bf16_bits(h32)), (l, fwd)
            assert torch.equal(lo, bf16_bits(full - h32)), (l, fwd)
            pad = torch.ones_like(hi, dtype=torch.bool)
            pad[:w.shape[0], :w.shape[1]] = False
            assert not bool(((hi != 0) & pad).any()) and not bool(((lo != 0) & pad).any()), (l, fwd)


def _planes(wst, key, k_bits, emu):
    from oracle.sf_mlp_bf16 import plane_agreement
    d, f, fr = plane_agreement(k_bits, emu)
    wst(key + '_diff', d), wst(key + '_far', f), wst(key + '_far_rel', fr)


def _check_case(name, B, H, W, monkeypatch, bench=False):
    from dvd_b200 import _lib, ops
    from oracle import sf_mlp_bf16 as E
    kw = _kw(name)
    td = kw['time_dependent']
    npx, hw = B * H * W, H * W
    L = E.Layout(npx=npx, **kw)
    assert L.kpad0 == KPAD0[name]
    lib = _lib.load()
    cfg = ops.make_mlp_cfg(**kw)
    assert lib.dvd_mlp_save_bytes_per_eval(ctypes.byref(cfg), npx) == L.save_total
    assert lib.dvd_mlp_dy_bytes(ctypes.byref(cfg), npx) == L.dy_total
    layers, p0, t0, g_acc, g_steps = make_case(name, B, H, W)
    ws = [w.cuda().contiguous() for w, _ in layers]
    bs = [b.cuda().contiguous() for _, b in layers]
    p0, t0, g_acc, g_steps = p0.cuda(), t0.cuda(), g_acc.cuda(), g_steps.cuda()
    pk = ops.PackedMlp(cfg, 'cuda').refresh(ws, bs)
    torch.cuda.synchronize()
    _check_pack(pk, ws, L)
    net = E.Net.from_images(pk.fwd, pk.bwd, bs, L, kw)
    wst, teeth = Worst(), Worst()
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    # ---- forward chain
    f = ops.mlp_chain_fwd(pk, p0, t0 if td else None, DT, N_EVAL, N_ACC, save=True)
    torch.cuda.synchronize()
    ps, ss, sv = f['p_steps'], f['s_steps'], f['save']
    # the kernel's own Euler bookkeeping, exactly: p_0 = p0, p_{e+1} = p_e + s_e, acc = s_0 + s_1 (fp32)
    assert torch.equal(ps[0], p0)
    for e in range(N_EVAL - 1):
        assert torch.equal(ps[e + 1], ps[e] + ss[e]), e
    assert torch.equal(f['acc'], ss[0] + ss[1])
    saves = [sv[e * L.save_total:(e + 1) * L.save_total] for e in range(N_EVAL)]
    dt32 = float(torch.tensor(DT, dtype=torch.float32))
    t_e = E.to_px(t0.double()).view(-1) if td else None
    for e in range(N_EVAL):
        p_e = E.to_px(ps[e].double())
        em = E.forward_eval(net, p_e, t_e, terms=3)
        masks = E.decode_masks(saves[e], L)[:, :npx]
        for l in range(6):
            xk = E.decode_x(saves[e], L, l)[:npx]
            n = L.nin if l == 0 else E.WIDTH
            _planes(wst, 'x', xk[:, :n], em['x'][l][0])
            if l == 0:
                assert not bool((xk[:, n:] != 0).any())
            if l < 5:
                flip = masks[l] != em['mask'][l]
                y = em['y'][l]
                band = float((y.abs() * flip).max()) / float(y.abs().max()) if flip.any() else 0.0
                wst('mask_flips', float(flip.double().mean())), wst('mask_band', band)
        wst('s_rel', E.rel_max(E.to_px(ss[e]), em['s']))
        # teeth: bf16x2 in the forward
        e2 = E.forward_eval(net, p_e, t_e, terms=2)
        teeth.low('fwd_bf16x2_s', E.rel_max(e2['s'], em['s']))
        teeth.low('fwd_bf16x2_x', max(E.plane_agreement(E.bf16_bits(e2['x'][l][0]), em['x'][l][0])[0] for l in range(1, 6)))
        if td:
            t_e = E.f32(t_e + dt32)

    # ---- data gradient and weight gradient of each eval, raw ABI
    valid = torch.arange(L.nq * 64, device='cuda') < npx
    a_in = None
    raw_w = [torch.zeros_like(w) for w in ws]
    raw_b = [torch.zeros_like(b) for b in bs]
    a_out0 = None
    for e in range(N_EVAL - 1, -1, -1):
        dy = torch.full((L.dy_total,), 0x55, dtype=torch.uint8, device='cuda')   # every element must be written
        gb5 = torch.zeros(3, device='cuda')
        a_out = torch.empty_like(p0)
        use_acc = int(e < N_ACC)
        save_e = ctypes.c_void_p(saves[e].data_ptr())
        _lib.check(lib.dvd_mlp_dgrad(ctypes.byref(cfg), ops._ptr(pk.bwd), ops._ptr(ps[e]), ops._ptr(t0) if td else None, DT, e,
                                     use_acc, ops._ptr(g_acc), ops._ptr(g_steps[e]), ops._ptr(a_in), ops._ptr(a_out), save_e,
                                     ops._ptr(dy), ops._ptr(gb5), npx, hw, ops._stream()), 'dvd_mlp_dgrad')
        torch.cuda.synchronize()
        masks = [m[:npx] for m in E.decode_masks(saves[e], L)]
        args = dict(a_in=E.to_px(a_in.double()) if a_in is not None else None, g_acc=E.to_px(g_acc.double()) if use_acc else None,
                    g_step=E.to_px(g_steps[e].double()))
        p_e = E.to_px(ps[e].double())
        dm = E.dgrad_eval(net, p_e, masks, terms=3, **args)
        dyk = [E.decode_dy(dy, L, l) for l in range(6)]
        for l in range(6):
            n = 3 if l == 5 else E.WIDTH
            _planes(wst, 'dy', dyk[l][:npx, :n], dm['dy'][l][0])
            assert not bool((dyk[l][npx:] != 0).any()), ('pad-pixel dY', l)
            assert not bool((dyk[l][:, n:] != 0).any()), ('padding channels of dY', l)
        wst('a_out_rel', E.rel_max(E.to_px(a_out), dm['a_out']))
        wst('gb5_rel', E.rel_max(gb5, dm['gb5']))
        d2 = E.dgrad_eval(net, p_e, masks, terms=2, **args)
        teeth.low('dgrad_bf16x2_a_out', E.rel_max(d2['a_out'], dm['a_out']))
        teeth.low('dgrad_bf16x2_dy', max(E.plane_agreement(E.bf16_bits(d2['dy'][l][0]), dm['dy'][l][0])[0] for l in range(5)))

        # weight gradient on zeroed buffers, then a second launch on top
        gw = [torch.zeros_like(w) for w in ws]
        gb = [torch.zeros_like(b) for b in bs]
        for rep in (1, 2):
            _lib.check(lib.dvd_mlp_wgrad(ctypes.byref(cfg), save_e, ops._ptr(dy), ops._ptr_array(gw), ops._ptr_array(gb), npx,
                                         ops._stream()), 'dvd_mlp_wgrad')
            torch.cuda.synchronize()
            if rep == 1:
                w1 = [g.clone() for g in gw]
                b1 = [g.clone() for g in gb]
        xs = [E.bits_to_f64(E.decode_x(saves[e], L, l))[:, :L.layer_in(l)] for l in range(6)]
        dys = [E.bits_to_f64(dyk[l])[:, :L.layer_out(l)] for l in range(6)]
        ew, eb = E.wgrad(xs, dys)
        for l in range(6):
            wst('wgrad_rel', E.rel_max(w1[l], ew[l]))
            wst('wgrad_rel_x2', E.rel_max(gw[l], 2 * ew[l]))
            teeth.low('wgrad_chunk', E.chunk_effect(xs[l], dys[l], ew[l], valid))
            if l < 5:
                wst('gb_rel', E.rel_max(b1[l], eb[l]))
                wst('gb_rel_x2', E.rel_max(gb[l], 2 * eb[l]))
                teeth.low('gb_chunk', E.chunk_effect(torch.ones_like(xs[l][:, :1]), dys[l], eb[l].view(-1, 1), valid))
            else:
                assert float(gb[5].abs().max()) == 0.0       # the output bias gradient comes from the data gradient
        for l in range(6):
            raw_w[l] += w1[l]
            raw_b[l] += b1[l] if l < 5 else gb5
        a_in = a_out
        a_out0 = a_out
        del dy, dyk, xs, dys

    # ---- autograd path: two-stream and one-stream backward
    res = {}
    for mode in ('overlap', 'serial'):
        if mode == 'serial':
            monkeypatch.setenv('DVD_BWD_OVERLAP', '0')
        else:
            monkeypatch.delenv('DVD_BWD_OVERLAP', raising=False)
        p = p0.clone().requires_grad_()
        wr = [w.clone().requires_grad_() for w in ws]
        br = [b.clone().requires_grad_() for b in bs]
        acc, s = ops.scene_flow_chain(p, t0 if td else None, pk, DT, N_EVAL, N_ACC, wr, br)
        ((acc * g_acc).sum() + (s * g_steps).sum()).backward()
        torch.cuda.synchronize()
        res[mode] = (p.grad, [w.grad for w in wr], [b.grad for b in br])
    monkeypatch.delenv('DVD_BWD_OVERLAP', raising=False)
    assert torch.equal(res['overlap'][0], res['serial'][0])
    assert torch.equal(res['overlap'][0], a_out0)
    for l in range(6):
        for i, raw in ((1, raw_w), (2, raw_b)):
            wst('autograd_atomic', E.rel_max(res['overlap'][i][l], res['serial'][i][l]))
            wst('autograd_atomic', E.rel_max(res['overlap'][i][l], raw[l]))
            wst('autograd_atomic', E.rel_max(res['serial'][i][l], raw[l]))

    # ---- report and bounds
    ksplit = min(max(sms // 12, 1), L.nq)
    per = (L.nq + ksplit - 1) // ksplit
    info = 'tiles %d on %d SMs, wgrad split-K %d (%d empty)' % (L.ntiles, sms, ksplit, ksplit - (L.nq + per - 1) // per)
    print('\n[%s %dx%dx%d] %s\n  measured: %s\n  defects:  %s' % (
        name, B, H, W, info, ' '.join('%s=%.2e' % kv for kv in sorted(wst.v.items())),
        ' '.join('%s=%.2e' % kv for kv in sorted(teeth.v.items()))))
    v, t = wst.v, teeth.v
    wb, bb = (WGRAD_REL_BENCH, GB_REL_BENCH) if bench else (WGRAD_REL, GB_REL)
    bounds = [('x_diff', X_DIFF), ('x_far', X_FAR), ('x_far_rel', X_FAR_REL), ('mask_flips', MASK_FLIPS),
              ('mask_band', MASK_BAND), ('s_rel', S_REL), ('dy_diff', DY_DIFF), ('dy_far', DY_FAR), ('dy_far_rel', DY_FAR_REL),
              ('a_out_rel', A_OUT_REL), ('gb5_rel', GB5_REL), ('wgrad_rel', wb), ('wgrad_rel_x2', wb), ('gb_rel', bb),
              ('gb_rel_x2', bb), ('autograd_atomic', ATOMIC_REL)]
    bad = [(k, v[k], b) for k, b in bounds if v[k] > b]
    assert not bad, bad
    # each bound is MARGIN below the effect of a dropped split product or a dropped chunk at this shape
    margins = [('fwd_bf16x2_s', S_REL), ('fwd_bf16x2_x', X_DIFF), ('dgrad_bf16x2_a_out', A_OUT_REL), ('dgrad_bf16x2_dy', DY_DIFF)]
    if not bench:
        margins += [('wgrad_chunk', WGRAD_REL), ('gb_chunk', GB_REL)]
    bad = [(k, t[k], b) for k, b in margins if t[k] < MARGIN * b]
    assert not bad, bad
    return L, sms


@pytest.mark.parametrize('shape', SHAPES, ids=['%dx%dx%d' % s for s in SHAPES])
@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_kernels_match_bf16_emulation(name, shape, monkeypatch):
    L, sms = _check_case(name, *shape, monkeypatch)
    if shape == (1, 27, 33):
        ksplit = min(max(sms // 12, 1), L.nq)
        per = (L.nq + ksplit - 1) // ksplit
        assert ksplit * per > L.nq and (ksplit - 1) * per >= L.nq, 'the shape must give empty weight-gradient splits'
    if shape == (1, 128, 192):
        assert L.ntiles > sms, 'the shape must make the chain kernels loop over tiles'


@pytest.mark.timeout(900)
def test_kernels_match_bf16_emulation_at_bench_resolution(monkeypatch):
    """The bench resolution: 1,344 tiles, 245 pixel chunks per weight-gradient CTA. One chunk of 2,688 is 2.1e-4 of dW here,
    within 3x of the fp32 accumulation noise of those long sums, so this case bounds dW / db by WGRAD_REL_BENCH / GB_REL_BENCH
    and leaves the one-chunk margin to the smaller shapes, which run the same split-K and stage-ring code."""
    _check_case('16-16-T', 2, 224, 384, monkeypatch, bench=True)


def test_acc_reg_at_bench_size():
    """dvd_acc_reg on more elements than its 1024 x 256 first-pass threads (grid-stride loop), a ragged count and exact ties:
    the value against fp64, the gradients exactly +-c (c = fp32(fp32(acc_mul / fp32(numel + 1e-6)) * gscale)) or 0 on ties"""
    from dvd_b200 import ops
    n = 8 * 3 * 224 * 384 + 77
    g = torch.Generator().manual_seed(5)
    s0 = torch.randn(n, generator=g) * 0.05
    s1 = s0 + torch.randn(n, generator=g) * 0.01
    tie = torch.rand(n, generator=g) < 0.05
    s1[tie] = s0[tie]
    acc_mul, gscale = 0.7, 3.0
    val, g0, g1 = ops.acc_reg(s0.cuda(), s1.cuda(), acc_mul, gscale)
    torch.cuda.synchronize()
    ref = acc_mul * float((s1.double() - s0.double()).abs().sum()) / (n + 1e-6)
    assert abs(val.item() - ref) <= 2e-6 * ref, (val.item(), ref)
    f = lambda x: torch.tensor(x, dtype=torch.float32)
    inv = f(1.0) / (f(float(n)) + f(1e-6))
    c = (f(acc_mul) * inv) * f(gscale)
    sgn = torch.sign(s1 - s0)
    assert int((sgn == 0).sum()) >= int(tie.sum())
    assert torch.equal(g1.cpu(), sgn * c)
    assert torch.equal(g0.cpu(), -sgn * c)
