"""The bf16 emulation of the scene-flow MLP kernels (oracle/sf_mlp_bf16.py), on the CPU: with rounding off it is
oracle.sf_mlp.sf_multi_step + autograd in fp64, so it cannot inherit a wiring error of the kernels it checks
(tests/test_mlp_bf16_emulation_gpu.py); its split2 is round-to-nearest-even; its layout decoders invert an element-by-element
encoder written from the C formulas and size the buffers as the library does; and the defects the GPU bounds must see (a
dropped split product, a dropped 64-pixel chunk of the weight gradient) change the result by at least 10x those bounds."""
import ctypes
import struct

import pytest
import torch

from conftest import rel_err
from test_mlp_bf16_emulation_gpu import (A_OUT_REL, CONFIGS, DY_DIFF, GB_REL, KPAD0, MARGIN, N_ACC, N_EVAL, S_REL, WGRAD_REL,
                                         X_DIFF, make_case)


def _kw(name):
    fx, ft, td = CONFIGS[name]
    return dict(n_freq_xyz=fx, n_freq_t=ft, time_dependent=td)


@pytest.mark.parametrize('name', ['16-16-T', '16-0-F', '8-4-T', '20-0-F'])
def test_unrounded_emulation_is_the_reference_structure(name):
    """value, dL/dp, every dW and db of a 3-eval chain (2 accumulated, cotangents on acc and on every step) to 1e-12"""
    from oracle import sf_mlp
    from oracle import sf_mlp_bf16 as E
    kw = _kw(name)
    B, H, W = 1, 9, 11
    layers, p0, t0, g_acc, g_steps = make_case(name, B, H, W, seed=3)
    layers = [(w.double(), b.double()) for w, b in layers]
    p0, t0, g_acc, g_steps = p0.double(), t0.double(), g_acc.double(), g_steps.double()
    dt = 1.0 / 80
    # reference: the reference's per-step field + torch autograd
    lw = [(w.clone().requires_grad_(), b.clone().requires_grad_()) for w, b in layers]
    p = p0.clone().requires_grad_()
    pp, tt, acc, loss = p, t0, 0.0, 0.0
    for e in range(N_EVAL):
        s = sf_mlp.sf_net(pp, tt, lw, sf_mag_div=100.0, **kw)
        loss = loss + (s * g_steps[e]).sum()
        if e < N_ACC:
            acc = acc + s
        pp, tt = pp + s, tt + dt
    (loss + (acc * g_acc).sum()).backward()
    # emulation without rounding
    net = E.Net.from_weights(layers, kw, rounding=False)
    r = E.chain(net, E.to_px(p0), E.to_px(t0).view(-1) if kw['time_dependent'] else None, dt, N_EVAL, N_ACC, E.to_px(g_acc),
                [E.to_px(g) for g in g_steps])
    assert rel_err(E.from_px(r['acc'], B, H, W), acc) < 1e-12
    assert rel_err(E.from_px(r['g_p'], B, H, W), p.grad) < 1e-12
    for l in range(6):
        assert float(lw[l][0].grad.abs().max()) > 0
        assert rel_err(r['g_w'][l], lw[l][0].grad) < 1e-12, ('dW', l)
        assert rel_err(r['g_b'][l], lw[l][1].grad) < 1e-12, ('db', l)


def test_split2_is_round_to_nearest_even():
    from oracle.sf_mlp_bf16 import split2
    u = 2.0 ** -7                   # bf16 spacing on [1, 2)
    x = torch.tensor([1 + u / 2, 1 + 3 * u / 2, -(1 + u / 2), 1 + u / 2 + 2 ** -20, 1 + 2 ** -9 + 2 ** -17,
                      1 + 2 ** -9 + 3 * 2 ** -17, 0.0], dtype=torch.float64)
    hi, lo = split2(x)
    assert hi.tolist() == [1.0, 1 + 2 * u, -1.0, 1 + u, 1.0, 1.0, 0.0]
    # the remainder is rounded to nearest even as well: 2^-9 + 2^-17 is a tie between 2^-9 and 2^-9 + 2^-16, and
    # -2^-8 + 2^-20 is nearer to -2^-8 than to the next bf16 value -2^-8 + 2^-16
    assert lo.tolist() == [u / 2, -u / 2, -u / 2, -u / 2, 2 ** -9, 2 ** -9 + 2 ** -15, 0.0]
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(100000, generator=g) * torch.exp(torch.randn(100000, generator=g) * 8)).float().double()
    hi, lo = split2(x)
    assert bool(((x - hi - lo).abs() <= 2.0 ** -17 * x.abs()).all())
    assert bool((hi.float().to(torch.bfloat16).double() == hi).all() and (lo.float().to(torch.bfloat16).double() == lo).all())


# ---- layouts ----------------------------------------------------------------------------------------------------------------
def _c_sw128(row, k):
    return (row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 3) ^ row) & 7) << 4) + (k & 7) * 2


def _c_mn128(mn, k):
    return (mn >> 6) * 8192 + (k >> 3) * 1024 + (k & 7) * 128 + (((((mn & 63) >> 3) ^ k) & 7) << 4) + (mn & 7) * 2


def test_layout_round_trip():
    """random bit patterns scattered element by element with the C formulas (pack_weights_kernel, the forward / data-gradient
    epilogues' act_offset and mask words) come back out of the vectorised decoders"""
    from oracle import sf_mlp_bf16 as E
    g = torch.Generator().manual_seed(1)
    for name, npx in (('16-16-T', 130), ('30-0-F', 200)):
        L = E.Layout(npx=npx, **_kw(name))
        # weight images
        for fwd in (True, False):
            buf = bytearray(L.wf_total if fwd else L.wb_total)
            for l in range(6):
                rows = L.rows_f(l) if fwd else L.rows_b(l)
                nkc = L.nkc_f(l) if fwd else L.nkc_b(l)
                base = L.wf_off[l] if fwd else L.wb_off[l]
                vals = torch.randint(-32768, 32768, (2, rows, nkc * 64), generator=g, dtype=torch.int16)
                vl = vals.tolist()
                for kc in range(nkc):
                    blk = base + kc * 2 * rows * 128
                    for row in range(rows):
                        for k in range(64):
                            off = blk + _c_sw128(row, k)
                            struct.pack_into('<h', buf, off, vl[0][row][kc * 64 + k])
                            struct.pack_into('<h', buf, off + rows * 128, vl[1][row][kc * 64 + k])
                hi, lo = E.decode_image(torch.frombuffer(buf, dtype=torch.uint8), L, l, fwd)
                assert torch.equal(hi, vals[0]) and torch.equal(lo, vals[1]), (name, fwd, l)
        # saved activations + masks, dY
        save, dy = bytearray(L.save_total), bytearray(L.dy_total)
        xs, dys = [], []
        for l in range(6):
            for which, buf, rows, off, out in ((0, save, L.rows_x(l), L.xs_off[l], xs), (1, dy, L.rows_dy(l), L.dy_off[l], dys)):
                vals = torch.randint(-32768, 32768, (L.nq * 64, rows), generator=g, dtype=torch.int16)
                vl = vals.tolist()
                for px in range(L.nq * 64):
                    chunk, row = px // 64, px % 64
                    for c in range(rows):
                        struct.pack_into('<h', buf, off + chunk * E.blk_bytes(rows) + _c_mn128(c, row), vl[px][c])
                out.append(vals)
        bits = torch.randint(0, 2, (5, L.ntiles * 128, 256), generator=g, dtype=torch.int64)
        bl = bits.tolist()
        for l in range(5):
            for tile in range(L.ntiles):
                for cw in range(2):
                    for row in range(64):
                        px = tile * 128 + cw * 64 + row
                        for q in range(8):
                            word = sum(bl[l][px][32 * q + b] << b for b in range(32))
                            struct.pack_into('<I', save, L.mask_off + (((l * L.ntiles + tile) * 128 + cw * 64 + row) * 32) + 4 * q,
                                             word)
        sv, dv = torch.frombuffer(save, dtype=torch.uint8), torch.frombuffer(dy, dtype=torch.uint8)
        for l in range(6):
            assert torch.equal(E.decode_x(sv, L, l), xs[l]), (name, 'x', l)
            assert torch.equal(E.decode_dy(dv, L, l), dys[l]), (name, 'dy', l)
        assert torch.equal(E.decode_masks(sv, L), bits.bool()), name


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_buffer_sizes_match_the_library(name):
    """the Python restatement of make_layout sizes the buffers as the library's host-side exports do"""
    from dvd_b200 import _lib, ops
    from oracle.sf_mlp_bf16 import Layout
    lib = _lib.load()
    cfg = ops.make_mlp_cfg(**_kw(name))
    for npx in (391, 891, 24576, 172032):
        L = Layout(npx=npx, **_kw(name))
        assert L.kpad0 == KPAD0[name]
        assert lib.dvd_mlp_save_bytes_per_eval(ctypes.byref(cfg), npx) == L.save_total, (name, npx)
        assert lib.dvd_mlp_dy_bytes(ctypes.byref(cfg), npx) == L.dy_total, (name, npx)
        assert lib.dvd_mlp_packed_weights_bytes(ctypes.byref(cfg)) == L.packed_weights_bytes(), name


# ---- teeth ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['16-16-T', '30-0-F'])
def test_defects_are_far_above_the_gpu_bounds(name):
    """At 128 x 192 pixels (the GPU test's inputs): what bf16x2 instead of bf16x3 changes in the forward (s, the saved X planes)
    and in the data gradient (a_out, the dY planes), and what one dropped 64-pixel chunk changes in dW and db, against the
    GPU bounds. One eval of the emulation with the weights split as pack_weights_kernel does."""
    from oracle import sf_mlp_bf16 as E
    torch.set_num_threads(max(torch.get_num_threads(), 1))
    kw = _kw(name)
    B, H, W = 1, 128, 192
    layers, p0, t0, g_acc, g_steps = make_case(name, B, H, W)
    net = E.Net.from_weights(layers, kw)
    p, t = E.to_px(p0.double()), E.to_px(t0.double()).view(-1) if kw['time_dependent'] else None
    f3, f2 = E.forward_eval(net, p, t, terms=3), E.forward_eval(net, p, t, terms=2)
    eff_s = E.rel_max(f2['s'], f3['s'])
    eff_x = min(E.plane_agreement(E.bf16_bits(f2['x'][l][0]), f3['x'][l][0])[0] for l in range(1, 6))
    args = dict(g_acc=E.to_px(g_acc.double()), g_step=E.to_px(g_steps[0].double()))
    d3 = E.dgrad_eval(net, p, f3['mask'], terms=3, **args)
    d2 = E.dgrad_eval(net, p, f3['mask'], terms=2, **args)
    eff_a = E.rel_max(d2['a_out'], d3['a_out'])
    eff_dy = min(E.plane_agreement(E.bf16_bits(d2['dy'][l][0]), d3['dy'][l][0])[0] for l in range(5))
    # weight gradient on the hi planes of the full 384 chunks (no pad pixels at this shape)
    xs = [x[0] for x in f3['x']]
    dys = [y[0] for y in d3['dy']]
    gw, gb = E.wgrad(xs, dys)
    valid = torch.ones(len(p), dtype=torch.bool)
    eff_w = min(E.chunk_effect(xs[l], dys[l], gw[l], valid) for l in range(6))
    eff_b = min(E.chunk_effect(torch.ones_like(xs[l][:, :1]), dys[l], gb[l].view(-1, 1), valid) for l in range(5))
    print('\n[%s] bf16x2 forward: s %.2e, X planes differ %.2e | bf16x2 data gradient: a_out %.2e, dY planes differ %.2e | '
          'one chunk: dW %.2e, db %.2e' % (name, eff_s, eff_x, eff_a, eff_dy, eff_w, eff_b))
    for eff, bound, what in ((eff_s, S_REL, 's'), (eff_x, X_DIFF, 'X'), (eff_a, A_OUT_REL, 'a_out'), (eff_dy, DY_DIFF, 'dY'),
                             (eff_w, WGRAD_REL, 'dW'), (eff_b, GB_REL, 'db')):
        assert eff >= MARGIN * bound, (what, eff, bound)
