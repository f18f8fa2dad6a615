"""The fp32 emulation of the re-projection kernels (oracle/reproject_fp32.py), checked without a GPU.

* `fma_f32` is the correctly rounded fused multiply-add: against exact rational arithmetic on random triples and on
  constructed cases whose fp64 sum lands exactly on an fp32 midpoint (where rounding twice gives the wrong answer).
* With rounding off, the emulation is plain fp64 arithmetic and must equal `oracle.geometry` to 1e-12 (relative to each
  tensor's maximum): the four loss scalars and the mask count, all nine materialised tensors, and the hand-written
  backward (g_sf, g_depth_2 and g_depth_1 = unproject_bwd(g_sf)) against autograd. That holds for every loss
  configuration the reference defines; the configurations only the C ABI reaches are checked against autograd of the same
  forward with the ABI's own choice of second term. The inputs plant every edge of the chain (oracle.reproject_fp32.edge_inputs).
* Defect sizes: each kernel defect the GPU test is meant to catch, applied to the emulation, changes a quantity that the GPU
  test checks exactly (mask count, bitwise per-pixel values, the non-zero pattern of g_depth_2) or changes g_depth_2 by
  more than 10x its bound.
"""
import random
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import geometry
from oracle import reproject_fp32 as R

SHAPE = (2, 12, 16)


def _round_fraction_f32(x):
    """x (a Fraction) rounded to the nearest fp32, ties to even"""
    r0 = np.float32(float(x))
    cands = [np.nextafter(r0, np.float32(-np.inf)), r0, np.nextafter(r0, np.float32(np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(np.array(c).view(np.uint32)) & 1))
    return best


def _exact_fma(a, b, c):
    return _round_fraction_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def test_fma_f32_is_correctly_rounded_on_random_triples():
    rng = random.Random(0)
    a, b, c = (np.array([np.float32(rng.uniform(-1, 1) * 2.0 ** rng.randint(-30, 30)) for _ in range(3000)], np.float32)
               for _ in range(3))
    c[:1000] = -(a[:1000].astype(np.float64) * b[:1000]).astype(np.float32)   # heavy cancellation
    got = R.fma_f32(a, b, c)
    want = np.array([_exact_fma(x, y, z) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_fma_f32_midpoint_ties():
    """641 * 6700417 = 2^32 + 1: the fp64 sum of 2^56 and that product is the fp32 midpoint 2^56 + 2^32 with a residual
    of 1, so rounding the fp64 sum again would round to even (2^56) instead of up. Scaled by powers of two and mirrored in
    sign, plus the residual -1 case whose even neighbour lies above, and exact ties (residual 0: ties to even)."""
    cases = []
    for s in (0, -40, -80, 20):
        sc = 2.0 ** s
        cases += [(641 * sc, 6700417.0, 2.0 ** 56 * sc, 2.0 ** 56 * sc + 2.0 ** 33 * sc),
                  (-641 * sc, 6700417.0, -2.0 ** 56 * sc, -(2.0 ** 56 * sc + 2.0 ** 33 * sc)),
                  (-641 * sc, 6700417.0, (2.0 ** 56 + 2.0 ** 34) * sc, (2.0 ** 56 + 2.0 ** 33) * sc),
                  (2.0 ** 16 * sc, 2.0 ** 16, 2.0 ** 56 * sc, 2.0 ** 56 * sc),                     # exact tie, even below
                  (2.0 ** 16 * sc, 2.0 ** 16 * 3, 2.0 ** 56 * sc, (2.0 ** 56 + 2.0 ** 34) * sc)]   # exact tie, even above
    a, b, c, want = (np.array(v, np.float32) for v in zip(*cases))
    got = R.fma_f32(a, b, c)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    for x, y, z, w in zip(a, b, c, want):
        assert _exact_fma(x, y, z) == w
    # rounding the fp64 result once more would get the residual cases wrong
    naive = (a.astype(np.float64) * b + c).astype(np.float32)
    assert not np.array_equal(naive, want)


def test_sgn_scale_signed_zeros():
    A = R.Fp32()
    v = np.array([1.0, -1.0, 0.0, -0.0, 2.0, -3.0], np.float32)
    c = np.array([0.0, 0.0, 5.0, 5.0, -2.0, -2.0], np.float32)
    got = A.sgn_scale(v, c)
    want = np.array([0.0, -0.0, 0.0, 0.0, -2.0, 2.0], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------

def _np(inp):
    return (inp['d1'][:, 0].numpy(), inp['d2'][:, 0].numpy(), inp['flow'].numpy(), inp['mask'].numpy(),
            inp['sf'].numpy())


@pytest.fixture(scope='module')
def inputs():
    inp = R.edge_inputs(*SHAPE, seed=0, sigma=3.0)
    A = R.Fp32(round=False)
    o = R.pixel_forward(A, R.derive_pose(A, inp['poses'].numpy()), inp['d2'][:, 0].numpy(), inp['flow'].numpy(),
                        inp['d1'][:, 0].numpy(), inp['sf'].numpy())
    # every edge is present
    assert (~o['zok']).any() and (o['p12'][2] < 1e-3).any()
    assert (o['wpc'][2] >= 100).any() and (o['d1'] >= 100).any() and (o['wpc'][2] < 1e-3).any()
    assert (o['sx1'] == 0).any() and (o['sy1'] == 0).any()
    return inp


def _close(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    err = np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)
    assert err <= 1e-12, (what, err)


def _calc_loss_abi(r, sf, batch, cfg):
    """geometry.calc_loss with the C ABI's free choice of disparity term (disp_mode) and second term (second_is_disp)"""
    mask = batch['mask_2'].reshape(r['dflow_1_2'].shape[0], 1, *r['dflow_1_2'].shape[2:]).to(sf.dtype)
    if cfg['midas']:
        mask = mask * (r['depth_1'] < 100).to(sf.dtype) * (r['warped_p2_camera_2'][:, 2:3] < 100).to(sf.dtype)
    n = mask.sum() + 1e-8
    diff = r['dflow_1_2'] - batch['flow_1_2'].permute(0, 3, 1, 2)
    flow_loss = (mask * (diff * diff if cfg['warm'] else diff.abs())).sum() / n
    za, zb = r['p1_camera_2'][:, 2:3], r['warped_p2_camera_2'][:, 2:3]
    a, b = za.clamp(min=1e-3), zb.clamp(min=1e-3)
    disp_pp = [100 * (1 / a - 1 / b).abs(), torch.maximum(a, b) / torch.minimum(a, b) - 1, (za - zb).abs()][cfg['disp_mode']]
    disp_loss = (mask * disp_pp).sum() / n
    sf_loss = (mask * (r['sf_by_depth'] - sf).abs()).sum() / n
    second = disp_loss if cfg['second_is_disp'] else sf_loss
    loss = cfg['flow_mul'] * flow_loss + cfg['disp_mul'] * second
    return loss, {'flow_loss_1_2': flow_loss, 'disp_loss_1_2': disp_loss, 'sf_loss': sf_loss, 'mask_sum': mask.sum()}


@pytest.mark.parametrize('cfg', R.all_cfgs(flow_mul=1.0, disp_mul=0.7), ids=lambda c: 'mi%d-wa%d-dm%d-sd%d' % (
    c['midas'], c['warm'], c['disp_mode'], c['second_is_disp']))
def test_unrounded_emulation_equals_fp64_oracle(inputs, cfg):
    inp = inputs
    A = R.Fp32(round=False)
    ps = R.derive_pose(A, inp['poses'].numpy())
    d1, d2, flow, mask, sf = _np(inp)
    b64 = {k: (v.double() if torch.is_tensor(v) else v) for k, v in inp['batch'].items()}
    d1o, d2o, sfo = (inp[k].double().requires_grad_() for k in ('d1', 'd2', 'sf'))
    kw = R.reference_kw(cfg)
    if kw is not None:
        loss_o, parts_o, r_o = geometry.reproject_and_loss(d1o, d2o, sfo, b64, **kw)
    else:
        r_o = geometry.reproject(d1o, d2o, sfo, b64)
        r_o['depth_1'] = d1o
        loss_o, parts_o = _calc_loss_abi(r_o, sfo, b64, cfg)
    g_o = torch.autograd.grad(loss_o, [d1o, d2o, sfo])
    f = R.loss_forward(A, cfg, ps, d1, d2, flow, mask, sf)
    s = f['scalars']
    for mine, key in ((s['flow'], 'flow_loss_1_2'), (s['disp'], 'disp_loss_1_2'), (s['sf'], 'sf_loss'),
                      (s['masksum'], 'mask_sum')):
        _close(mine, float(parts_o[key].detach()), key)
    _close(s['loss'], float(loss_o.detach()), 'loss')
    gv, h = R.pixel_backward(A, cfg, ps, f['o'], f['m'], s['cf'], s['cd'])
    taps = R.tap_grads(A, f['o'], *h)
    g_sf = np.stack(gv, 1)
    B, H, W = d1.shape
    g_d2 = R.scatter(f['o'], taps, B, H * W)[0].reshape(B, 1, H, W)
    g_d1 = R.unproject_bwd(A, g_sf, inp['poses'].numpy(), 1)[:, None]
    _close(g_sf, g_o[2].numpy(), 'g_sf')
    _close(g_d2, g_o[1].numpy(), 'g_d2')
    _close(g_d1, g_o[0].numpy(), 'g_d1')


def test_unrounded_materialize_and_unproject_equal_fp64_oracle(inputs):
    inp = inputs
    A = R.Fp32(round=False)
    ps = R.derive_pose(A, inp['poses'].numpy())
    d1, d2, flow, mask, sf = _np(inp)
    b64 = {k: (v.double() if torch.is_tensor(v) else v) for k, v in inp['batch'].items()}
    d1o, d2o, sfo = (inp[k].double().requires_grad_() for k in ('d1', 'd2', 'sf'))
    r_o = geometry.reproject(d1o, d2o, sfo, b64)
    mat = R.materialize(A, ps, d1, d2, flow, sf)
    for k, v in mat.items():
        _close(v, r_o[k].detach().numpy(), k)
    R1, R2, t1, t2, K, Kinv = geometry._poses(b64)
    for which, Rw, tw in ((1, R1, t1), (2, R2, t2)):
        _close(R.unproject_fwd(A, d1, inp['poses'].numpy(), which), geometry.unproject(d1o.detach(), Rw, tw, Kinv).numpy(),
               'unproject_fwd')
    # materialise adjoint against autograd for random cotangents on all nine outputs
    gen = torch.Generator().manual_seed(5)
    G = {k: torch.randn(r_o[k].shape, generator=gen, dtype=torch.float64) for k in mat}
    g_o = torch.autograd.grad(sum((r_o[k] * G[k]).sum() for k in mat), [d1o, d2o, sfo])
    g_d1, g_d2, g_sf = R.materialize_bwd(A, ps, d1, d2, flow, sf, {k: v.numpy() for k, v in G.items()})
    _close(g_d1[:, None], g_o[0].numpy(), 'mat g_d1')
    _close(g_d2[:, None], g_o[1].numpy(), 'mat g_d2')
    _close(g_sf, g_o[2].numpy(), 'mat g_sf')
    gP = torch.randn(d1o.shape[0], 3, *d1.shape[1:], generator=gen, dtype=torch.float64)
    P = geometry.unproject(d1o, R1, t1, Kinv)
    _close(R.unproject_bwd(A, gP.numpy(), inp['poses'].numpy(), 1)[:, None],
           torch.autograd.grad((P * gP).sum(), d1o)[0].numpy(), 'unproject_bwd')


# ---------------------------------------------------------------------------------------------------------------------
# defect sizes, in the fp32 emulation itself

@pytest.fixture(scope='module')
def rounded(inputs):
    inp = inputs
    A = R.Fp32()
    ps = R.derive_pose(A, inp['poses'].numpy())
    d1, d2, flow, mask, sf = _np(inp)
    return A, ps, R.pixel_forward(A, ps, d2, flow, d1, sf), mask


def test_defect_mask_ignoring_warped_depth_changes_the_mask_count(rounded):
    A, ps, o, mask = rounded
    cfg = R.cfg_dict(1, 0, 0, 1)
    m = R.mask_of(A, cfg, mask, o)
    m_mut = np.where(o['d1'] < 100, A.f(mask), 0)
    assert m_mut.sum() - m.sum() >= 1


def test_defect_tap_grads_sizes(rounded):
    """tap_grads using `base` for the ne tap changes g_depth_2 by more than 10x the GPU test's per-element bound
    (k · 2^-24 · sum |contributions|); a one-lane shift of the odd-column vector reduction moves non-zero contributions,
    which the exact non-zero pattern check sees, as long as such pixels exist. Only the scene-flow term gives the ne tap a
    gradient of its own (hu = Kinv[6] g_wpc.z = 0 under the disparity terms), so the GPU test needs second_is_disp = 0."""
    A, ps, o, mask = rounded
    for cfg in (R.cfg_dict(1, 0, 2, 0), R.cfg_dict(0, 1, 1, 0)):
        m = R.mask_of(A, cfg, mask, o)
        gv, (hu, hv, h1) = R.pixel_backward(A, cfg, ps, o, m, np.float32(1e-2), np.float32(1e-2))
        taps = R.tap_grads(A, o, hu, hv, h1)
        B, H, W = o['d1'].shape
        tot, ab, cnt = R.scatter(o, taps, B, H * W)
        base = A.fma(hu, o['x0f'], A.fma(hv, o['y0f'], h1))
        mut = [taps[0], A.mul(o['w'][1], base), taps[2], taps[3]]
        tot_m = R.scatter(o, mut, B, H * W)[0]
        assert (np.abs(tot_m - tot) > 10 * cnt * 2.0 ** -24 * ab).any()
        odd = (o['i00'] % 4 == 1) & (o['sx1'] == 1) & ((taps[0] != 0) | (taps[1] != 0))
        assert odd.any()


def test_defect_swapped_ratio_gradients_change_g_sf(rounded):
    """disp_mode 1 with second_is_disp (reachable only through the C ABI): swapping the two ratio gradients changes g_sf,
    which the GPU test compares bit for bit."""
    A, ps, o, mask = rounded
    cfg = R.cfg_dict(0, 0, 1, 1)
    m = R.mask_of(A, cfg, mask, o)
    gv, _ = R.pixel_backward(A, cfg, ps, o, m, np.float32(1e-2), np.float32(1e-2))
    za, zb = o['p12'][2], o['wpc'][2]
    a, bb = A.fmax(za, A.f(1e-3)), A.fmax(zb, A.f(1e-3))
    ra, rb = A.rcp(a), A.rcp(bb)
    ga = np.where(a >= bb, rb, A.mul(A.mul(-bb, ra), ra))
    gb = np.where(a >= bb, A.mul(A.mul(-a, rb), rb), ra)
    # ga enters g_p12.z, so g_sf = R2 g_p12 moves by R2[:, 2] (gb - ga) mc wherever za >= 1e-3 and the pixel counts
    moved = (za >= 1e-3) & (m != 0) & (ga != gb)
    assert moved.sum() >= 10
