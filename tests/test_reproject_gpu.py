"""GPU parity: fused re-projection kernels (through the C ABI) vs the reference-generated fixtures
and vs the CPU oracle on seeded inputs. Tolerance: 1e-3 tensor-normalised;
observed errors are ~1e-6 (fp32 rounding order only)."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-3
TIGHT = 5e-5


def _dev(batch):
    return {k: (v.cuda().float().contiguous() if torch.is_tensor(v) else v) for k, v in batch.items()}


def _cfg(kw):
    from dvd_b200 import ops
    return ops.make_loss_cfg(midas=kw['midas'], warm=kw['warm'], use_disp=kw['use_disp'],
                             use_disp_ratio=kw['use_disp_ratio'], flow_mul=kw.get('flow_mul', 1.0),
                             disp_mul=kw.get('disp_mul', 1.0))


def test_materialize_matches_reference_fixture(reproject_golden):
    from dvd_b200 import ops
    g = reproject_golden
    i = g['inputs']
    b = _dev(i['batch'])
    poses = ops.pack_poses_from_batch(b)
    out = ops.reproject_materialize(i['d1'].cuda(), i['d2'].cuda(), b['flow_1_2'], i['sf'].cuda(), poses)
    for k, ref in g['tensors'].items():
        assert rel_err(out[k], ref) < TIGHT, k


def test_unproject_matches_fixture_and_adjoint(reproject_golden):
    from dvd_b200 import ops
    g = reproject_golden
    i = g['inputs']
    b = _dev(i['batch'])
    poses = ops.pack_poses_from_batch(b)
    d1 = i['d1'].cuda()
    P = ops.unproject_fwd(d1, poses, 1)
    assert rel_err(P, g['tensors']['global_p1']) < TIGHT
    # adjoint identity <gP, J d> == <J^T gP, d> (P is affine in d: subtract the offset)
    gP = torch.randn_like(P)
    P0 = ops.unproject_fwd(torch.zeros_like(d1), poses, 1)
    lhs = ((P - P0) * gP).sum().item()
    rhs = (ops.unproject_bwd(gP, poses, 1) * d1).sum().item()
    assert abs(lhs - rhs) <= 1e-4 * abs(lhs)


@pytest.mark.parametrize('mode', ['joint_disp', 'warm_disp', 'joint_sf', 'joint_ratio_nomidas'])
def test_fused_loss_and_grads_match_reference_fixture(reproject_golden, mode):
    from dvd_b200 import ops
    g = reproject_golden
    i = g['inputs']
    m = g['modes'][mode]
    b = _dev(i['batch'])
    poses = ops.pack_poses_from_batch(b)
    d1 = i['d1'].cuda().requires_grad_()
    d2 = i['d2'].cuda().requires_grad_()
    sf = i['sf'].cuda().requires_grad_()
    mask = b['mask_2'].reshape(d1.shape[0], *d1.shape[2:]).contiguous()
    loss, scal = ops.reproject_loss(d1, d2, sf, b['flow_1_2'], mask, poses, _cfg(m['kw']))
    s = scal.cpu()
    assert abs(loss.item() - m['loss']) <= TOL * abs(m['loss'])
    assert abs(loss.item() - m['loss']) <= 2e-5 * abs(m['loss'])
    assert abs(s[0].item() - m['loss_data']['flow_loss_1_2']) <= 2e-5 * abs(m['loss_data']['flow_loss_1_2'])
    assert abs(s[1].item() - m['loss_data']['disp_loss_1_2']) <= 2e-5 * abs(m['loss_data']['disp_loss_1_2'])
    assert abs(s[2].item() - m['loss_data']['sf_loss']) <= 2e-5 * abs(m['loss_data']['sf_loss'])
    loss.backward()
    # reference autograd gives d1 the direct-path gradient only here (sf is a leaf), like ours
    assert rel_err(sf.grad, m['g_sf']) < 1e-4
    assert rel_err(d2.grad, m['g_d2']) < 1e-4
    assert rel_err(d1.grad, m['g_d1']) < 1e-4


@pytest.mark.parametrize('shape', [(1, 32, 48), (3, 30, 50), (2, 17, 23), (5, 64, 96), (65, 6, 10), (65, 96, 128)])
def test_fused_matches_oracle_on_seeded_inputs(shape):
    """Odd and small shapes run the generic kernels, (65, 96, 128) the staged ones (the size condition holds up to
    390 SMs); B = 65 crosses the 64-pair chunk of constant-bank poses of the staged path."""
    from dvd_b200 import ops, synthetic
    from oracle import geometry
    B, H, W = shape
    pairs = [(2 * k, 2 * k + 1 + (k % 3)) for k in range(B)]
    batch = synthetic.make_batch(pairs, H=H, W=W, seed=B + H, leading_dim=False, flow_sigma=5.0)
    d1 = synthetic.make_depths(B, H, W, seed=1)
    d2 = synthetic.make_depths(B, H, W, seed=2)
    sf = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(7)) * 0.05
    kw = dict(midas=True, warm=False, use_disp=True, use_disp_ratio=False, flow_mul=1.0, disp_mul=1.0)
    b64 = {k: (v.double() if torch.is_tensor(v) else v) for k, v in batch.items()}
    d1o, d2o, sfo = (t.double().requires_grad_() for t in (d1, d2, sf))
    loss_o, parts_o, r_o = geometry.reproject_and_loss(d1o, d2o, sfo, b64, **kw)
    go = torch.autograd.grad(loss_o, [d1o, d2o, sfo])
    b = _dev(batch)
    poses = ops.pack_poses_from_batch(b)
    d1g, d2g, sfg = (t.cuda().requires_grad_() for t in (d1, d2, sf))
    mask = b['mask_2'].reshape(B, H, W).contiguous()
    loss, scal = ops.reproject_loss(d1g, d2g, sfg, b['flow_1_2'], mask, poses, _cfg(kw))
    assert abs(loss.item() - float(loss_o)) <= 1e-4 * abs(float(loss_o))
    loss.backward()
    for mine, ref, name in ((d1g.grad, go[0], 'g_d1'), (d2g.grad, go[1], 'g_d2'), (sfg.grad, go[2], 'g_sf')):
        assert rel_err(mine, ref) < TOL, name
        assert rel_err(mine, ref) < 2e-4, name
    out = ops.reproject_materialize(d1g.detach(), d2g.detach(), b['flow_1_2'], sfg.detach(), poses)
    for k in ('global_p1', 'sf_by_depth', 'warped_p2_camera_2', 'p1_camera_2', 'dflow_1_2', 'depth_warp_1_2'):
        assert rel_err(out[k], r_o[k]) < 1e-4, k


@pytest.mark.parametrize('case', [(4, 224, 384, 3.0, 'joint_disp'), (4, 224, 384, 14.0, 'joint_sf'),
                                  (5, 203, 384, 9.0, 'warm_disp'), (4, 224, 384, 40.0, 'joint_ratio_nomidas')])
def test_staged_path_matches_oracle(case):
    """The staged kernels (bulk-async staged inputs, vector reductions for the scatter) against the oracle. Small and
    very large flows (border clamps), H = 203 leaves a ragged last tile; every loss mode of the reference is covered
    (smf.py:285-324,140-150). The same inputs through the generic kernels (16-byte misaligned copies) give a bitwise
    equal g_sf: both paths run the same per-pixel functions."""
    from dvd_b200 import ops, synthetic
    from oracle import geometry
    B, H, W, sigma, mode = case
    kw = {'joint_disp': dict(midas=True, warm=False, use_disp=True, use_disp_ratio=False),
          'warm_disp': dict(midas=True, warm=True, use_disp=True, use_disp_ratio=False),
          'joint_sf': dict(midas=True, warm=False, use_disp=False, use_disp_ratio=False),
          'joint_ratio_nomidas': dict(midas=False, warm=False, use_disp=False, use_disp_ratio=True)}[mode]
    kw.update(flow_mul=1.0, disp_mul=0.7)
    pairs = [(3 * k, 3 * k + 1 + (k % 4)) for k in range(B)]
    batch = synthetic.make_batch(pairs, H=H, W=W, seed=11 + B, leading_dim=False, flow_sigma=sigma)
    d1 = synthetic.make_depths(B, H, W, seed=1)
    d2 = synthetic.make_depths(B, H, W, seed=2)
    sf = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(7)) * 0.05
    b64 = {k: (v.double() if torch.is_tensor(v) else v) for k, v in batch.items()}
    d1o, d2o, sfo = (t.double().requires_grad_() for t in (d1, d2, sf))
    loss_o, parts_o, _ = geometry.reproject_and_loss(d1o, d2o, sfo, b64, **kw)
    go = torch.autograd.grad(loss_o, [d1o, d2o, sfo])
    b = _dev(batch)
    poses = ops.pack_poses_from_batch(b)
    d1g, d2g, sfg = (t.cuda().requires_grad_() for t in (d1, d2, sf))
    mask = b['mask_2'].reshape(B, H, W).contiguous()
    loss, scal = ops.reproject_loss(d1g, d2g, sfg, b['flow_1_2'], mask, poses, _cfg(kw))
    assert abs(loss.item() - float(loss_o)) <= 1e-4 * abs(float(loss_o))
    loss.backward()
    for mine, ref, name in ((d1g.grad, go[0], 'g_d1'), (d2g.grad, go[1], 'g_d2'), (sfg.grad, go[2], 'g_sf')):
        assert rel_err(mine, ref) < 2e-4, name

    def misaligned(t):   # contiguous copy whose data pointer sits 4 bytes past a 16-byte boundary
        buf = torch.empty(t.numel() + 4, dtype=t.dtype, device=t.device)
        out = buf[1:1 + t.numel()].view(t.shape)
        out.copy_(t)
        return out

    cfg = _cfg(kw)
    ins = (d1g.detach(), d2g.detach(), b['flow_1_2'], mask, sfg.detach(), poses)
    s_st = ops.reproject_loss_fwd(*ins, cfg)
    g_st, gd_st = ops.reproject_loss_bwd(*ins, cfg, s_st)
    mis = [misaligned(t) for t in ins[:5]] + [poses]
    s_gen = ops.reproject_loss_fwd(*mis, cfg)
    g_gen, gd_gen = ops.reproject_loss_bwd(*mis, cfg, s_st)
    assert torch.equal(g_gen, g_st)
    assert abs(s_gen[3].item() - s_st[3].item()) <= 1e-6 * abs(s_st[3].item())
    assert rel_err(gd_gen, gd_st) < 1e-6


def test_border_and_empty_mask_edge_cases():
    """Flow pushing every sample out of the image (border clamp) and an all-zero mask (N = 1e-8)."""
    from dvd_b200 import ops, synthetic
    from oracle import geometry
    B, H, W = 2, 16, 24
    batch = synthetic.make_batch([(0, 1), (5, 9)], H=H, W=W, seed=3, leading_dim=False, flow_sigma=60.0)
    batch['mask_2'].zero_()
    d1 = synthetic.make_depths(B, H, W, seed=1)
    d2 = synthetic.make_depths(B, H, W, seed=2)
    sf = torch.zeros(B, 3, H, W)
    kw = dict(midas=True, warm=True, use_disp=True, use_disp_ratio=False)
    loss_o, _, r_o = geometry.reproject_and_loss(d1, d2, sf, batch, **kw)
    b = _dev(batch)
    poses = ops.pack_poses_from_batch(b)
    scal = ops.reproject_loss_fwd(d1.cuda(), d2.cuda(), b['flow_1_2'], b['mask_2'].reshape(B, H, W).contiguous(),
                                  sf.cuda(), poses, _cfg(kw))
    assert scal[3].item() == 0.0 and float(loss_o) == 0.0
    out = ops.reproject_materialize(d1.cuda(), d2.cuda(), b['flow_1_2'], sf.cuda(), poses)
    assert rel_err(out['warped_p2_camera_2'], r_o['warped_p2_camera_2']) < TIGHT
    assert rel_err(out['depth_warp_1_2'], r_o['depth_warp_1_2']) < TIGHT


def test_large_batch_properties():
    """BASELINE size (384x224) x 8 pairs: size-independent properties — the loss of a batch made of
    8 copies of one pair equals the single-pair loss, and the gradients are the single-pair ones / 8."""
    from dvd_b200 import ops, synthetic
    H, W = 224, 384
    one = synthetic.make_batch([(4, 8)], H=H, W=W, seed=0, leading_dim=False)
    b1 = _dev(one)
    d1 = synthetic.make_depths(1, H, W, seed=1).cuda()
    d2 = synthetic.make_depths(1, H, W, seed=2).cuda()
    sf = (torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(1)) * 0.05).cuda()
    cfg = ops.make_loss_cfg()
    p1 = ops.pack_poses_from_batch(b1)
    m1 = b1['mask_2'].reshape(1, H, W).contiguous()
    s1 = ops.reproject_loss_fwd(d1, d2, b1['flow_1_2'], m1, sf, p1, cfg)
    g1, gd1 = ops.reproject_loss_bwd(d1, d2, b1['flow_1_2'], m1, sf, p1, cfg, s1)
    rep = lambda t: t.repeat(8, *([1] * (t.dim() - 1))).contiguous()  # noqa: E731
    s8 = ops.reproject_loss_fwd(rep(d1), rep(d2), rep(b1['flow_1_2']), rep(m1), rep(sf), rep(p1), cfg)
    g8, gd8 = ops.reproject_loss_bwd(rep(d1), rep(d2), rep(b1['flow_1_2']), rep(m1), rep(sf), rep(p1), cfg, s8)
    assert abs(s8[3].item() - s1[3].item()) <= 1e-5 * abs(s1[3].item())
    assert abs(s8[4].item() - 8 * s1[4].item()) <= 1e-6 * abs(8 * s1[4].item())
    assert rel_err(g8[3] * 8, g1[0]) < 1e-5
    assert rel_err(gd8[5] * 8, gd1[0]) < 1e-4   # atomics: summation order differs


def test_operator_mirrors_are_differentiable_for_arbitrary_losses():
    """A user-defined loss on the mirrors' result dicts back-propagates like the reference modules would
    (oracle autograd, fp64) — dvd_reproject_materialize_bwd."""
    from dvd_b200 import synthetic
    from dvd_b200.losses import scene_flow_projection as sfp
    from oracle import geometry
    B, H, W = 2, 20, 28
    batch = synthetic.make_batch([(2, 5), (9, 10)], H=H, W=W, seed=4, leading_dim=False, flow_sigma=3.0)
    d1 = synthetic.make_depths(B, H, W, seed=1)
    d2 = synthetic.make_depths(B, H, W, seed=2)
    sf = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(7)) * 0.05
    gen = torch.Generator().manual_seed(8)
    keys = ['global_p1', 'sf_by_depth', 'warped_global_p2', 'warped_p2_camera_2', 'p1_camera_2', 'dflow_1_2',
            'staticflow_1_2', 'depth_image_1_2', 'depth_warp_1_2']
    b64 = {k: (v.double() if torch.is_tensor(v) else v) for k, v in batch.items()}
    d1o, d2o, sfo = (t.double().requires_grad_() for t in (d1, d2, sf))
    ro = geometry.reproject(d1o, d2o, sfo, b64)
    cots = {k: torch.randn(ro[k].shape, generator=gen) for k in keys}
    sum((ro[k] * cots[k].double()).sum() for k in keys).backward()
    b = _dev(batch)
    pose = {k: b[k] for k in ('R_1', 'R_2', 'R_1_T', 'R_2_T', 't_1', 't_2', 'K', 'K_inv')}
    d1g, d2g, sfg = (t.cuda().requires_grad_() for t in (d1, d2, sf))
    sfl = sfg.permute(0, 2, 3, 1)[..., None, :]
    r1 = sfp.flow_by_depth()(depth_1=d1g, depth_2=d2g, flow_1_2=b['flow_1_2'], **pose)
    r2 = sfp.scene_flow_projection_slack()(depth_1=d1g, depth_2=d2g, flow_1_2=b['flow_1_2'], flow_2_1=b['flow_2_1'],
                                           sflow_1_2=sfl, sflow_2_1=sfl, **pose)
    cf = lambda x: x.squeeze(3).permute(0, 3, 1, 2)  # noqa: E731
    mine = {'global_p1': cf(r2['global_p1']), 'sf_by_depth': cf(r1['sf_by_depth']), 'warped_global_p2': cf(r1['warped_global_p2']),
            'warped_p2_camera_2': cf(r2['warped_p2_camera_2']), 'p1_camera_2': cf(r2['p1_camera_2']),
            'dflow_1_2': r2['dflow_1_2'].permute(0, 3, 1, 2), 'staticflow_1_2': r2['staticflow_1_2'].permute(0, 3, 1, 2),
            'depth_image_1_2': r2['depth_image_1_2'], 'depth_warp_1_2': r2['depth_warp_1_2']}
    sum((mine[k] * cots[k].cuda()).sum() for k in keys).backward()
    assert rel_err(d1g.grad, d1o.grad) < 2e-4
    assert rel_err(d2g.grad, d2o.grad) < 2e-4
    assert rel_err(sfg.grad, sfo.grad) < 2e-4
