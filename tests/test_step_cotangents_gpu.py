"""The whole training step's gradients against fp64, teacher-forced at the depth maps and at the scene flow.

Every kernel family of the step is held to a reference of its own arithmetic in isolation; this module checks the glue
`Model._step_body` composes them with: which cotangents reach the depth net and the MLP, with which scales and masks. One
eager step (`cuda_graph=False`) runs with wrappers that keep the step's own internal tensors and hook their cotangents: `d1`,
`d2` (from `_depths`), `P1` (from `ops.unproject`), `acc`, `s_steps` (from `net_sceneflow.chain`), `dL/dp0` (from
`ops.mlp_chain_bwd`), the MLP parameters' gradients as autograd delivers them, and, after the MiDaS forward, the engine's saved
tensors and packed weight images. Then:

* reference A: the step's composition in the order of oracle/step.py (`geometry.unproject`, `sf_mlp.sf_multi_step`, motion
  segmentation, `geometry.reproject_and_loss`, the `--weight_steps` scale, `sf_mlp.acc_reg`), in fp64 on the GPU from the
  step's own `d1`, `d2` and the pre-step MLP weights, one backward. Against it: the five logged losses, `dL/dd1`, `dL/dd2`
  and every MLP parameter gradient;
* reference B, loss -> MLP: `dL/dacc` restated with oracle/reproject_fp32.py (the hardware rcp) on the step's own `d1`, `d2`,
  `sf`, flow, mask and poses, the loss configuration and `gscale` taken from the options, times `motion_seg_1` where it
  applies: bit for bit;
* reference B, MLP -> depth: `dL/dP1` as the fp64 VJP of the Euler chain at the step's own `P1`, fed the step's own
  `dL/dacc` and `dL/ds_steps`;
* the depth net (MiDaS, joint phase): the engine emulation of tests/test_depth_engine_tf32_gpu.py, fed the step's anchors,
  images and the cotangent `cat(dL/dd1, dL/dd2)` a real loss produces (sparse, masked, L1 signs), with that test's bounds.

Every gradient tensor is compared over all its elements by slope, relative L2 and max-norm (conftest.grad_agreement). Only the
max-norm of the per-pixel cotangents leaves out a band of pixels where two correct implementations may take different sides of
a kink, found from reference A: an L1 residual (flow, disparity, scene flow) within a small distance of 0, |s_1 - s_0| near 0,
a value near a clamp(1e-3) or the < 100 mask threshold, and the LeakyReLU kink band (`sf_mlp.kink_band`). The band's share is
bounded. `.grad` still holds the pre-Adam gradients after the step: the MLP's equal what autograd delivered bit for bit, and
Adam's first step moved every parameter of both nets against the sign of its `.grad` and none whose `.grad` is 0.

Teeth: in every case, defects planted on the reference side (the depth cotangent and all gradients scaled by 1.01, the MLP path
into dL/dd1 removed, the regulariser's gradient removed, `gscale` missing, `motion_seg_1` not applied in the backward, the
`d1` / `d2` halves swapped, the pairs rolled by one) change some compared quantity by at least MARGIN times its bound.

Bounds: measured on an NVIDIA H100 80GB HBM3 with a 700 W power limit, set at about 3x the largest value observed over all
cases; observed maxima in the comments. The kink band holds about a fifth of the pixels for two chain evaluations and 49 % for
eight (gap 8: each evaluation adds its own LeakyReLU kinks); outside it dL/dd agrees to 8e-6 of its maximum, inside it single
pixels differ by up to 53 % (an L1 sign taken the other way), which the slope and L2 figures over all elements absorb. The
depth-net gradients stay within the bounds of tests/test_depth_engine_tf32_gpu.py: observed |slope - 1| 4.2e-4, relative L2
1.5e-3, max-norm 2.5e-3. What the defects change, in units of the bound that sees them best: the 1.01 scale 400 (dL/dd, max),
25 in the warm phase (MLP gradients, slope); the MLP path into dL/dd1 1,500-19,000 (it is 4-48 % of dL/dd1's maximum); the
regulariser 20-73 (dL/dd1, max-norm), but 0.8 with the hourglass depth net, whose dL/dd1 is dominated by the loss (the
regulariser moves it by 2e-5 of its maximum, under the noise): that one pair is reported, not asserted; gscale 20,000; the
motion segmentation 7,700; swapped halves and rolled pairs above 45,000. Peak memory 34 GB for the references at 4 x 224 x
384, then 21 GB for the engine emulation. The module runs in about 35 s on that H100.
"""
import numpy as np
import pytest
import torch

from conftest import grad_agreement
from test_depth_engine_tf32_gpu import capture_engine, check_engine_against_emulation
from test_reproject_fp32_emulation_gpu import emu  # noqa: F401  (fixture: the fp32 emulation with the hardware rcp)
from test_step_variants_gpu import _build

pytestmark = pytest.mark.gpu

# relative error of the five logged losses against reference A
LOSS_REL = 4e-5                                    # observed 1.3e-5 (time_independent)
# dL/dd1, dL/dd2 against reference A: |slope - 1|, relative L2, max-norm outside the kink band (relative to the tensor's max);
#   observed 1.4e-5 (portrait-2x384x224), 3.4e-3 (portrait: L1 signs taken the other way inside the band), 8.1e-6 (4x224x384, dL/dd2)
D_SLOPE, D_L2, D_MAX = 3e-5, 7.5e-3, 2.5e-5
# MLP parameter gradients against reference A; observed 1.4e-4 (4x224x384), 7.7e-4 (gap 1), 7.3e-4 (hourglass)
MLP_SLOPE, MLP_L2, MLP_MAX = 4e-4, 2.5e-3, 2.2e-3
# dL/dP1 against the fp64 VJP of the chain (reference B); observed 3.9e-5 (smallest-2x32x32), 4.5e-3 (gap 1), 1.4e-5 (hourglass)
P1_SLOPE, P1_L2, P1_MAX = 6e-5, 1.5e-2, 4e-5
# share of pixels in the kink band; observed 0.49 (gap 8, eight chain evaluations)
BAND_SHARE = 0.6
# every planted defect changes some compared quantity by at least this many times its bound
MARGIN = 10.0
# (case, defect) whose effect is under MARGIN times the noise there: reported, not asserted (see the module docstring)
WEAK = {('hourglass', 'no_reg')}

# half-widths of the kink band: flow residual (pixels), disparity residual and |s1 - s0| (relative to the larger side / to
# max |s0|), scene-flow residual (relative to max |sf_by_depth|), clamp(1e-3) and the < 100 threshold (relative)
DELTA_FLOW, DELTA_DISP, DELTA_S, DELTA_SF, DELTA_EDGE = 1e-3, 1e-4, 2e-4, 1e-4, 1e-4
# LeakyReLU kink band: |pre-activation| below this in some hidden layer of some evaluation (1e-5 is too narrow: at gap 8 a
# kink between the two moves dL/dP1 by 4.8e-4 of its maximum)
KINK_WIDTH = 3e-5

_GAP2 = [(10, 12), (30, 32)]
CASES = {
    'joint-2x64x96-gap1': dict(pairs=[(10, 11), (30, 31)], H=64, W=96, epoch=6, over={}),
    'joint-2x64x96-gap8': dict(pairs=[(10, 18), (30, 38)], H=64, W=96, epoch=6, over={}),
    'weight_steps-motion_seg': dict(pairs=_GAP2, H=64, W=96, epoch=6, over=dict(weight_steps=True, use_motion_seg=True)),
    'sf_loss': dict(pairs=_GAP2, H=64, W=96, epoch=6, over=dict(use_disp=False)),
    'disp_ratio-warm_reg': dict(pairs=_GAP2, H=64, W=96, epoch=6, over=dict(use_disp=False, use_disp_ratio=True, warm_reg=True)),
    'time_independent': dict(pairs=_GAP2, H=64, W=96, epoch=6, over=dict(time_dependent=False, n_freq_t=0)),
    'warm': dict(pairs=_GAP2, H=64, W=96, epoch=1, over={}),
    'hourglass': dict(pairs=_GAP2, H=64, W=96, epoch=6, over=dict(midas=False)),
    # working sizes that are not landscape: a ShutterStock portrait frame, a very wide frame (layer4 grid 1 x 12) and the
    # smallest size the engine runs (layer4 grid 1 x 1)
    'portrait-2x384x224': dict(pairs=_GAP2, H=384, W=224, epoch=6, over={}),
    'wide-2x32x384': dict(pairs=_GAP2, H=32, W=384, epoch=6, over={}),
    'smallest-2x32x32': dict(pairs=_GAP2, H=32, W=32, epoch=6, over={}),
}
BENCH_CASE = dict(pairs=[(5, 6), (12, 13), (19, 20), (26, 27)], H=224, W=384, epoch=6, over={})


class _Capture:
    """Wrappers that keep the step's own tensors (`t`) and the cotangents autograd delivers to them (`g`)."""

    def __init__(self, model, monkeypatch):
        from dvd_b200 import ops
        self.t, self.g, self.engine = {}, {}, None
        depths, unproject, chain, chain_bwd = model._depths, ops.unproject, model.net_sceneflow.chain, ops.mlp_chain_bwd

        def keep(name, t):
            self.t[name] = t.detach().clone()
            if t.requires_grad:
                # an output the loss does not use (s_steps without the regulariser) gets no cotangent
                t.register_hook(lambda g: None if g is None else self.g.__setitem__(name, g.detach().clone()))

        def _depths(img_1, img_2):
            d1, d2 = depths(img_1, img_2)
            keep('d1', d1), keep('d2', d2)
            if model.opt.midas and d1.requires_grad:
                self.engine = capture_engine(model.net_depth)
            return d1, d2

        def _unproject(depth, poses, which=1):
            P = unproject(depth, poses, which)
            keep('P1', P)
            self.t['poses'] = poses.clone()
            return P

        def _chain(*args):
            acc, s = chain(*args)
            keep('acc', acc), keep('s_steps', s)
            return acc, s

        def _chain_bwd(*args):
            gp = chain_bwd(*args)
            self.g['p0'] = gp.clone()
            return gp

        monkeypatch.setattr(model, '_depths', _depths)
        monkeypatch.setattr(ops, 'unproject', _unproject)
        monkeypatch.setattr(model.net_sceneflow, 'chain', _chain)
        monkeypatch.setattr(ops, 'mlp_chain_bwd', _chain_bwd)
        for k, p in model.net_sceneflow.named_parameters():
            p.register_hook(lambda g, k=k: self.g.__setitem__('mlp.' + k, g.detach().clone()))


def _kw(opt):
    return dict(n_freq_xyz=opt.n_freq_xyz, n_freq_t=opt.n_freq_t, time_dependent=opt.time_dependent, sf_mag_div=opt.sf_mag_div)


def _use_reg(opt, warm):
    return opt.interp_steps > 0 and (not warm or opt.warm_reg) and opt.acc_mul > 0


def _reference_a(cap, b, opt, steps, dt, warm, sd_m, defect=None):
    """fp64 restatement of the step from the step's own d1, d2 (oracle/step.py order), one backward. `defect` plants one
    error in it. Returns the losses, dL/dd1, dL/dd2, the MLP gradients and what the kink band needs."""
    from oracle import geometry, sf_mlp
    D1 = cap.t['d1'].double().requires_grad_(not warm)
    D2 = cap.t['d2'].double().requires_grad_(not warm)
    sd = {k: v.detach().cuda().double().requires_grad_() for k, v in sd_m.items()}
    layers = sf_mlp.layers_from_state_dict(sd)
    kw = _kw(opt)
    B, _, H, W = D1.shape
    R1, R2, t1, t2, K, Kinv = geometry._poses(b)
    P1 = geometry.unproject(D1, R1, t1, Kinv)
    if defect == 'detach_p1':
        P1 = P1.detach()
    ts1 = b['time_stamp_1']
    acc = sf_mlp.sf_multi_step(P1, ts1, dt, steps, layers, **kw)
    sf = acc
    if opt.use_motion_seg:
        ms = b['motion_seg_1'].reshape(B, 1, H, W)
        sf = acc * ms if defect != 'no_mseg_bwd' else acc + (acc * ms - acc).detach()
    loss, parts, r = geometry.reproject_and_loss(D1, D2, sf, b, midas=opt.midas, warm=warm, use_disp=opt.use_disp,
                                                 use_disp_ratio=opt.use_disp_ratio, flow_mul=opt.flow_mul,
                                                 disp_mul=opt.disp_mul)
    total = loss * steps if (opt.weight_steps and defect != 'no_gscale') else loss
    reg = None
    if _use_reg(opt, warm) and defect != 'no_reg':
        reg = sf_mlp.acc_reg(P1, ts1, dt, layers, acc_mul=opt.acc_mul, **kw)
        total = total + reg
    total.backward()
    out = {'losses': {'loss': float(loss.detach()), 'flow_loss_1_2': float(parts['flow_loss_1_2'].detach()),
                      'disp_loss_1_2': float(parts['disp_loss_1_2'].detach()), 'sf_loss': float(parts['sf_loss'].detach()),
                      'acc_reg': float(reg.detach()) if reg is not None else 0.0},
           'g_d1': D1.grad, 'g_d2': D2.grad, 'mlp': {k: v.grad for k, v in sd.items()}}
    if defect is None:
        out['r'] = {k: r[k].detach() for k in ('dflow_1_2', 'p1_camera_2', 'warped_p2_camera_2', 'sf_by_depth')}
        out['sf'] = sf.detach()
    return out


def _chain64(P, ts, dt, n_eval, n_acc, layers, kw):
    """(acc, s_steps) of the Euler chain in the precision of P (Model.forward_sf_net_multi_step with every step exposed)"""
    from oracle import sf_mlp
    s_all, p, t = [], P, ts
    for _ in range(n_eval):
        s = sf_mlp.sf_net(p, t, layers, **kw)
        s_all.append(s)
        p, t = p + s, t + dt
    return sum(s_all[:n_acc]), torch.stack(s_all)


def _band(ref, cap, b, opt, steps, dt, warm, sd_m, n_eval):
    """Kink band from reference A: (pixels of dL/dd1 [B,H,W], elements of dL/dd2 [B,H,W], pixels of dL/dP1 [B,H,W])."""
    from oracle import sf_mlp
    r, sf = ref['r'], ref['sf']
    d1 = cap.t['d1'].double()[:, 0]
    B, H, W = d1.shape
    flow = b['flow_1_2'].permute(0, 3, 1, 2)
    za, zb = r['p1_camera_2'][:, 2], r['warped_p2_camera_2'][:, 2]
    # the flow term reaches d1 only (through P1 + sf); the others reach d2 as well
    loss_band = torch.zeros(B, H, W, dtype=torch.bool, device=d1.device)
    if opt.use_disp:
        a, c = za.clamp(min=1e-3), zb.clamp(min=1e-3)
        loss_band |= (a - c).abs() < DELTA_DISP * torch.maximum(a, c)
    else:
        e = r['sf_by_depth'] - sf
        loss_band |= (e.abs() < DELTA_SF * float(r['sf_by_depth'].abs().max())).any(1)
    for z in (za, zb):
        loss_band |= (z - 1e-3).abs() < DELTA_EDGE * 1e-3
    if opt.midas:
        for z in (d1, zb):
            loss_band |= (z - 100).abs() < DELTA_EDGE * 100
    layers = sf_mlp.layers_from_state_dict({k: v.cuda().double() for k, v in sd_m.items()})
    kw = _kw(opt)
    P1, ts1 = cap.t['P1'].double(), b['time_stamp_1']
    mlp_band = sf_mlp.kink_band(P1, ts1, dt, n_eval, layers, width=KINK_WIDTH, **kw)
    if _use_reg(opt, warm):
        with torch.no_grad():
            _, s = _chain64(P1, ts1, dt, 2, 1, layers, kw)
        mlp_band |= ((s[1] - s[0]).abs() < DELTA_S * float(s[0].abs().max())).any(1)
    # dL/dd2 of a band pixel lands on its four bilinear taps
    ys, xs = torch.meshgrid(torch.arange(H, device=d1.device), torch.arange(W, device=d1.device), indexing='ij')
    ix = (xs + b['flow_1_2'][..., 0]).clamp(0, W - 1)
    iy = (ys + b['flow_1_2'][..., 1]).clamp(0, H - 1)
    x0, y0 = ix.floor().long(), iy.floor().long()
    d2_band = torch.zeros(B, H * W, dtype=torch.bool, device=d1.device)
    bi = torch.arange(B, device=d1.device).view(B, 1, 1).expand(B, H, W)
    for xx in (x0, (x0 + 1).clamp(max=W - 1)):
        for yy in (y0, (y0 + 1).clamp(max=H - 1)):
            idx = (yy * W + xx)[loss_band]
            d2_band[bi[loss_band], idx] = True
    flow_band = ((r['dflow_1_2'] - flow).abs() < DELTA_FLOW).any(1) if not warm else torch.zeros_like(loss_band)
    return loss_band | flow_band | mlp_band, d2_band.view(B, H, W), mlp_band


def _agree(g, ref, band=None):
    """(|slope - 1|, relative L2, max-norm) over all elements; the max-norm outside `band` if given"""
    slope, l2, mx = grad_agreement(g, ref)
    if band is not None:
        a = g.detach().double().reshape(band.shape[0], -1, *band.shape[1:])
        b_ = ref.detach().double().reshape(a.shape)
        keep = ~band.unsqueeze(1).expand_as(a)
        mx = float((a - b_).abs()[keep].max() / b_.abs().max())
    return abs(slope), l2, mx


def _effect(bad, good, keys):
    """largest (metric / its bound) by which a defective reference result differs from the honest one, and where"""
    best = (0.0, None)
    for k, (sb, lb, mb) in keys.items():
        a, r = (bad[k], good[k]) if not k.startswith('mlp.') else (bad['mlp'][k[4:]], good['mlp'][k[4:]])
        m = _agree(a, r)
        for v, bound, what in zip(m, (sb, lb, mb), ('slope', 'L2', 'max')):
            if v / bound > best[0]:
                best = (v / bound, '%s %s %.2e' % (k, what, v))
    return best


def _run_case(c, emu, monkeypatch):
    from dvd_b200 import ops, synthetic
    from oracle import reproject_fp32 as R
    from oracle import sf_mlp
    model, opt, sd_d, sd_m = _build(dict(lr=1e-4, cuda_graph=False, **c['over']))
    B, H, W = len(c['pairs']), c['H'], c['W']
    batch = synthetic.make_batch(c['pairs'], H=H, W=W, seed=11, smooth_flow=True, flow_sigma=2.0)
    batch['motion_seg_1'] = (torch.rand(batch['motion_seg_1'].shape, generator=torch.Generator().manual_seed(5)) > 0.3).float()
    epoch = c['epoch']
    warm = epoch <= opt.warm_sf
    cap = _Capture(model, monkeypatch)
    log = model._train_on_batch(epoch, 0, batch)
    torch.cuda.synchronize()
    monkeypatch.undo()
    steps, dt = model.steps, float(batch['time_step'].reshape(-1)[0])
    use_reg = _use_reg(opt, warm)
    n_eval = max(steps, 2) if use_reg else steps
    depth_grads = not warm
    b = {k: v.squeeze(0).cuda() for k, v in batch.items() if torch.is_tensor(v) and v.dim() > 1}
    b64 = {k: v.double() for k, v in b.items()}
    meas, teeth = {}, {}

    # ---- .grad holds the pre-Adam gradients
    for k, p in model.net_sceneflow.named_parameters():
        assert torch.equal(p.grad, cap.g['mlp.' + k]), k
    nets = [('mlp', model.net_sceneflow, sd_m)] + ([('depth', model.net_depth, sd_d)] if depth_grads else [])
    for name, net, sd in nets:
        moved = n = 0
        for k, p in net.named_parameters():
            d = p.detach() - sd[k].cuda()
            assert not bool(((d != 0) & ~(d * p.grad < 0)).any()), (name, k)
            moved, n = moved + int((d != 0).sum()), n + d.numel()
        assert moved > 0.5 * n, (name, moved, n)
    if warm:
        for k, p in model.net_depth.named_parameters():
            assert torch.equal(p.detach().cpu(), sd_d[k]), k

    # ---- reference B, loss -> MLP: dL/dacc bit for bit
    A = emu
    poses = ops.pack_poses_from_batch(b)
    assert torch.equal(poses, cap.t['poses'])
    ms = b['motion_seg_1'].reshape(B, 1, H, W).cpu().numpy()
    acc = cap.t['acc'].cpu().numpy()
    sf = acc * ms if opt.use_motion_seg else acc
    cfg = R.cfg_dict(opt.midas, warm, 0 if opt.use_disp else (1 if opt.use_disp_ratio else 2), opt.use_disp, opt.flow_mul,
                     opt.disp_mul)
    ps = R.derive_pose(A, poses.cpu().numpy())
    f = R.loss_forward(A, cfg, ps, cap.t['d1'][:, 0].cpu().numpy(), cap.t['d2'][:, 0].cpu().numpy(),
                       b['flow_1_2'].cpu().numpy(), b['mask_2'].reshape(B, H, W).cpu().numpy(), sf)
    gs = np.float32(np.float32(steps if opt.weight_steps else 1.0) * np.float32(1.0))
    gv, _ = R.pixel_backward(A, cfg, ps, f['o'], f['m'], np.float32(f['scalars']['cf'] * gs),
                             np.float32(f['scalars']['cd'] * gs))
    want = np.stack(gv, 1)
    if opt.use_motion_seg:
        want = want * ms
    got = cap.g['acc'].cpu().numpy()
    n_bits = int((got.view(np.int32) != np.ascontiguousarray(want, np.float32).view(np.int32)).sum())
    assert n_bits == 0, ('dL/dacc bits', n_bits)

    # ---- reference A
    torch.cuda.reset_peak_memory_stats()
    ref = _reference_a(cap, b64, opt, steps, dt, warm, sd_m)
    d1_band, d2_band, mlp_band = _band(ref, cap, b64, opt, steps, dt, warm, sd_m, n_eval)
    meas['band_d1'], meas['band_d2'], meas['band_mlp'] = (float(x.double().mean()) for x in (d1_band, d2_band, mlp_band))
    meas['loss_rel'] = max(abs(log[k] - v) / max(abs(v), 1e-30) for k, v in ref['losses'].items() if (k != 'acc_reg' or use_reg))
    keys = {}
    if depth_grads:
        for k, g, band in (('g_d1', cap.g['d1'], d1_band), ('g_d2', cap.g['d2'], d2_band)):
            meas[k] = _agree(g, ref[k], band)
            meas[k + '_max_all'] = _agree(g, ref[k])[2]
            keys[k] = (D_SLOPE, D_L2, D_MAX)
    mlp = [_agree(p.grad, ref['mlp'][k]) for k, p in model.net_sceneflow.named_parameters()]
    meas['mlp'] = tuple(max(m[i] for m in mlp) for i in range(3))
    keys.update({'mlp.' + k: (MLP_SLOPE, MLP_L2, MLP_MAX) for k in ref['mlp']})

    # ---- reference B, MLP -> depth: dL/dP1 as the fp64 VJP of the chain
    if depth_grads:
        assert torch.equal(cap.g['P1'], cap.g['p0'])
    layers = sf_mlp.layers_from_state_dict({k: v.cuda().double() for k, v in sd_m.items()})
    P = cap.t['P1'].double().requires_grad_()
    a64, s64 = _chain64(P, b64['time_stamp_1'], dt, n_eval, steps, layers, _kw(opt))
    g_steps = cap.g.get('s_steps', torch.zeros_like(cap.t['s_steps']))
    ((a64 * cap.g['acc'].double()).sum() + (s64 * g_steps.double()).sum()).backward()
    meas['g_P1'] = _agree(cap.g['p0'], P.grad, mlp_band)
    meas['g_P1_max_all'] = _agree(cap.g['p0'], P.grad)[2]
    del a64, s64, P

    # ---- teeth: defects planted in reference A
    defects = ['scale']
    if depth_grads:
        defects += ['detach_p1', 'swap_halves', 'roll_pairs']
    if use_reg:
        defects.append('no_reg')
    if opt.weight_steps and steps != 1:
        defects.append('no_gscale')
    if opt.use_motion_seg:
        defects.append('no_mseg_bwd')
    for d in defects:
        if d == 'scale':
            bad = {'g_d1': ref['g_d1'] * 1.01 if depth_grads else None, 'g_d2': ref['g_d2'] * 1.01 if depth_grads else None,
                   'mlp': {k: v * 1.01 for k, v in ref['mlp'].items()}}
        elif d == 'swap_halves':
            bad = dict(ref, g_d1=ref['g_d2'], g_d2=ref['g_d1'])
        elif d == 'roll_pairs':
            bad = dict(ref, g_d1=ref['g_d1'].roll(1, 0), g_d2=ref['g_d2'].roll(1, 0))
        else:
            bad = _reference_a(cap, b64, opt, steps, dt, warm, sd_m, defect=d)
        teeth[d] = _effect(bad, ref, keys)
        del bad
    meas['peak_gb'] = torch.cuda.max_memory_allocated() / 2 ** 30

    print('\n[%s] steps %d, n_eval %d, losses %s' % (c.get('name'), steps, n_eval,
                                                     ' '.join('%s=%.6g' % (k, log[k]) for k in sorted(ref['losses']))))
    print('  measured (|slope-1|, rel L2, max-norm outside the band): %s' % ' '.join(
        '%s=%s' % (k, ('(%.2e, %.2e, %.2e)' % v) if isinstance(v, tuple) else '%.2e' % v) for k, v in sorted(meas.items())))
    print('  defects (effect / bound, where): %s' % ' '.join('%s=%.1f [%s]' % (k, v[0], v[1]) for k, v in teeth.items()))

    # ---- the depth net's parameter gradients: the engine emulation fed the step's cotangent
    if opt.midas and depth_grads:
        del ref
        A_eng, images = cap.engine
        cap.engine = None
        x = torch.cat([b['img_1'], b['img_2']], 0)
        check_engine_against_emulation(sd_d, x, torch.cat([cap.t['d1'], cap.t['d2']], 0),
                                       torch.cat([cap.g['d1'], cap.g['d2']], 0), A_eng, images,
                                       {k: p.grad for k, p in model.net_depth.named_parameters()}, c.get('name'))

    # ---- bounds
    bad = [(k, meas[k], lim) for k, lim in (('band_d1', BAND_SHARE), ('band_d2', BAND_SHARE), ('band_mlp', BAND_SHARE),
                                            ('loss_rel', LOSS_REL)) if meas[k] > lim]
    for k, lims in (('g_d1', (D_SLOPE, D_L2, D_MAX)), ('g_d2', (D_SLOPE, D_L2, D_MAX)), ('mlp', (MLP_SLOPE, MLP_L2, MLP_MAX)),
                    ('g_P1', (P1_SLOPE, P1_L2, P1_MAX))):
        if k in meas:
            bad += [(k, what, v, lim) for v, lim, what in zip(meas[k], lims, ('slope', 'L2', 'max')) if v > lim]
    assert not bad, bad
    bad = [(d, v) for d, v in teeth.items() if v[0] < MARGIN and (c['name'], d) not in WEAK]
    assert not bad, bad


@pytest.mark.parametrize('name', list(CASES))
def test_step_cotangents_match_fp64(name, emu, monkeypatch):   # noqa: F811
    monkeypatch.delenv('DVD_BWD_OVERLAP', raising=False)
    _run_case(dict(CASES[name], name=name), emu, monkeypatch)


@pytest.mark.timeout(1200)
def test_step_cotangents_match_fp64_at_bench_resolution(emu, monkeypatch):   # noqa: F811
    """4 pairs at 224 x 384, gap 1: 8 images through the depth net, whose fp64 emulation needs 17-19 GB."""
    monkeypatch.delenv('DVD_BWD_OVERLAP', raising=False)
    _run_case(dict(BENCH_CASE, name='joint-4x224x384-gap1'), emu, monkeypatch)
