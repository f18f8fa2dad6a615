"""Cost of the ordered reductions that torch.use_deterministic_algorithms(True) selects (DESIGN.md 2.11).

One call on one GPU reports, as one JSON object:
  * the card: name, power limit and maximum SM clock (nvidia-smi, read in the same call);
  * whole steps at 384x224 with 1 and 8 pairs per step, bench.py's gap cycle 8, 6, 4, 2, 1, step graphs on: every gap is
    warmed up (two eager steps and the capture) in both modes, then timed rounds alternate between the modes; step time is
    a host clock around `--steps` steps ending in a device synchronise, frame-pairs/s = pairs * steps / time;
  * per site, the ordered launch against the atomic one on the same inputs: CUDA events around `--launches` back-to-back calls
    of the Python wrapper, after a warm-up (the conv rows are single layers of an 8-pair step);
  * the workspace bytes of every site, and the per-call sort buffers of the re-projection backward at 1 and 8 pairs.

Usage: python tools/bench_deterministic.py [--steps 10] [--rounds 3] [--launches 50]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, N_FRAMES, GAPS = 224, 384, 80, (8, 6, 4, 2, 1)


@contextlib.contextmanager
def mode(flag):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(flag)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().split(',')]
    return {'name': name, 'power_limit': power, 'max_sm_clock': clock}


def steps_arm(B, n_steps, rounds):
    from dvd_b200 import synthetic
    from dvd_b200.models import get_model
    dev = torch.device('cuda:0')
    opt = synthetic.default_opt()
    model = get_model('scene_flow_motion_field')(opt, None)
    synthetic.seed_net_(model.net_depth, 0, 2000.0)
    synthetic.seed_net_(model.net_sceneflow, 1)
    model.to(dev)
    epoch = opt.warm_sf + 1
    batches = {}
    for gi, gap in enumerate(GAPS):
        pairs = [((5 * gi + j) % (N_FRAMES - 1 - gap), (5 * gi + j) % (N_FRAMES - 1 - gap) + gap) for j in range(B)]
        hb = synthetic.make_batch(pairs, H=H, W=W, n_frames=N_FRAMES, seed=gi)
        batches[gap] = {k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in hb.items()}
    for flag in (False, True):               # two eager steps and the capture of every gap, in both modes
        with mode(flag):
            for _ in range(3):
                for gap in GAPS:
                    model._train_on_batch(epoch, 0, batches[gap])
    torch.cuda.synchronize()
    assert not getattr(model, '_graph_broken', False), getattr(model, 'graph_error', None)
    res = {False: [], True: []}
    for _ in range(rounds):
        for flag in (False, True):
            with mode(flag):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(n_steps):
                    model._train_on_batch(epoch, 0, batches[GAPS[i % len(GAPS)]])
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
            res[flag].append({'step_ms': 1e3 * dt / n_steps, 'pairs_per_s': B * n_steps / dt})
    return {'default': res[False], 'ordered': res[True], 'graph_stats': dict(model.graph_stats)}


def ev_ms(fn, n):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def sites(n):
    from dvd_b200 import conv_ops as co, ops
    from oracle import sf_mlp
    dev = torch.device('cuda:0')
    g = torch.Generator(device='cuda').manual_seed(0)
    cl = torch.channels_last
    out = {}

    def both(name, fn):
        t = {}
        for flag in (False, True, False, True):
            with mode(flag):
                t.setdefault('ordered_ms' if flag else 'atomic_ms', []).append(ev_ms(fn, n))
        out[name] = {k: min(v) for k, v in t.items()}

    # depth-net weight gradients of an 8-pair step (16 images)
    for (N, h, w, ci, co_, k, groups) in [(16, 14, 24, 1024, 1024, 1, 1), (16, 56, 96, 256, 256, 3, 1), (16, 14, 24, 1024, 1024, 3, 32),
                                          (16, 112, 192, 256, 128, 3, 1), (16, 7, 12, 2048, 2048, 1, 1)]:
        conv = torch.nn.Conv2d(ci, co_, k, padding=k // 2, groups=groups, bias=False).cuda()
        bn = torch.nn.BatchNorm2d(co_).eval().cuda()
        conv.weight.grad, bn.weight.grad, bn.bias.grad = (torch.zeros_like(t) for t in (conv.weight, bn.weight, bn.bias))
        x = co.round_tf32(torch.randn(N, ci, h, w, generator=g, device=dev).contiguous(memory_format=cl))
        gm = co.round_tf32(torch.randn(N, co_, h, w, generator=g, device=dev).contiguous(memory_format=cl))
        c = co.Conv(conv, bn)
        both('conv_wgrad %dx%d %d->%d k%d g%d' % (h, w, ci, co_, k, groups), lambda c=c, x=x, gm=gm: c.wgrad(x, gm, sums=True))
    # scene-flow MLP backward (data gradient + weight gradient per evaluation), 8 pairs, 2 evaluations
    layers = sf_mlp.init_layers(seed=1)
    ws = [w_.cuda().contiguous() for w_, _ in layers]
    bs = [b_.cuda().contiguous() for _, b_ in layers]
    pk = ops.PackedMlp(ops.make_mlp_cfg(), 'cuda').refresh(ws, bs)
    p0 = (torch.randn(8, 3, H, W, generator=g, device=dev) * 3)
    t0 = torch.full((8, 1, H, W), 0.25, device=dev)
    f = ops.mlp_chain_fwd(pk, p0, t0, 1 / 80, 2, 2, save=True)
    gacc = torch.randn(8, 3, H, W, generator=g, device=dev)
    gw = [torch.zeros_like(w_) for w_ in ws]
    gb = [torch.zeros_like(b_) for b_ in bs]
    both('mlp_backward 8x224x384 2 evals', lambda: ops.mlp_chain_bwd(pk, f, t0, 1 / 80, 2, gacc, None, gw, gb))
    # re-projection backward with g_depth_2, 8 pairs and 1 pair
    from dvd_b200 import synthetic
    for B in (8, 1):
        batch = synthetic.make_batch([(j, j + 4) for j in range(B)], H=H, W=W, seed=3, leading_dim=False)
        bd = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
        poses = ops.pack_poses_from_batch(bd)
        d1, d2 = synthetic.make_depths(B, H, W, seed=1).cuda(), synthetic.make_depths(B, H, W, seed=2).cuda()
        sf = torch.randn(B, 3, H, W, generator=g, device=dev) * 0.05
        mask = bd['mask_2'].reshape(B, H, W).contiguous()
        lc = ops.make_loss_cfg()
        sc = ops.reproject_loss_fwd(d1, d2, bd['flow_1_2'], mask, sf, poses, lc)
        both('reproject_loss_bwd %dx224x384' % B, lambda d1=d1, d2=d2, bd=bd, mask=mask, sf=sf, poses=poses, lc=lc, sc=sc:
             ops.reproject_loss_bwd(d1, d2, bd['flow_1_2'], mask, sf, poses, lc, sc))
    # CUDA-core sites of an 8-pair step
    conv = torch.nn.Conv2d(3, 64, 7, 2, 3, bias=False).cuda()
    bn = torch.nn.BatchNorm2d(64).eval().cuda()
    for p in (conv.weight, bn.weight, bn.bias):
        p.grad = torch.zeros_like(p)
    x = torch.rand(16, 3, H, W, generator=g, device=dev)
    a0 = co.stem_fwd(x, conv, bn)
    ga = torch.randn(a0.shape, generator=g, device=dev).contiguous(memory_format=cl)
    both('stem_wgrad 16x224x384', lambda: co.stem_wgrad(x, ga, a0, conv, bn))
    hx = torch.relu(torch.randn(16, 32, H, W, generator=g, device=dev)).contiguous(memory_format=cl)
    hw_, hb_ = torch.randn(32, generator=g, device=dev) * 0.1, torch.full((1,), 0.5, device=dev)
    gd = torch.randn(16, 1, H, W, generator=g, device=dev)
    gw_, gb_ = torch.zeros(32, device=dev), torch.zeros(1, device=dev)
    both('head_bwd 16x224x384', lambda: co.head_bwd(hx, hw_, hb_, gd, gw_, gb_))
    gc = torch.randn(16, 256, 56, 96, generator=g, device=dev).contiguous(memory_format=cl)
    mean, var = torch.zeros(256, device=dev), torch.ones(256, device=dev)
    cs, dg = torch.zeros(256, device=dev), torch.zeros(256, device=dev)
    both('relu_bwd_colsum 16x56x96x256', lambda: co.relu_bwd_colsum(gc, colsum=cs, bn=(mean, var, 1e-5), dgamma=dg, round_out=False))
    bnh = torch.nn.BatchNorm2d(128).eval().cuda()
    xb = torch.randn(16, 128, 56, 96, generator=g, device=dev).contiguous(memory_format=cl).requires_grad_()
    gy = torch.randn(16, 128, 56, 96, generator=g, device=dev).contiguous(memory_format=cl)

    def bn_step():
        ops.bn_act(xb, bnh, None, True).backward(gy)
    both('bn_act fwd+bwd 16x56x96x128 (hourglass)', bn_step)
    return out


def workspaces():
    from dvd_b200 import _lib
    lib = _lib.load()
    names = ['conv_wgrad', 'mlp_wgrad', 'mlp_dgrad', 'channel_sums', 'stem', 'head']
    out = {n: int(lib.dvd_ordered_workspace_bytes(i)) for i, n in enumerate(names)}
    out['total_per_device'] = sum(out.values())
    for B in (1, 8):
        out['reproject_sort_per_call_%dx224x384' % B] = int(lib.dvd_reproject_ordered_bytes(B, H, W))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--launches', type=int, default=50)
    args = ap.parse_args()
    os.environ.setdefault('CUBLAS_WORKSPACE_CONFIG', ':4096:8')
    torch.cuda.set_device(0)
    res = {'card': card(), 'workspace_bytes': workspaces()}
    res['steps'] = {'%d_pairs' % B: steps_arm(B, args.steps, args.rounds) for B in (8, 1)}
    res['sites'] = sites(args.launches)
    res['card_after'] = card()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
