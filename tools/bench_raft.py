"""Timing of the RAFT forward (dvd_b200/raft.py) on the GPU, at the reference's 288x512 with seeded weights.

    python tools/bench_raft.py [--frames 80] [--gaps 8] [--iters 20] [--eager_pairs 6]

CUDA events around warmed-up work; FLOPs and bytes are computed from the layer shapes; the card's name and power limit are read
in the same run. The eager baseline is oracle/raft.py in PyTorch on the same GPU, one pair per call with both encoders
recomputed, as the reference does; it alternates with the native path. Fails without a GPU. Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps / 1e3


def iteration_flops(plan, npx):
    """FLOPs of one update iteration over npx 1/8-resolution pixels, from the layer shapes (mask head excluded: once per pair)"""
    convs = [plan.convc1, plan.convc2, plan.convf2, plan.conv_flo, plan.conv_cor, plan.fh1] + [c for pair in plan.gru for c in pair]
    f = sum(c.flops(npx) for c in convs)
    f -= 2.0 * npx * 256 * (352 - 324)                     # convc1's zero tail is not work the algorithm needs
    f -= 2.0 * npx * 2 * 256 * 9                           # nor the two pad outputs of the motion encoder's last convolution
    return f + 2.0 * npx * (128 * 2 * 49 + 2 * 256 * 9)    # convf1 and the flow head's last convolution (CUDA cores)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=80)
    ap.add_argument('--gaps', type=int, default=8)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--chunk', type=int, default=32)
    ap.add_argument('--eager_pairs', type=int, default=6)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_raft.py measures on a GPU; none is available')
    from dvd_b200 import ops, raft
    from dvd_b200.flow_pairs import finish_flows, pair_list
    from oracle import raft as oracle_raft
    H, W = 288, 512
    h, w = H // 8, W // 8
    sd = oracle_raft.seeded_state_dict(0, 0.7)
    net = raft.RaftNet()
    net.load_state_dict(sd)
    net = net.cuda()
    sdg = oracle_raft.cast(sd, torch.float32, 'cuda')
    images = torch.cat([oracle_raft.seeded_pair(H, W, s)[0] for s in range(8)]).cuda()
    res = {'gpu': torch.cuda.get_device_name(0), 'size': [H, W], 'iters': a.iters}
    q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True)
    res['power_limit_and_max_sm_clock'] = q.stdout.strip()
    res['encode_s_per_frame'] = timed(lambda: net.encode(images), 5) / len(images)
    feats = net.encode(images)
    P = net.plan()
    for B in (1, 8, 32):
        idx = [i % 8 for i in range(B)]
        fa, fb = feats.index(idx), feats.index([(i + 1) % 8 for i in idx])
        t = timed(lambda: raft.corr_pyramid(fa.fmap, fb.fmap), 10)
        npx = h * w
        pyr_bytes = 4.0 * (2 * npx * 256 + sum(npx * (h >> l) * (w >> l) * (2 if l in (1, 2) else 1) for l in range(4)) + npx * npx)
        res['corr_pyramid_B%d' % B] = {'s_per_pair': t / B, 'GB_per_s': B * pyr_bytes / t / 1e9, 'TFLOP_per_s_fp32': B * 2.0 * npx * npx * 256 / t / 1e12}
        pyr = raft.corr_pyramid(fa.fmap, fb.fmap)
        state = net.init_state(fa.cnet)
        coords1 = raft.coords_grid(B, h, w, 'cuda')
        t = timed(lambda: net.update_step(P, pyr, coords1, *state), 20)
        fl = iteration_flops(P, B * npx)
        res['update_iteration_B%d' % B] = {'s': t, 's_per_pair': t / B, 'GFLOP_per_pair': fl / B / 1e9, 'TFLOP_per_s': fl / t / 1e12}

    # the whole workload: every frame encoded once, both directions of every pair, resize to the frame size and masks
    pairs = pair_list(a.frames, range(1, a.gaps + 1))
    frames = images[[i % 8 for i in range(a.frames)]]

    def native():
        fs = [net.encode(frames[i:i + a.chunk]) for i in range(0, a.frames, a.chunk)]
        fs = raft.FrameFeatures(torch.cat([f.fmap for f in fs]), torch.cat([f.cnet for f in fs]))
        for i0 in range(0, len(pairs), a.chunk):
            pa, pb = [p[0] for p in pairs[i0:i0 + a.chunk]], [p[1] for p in pairs[i0:i0 + a.chunk]]
            fa, fb = fs.index(pa), fs.index(pb)
            finish_flows(net.flow(fa, fb, a.iters), net.flow(fb, fa, a.iters), 224, 384)

    def eager():
        with torch.no_grad():
            for k in range(a.eager_pairs):
                i1, i2 = images[k % 8:k % 8 + 1], images[(k + 1) % 8:(k + 1) % 8 + 1]
                f12 = oracle_raft.raft_forward(sdg, i1, i2, a.iters)[1].permute(0, 2, 3, 1).contiguous()
                f21 = oracle_raft.raft_forward(sdg, i2, i1, a.iters)[1].permute(0, 2, 3, 1).contiguous()
                finish_flows(f12, f21, 224, 384)
    torch.backends.cudnn.allow_tf32 = True          # the reference's own GPU path
    tn, te = [], []
    for _ in range(2):
        tn.append(timed(native, 1))
        te.append(timed(eager, 1))
    n_eval = 2 * len(pairs)
    res['workload'] = {'frames': a.frames, 'gaps': a.gaps, 'evaluations': n_eval, 'native_s': tn, 'native_evaluations_per_s': n_eval / min(tn),
                       'eager_s_for_%d_evaluations' % (2 * a.eager_pairs): te, 'eager_evaluations_per_s': 2 * a.eager_pairs / min(te)}
    res['speedup_over_eager'] = res['workload']['native_evaluations_per_s'] / res['workload']['eager_evaluations_per_s']
    print(json.dumps(res))


if __name__ == '__main__':
    main()
