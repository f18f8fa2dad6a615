"""Point-cloud export (dvd_b200.points, csrc/points.cu): device time per stage for a whole video, against the numpy oracle.

    python tools/bench_points.py [--configs 200x288x512,80x224x384] [--skip_cpu] [--out results/points.json]

Per configuration (frames x H x W), synthetic frames are built on the device (smooth depth in [2, 8] with a 5 % step edge,
random colours, the synthetic cameras). After a warm-up pass, CUDA events time one pass over all frames at once: the
unprojection, dvd_points_select, the stable key sort, dvd_voxel_reduce; then the D2H copy of the fused cloud and the PLY write
(host clocks). The selection and the reduction wait for their counts, so their times include one stream synchronisation.
GB/s is the compulsory traffic stated below divided by the stage's time, next to the 3.35 TB/s data-sheet HBM3 peak of an H100
SXM. The CPU column is oracle/points.py (numpy) on the same fp32 points: selection with keys, then the reduction.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK_GBS = 3350.0


def frames(N, H, W, dev):
    from dvd_b200 import points, synthetic
    depth = synthetic.make_depths(N, H, W, seed=1).to(dev)[:, 0].contiguous()
    depth[:, :, W // 2:] *= 1.05
    img = torch.rand(N, 3, H, W, generator=torch.Generator().manual_seed(2)).to(dev)
    K, c2w = [], []
    for i in range(N):
        R, t, k = synthetic.camera(i, H, W)
        m = np.eye(4)
        m[:3, :3], m[:3, 3] = R.numpy(), t.numpy()
        K.append(k.numpy()), c2w.append(m)
    K, c2w = np.stack(K).astype(np.float32), np.stack(c2w).astype(np.float32)
    return depth, img, K, c2w, torch.from_numpy(points.camera_block(K, c2w)).to(dev)


def one_pass(depth, img, cam, voxel, origin):
    from dvd_b200 import ops, points
    N, H, W = depth.shape
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    torch.cuda.synchronize()
    ev[0].record()
    P = points.world_points(depth, cam)
    ev[1].record()
    sel = ops.points_select(depth, img, P, points.EDGE_TOL, voxel, origin)
    ev[2].record()
    skey, order = torch.sort(sel['key'], stable=True)
    ev[3].record()
    res = ops.voxel_reduce(skey, order, sel['index'], sel['xyz'], sel['rgb'], H * W, 2)
    ev[4].record()
    torch.cuda.synchronize()
    ms = [ev[i].elapsed_time(ev[i + 1]) for i in range(4)]
    return ms, sel, res, P


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--configs', default='200x288x512,80x224x384')
    p.add_argument('--skip_cpu', action='store_true')
    p.add_argument('--out', default=None)
    a = p.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    from dvd_b200 import points
    from oracle import points as op
    res = dict(gpu=torch.cuda.get_device_name(0), peak_gbs=PEAK_GBS, runs=[])
    try:
        res['nvidia_smi'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm,clocks.sm,clocks.mem',
                                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        res['nvidia_smi'] = repr(e)
    dev = torch.device('cuda')
    for cfg in a.configs.split(','):
        N, H, W = (int(x) for x in cfg.split('x'))
        depth, img, K, c2w, cam = frames(N, H, W, dev)
        voxel = points.default_voxel(depth.cpu().numpy())
        origin = points.default_origin(c2w, voxel)
        one_pass(depth, img, cam, voxel, origin)                              # warm-up: allocator, sort plan
        best = None
        for _ in range(3):
            ms, sel, red, P = one_pass(depth, img, cam, voxel, origin)
            best = ms if best is None else [min(x, y) for x, y in zip(best, ms)]
        n, M, R = N * H * W, sel['index'].numel(), red['count'].numel()
        t0 = time.perf_counter()
        xyz, rgb = red['xyz'].cpu().numpy(), red['rgb'].cpu().numpy()
        t1 = time.perf_counter()
        with tempfile.TemporaryDirectory() as tmp:
            points.write_ply(os.path.join(tmp, 's.ply'), xyz, points.mean_rgb_to_u8(rgb))
        t2 = time.perf_counter()
        # compulsory traffic: select reads depth twice (count + scatter), writes the mask, and per kept pixel reads P and img
        # and writes key, index, xyz, rgb; reduce reads the keys twice, per point order + index (views) and order + xyz + rgb
        # (sums), and writes run starts and the R kept runs
        sel_bytes = n * (4 + 4 + 1) + M * (12 + 12 + 8 + 8 + 12 + 3)
        red_bytes = M * (8 + 8 + 8 + 8 + 8 + 12 + 3) + R * (8 * 6 + 4 + 4)
        run = dict(frames=N, H=H, W=W, pixels=n, kept=M, voxels=R, voxel=voxel, unproject_ms=best[0], select_ms=best[1],
                   sort_ms=best[2], reduce_ms=best[3], device_ms=sum(best), d2h_ms=1e3 * (t1 - t0), ply_ms=1e3 * (t2 - t1),
                   select_gbs=sel_bytes / best[1] / 1e6, reduce_gbs=red_bytes / best[3] / 1e6)
        if not a.skip_cpu:
            dh, ih, Ph = depth.cpu().numpy(), img.cpu().numpy(), P.cpu().numpy()
            t0 = time.perf_counter()
            s = op.select(dh, ih, Ph, points.EDGE_TOL, voxel, origin)
            t1 = time.perf_counter()
            r = op.reduce(s['key'], s['index'], s['xyz'], s['rgb'], H * W, 2)
            t2 = time.perf_counter()
            run.update(cpu_select_s=t1 - t0, cpu_reduce_s=t2 - t1, cpu_s=t2 - t0,
                       cpu_equal=bool(np.array_equal(r['xyz'], xyz) and np.array_equal(r['views'], red['views'].cpu().numpy())))
        res['runs'].append(run)
        print(json.dumps(run), flush=True)
        del depth, img, cam, sel, red, P
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
