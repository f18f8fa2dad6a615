"""COLMAP frame preparation (dvd_b200.frames.read_colmap_model, ColmapFrameBuilder's calibration): the host time to read a
binary sparse model, and the device time of the scale calibration per video, at two model sizes.

    python tools/bench_prepare_colmap.py [--frames 80] [--points 50000,500000] [--memory_frames 200] [--out results/colmap.json]

Per point count V, a binary model of --frames registered 1080x1920 images (one PINHOLE camera, 2000 2-D points per image, a
3-image track per point) is written to a temporary directory and read three times (the best is kept). The calibration is
the one FrameBuilder._run makes, on synthetic full-resolution depth and mask maps already on the device: per chunk of 8 the
two spline prefilters and dvd_calib_ratios, then the row medians over [frames, V]; CUDA events, after a warm-up pass. Last,
the medians of a [--memory_frames, max V] ratio buffer: their time and the peak device memory, the bound the builder's
docstring states.
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

H, W, CHUNK = 1080, 1920, 8


def write_model(d, n, V, seed=0):
    g = np.random.default_rng(seed)
    fx = 1.1 * W
    with open(os.path.join(d, 'cameras.bin'), 'wb') as f:
        f.write(np.uint64(1).tobytes())
        f.write(np.array([1, 1], '<i4').tobytes() + np.array([W, H], '<u8').tobytes() +
                np.array([fx, fx, W / 2, H / 2], '<f8').tobytes())
    p2d = np.zeros(2000, [('xy', '<f8', 2), ('id', '<i8')])
    p2d['xy'] = g.uniform(0, W, (2000, 2))
    p2d['id'] = g.integers(1, V + 1, 2000)
    with open(os.path.join(d, 'images.bin'), 'wb') as f:
        f.write(np.uint64(n).tobytes())
        for i in range(n):
            f.write(np.array([i + 1], '<i4').tobytes() + np.array([1, 0, 0, 0, -0.02 * i, 0, 0], '<f8').tobytes() +
                    np.array([1], '<i4').tobytes() + b'%05d.jpg\0' % i + np.uint64(len(p2d)).tobytes() + p2d.tobytes())
    rec = np.zeros(V, [('id', '<u8'), ('xyz', '<f8', 3), ('rgb', 'u1', 3), ('err', '<f8'), ('n', '<u8'), ('track', '<i4', (3, 2))])
    rec['id'] = g.permutation(V) + 1
    rec['xyz'] = np.stack([g.uniform(-6, 6, V), g.uniform(-3.5, 3.5, V), g.uniform(2, 12, V)], 1)
    rec['n'] = 3
    rec['track'][:, :, 0] = g.integers(1, n + 1, (V, 3))
    with open(os.path.join(d, 'points3D.bin'), 'wb') as f:
        f.write(np.uint64(V).tobytes() + rec.tobytes())


def maps(dev, n, f0):
    yy = torch.arange(H, device=dev, dtype=torch.float32)[:, None]
    xx = torch.arange(W, device=dev, dtype=torch.float32)[None]
    f = torch.arange(f0, f0 + n, device=dev, dtype=torch.float32)[:, None, None]
    depth = 3 + torch.sin(xx / 90 + 0.1 * f) * torch.cos(yy / 70)
    mask = ((xx > 700 + 4 * f) & (xx < 1200 + 4 * f) & (yy > 300) & (yy < 700)).float()
    return depth.contiguous(), mask.contiguous()


def calibration(ops, K, E, h_pt, dev):
    """ms of the prefilters and selection over all chunks, and of the medians"""
    N, V = E.shape[0], h_pt.shape[1]
    pts = torch.from_numpy(np.ascontiguousarray(h_pt[:3].T)).to(dev)
    w2c = torch.from_numpy(np.ascontiguousarray(E)).to(dev)
    ratio = torch.empty(N, V, dtype=torch.float64, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    t_sel = 0.0
    for a in range(0, N, CHUNK):
        depth, mask = maps(dev, min(CHUNK, N - a), a)
        torch.cuda.synchronize()
        ev[0].record()
        ops.calib_ratios(ops.spline_prefilter(depth), ops.spline_prefilter(mask), w2c[a:a + CHUNK], pts, K[0, 0], K[1, 1],
                         K[0, 2], K[1, 2], out=ratio[a:a + CHUNK])
        ev[1].record()
        torch.cuda.synchronize()
        t_sel += ev[0].elapsed_time(ev[1])
    ev[2].record()
    med, cnt = ops.row_medians(ratio)
    ev[3].record()
    torch.cuda.synchronize()
    return t_sel, ev[2].elapsed_time(ev[3]), cnt.cpu().numpy()


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--frames', type=int, default=80)
    p.add_argument('--points', default='50000,500000')
    p.add_argument('--memory_frames', type=int, default=200)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    from dvd_b200 import frames as fr, ops
    res = dict(gpu=torch.cuda.get_device_name(0), frames=a.frames, size=[H, W])
    try:
        res['nvidia_smi'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        res['nvidia_smi'] = repr(e)
    dev = torch.device('cuda')
    res['models'] = []
    for V in (int(v) for v in a.points.split(',')):
        with tempfile.TemporaryDirectory() as tmp:
            write_model(tmp, a.frames, V)
            size = sum(os.path.getsize(os.path.join(tmp, f)) for f in os.listdir(tmp))
            reads = []
            for _ in range(3):
                t0 = time.perf_counter()
                K, names, E, h_pt = fr.read_colmap_model(tmp)
                reads.append(time.perf_counter() - t0)
        calibration(ops, K, E, h_pt, dev)                                         # warm-up: allocator, sort plan
        sel_ms, med_ms, cnt = calibration(ops, K, E, h_pt, dev)
        res['models'].append(dict(points=V, model_mb=size / 1e6, read_s=min(reads), selection_ms=sel_ms, medians_ms=med_ms,
                                  calibration_ms=sel_ms + med_ms, selected_per_frame=float(cnt.mean())))
    V = h_pt.shape[1]
    ratio = torch.rand(a.memory_frames, V, dtype=torch.float64, device=dev)
    ratio[ratio < 0.3] = float('nan')
    ops.row_medians(ratio)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    ops.row_medians(ratio)
    ev[1].record()
    torch.cuda.synchronize()
    res['medians_at_scale'] = dict(frames=a.memory_frames, points=V, ratio_gb=ratio.numel() * 8 / 1e9,
                                   sort_extra_gb=(torch.cuda.max_memory_allocated() - base) / 1e9,
                                   ms=ev[0].elapsed_time(ev[1]))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
