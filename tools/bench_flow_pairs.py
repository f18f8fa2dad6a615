"""Throughput of the flow-pair kernels and wall time of preparing a whole video's pairs.

  kernels   dvd_flow_resize_cubic (64 pairs, 288x512 -> 224x384, the RAFT size to the working size) and dvd_flow_pair_masks
            (64 pairs of 224x384, both conventions): CUDA events over many launches, GB/s from the algorithmic traffic
            (DESIGN.md §2.4: resize 8 h w / (H W) B read + 8 B written per output pixel; masks 16 B read + 2 B (uint8) or 8 B
            (fp32) written per pixel) against the card's HBM3 peak. 64 pairs of flows are 44 MB per direction, more than
            twice the 50 MB L2.
  video     every pair of an 80-frame video at gaps 1-8 (596 pairs): raw 288x512 flows of one gap per call to
            flow_pairs.process_raw_flows (host -> device, resize, masks, device -> host), against the reference's per-pair CPU
            path (cv2.resize + F.grid_sample + numpy, generate_flows.py:44-82,139-148, restated here) timed on a subset of
            pairs and scaled to 596, on the host's cores (count printed).

Prints one JSON object (and writes it to --json PATH when given). Needs a GPU.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12      # H100 SXM data sheet, bytes/s


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:       # noqa: BLE001 - informational only
        return 'unknown (%s)' % e


def time_launches(fn, iters=200, warmup=20):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = []
    for _ in range(3):
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        best.append(e0.elapsed_time(e1) / iters * 1e-3)
    return min(best), max(best)


def smooth_flows(B, h, w, g, seed):
    gen = torch.Generator(device='cuda').manual_seed(seed)
    lo = torch.randn(B, 2, 9, 16, device='cuda', generator=gen) * 3
    f12 = F.interpolate(lo, size=(h, w), mode='bilinear', align_corners=False).permute(0, 2, 3, 1).contiguous()
    f21 = -f12 + torch.randn(f12.shape, device='cuda', generator=gen) * 0.3
    return f12, f21.contiguous()


def reference_cpu_pair(f12, f21, H, W, resize):
    """the reference's per-pair CPU path: resize both flows, then backward warp + L2 error + out-of-bounds masks"""
    def warp(im2, fl):
        h, w, _ = im2.shape
        hh, ww = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing='ij')
        grid = torch.stack([ww, hh], -1)[None] + torch.from_numpy(fl)[None]
        grid[..., 0] /= (w - 1) / 2
        grid[..., 1] /= (h - 1) / 2
        grid -= 1
        out = F.grid_sample(torch.from_numpy(im2).permute(2, 0, 1)[None], grid, align_corners=True)
        return out[0].permute(1, 2, 0).numpy()

    def oob(fl):
        h, w, _ = fl.shape
        hh, ww = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing='ij')
        tx, ty = ww + fl[..., 0], hh + fl[..., 1]
        return ((tx < 0) | (tx > w - 1) | (ty < 0) | (ty > h - 1)).astype(np.float32)
    a, b = resize(f12, H, W), resize(f21, H, W)
    m1 = np.clip(np.where(np.linalg.norm(warp(a, b) + b, axis=-1) > 1, 1, 0) + oob(b), 0, 1)
    m2 = np.clip(np.where(np.linalg.norm(warp(b, a) + a, axis=-1) > 1, 1, 0) + oob(a), 0, 1)
    return a, b, m1.astype(np.uint8), m2.astype(np.uint8)


def main():
    import argparse
    ap = argparse.ArgumentParser(description='flow-pair kernel throughput and whole-video preparation time')
    ap.add_argument('--json', default=None, help='also write the results to this file')
    args = ap.parse_args()
    from dvd_b200 import ops
    from dvd_b200.flow_pairs import pair_list, process_raw_flows
    assert torch.cuda.is_available(), 'bench_flow_pairs needs a GPU'
    res = {'gpu': gpu_info(), 'host_cores': os.cpu_count(), 'torch_threads': torch.get_num_threads()}
    B, h, w, H, W = 64, 288, 512, 224, 384
    f12, f21 = smooth_flows(B, H, W, 1, 0)
    raw, _ = smooth_flows(B, h, w, 1, 1)
    t_lo, t_hi = time_launches(lambda: ops.flow_resize_cubic(raw, H, W))
    npx = B * H * W
    by = npx * (8.0 * h * w / (H * W) + 8)
    res['resize'] = {'ms': [t_lo * 1e3, t_hi * 1e3], 'GBps': by / t_lo / 1e9, 'of_hbm_peak': by / t_lo / HBM_PEAK}
    for conv, wb in (('flowpair', 2), ('pair_file', 8)):
        t_lo, t_hi = time_launches(lambda: ops.flow_pair_masks(f12, f21, convention=conv))
        by = npx * (16.0 + wb)
        res['masks_' + conv] = {'ms': [t_lo * 1e3, t_hi * 1e3], 'GBps': by / t_lo / 1e9, 'of_hbm_peak': by / t_lo / HBM_PEAK}
    # an 80-frame video, gaps 1-8: all pairs of one gap per call, host arrays in and out
    n_frames, gaps = 80, list(range(1, 9))
    pairs = pair_list(n_frames, gaps)
    per_gap = {g: sum(1 for p in pairs if p[1] - p[0] == g) for g in gaps}
    r12, r21 = smooth_flows(max(per_gap.values()), h, w, 1, 2)
    r12, r21 = r12.cpu().numpy(), r21.cpu().numpy()
    process_raw_flows(r12[:4], r21[:4], H, W)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for g in gaps:
        process_raw_flows(r12[:per_gap[g]], r21[:per_gap[g]], H, W)
    torch.cuda.synchronize()
    gpu_s = time.perf_counter() - t0
    try:
        import cv2

        def resize(fl, Ho, Wo):
            out = cv2.resize(fl, dsize=(Wo, Ho), interpolation=cv2.INTER_CUBIC)
            out *= np.array((Wo / float(fl.shape[1]), Ho / float(fl.shape[0]))).reshape(1, 1, -1)
            return out
        resizer = 'cv2'
    except ImportError:
        from oracle.flow_pairs import resize_flow_cubic as resize
        resizer = 'numpy restatement (cv2 not installed)'
    n_cpu = 12
    reference_cpu_pair(r12[0], r21[0], H, W, resize)
    t0 = time.perf_counter()
    for j in range(n_cpu):
        reference_cpu_pair(r12[j], r21[j], H, W, resize)
    cpu_pair_s = (time.perf_counter() - t0) / n_cpu
    res['video'] = {'frames': n_frames, 'pairs': len(pairs), 'gpu_s': gpu_s, 'cpu_reference_s_per_pair': cpu_pair_s,
                    'cpu_reference_s_scaled': cpu_pair_s * len(pairs), 'cpu_pairs_timed': n_cpu, 'cpu_resize': resizer,
                    'speedup': cpu_pair_s * len(pairs) / gpu_s}
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
