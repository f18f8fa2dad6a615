"""Evaluation of a test export (dvd_b200.evaluate, csrc/depth_metrics.cu): per-kernel times for a whole video, bytes moved
against the HBM bound, and one whole command with its file reading shown apart.

    python tools/bench_evaluate.py [--configs 200x224x384,200x448x768] [--gaps 1,2,4,8] [--e2e 200x224x384] [--out FILE.json]

Kernels. Per configuration (frames x H x W) the three depth maps and, for every pair of the gaps, flow_1_2 and mask_2 are
seeded on the device and stay resident. After a warm-up, CUDA events time, best of 5: the four masked selections of the
accuracy pass (median of depth_gt and of each source, per frame and pooled), dvd_depth_metrics over all frames, and
dvd_pair_consistency over all pairs in launches of 64 pairs. Bytes are the compulsory traffic from the shapes: a selection
reads its two maps once per radix pass (4 passes, 8 B per pixel each); the metrics read 12 B per pixel; the consistency reads
per pixel pair 8 B of flow, 1 B of mask, 1 B of motion_seg and 4 B of D_a and of D_b per source (26 B; the four bilinear taps
of D_b come from L2 after their first read). GB/s is those bytes over the kernel time, against the 3.35 TB/s data-sheet HBM3
bandwidth of the H100 SXM.

Command. For `--e2e` a seeded video is written to a temporary directory (export, frame files with motion_seg, finished
flowpair files) and `python -m dvd_b200.evaluate` runs once as a subprocess; its wall time is reported with the split it
prints (reading the export, reading the flows, the device pass).
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
F32 = np.float32
HBM_BPS = 3.35e12
PAIR_CHUNK = 64


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'nvidia-smi unavailable'


def timed(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    best = float('inf')
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b) / 1e3)
    return best


def kernels(N, H, W, gaps):
    from dvd_b200 import ops
    from dvd_b200.flow_pairs import pair_list
    from dvd_b200.points import camera_block
    g = torch.Generator(device='cuda').manual_seed(0)
    base = 2 + torch.rand(N, H, W, device='cuda', generator=g)
    d, dn, gt = base * 1.01, base * 1.1, base.clone()
    scales = torch.ones(N, 2, 3, dtype=torch.float64, device='cuda')
    pairs = pair_list(N, gaps)
    P = len(pairs)
    flow = torch.randn(P, H, W, 2, device='cuda', generator=g) * 0.5
    mask = (torch.rand(P, H, W, device='cuda', generator=g) < 0.1).to(torch.uint8)
    seg = (torch.rand(N, H, W, device='cuda', generator=g) < 0.2).to(torch.uint8)
    K = np.tile(np.array([[0.9 * W, 0, W / 2], [0, 0.9 * W, H / 2], [0, 0, 1]], F32), (N, 1, 1))
    c2w = np.tile(np.eye(4, dtype=F32)[:3], (N, 1, 1))
    c2w[:, 0, 3] = 0.01 * np.arange(N)
    cam = torch.from_numpy(camera_block(K, c2w)).cuda()
    ia = torch.tensor([a for a, _ in pairs], dtype=torch.int32, device='cuda')
    ib = torch.tensor([b for _, b in pairs], dtype=torch.int32, device='cuda')

    def select():
        for v, o in ((gt, d), (d, gt), (gt, dn), (dn, gt)):
            ops.masked_select_median(v, o)

    def consistency():
        for s in range(0, P, PAIR_CHUNK):
            ops.pair_consistency(d, dn, cam, ia[s:s + PAIR_CHUNK], ib[s:s + PAIR_CHUNK], flow[s:s + PAIR_CHUNK],
                                 mask[s:s + PAIR_CHUNK], seg)

    px = N * H * W
    out = {'frames': N, 'H': H, 'W': W, 'pairs': P, 'gaps': list(gaps)}
    for name, fn, nbytes in (('masked_select_x4', select, 4 * 4 * 8 * px), ('depth_metrics', lambda: ops.depth_metrics(d, dn, gt, scales), 12 * px),
                             ('pair_consistency', consistency, 26 * P * H * W)):
        t = timed(fn)
        out[name] = {'ms': t * 1e3, 'bytes': nbytes, 'GBps': nbytes / t / 1e9, 'share_of_hbm_bound': nbytes / t / HBM_BPS}
    del flow, mask
    torch.cuda.empty_cache()
    return out


def write_video(root, N, H, W, gaps):
    from dvd_b200.flow_pairs import pair_list
    rng = np.random.default_rng(0)
    fdir, pdir, tdir = (os.path.join(root, k) for k in ('frames', 'flows', 'export'))
    for k in (fdir, pdir, tdir):
        os.makedirs(k)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    K = np.array([[0.9 * W, 0, W / 2], [0, 0.9 * W, H / 2], [0, 0, 1]])
    truth = (2.0 + 1.5 * x / W + 0.3 * y / H).astype(F32)
    seg = np.zeros((H, W), F32)
    seg[H // 3:H // 2, W // 3:W // 2] = 1
    for f in range(N):
        pose = np.eye(4)
        pose[0, 3] = 0.01 * f
        np.savez(os.path.join(fdir, 'frame_%05d.npz' % f), img=np.zeros((H, W, 3), F32), pose_c2w=pose, intrinsics=K,
                 depth_mvs=truth, depth_pred=truth, motion_seg=seg)
    for a, b in pair_list(N, gaps):
        f12 = np.zeros((H, W, 2), F32)
        f12[..., 0] = -0.9 * W * 0.01 * (b - a) / truth + rng.standard_normal((H, W)).astype(F32) * 0.3
        m = (rng.random((H, W)) < 0.1).astype(np.uint8)
        np.savez(os.path.join(pdir, 'flowpair_%05d_%05d.npz' % (a, b)), flow_1_2=f12, flow_2_1=-f12, mask_1=m, mask_2=m)
    for s in range(0, N, 8):
        e = min(s + 8, N)
        B = e - s
        dep = np.broadcast_to(truth, (B, 1, H, W))
        c2w = np.tile(np.eye(4, dtype=F32), (B, 1, 1))
        c2w[:, 0, 3] = 0.01 * np.arange(s, e)
        np.savez(os.path.join(tdir, 'batch%04d.npz' % (s // 8)), depth=(dep * 1.01).astype(F32), depth_nn=(dep * 1.1).astype(F32),
                 depth_gt=dep.astype(F32), img_1=np.zeros((B, 3, H, W), F32), K=np.broadcast_to(K.T, (B, 1, 1, 3, 3)).astype(F32),
                 cam_c2w=c2w, pair_path=np.asarray([os.path.join(fdir, 'frame_%05d.npz' % f) for f in range(s, e)]))
    return fdir, pdir, tdir


def e2e(N, H, W, gaps):
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        fdir, pdir, tdir = write_video(tmp, N, H, W, gaps)
        t_write = time.perf_counter() - t0
        t0 = time.perf_counter()
        r = subprocess.run([sys.executable, '-m', 'dvd_b200.evaluate', '--test_dir', tdir, '--frames', fdir, '--flows', pdir,
                            '--gaps', ','.join(map(str, gaps)), '--out', os.path.join(tmp, 'out')], cwd=ROOT, capture_output=True,
                           text=True)
        wall = time.perf_counter() - t0
        if r.returncode != 0:
            raise RuntimeError(r.stderr)
        m = re.search(r'in [^(]*\(([\d.]+) s: reading ([\d.]+) s, flows ([\d.]+) s, device ([\d.]+) s\)', r.stdout)
        return {'frames': N, 'H': H, 'W': W, 'gaps': list(gaps), 'write_inputs_s': t_write, 'command_wall_s': wall,
                'evaluate_total_s': float(m.group(1)), 'read_export_s': float(m.group(2)), 'read_flows_s': float(m.group(3)),
                'device_s': float(m.group(4)), 'stdout': r.stdout}


def main():
    p = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    p.add_argument('--configs', default='200x224x384,200x448x768')
    p.add_argument('--gaps', default='1,2,4,8')
    p.add_argument('--e2e', default='200x224x384', help='configurations of the whole command ("" for none)')
    p.add_argument('--out', default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_evaluate needs a CUDA device')
    gaps = [int(g) for g in a.gaps.split(',')]
    res = {'gpu': gpu_info(), 'kernels': [], 'command': []}
    print('GPU:', res['gpu'])
    for c in a.configs.split(','):
        N, H, W = (int(v) for v in c.split('x'))
        k = kernels(N, H, W, gaps)
        res['kernels'].append(k)
        print('%d frames %dx%d, %d pairs:' % (N, H, W, k['pairs']))
        for name in ('masked_select_x4', 'depth_metrics', 'pair_consistency'):
            v = k[name]
            print('  %-18s %8.3f ms  %7.1f MB  %7.1f GB/s  (%.1f %% of 3.35 TB/s)' % (name, v['ms'], v['bytes'] / 1e6, v['GBps'],
                                                                                     100 * v['share_of_hbm_bound']))
    for c in filter(None, a.e2e.split(',')):
        N, H, W = (int(v) for v in c.split('x'))
        r = e2e(N, H, W, gaps)
        res['command'].append(r)
        print('command, %d frames %dx%d: wall %.2f s (evaluate %.2f s: export read %.2f s, flows read %.2f s, device %.2f s)'
              % (N, H, W, r['command_wall_s'], r['evaluate_total_s'], r['read_export_s'], r['read_flows_s'], r['device_s']))
        print(r['stdout'])
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
