"""Synthetic depth of field (dvd_b200.refocus, csrc/refocus.cu): kernel time per blur radius for a whole video, the host
stages, one whole call, and the numpy oracle.

    python tools/bench_refocus.py [--configs 80x224x384,200x288x512] [--radii 8,16,32] [--oracle_frames 1] [--out FILE.json]

Per configuration (frames x H x W) a synthetic export is written to a temporary directory: a sloped plane from 1.5 to 6 with
a near square moving across it, random colours, and a depth_nn that flickers (each frame's depth scaled and warped a
little). The focus is a rack focus from 0.4 to 2.5 times the median depth (`--focus_pull 0.4:2.5`), aperture 8. The frames
are uploaded in chunks of 16 once. Per radius R, after a warm-up pass, CUDA events time the dvd_refocus launches summed over
the chunks, best of 3 passes: the refined source alone, and a whole chunk's three launches (the frame itself, the initial and
the refined render). Rule taps/s counts, from the shapes, every tap of the R disc whose q lies inside the image, per pixel and
source, over the refined launches' time; the kernel walks fewer (it skips the taps beyond a tile's largest blur radius, which
weigh 0), so this is the rate of the rule, not of the loop. Host clocks time the per-chunk D2H copies, the PNG writes (thread
pool), the two mp4 files, and one whole `refocus` call. The oracle renders the first `--oracle_frames` refined frames on
the CPU; its time is scaled to the whole video, and its frames must equal the device's bit for bit.
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
F32 = np.float32
PULL = (0.4, 2.5)
APERTURE = 8.0
CHUNK = 16


def synth_export(d, N, H, W, per_file=8):
    rng = np.random.default_rng(0)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    base = 1.5 + 4.5 * x / W + 0.5 * y / H
    for s in range(0, N, per_file):
        e = min(s + per_file, N)
        depth = np.empty((e - s, 1, H, W), F32)
        nn = np.empty((e - s, 1, H, W), F32)
        for j, i in enumerate(range(s, e)):
            dep = base.copy()
            x0 = (2 * i) % (W - W // 4)
            dep[H // 3:H // 3 + H // 4, x0:x0 + W // 4] = 1.2
            depth[j, 0] = dep
            nn[j, 0] = dep * (1 + 0.15 * rng.uniform(-1, 1)) * (1 + 0.1 * np.sin(x / 11 + i))
        img = rng.uniform(0, 1, (e - s, 3, H, W)).astype(F32)
        np.savez(os.path.join(d, 'batch%04d.npz' % (s // per_file)), depth=depth, depth_nn=nn, img_1=img,
                 K=np.tile(np.eye(3, dtype=F32), (e - s, 1, 1)), cam_c2w=np.tile(np.eye(4, dtype=F32), (e - s, 1, 1)))


def rule_taps(H, W, R):
    """taps of the R disc that land inside an H x W image, summed over its pixels"""
    return sum((W - abs(dx)) * (H - abs(dy)) for dy in range(-R, R + 1) for dx in range(-R, R + 1)
               if dx * dx + dy * dy <= R * R and abs(dx) < W and abs(dy) < H)


def device_pass(chunks, scales, R):
    """CUDA-event times of the refined launches and of all three launches of every chunk; the chunks' output buffers"""
    from dvd_b200 import ops
    ms_ref = ms_all = 0.0
    outs = []
    for depth, nn, img, phi, phi_nn in chunks:
        n, H, W = depth.shape
        buf = torch.empty(3, n, H, W, 3, dtype=torch.uint8, device=depth.device)
        a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        a.record()
        ops.refocus(depth, img, phi, 0.0, 0, out=buf[0])
        ops.refocus(nn, img, phi_nn, scales['initial'], R, out=buf[1])
        b.record()
        ops.refocus(depth, img, phi, scales['refined'], R, out=buf[2])
        c.record()
        torch.cuda.synchronize()
        ms_ref += b.elapsed_time(c)
        ms_all += a.elapsed_time(c)
        outs.append(buf)
    return ms_ref, ms_all, outs


def run(N, H, W, radii, oracle_frames, workdir):
    from dvd_b200 import refocus as rf
    from dvd_b200.export_io import Frames, Writer, list_files
    from oracle import refocus as orf
    d = os.path.join(workdir, 'exp_%dx%dx%d' % (N, H, W))
    os.makedirs(d)
    synth_export(d, N, H, W)
    dev = torch.device('cuda')
    ex = Frames(list_files(d), optional=('depth_nn',))
    depth, nn = ex.depth, ex.depth_nn
    m, m_nn = rf.source_median(depth, 'refined'), rf.source_median(nn, 'initial')
    phi, phi_nn = rf.focus_disparities(depth, m, focus_pull=PULL), rf.focus_disparities(nn, m_nn, focus_pull=PULL)
    scales = {'refined': float(F32(APERTURE * m)), 'initial': float(F32(APERTURE * m_nn))}
    chunks = []
    for s in range(0, N, CHUNK):
        e = min(s + CHUNK, N)
        chunks.append(tuple(torch.from_numpy(np.ascontiguousarray(a)).to(dev)
                            for a in (depth[s:e], nn[s:e], ex.images(s, e), phi[s:e], phi_nn[s:e])))
    out = {'frames': N, 'H': H, 'W': W, 'median_depth': m, 'radii': {}}
    for R in radii:
        device_pass(chunks, scales, R)                                                  # warm-up
        best = min((device_pass(chunks, scales, R) for _ in range(3)), key=lambda r: r[0])
        ms_ref, ms_all, outs = best
        taps = rule_taps(H, W, R) * N
        mean_c = float(np.mean(rf.mean_blur(depth, phi, scales['refined'], R)))
        t0 = time.perf_counter()
        host = [b.cpu().numpy() for b in outs]
        d2h = time.perf_counter() - t0
        frames = np.concatenate([h[2] for h in host])
        cmp = np.concatenate([np.concatenate([h[0], h[1], h[2]], 2) for h in host])
        o = os.path.join(workdir, 'out_%dx%dx%d_%d' % (N, H, W, R))
        os.makedirs(o)
        t0 = time.perf_counter()
        with Writer() as w:
            for j in range(N):
                w.png(os.path.join(o, 'dof_%05d.png' % j), frames[j])
        png = time.perf_counter() - t0
        t0 = time.perf_counter()
        with Writer() as w:
            v1, v2 = w.video(os.path.join(o, 'dof.mp4'), 30, (H, W)), w.video(os.path.join(o, 'compare.mp4'), 30, (H, 3 * W))
            for j in range(N):
                v1.write(frames[j])
                v2.write(cmp[j])
        mp4 = time.perf_counter() - t0
        t0 = time.perf_counter()
        rf.refocus(d, os.path.join(workdir, 'cli_%dx%dx%d_%d' % (N, H, W, R)), aperture=APERTURE, max_blur=R, focus_pull=PULL)
        torch.cuda.synchronize()
        whole = time.perf_counter() - t0
        k = min(oracle_frames, N)
        t0 = time.perf_counter()
        ref = orf.render(depth[:k], ex.images(0, k), phi[:k], F32(scales['refined']), R)
        cpu_per_frame = (time.perf_counter() - t0) / k
        out['radii'][R] = {'refined_kernel_ms': ms_ref, 'three_launches_ms': ms_all, 'rule_taps': taps,
                           'rule_taps_per_s': taps / (ms_ref / 1e3), 'mean_blur_radius': mean_c, 'd2h_ms': d2h * 1e3,
                           'png_ms': png * 1e3, 'mp4_ms': mp4 * 1e3, 'refocus_call_s': whole,
                           'oracle_s_per_frame': cpu_per_frame, 'oracle_s_video': cpu_per_frame * N, 'oracle_frames': k,
                           'oracle_equal': bool(np.array_equal(ref, frames[:k]))}
        print(json.dumps({'config': '%dx%dx%d' % (N, H, W), 'R': R, **out['radii'][R]}), flush=True)
    return out


def main():
    p = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    p.add_argument('--configs', default='80x224x384,200x288x512')
    p.add_argument('--radii', default='8,16,32')
    p.add_argument('--oracle_frames', type=int, default=1)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_refocus needs a CUDA device')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    results = {'gpu': gpu[0] if gpu else torch.cuda.get_device_name(), 'runs': []}
    print(results['gpu'], flush=True)
    radii = [int(r) for r in a.radii.split(',')]
    with tempfile.TemporaryDirectory() as workdir:
        for c in a.configs.split(','):
            N, H, W = (int(v) for v in c.split('x'))
            results['runs'].append(run(N, H, W, radii, a.oracle_frames, workdir))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
