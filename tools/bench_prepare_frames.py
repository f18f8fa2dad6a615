"""Frame preparation of one video (dvd_b200.frames.FrameBuilder): time per stage and for the whole video, against the
reference's path on the same GPU (eager PyTorch MiDaS, then scipy on the CPU for the calibration and the resizes), a few
frames timed and scaled to the video.

    python tools/bench_prepare_frames.py [--frames 80] [--points 50000] [--ref_frames 3] [--out results/bench_frames.json]

Synthetic 1080x1920 JPEG frames, masks and a reconstruction with --points vertices are written to a temporary directory;
MiDaS has seeded weights. Device stages are timed with CUDA events on one pass over the video, after a warm-up chunk.
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_video(root, n, H, W, n_points, seed=0):
    g = np.random.default_rng(seed)
    jd, md, td = (os.path.join(root, d) for d in ('JPEGImages/1080p/v', 'Annotations/1080p/v', 'triangulation'))
    for d in (jd, md, td):
        os.makedirs(d, exist_ok=True)
    yy, xx = np.mgrid[0:H, 0:W]
    for f in range(n):
        base = np.stack([np.sin(xx / (60.0 + 9 * c) + 0.05 * f) * np.cos(yy / (40.0 + 5 * c)) for c in range(3)], -1)
        Image.fromarray(np.clip(127.5 + 100 * base, 0, 255).astype(np.uint8)).save(os.path.join(jd, '%05d.jpg' % f), quality=90)
        m = np.zeros((H, W, 3), np.uint8)
        m[300 + 2 * f:700 + 2 * f, 700 + 4 * f:1200 + 4 * f, 0] = 255
        Image.fromarray(m).save(os.path.join(md, '%05d.png' % f))
    fx = 1.1 * W
    with open(os.path.join(td, 'v.intrinsics.txt'), 'w') as fh:
        fh.writelines('%d %f %f %f %f\n' % (f, fx, fx, W / 2, H / 2) for f in range(n))
    with open(os.path.join(td, 'v.matrices.txt'), 'w') as fh:
        for f in range(n):
            c2w = np.eye(4)
            c2w[:3, 3] = [0.02 * f, 0, 0]
            fh.write('%d ' % f + ' '.join('%.12g' % v for v in c2w.reshape(-1)) + '\n')
    pts = np.stack([g.uniform(-6, 6, n_points), g.uniform(-3.5, 3.5, n_points), g.uniform(-12, -2, n_points)], 1)
    with open(os.path.join(td, 'v.obj'), 'w') as fh:
        fh.writelines('v %.9g %.9g %.9g\n' % tuple(p) for p in pts)


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--frames', type=int, default=80)
    p.add_argument('--points', type=int, default=50000)
    p.add_argument('--chunk', type=int, default=8)
    p.add_argument('--ref_frames', type=int, default=3)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    from dvd_b200 import frames as fr, ops, synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    from oracle import depth_nets, frames as oracle_frames
    H, W = 1080, 1920
    res = dict(gpu=torch.cuda.get_device_name(0), frames=a.frames, points=a.points, size=[H, W])
    try:
        res['nvidia_smi'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        res['nvidia_smi'] = repr(e)
    net = synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True, resize=[256, 512]), 0, 2000.0).cuda().eval()
    with tempfile.TemporaryDirectory() as tmp:
        make_video(tmp, a.frames, H, W, a.points)
        fr.FrameBuilder(tmp, 'v', net, chunk=a.chunk)                     # warm-up: engine plan, allocator
        torch.cuda.synchronize()
        # per stage, on the same work FrameBuilder does
        K, E, h_pt = fr.read_cameras(tmp, 'v')
        jpgs = sorted(os.listdir(os.path.join(tmp, 'JPEGImages/1080p/v')))
        pngs = sorted(os.listdir(os.path.join(tmp, 'Annotations/1080p/v')))
        t0 = time.perf_counter()
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(8) as pool:
            imgs = list(pool.map(fr.decode_image, [os.path.join(tmp, 'JPEGImages/1080p/v', j) for j in jpgs]))
            masks = list(pool.map(fr.decode_mask, [os.path.join(tmp, 'Annotations/1080p/v', q) for q in pngs]))
        res['decode_s'] = time.perf_counter() - t0
        dev = torch.device('cuda')
        pts = torch.from_numpy(np.ascontiguousarray(h_pt[:3].T)).to(dev)
        w2c = torch.from_numpy(np.ascontiguousarray(E)).to(dev)
        ratio = torch.empty(a.frames, a.points, dtype=torch.float64, device=dev)
        th, tw = fr.working_size(H, W)
        wts = [torch.from_numpy(ops.gaussian_weights(i, o)[1]).to(dev) for i, o in ((H, th), (W, tw))]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        t_midas = t_cal = t_aa = 0.0
        for c in range(0, a.frames, a.chunk):
            img = torch.from_numpy(np.stack(imgs[c:c + a.chunk])).to(dev)
            mask = torch.from_numpy(np.stack(masks[c:c + a.chunk])).to(dev)
            n = img.shape[0]
            ev[0].record()
            x = ops.resize_bicubic_ac(img.permute(0, 3, 1, 2).contiguous(), 256, 512)
            full = ops.resize_bicubic_ac(net.engine().forward(x, train=False).contiguous(), H, W).reshape(n, H, W)
            ev[1].record()
            ops.calib_ratios(ops.spline_prefilter(full), ops.spline_prefilter(mask), w2c[c:c + n], pts, K[0, 0], K[1, 1], K[0, 2],
                             K[1, 2], out=ratio[c:c + n])
            ev[2].record()
            for t in (img, full.reshape(n, H, W, 1), mask.reshape(n, H, W, 1)):
                ops.aa_resize(t, th, tw, wts)
            ev[3].record()
            torch.cuda.synchronize()
            t_midas += ev[0].elapsed_time(ev[1]) / 1e3
            t_cal += ev[1].elapsed_time(ev[2]) / 1e3
            t_aa += ev[2].elapsed_time(ev[3]) / 1e3
        ev[0].record()
        ops.row_medians(ratio)
        ev[1].record()
        torch.cuda.synchronize()
        res.update(midas_with_resizes_s=t_midas, calibration_s=t_cal + ev[0].elapsed_time(ev[1]) / 1e3, aa_resize_s=t_aa)
        # whole video: construction (decode, device passes, medians) and write
        t0 = time.perf_counter()
        b = fr.FrameBuilder(tmp, 'v', net, chunk=a.chunk)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        b.write(os.path.join(tmp, 'out'))
        t2 = time.perf_counter()
        res.update(build_s=t1 - t0, write_s=t2 - t1, video_s=t2 - t0, scale=float(b.scale))
        # the reference's path: eager MiDaS on the GPU, scipy on the CPU, per frame
        sd = {k: v.to(dev) for k, v in net.state_dict().items()}
        k = a.ref_frames
        torch.cuda.synchronize()
        with torch.no_grad():
            depth_nets.midas_forward(sd, torch.from_numpy(imgs[0]).permute(2, 0, 1)[None].to(dev), True, [256, 512])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        deps = []
        with torch.no_grad():
            for f in range(k):
                d = depth_nets.midas_forward(sd, torch.from_numpy(imgs[f]).permute(2, 0, 1)[None].to(dev), True, [256, 512])
                deps.append(d[0, 0].cpu().numpy())
        t1 = time.perf_counter()
        oracle_frames.calibrate(E[:k], K, h_pt, masks[:k], deps)
        t2 = time.perf_counter()
        for f in range(k):
            oracle_frames.frame_outputs(imgs[f], masks[f], deps[f], E[f], K, 1.0)
        t3 = time.perf_counter()
        sc = a.frames / k
        res.update(ref_midas_s=(t1 - t0) * sc, ref_calibration_s=(t2 - t1) * sc, ref_resize_s=(t3 - t2) * sc,
                   ref_video_s=(t3 - t0) * sc + res['decode_s'] + res['write_s'])
    res['speedup_video'] = res['ref_video_s'] / res['video_s']
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
