"""Novel-view rendering (dvd_b200.render_views, csrc/render_views.cu): device time per stage for a whole video, the host
stages, and the numpy oracle.

    python tools/bench_render_views.py [--configs 80x224x384,200x288x512] [--splat 1] [--oracle_frames 4] [--out FILE.json]

Per configuration (frames x H x W) a synthetic export is written to a temporary directory: a sloped background plane seen by
nearly still cameras with a near square moving across it, random colours. The frames are uploaded in chunks of 16 once, then,
after a warm-up pass, CUDA events time each stage summed over the chunks: selection (unprojection + dvd_points_select, which
waits for its count), static fusion (points.Fuser over all frames, default voxel, min_views 2), the frame splat (key buffer
fill + dvd_splat_views of each frame's points), the static splat (every static point into every view of the chunk) and the
resolve (dvd_resolve_views + the original frames). The static splat is repeated with chunks of 64 and of all frames, whose key
buffers do not stay in the 50 MB L2, to show whether L2 residency or the atomics bound it. Host clocks time the per-chunk D2H
copies, the PNG writes (thread pool) and the two mp4 files, and one whole `render_views` call (`--static auto`, wiggle path).
The oracle (oracle/render_views.py) renders the first `--oracle_frames` frames on the CPU from the same points and static
cloud; its per-frame time is scaled to the whole video, and its views must equal the device's bit for bit.
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


def synth_export(d, N, H, W, per_file=8):
    rng = np.random.default_rng(0)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    base = 3.0 + 0.5 * x / W + 0.2 * y / H
    f = 0.8 * W
    K = np.array([[f, 0, (W - 1) / 2], [0, f, (H - 1) / 2], [0, 0, 1]], F32)
    for s in range(0, N, per_file):
        e = min(s + per_file, N)
        depth = np.empty((e - s, 1, H, W), F32)
        c2w = np.tile(np.eye(4, dtype=F32), (e - s, 1, 1))
        for j, i in enumerate(range(s, e)):
            dep = base.copy()
            x0 = (2 * i) % (W - W // 4)
            dep[H // 3:H // 3 + H // 4, x0:x0 + W // 4] = 1.5
            depth[j, 0] = dep
            a = 0.001 * i
            c2w[j, :3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
            c2w[j, :3, 3] = [1e-3 * i, 0, 0]
        img = rng.uniform(0, 1, (e - s, 3, H, W)).astype(F32)
        np.savez(os.path.join(d, 'batch%04d.npz' % (s // per_file)), depth=depth, img_1=img,
                 K=np.tile(K.T, (e - s, 1, 1)), cam_c2w=c2w)


class Timer:
    def __init__(self):
        self.ms = {}

    def __call__(self, name, fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r = fn()
        b.record()
        torch.cuda.synchronize()
        self.ms[name] = self.ms.get(name, 0.0) + a.elapsed_time(b)
        return r


def device_pass(chunks, ex, splat, static, sxyz, srgb, vox, origin):
    from dvd_b200 import ops, points
    H, W, HW = ex.H, ex.W, ex.H * ex.W
    t = Timer()
    if static:
        def fuse():
            fz = points.Fuser(H, W, vox, origin, points.EDGE_TOL, 2)
            for depth, img, cam, _ in chunks:
                fz.add(depth, img, cam)
            return fz.result()
        t('fusion', fuse)
    n_frame_pts, outs = 0, []
    for depth, img, cam, vc in chunks:
        n = depth.shape[0]
        sel = t('select', lambda: ops.points_select(depth, img, points.world_points(depth, cam), points.EDGE_TOL))
        n_frame_pts += sel['xyz'].shape[0]
        keys = t('splat_frame', lambda: ops.splat_views(ops.view_keys(n, H, W, depth.device), sel['xyz'], vc, splat, index=sel['index']))
        if static:
            t('splat_static', lambda: ops.splat_views(keys, sxyz, vc, splat))
        buf = torch.empty(4 * n + 2 * n * HW * 3, dtype=torch.uint8, device=depth.device)

        def resolve():
            ops.resolve_views(keys, img, srgb if static else None, out=buf[4 * n:4 * n + n * HW * 3].view(n, H, W, 3),
                              coverage=buf[:4 * n].view(torch.int32))
            ops.vis_panels(torch.zeros(H, W, 3, dtype=torch.uint8, device=depth.device),
                           [ops.vis_panel(img, 'rgb', H, W, 0, 0, (3 * HW, W, 1, HW))], None, buf[4 * n + n * HW * 3:].view(n, H, W, 3))
        t('resolve', resolve)
        outs.append((n, buf))
    return t.ms, n_frame_pts, outs


def static_splat_ms(ex, vcams_dev, sxyz, splat, chunk, dev):
    """static splat alone over all frames with a given chunk (key buffers filled outside the timed window)"""
    from dvd_b200 import ops
    ms = 0.0
    for s in range(0, ex.N, chunk):
        e = min(s + chunk, ex.N)
        keys = ops.view_keys(e - s, ex.H, ex.W, dev)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ops.splat_views(keys, sxyz, vcams_dev[s:e], splat)
        b.record()
        torch.cuda.synchronize()
        ms += a.elapsed_time(b)
        del keys
    return ms


def run(N, H, W, splat, oracle_frames, workdir):
    from dvd_b200 import points, render_views as rv
    from dvd_b200.export_io import Frames, Writer, list_files, to_device
    from oracle import render_views as orv
    d = os.path.join(workdir, 'exp_%dx%dx%d' % (N, H, W))
    os.makedirs(d)
    synth_export(d, N, H, W)
    dev = torch.device('cuda')
    ex = Frames(list_files(d))
    HW = H * W
    vK, vc2w = rv.camera_path(ex.K, ex.c2w, ex.ids, 'wiggle', median=rv.median_depth(ex.depth))
    vcams = rv.view_cams(vK, vc2w)
    cam30 = points.camera_block(ex.K, ex.c2w)
    chunk = 16
    chunks = [to_device(dev, ex.depth[s:s + chunk], ex.images(s, min(s + chunk, N)), cam30[s:s + chunk],
                        vcams[s:s + chunk]) for s in range(0, N, chunk)]
    vox = points.default_voxel(ex.depth)
    origin = points.default_origin(ex.c2w, vox)
    fz = points.Fuser(H, W, vox, origin, points.EDGE_TOL, 2)
    for depth, img, cam, _ in chunks:
        fz.add(depth, img, cam)
    res = fz.result()
    del fz
    sxyz = res['xyz'].float().contiguous()
    srgb_h = points.mean_rgb_to_u8(res['rgb'].cpu().numpy())
    srgb = torch.from_numpy(srgb_h).to(dev)
    R = sxyz.shape[0]
    device_pass(chunks, ex, splat, True, sxyz, srgb, vox, origin)                      # warm-up
    best = None
    for _ in range(3):
        ms, n_frame_pts, outs = device_pass(chunks, ex, splat, True, sxyz, srgb, vox, origin)
        best = ms if best is None or sum(ms.values()) < sum(best.values()) else best
    vcams_dev = torch.from_numpy(vcams).to(dev)
    residency = {}
    for c in (16, 64, N):
        static_splat_ms(ex, vcams_dev, sxyz, splat, c, dev)
        t = min(static_splat_ms(ex, vcams_dev, sxyz, splat, c, dev) for _ in range(3))
        residency[c] = {'ms': t, 'key_buffer_MB': min(c, N) * HW * 8 / 1e6, 'pairs_per_s': R * N / (t / 1e3)}
    # host stages: D2H per chunk, PNG, mp4
    t0 = time.perf_counter()
    host = [(n, b.cpu().numpy()) for n, b in outs]
    d2h = time.perf_counter() - t0
    views = np.concatenate([h[4 * n:4 * n + n * HW * 3].reshape(n, H, W, 3) for n, h in host])
    origs = np.concatenate([h[4 * n + n * HW * 3:].reshape(n, H, W, 3) for n, h in host])
    out = os.path.join(workdir, 'out_%dx%dx%d' % (N, H, W))
    os.makedirs(out)
    t0 = time.perf_counter()
    with Writer() as w:
        for j in range(N):
            w.png(os.path.join(out, 'view_%05d.png' % j), views[j])
    png = time.perf_counter() - t0
    t0 = time.perf_counter()
    with Writer() as w:
        v1, v2 = w.video(os.path.join(out, 'views.mp4'), 30, (H, W)), w.video(os.path.join(out, 'compare.mp4'), 30, (H, 2 * W))
        for j in range(N):
            v1.write(views[j])
            v2.write(np.concatenate([origs[j], views[j]], 1))
    mp4 = time.perf_counter() - t0
    # one whole call of the command's function
    t0 = time.perf_counter()
    rv.render_views(d, os.path.join(workdir, 'cli_%dx%dx%d' % (N, H, W)), path='wiggle', splat=splat)
    torch.cuda.synchronize()
    whole = time.perf_counter() - t0
    # the oracle on the first frames, from the same points and static cloud
    k = min(oracle_frames, N)
    P = points.world_points(chunks[0][0][:k].contiguous(), chunks[0][2][:k].contiguous()).cpu().numpy()
    t0 = time.perf_counter()
    ref, _ = orv.render(ex.depth[:k], ex.images(0, k), P, vK[:k], vc2w[:k], splat, (sxyz.cpu().numpy(), srgb_h))
    cpu_per_frame = (time.perf_counter() - t0) / k
    equal = bool(np.array_equal(ref, views[:k]))
    splat_ms = best['splat_frame'] + best['splat_static']
    return {'frames': N, 'H': H, 'W': W, 'splat': splat, 'frame_points': int(n_frame_pts), 'static_points': int(R),
            'device_ms': best, 'device_total_ms': sum(best.values()),
            'splats_per_s': (n_frame_pts + R * N) / (splat_ms / 1e3),
            'static_splat_by_chunk': residency,
            'd2h_ms': d2h * 1e3, 'png_ms': png * 1e3, 'mp4_ms': mp4 * 1e3, 'render_views_call_s': whole,
            'oracle_s_per_frame': cpu_per_frame, 'oracle_s_video': cpu_per_frame * N, 'oracle_frames': k,
            'oracle_equal': equal}


def main():
    p = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    p.add_argument('--configs', default='80x224x384,200x288x512')
    p.add_argument('--splat', type=int, default=1)
    p.add_argument('--oracle_frames', type=int, default=4)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_render_views needs a CUDA device')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    results = {'gpu': gpu[0] if gpu else torch.cuda.get_device_name(), 'runs': []}
    print(results['gpu'])
    with tempfile.TemporaryDirectory() as workdir:
        for c in a.configs.split(','):
            N, H, W = (int(v) for v in c.split('x'))
            r = run(N, H, W, a.splat, a.oracle_frames, workdir)
            results['runs'].append(r)
            print(json.dumps(r, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
