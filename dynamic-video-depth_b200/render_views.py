"""Novel views of a test export: `python -m dvd_b200.render_views --test_dir OUT/<net>_<dataset>/epochbest_test --out DIR
[--path lock|wiggle] [--ref_frame K] [--amplitude 0.03] [--period 60] [--cameras FILE.npy] [--static auto|none|FILE.ply]
[--voxel V] [--min_views 2] [--edge_tol 0.05] [--splat 1] [--frames a:b] [--chunk 16] [--gpu 0]`.

Reads `depth`, `img_1`, `K` and `cam_c2w` of the `batch%04d.npz` files as `export_points` does (export_io.Frames, same
`--frames`, `--voxel`, `--edge_tol` and `--min_views`) and renders every selected frame t from a virtual camera. Output frame
t shows the kept pixels of frame t (`ops.points_select`: finite depth > 1e-2, no flying pixel; colour floor(255 clip(img))) and, unless
`--static none`, the fused static cloud: `auto` fuses it from the selected frames with `points.Fuser` (positions rounded to
fp32, colours through `points.mean_rgb_to_u8`, what `export_points` writes), a PLY file is read as `export_points` wrote it.
Moving objects therefore appear only in their own frame; the static cloud fills the background they and the camera motion
uncover, and what neither covers stays black. It writes DIR/view_%05d.png (numbered like `export_points`' per-frame files:
frame numbers count from the first file), DIR/views.mp4 and DIR/compare.mp4 (the frame and its view side by side, 30 fps,
`mp4v`) and DIR/render.json (the virtual cameras, the options and each view's coverage).

Camera paths, computed on the host in fp64 from the fp32 cameras and rounded to fp32 once; the views are H x W, t is the frame
number:
  lock    every frame is seen from frame k's camera, c2w(k) and K(k) (k = --ref_frame, default the middle selected frame);
  wiggle  c2w(t) with its centre moved to c(t) + R(t) (a m cos phi, a m sin phi, 0), phi = 2 pi t / period, a = --amplitude,
          m = the median valid depth (finite and > 1e-2) of the selected frames; K(t);
  --cameras FILE.npy  [N,3,4] or [N,4,4] camera-to-world matrices, one per selected frame, with K(t); overrides --path.

Rendering rule (csrc/render_views.cu), exact and order-independent, so the views are bitwise reproducible: w2c = (R^T, -R^T c)
in fp64 rounded to fp32; q = w2c P, h = K q, u = h0 / h2, v = h1 / h2 with every operation rounded on its own; a point with
q2 <= 1e-2 or a non-finite coordinate is dropped; it covers the s x s pixels (s = --splat) from floor(u + 0.5) - (s - 1) // 2;
each pixel keeps the minimum of (bits(q2) << 32) | index, index = the source pixel y W + x for frame t's points and H W + r
for static point r (nearest wins, then the frame's own point, then the lower index); the colour is the winner's.

The frames go to the device `--chunk` at a time, one host-to-device copy per chunk and pass (`auto` reads them twice: once to
fuse the static cloud, once to render), and each chunk's views come back in one copy. The key buffer of a chunk is
chunk x H x W x 8 bytes: 16 frames of 384 x 224 take 11 MB, which stays in the H100's 50 MB L2 while the points are splatted.
"""
import argparse
import json
import os
import time

import numpy as np
import torch

from . import ops, points
from .export_io import Frames, Writer, chunk_size, cuda_device, frame_range, list_files, to_device

PATHS = ('lock', 'wiggle')
FPS = 30
SPLAT_MAX = 4
INDEX_LIMIT = 2 ** 32


def median_depth(depth):
    """The median of the valid (finite, > 1e-2) depths of a host array, computed as points.default_voxel computes it."""
    d = np.asarray(depth, dtype=np.float32)
    valid = d[np.isfinite(d) & (d > np.float32(1e-2))]
    if valid.size == 0:
        raise ValueError('no valid depth (finite and > 1e-2) to derive the wiggle amplitude from')
    return float(np.median(valid))


def load_cameras(path, n):
    """[n,3,4] fp32 camera-to-world matrices of a .npy file holding [n,3,4] or [n,4,4]; ValueError otherwise."""
    try:
        c = np.load(path, allow_pickle=False)
    except (OSError, ValueError) as e:
        raise ValueError('cannot read the camera file %s: %s' % (path, e)) from None
    if c.ndim != 3 or c.shape[1:] not in ((3, 4), (4, 4)) or c.shape[0] != n:
        raise ValueError('%s holds cameras of shape %s; expected [%d,3,4] or [%d,4,4], one per selected frame' % (path, c.shape, n, n))
    if not np.issubdtype(c.dtype, np.floating) or not np.isfinite(c[:, :3]).all():
        raise ValueError('%s must hold finite floating-point matrices, got %s' % (path, c.dtype))
    return np.asarray(c[:, :3], dtype=np.float32)


def camera_path(K, c2w, ids, path='lock', ref_frame=None, amplitude=0.03, period=60.0, median=None, cameras=None):
    """The virtual cameras of the frames `ids` (frame numbers) whose fp32 K [N,3,3] and c2w [N,3,4] are given: (K [N,3,3],
    c2w [N,3,4]) fp32. `median` is median_depth of the selected frames (wiggle only); `cameras` a [N,3,4] array that overrides
    the path (load_cameras)."""
    K = np.asarray(K, dtype=np.float32)
    c2w = np.asarray(c2w, dtype=np.float32)[:, :3]
    ids = np.asarray(ids)
    N = ids.shape[0]
    if cameras is not None:
        cameras = np.asarray(cameras, dtype=np.float32)
        if cameras.shape != (N, 3, 4):
            raise ValueError('cameras must be [%d,3,4], got %s' % (N, cameras.shape))
        return K.copy(), cameras.copy()
    if path == 'lock':
        k = int(ids[N // 2]) if ref_frame is None else int(ref_frame)
        hit = np.flatnonzero(ids == k)
        if hit.size == 0:
            raise ValueError('--ref_frame %d is not among the selected frames %d..%d' % (k, ids[0], ids[-1]))
        return np.repeat(K[hit[:1]], N, 0), np.repeat(c2w[hit[:1]], N, 0)
    if path == 'wiggle':
        if not (period > 0 and np.isfinite(period)) or not np.isfinite(amplitude):
            raise ValueError('wiggle needs a positive period and a finite amplitude, got %r and %r' % (period, amplitude))
        if median is None:
            raise ValueError('wiggle needs the median valid depth')
        c = c2w.astype(np.float64)
        phi = 2 * np.pi * ids.astype(np.float64) / float(period)
        am = float(amplitude) * float(median)
        off = np.stack([am * np.cos(phi), am * np.sin(phi), np.zeros(N)], 1)
        out = c.copy()
        out[:, :, 3] = c[:, :, 3] + np.einsum('nij,nj->ni', c[:, :, :3], off)
        return K.copy(), out.astype(np.float32)
    raise ValueError('path must be one of %s, got %r' % (PATHS, path))


def view_cams(K, c2w):
    """fp32 K [N,3,3] and c2w [N,3,4] -> the [N,21] fp32 blocks of dvd_splat_views: w2c = (R^T | -R^T c) in fp64 rounded to
    fp32, then K, both row-major."""
    K = np.asarray(K, dtype=np.float32).reshape(-1, 3, 3)
    c = np.asarray(c2w, dtype=np.float64).reshape(K.shape[0], -1, 4)
    Rt = c[:, :3, :3].transpose(0, 2, 1)
    w2c = np.concatenate([Rt, -np.einsum('nij,nj->ni', Rt, c[:, :3, 3])[:, :, None]], 2).astype(np.float32)
    return np.concatenate([w2c.reshape(-1, 12), K.reshape(-1, 9)], 1)


def check_index_range(H, W, n_static):
    """The key's 32-bit index holds pixel indices below H W and static indices H W + r: H W + R must stay below 2^32."""
    if H * W + int(n_static) >= INDEX_LIMIT:
        raise ValueError('%dx%d views and %d static points need indices up to %d, beyond the key\'s 32 bits; use a larger --voxel '
                         'or a smaller static cloud' % (H, W, n_static, H * W + n_static - 1))


def record(test_dir, ids, K, c2w, coverage, options, H, W, n_static):
    """The contents of render.json: per output frame its number, virtual camera (c2w 3x4, K 3x3, the fp32 values) and
    coverage (the fraction of its H W pixels that received a point), and the options."""
    return {'test_dir': os.path.abspath(test_dir), 'height': int(H), 'width': int(W), 'static_points': int(n_static),
            'options': options,
            'views': [{'frame': int(i), 'c2w': np.asarray(c, np.float32).astype(np.float64).tolist(),
                       'K': np.asarray(k, np.float32).astype(np.float64).tolist(), 'coverage': float(n) / (H * W)}
                      for i, c, k, n in zip(ids, c2w, K, coverage)]}


def render_views(test_dir, out, path='lock', ref_frame=None, amplitude=0.03, period=60.0, cameras=None, static='auto',
                 voxel=None, min_views=2, edge_tol=points.EDGE_TOL, splat=1, frames=None, chunk=16, device=None):
    """Renders the test export in `test_dir` into `out` (see the module docstring) on CUDA device `device` (default: the
    current one). `cameras` is a .npy path or an [N,3,4] / [N,4,4] array; `static` is 'auto', 'none' or a PLY path. Every
    argument and file is checked before the device is touched. Returns a dict of the written paths, the frame numbers, the
    per-view coverage counts and the record written to render.json."""
    if not 1 <= int(splat) <= SPLAT_MAX:
        raise ValueError('splat must be in [1, %d], got %r' % (SPLAT_MAX, splat))
    chunk_size(chunk)
    if not edge_tol >= 0:
        raise ValueError('edge_tol must be >= 0, got %r' % edge_tol)
    if int(min_views) < 1:
        raise ValueError('min_views must be >= 1, got %r' % min_views)
    if voxel is not None and not (voxel > 0 and np.isfinite(voxel)):
        raise ValueError('voxel must be positive, got %r' % voxel)
    splat, chunk = int(splat), int(chunk)
    ex = Frames(list_files(test_dir), frames)
    N, H, W = ex.N, ex.H, ex.W
    if isinstance(cameras, str):
        cameras = load_cameras(cameras, N)
    elif cameras is not None:
        cameras = np.asarray(cameras)
        if cameras.ndim != 3 or cameras.shape[1:] not in ((3, 4), (4, 4)) or cameras.shape[0] != N:
            raise ValueError('cameras must be [%d,3,4] or [%d,4,4], got %s' % (N, N, cameras.shape))
        cameras = cameras[:, :3]
    median = median_depth(ex.depth) if cameras is None and path == 'wiggle' else None
    vK, vc2w = camera_path(ex.K, ex.c2w, ex.ids, path, ref_frame, amplitude, period, median, cameras)
    vcams = view_cams(vK, vc2w)
    static_host = None
    if static not in ('auto', 'none'):
        if not os.path.isfile(static):
            raise ValueError('--static must be auto, none or a PLY file; %s is not a file' % static)
        static_host = points.read_ply(static)
        check_index_range(H, W, static_host[0].shape[0])
    HW = H * W
    cam30 = points.camera_block(ex.K, ex.c2w)
    dev = cuda_device(device)

    def upload(s, e):
        """the chunk's one host-to-device copy: depth [n,H,W], img [n,3,H,W], camera_block [n,30], view cams [n,21]"""
        return to_device(dev, ex.depth[s:e], ex.images(s, e), cam30[s:e], vcams[s:e])

    sxyz = srgb = None
    if static == 'auto':
        vox = voxel if voxel is not None else points.default_voxel(ex.depth)
        fz = points.Fuser(H, W, vox, points.default_origin(ex.c2w, vox), edge_tol, min_views)
        for s in range(0, N, chunk):
            depth, img, cam, _ = upload(s, min(s + chunk, N))
            fz.add(depth, img, cam)
        res = fz.result()
        del fz
        check_index_range(H, W, res['xyz'].shape[0])
        sxyz = res['xyz'].float().contiguous()
        srgb = torch.from_numpy(points.mean_rgb_to_u8(res['rgb'].cpu().numpy())).to(dev)
    elif static_host is not None:
        sxyz = torch.from_numpy(np.ascontiguousarray(static_host[0], dtype=np.float32)).to(dev)
        srgb = torch.from_numpy(np.ascontiguousarray(static_host[1], dtype=np.uint8)).to(dev)
    n_static = 0 if sxyz is None else int(sxyz.shape[0])

    os.makedirs(out, exist_ok=True)
    rgb_tmpl = torch.zeros(H, W, 3, dtype=torch.uint8, device=dev)
    coverage = np.zeros(N, dtype=np.int64)
    written = []
    vids = {'views': os.path.join(out, 'views.mp4'), 'compare': os.path.join(out, 'compare.mp4')}
    with Writer() as wr:
        v_views, v_cmp = wr.video(vids['views'], FPS, (H, W)), wr.video(vids['compare'], FPS, (H, 2 * W))
        for s in range(0, N, chunk):
            e = min(s + chunk, N)
            n = e - s
            depth, img, cam, vc = upload(s, e)
            sel = ops.points_select(depth, img, points.world_points(depth, cam), edge_tol)
            keys = ops.view_keys(n, H, W, dev)
            ops.splat_views(keys, sel['xyz'], vc, splat, index=sel['index'])
            if n_static:
                ops.splat_views(keys, sxyz, vc, splat)
            buf = torch.empty(4 * n + 2 * n * HW * 3, dtype=torch.uint8, device=dev)
            views = buf[4 * n:4 * n + n * HW * 3].view(n, H, W, 3)
            ops.resolve_views(keys, img, srgb, out=views, coverage=buf[:4 * n].view(torch.int32))
            ops.vis_panels(rgb_tmpl, [ops.vis_panel(img, 'rgb', H, W, 0, 0, (3 * HW, W, 1, HW))], None,
                           buf[4 * n + n * HW * 3:].view(n, H, W, 3))
            hb = buf.cpu().numpy()                                              # the chunk's one device-to-host copy
            coverage[s:e] = hb[:4 * n].view(np.int32)
            views_h = hb[4 * n:4 * n + n * HW * 3].reshape(n, H, W, 3)
            orig_h = hb[4 * n + n * HW * 3:].reshape(n, H, W, 3)
            for j in range(n):
                p = os.path.join(out, 'view_%05d.png' % ex.ids[s + j])
                written.append(p)
                wr.png(p, views_h[j])
                v_views.write(views_h[j])
                v_cmp.write(np.concatenate([orig_h[j], views_h[j]], 1))
    options = {'path': 'cameras' if cameras is not None else path, 'ref_frame': ref_frame, 'amplitude': amplitude,
               'period': period, 'median_depth': median, 'static': static, 'voxel': voxel, 'min_views': min_views,
               'edge_tol': edge_tol, 'splat': splat, 'frames': frames, 'chunk': chunk}
    if path == 'lock' and cameras is None:
        options['ref_frame'] = int(ex.ids[N // 2]) if ref_frame is None else int(ref_frame)
    rec = record(test_dir, ex.ids, vK, vc2w, coverage, options, H, W, n_static)
    with open(os.path.join(out, 'render.json'), 'w') as f:
        json.dump(rec, f, indent=1)
    return {'views': written, 'videos': vids, 'json': os.path.join(out, 'render.json'), 'frames': [int(i) for i in ex.ids],
            'coverage': coverage, 'record': rec}


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog='python -m dvd_b200.render_views', description=__doc__.split('\n\n')[0])
    p.add_argument('--test_dir', required=True, help='directory of the batch%%04d.npz files the test driver wrote')
    p.add_argument('--out', required=True, help='output directory (view_%%05d.png, views.mp4, compare.mp4, render.json)')
    p.add_argument('--path', choices=PATHS, default='lock', help='camera path: lock (one frame\'s camera) or wiggle (a circle '
                   'around each frame\'s camera)')
    p.add_argument('--ref_frame', type=int, default=None, help='frame number whose camera lock uses (default: the middle '
                   'selected frame)')
    p.add_argument('--amplitude', type=float, default=0.03, help='wiggle radius as a fraction of the median valid depth')
    p.add_argument('--period', type=float, default=60, help='wiggle period in frames')
    p.add_argument('--cameras', default=None, help='.npy of [N,3,4] or [N,4,4] camera-to-world matrices, one per selected '
                   'frame (overrides --path)')
    p.add_argument('--static', default='auto', help='static cloud: auto (fused from the selected frames), none, or a PLY '
                   'file export_points wrote')
    p.add_argument('--voxel', type=float, default=None,
                   help='voxel edge of the auto static cloud (default: %g x the median valid depth)' % points.VOXEL_DEPTH_FRACTION)
    p.add_argument('--min_views', type=int, default=2, help='auto static cloud: keep voxels seen in at least this many frames')
    p.add_argument('--edge_tol', type=float, default=points.EDGE_TOL,
                   help='drop a pixel when |d - d_n| / d exceeds this for one of its 4-neighbours (flying pixels)')
    p.add_argument('--splat', type=int, default=1, help='footprint of a point: splat x splat pixels (1 to %d)' % SPLAT_MAX)
    p.add_argument('--frames', type=frame_range, default=None, help='frames a:b (Python slice of the frames in file order)')
    p.add_argument('--chunk', type=int, default=16, help='frames per device chunk')
    p.add_argument('--gpu', type=int, default=0)
    return p.parse_args(argv)


def main(argv=None):
    a = parse_args(argv)
    t0 = time.perf_counter()
    res = render_views(a.test_dir, a.out, a.path, a.ref_frame, a.amplitude, a.period, a.cameras, a.static, a.voxel, a.min_views,
                       a.edge_tol, a.splat, a.frames, a.chunk, device=a.gpu)
    cov = res['coverage'] / (res['record']['height'] * res['record']['width'])
    print('rendered %d views (coverage %.3f to %.3f, %d static points) into %s in %.2f s'
          % (len(res['views']), cov.min(), cov.max(), res['record']['static_points'], a.out, time.perf_counter() - t0))
    return res


if __name__ == '__main__':
    main()
