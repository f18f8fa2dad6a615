"""Point clouds of a test export: `python -m dvd_b200.export_points --test_dir OUT/<net>_<dataset>/epochbest_test --out scene.ply
[--per_frame DIR] [--voxel V] [--edge_tol 0.05] [--min_views 2] [--frames a:b] [--chunk 16] [--gpu 0]`.

Reads `depth`, `img_1`, `K` and `cam_c2w` of the `batch%04d.npz` files (in index order; a file may hold several frames),
works on `--chunk` frames at a time with one host-to-device copy per chunk, and writes the fused cloud of the voxels seen in
at least `--min_views` frames to `--out` and, with `--per_frame`, each frame's cloud to DIR/frame_%05d.ply (frame numbers
count from the first file). Files are binary little-endian PLY with float x, y, z and uchar red, green, blue; the fused
colours are the mean colours rounded half up. See dvd_b200/points.py for the conventions.
"""
import argparse
import glob
import os
import re
import time

import numpy as np
import torch

from . import points

KEYS = ('depth', 'img_1', 'K', 'cam_c2w')


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog='python -m dvd_b200.export_points', description=__doc__.split('\n\n')[0])
    p.add_argument('--test_dir', required=True, help='directory of the batch%%04d.npz files the test driver wrote')
    p.add_argument('--out', required=True, help='PLY file of the fused cloud')
    p.add_argument('--per_frame', default=None, help='directory for one PLY file per frame (frame_%%05d.ply)')
    p.add_argument('--voxel', type=float, default=None,
                   help='voxel edge in world units (default: %g x the median valid depth of the selected frames)'
                   % points.VOXEL_DEPTH_FRACTION)
    p.add_argument('--edge_tol', type=float, default=points.EDGE_TOL,
                   help='drop a pixel when |d - d_n| / d exceeds this for one of its 4-neighbours (flying pixels)')
    p.add_argument('--min_views', type=int, default=2, help='keep voxels seen in at least this many frames')
    p.add_argument('--frames', default=None, help='frames a:b (Python slice of the frames in file order)')
    p.add_argument('--chunk', type=int, default=16, help='frames per device chunk')
    p.add_argument('--gpu', type=int, default=0)
    a = p.parse_args(argv)
    if a.voxel is not None and not (a.voxel > 0 and np.isfinite(a.voxel)):
        p.error('--voxel must be positive')
    if not a.edge_tol >= 0:
        p.error('--edge_tol must be >= 0')
    if a.min_views < 1:
        p.error('--min_views must be >= 1')
    if a.chunk < 1:
        p.error('--chunk must be >= 1')
    if a.frames is not None and not re.fullmatch(r'-?\d*:-?\d*', a.frames):
        p.error('--frames must look like a:b, got %r' % a.frames)
    return a


def list_files(test_dir):
    files = glob.glob(os.path.join(test_dir, 'batch*.npz'))
    files = sorted((int(m.group(1)), f) for f in files for m in [re.fullmatch(r'batch(\d+)\.npz', os.path.basename(f))] if m)
    if not files:
        raise ValueError('no batch%%04d.npz files in %s' % test_dir)
    return [f for _, f in files]


class Frames:
    """The frames of the files, flattened in file order: depth, K and c2w are read up front, images per chunk."""

    def __init__(self, files, sel=None):
        self.files, depth, K, c2w, self.where = files, [], [], [], []
        for fi, f in enumerate(files):
            z = np.load(f)
            missing = [k for k in KEYS if k not in z.files]
            if missing:
                raise ValueError('%s lacks %s' % (f, ', '.join(missing)))
            d = np.asarray(z['depth'], dtype=np.float32)
            B = d.shape[0]
            if d.ndim != 4 or d.shape[1] != 1:
                raise ValueError('%s: depth must be [B,1,H,W], got %s' % (f, d.shape))
            if depth and d.shape[2:] != depth[0].shape[1:]:
                raise ValueError('%s: frames of %dx%d, the first file has %dx%d' % (f, d.shape[2], d.shape[3], *depth[0].shape[1:]))
            if z['K'].size != 9 * B or z['cam_c2w'].size not in (12 * B, 16 * B):
                raise ValueError('%s: K %s / cam_c2w %s do not hold %d frames' % (f, z['K'].shape, z['cam_c2w'].shape, B))
            depth.append(d[:, 0])
            K.append(np.asarray(z['K'], dtype=np.float32).reshape(B, 3, 3).transpose(0, 2, 1))   # the files hold K^T
            cw = np.asarray(z['cam_c2w'], dtype=np.float32)
            c2w.append(cw.reshape(B, -1, 4)[:, :3])
            self.where += [(fi, b) for b in range(B)]
        self.depth, self.K, self.c2w = np.concatenate(depth), np.concatenate(K), np.concatenate(c2w)
        self.ids = np.arange(len(self.where))
        if sel is not None:
            a, b = sel.split(':')
            sl = slice(int(a) if a else None, int(b) if b else None)
            self.depth, self.K, self.c2w, self.ids = self.depth[sl], self.K[sl], self.c2w[sl], self.ids[sl]
        if len(self.ids) == 0:
            raise ValueError('the frame selection %r is empty (%d frames)' % (sel, len(self.where)))
        self.N, self.H, self.W = self.depth.shape

    def images(self, s, e):
        out = np.empty((e - s, 3, self.H, self.W), dtype=np.float32)
        cache = {}
        for j, i in enumerate(self.ids[s:e]):
            fi, b = self.where[i]
            if fi not in cache:
                z = np.load(self.files[fi])
                img = np.asarray(z['img_1'], dtype=np.float32)
                if img.shape[1:] != (3, self.H, self.W):
                    raise ValueError('%s: img_1 %s does not match the depth of %dx%d' % (self.files[fi], img.shape, self.H, self.W))
                cache[fi] = img
            out[j] = cache[fi][b]
        return out


def main(argv=None):
    a = parse_args(argv)
    t0 = time.perf_counter()
    fr = Frames(list_files(a.test_dir), a.frames)
    voxel = a.voxel if a.voxel is not None else points.default_voxel(fr.depth)
    origin = points.default_origin(fr.c2w, voxel)
    dev = torch.device('cuda', a.gpu)
    torch.cuda.set_device(dev)
    fz = points.Fuser(fr.H, fr.W, voxel, origin, a.edge_tol, a.min_views)
    if a.per_frame:
        os.makedirs(a.per_frame, exist_ok=True)
    hw = fr.H * fr.W
    cam = points.camera_block(fr.K, fr.c2w)
    for s in range(0, fr.N, a.chunk):
        e = min(s + a.chunk, fr.N)
        n = e - s
        buf = np.concatenate([fr.depth[s:e].reshape(-1), fr.images(s, e).reshape(-1), cam[s:e].reshape(-1)])
        g = torch.from_numpy(buf).to(dev)                                    # the chunk's one host-to-device copy
        depth = g[:n * hw].view(n, fr.H, fr.W)
        img = g[n * hw:4 * n * hw].view(n, 3, fr.H, fr.W)
        per = fz.add(depth, img, g[4 * n * hw:].view(n, 30))
        if a.per_frame:
            for j, (xyz, rgb) in enumerate(per):
                points.write_ply(os.path.join(a.per_frame, 'frame_%05d.ply' % fr.ids[s + j]), xyz.cpu().numpy(), rgb.cpu().numpy())
    res = fz.result()
    xyz, rgb = res['xyz'].cpu().numpy(), res['rgb'].cpu().numpy()
    points.write_ply(a.out, xyz, points.mean_rgb_to_u8(rgb))
    print('fused %d voxels of %g from %d frames of %dx%d into %s in %.2f s' % (xyz.shape[0], voxel, fr.N, fr.H, fr.W, a.out,
                                                                              time.perf_counter() - t0))
    return res


if __name__ == '__main__':
    main()
