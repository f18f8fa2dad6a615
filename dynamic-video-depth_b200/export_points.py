"""Point clouds of a test export: `python -m dvd_b200.export_points --test_dir OUT/<net>_<dataset>/epochbest_test --out scene.ply
[--per_frame DIR] [--voxel V] [--edge_tol 0.05] [--min_views 2] [--frames a:b] [--chunk 16] [--gpu 0]`.

Reads `depth`, `img_1`, `K` and `cam_c2w` of the `batch%04d.npz` files with export_io.Frames (in index order; a file
may hold several frames), works on `--chunk` frames at a time with one host-to-device copy per chunk, and writes the fused
cloud of the voxels seen in at least `--min_views` frames to `--out` and, with `--per_frame`, each frame's cloud to
DIR/frame_%05d.ply (frame numbers count from the first file). Files are binary little-endian PLY with float x, y, z and uchar red, green, blue; the fused
colours are the mean colours rounded half up. See dvd_b200/points.py for the conventions.
"""
import argparse
import os
import time

import numpy as np

from . import points
from .export_io import Frames, chunk_size, cuda_device, frame_range, list_files, to_device


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
    p.add_argument('--frames', type=frame_range, default=None, help='frames a:b (Python slice of the frames in file order)')
    p.add_argument('--chunk', type=chunk_size, default=16, help='frames per device chunk')
    p.add_argument('--gpu', type=int, default=0)
    a = p.parse_args(argv)
    if a.voxel is not None and not (a.voxel > 0 and np.isfinite(a.voxel)):
        p.error('--voxel must be positive')
    if not a.edge_tol >= 0:
        p.error('--edge_tol must be >= 0')
    if a.min_views < 1:
        p.error('--min_views must be >= 1')
    return a


def main(argv=None):
    a = parse_args(argv)
    t0 = time.perf_counter()
    ex = Frames(list_files(a.test_dir), a.frames)
    voxel = a.voxel if a.voxel is not None else points.default_voxel(ex.depth)
    origin = points.default_origin(ex.c2w, voxel)
    dev = cuda_device(a.gpu)
    fz = points.Fuser(ex.H, ex.W, voxel, origin, a.edge_tol, a.min_views)
    if a.per_frame:
        os.makedirs(a.per_frame, exist_ok=True)
    cam = points.camera_block(ex.K, ex.c2w)
    for s in range(0, ex.N, a.chunk):
        e = min(s + a.chunk, ex.N)
        per = fz.add(*to_device(dev, ex.depth[s:e], ex.images(s, e), cam[s:e]))
        if a.per_frame:
            for j, (xyz, rgb) in enumerate(per):
                points.write_ply(os.path.join(a.per_frame, 'frame_%05d.ply' % ex.ids[s + j]), xyz.cpu().numpy(), rgb.cpu().numpy())
    res = fz.result()
    xyz, rgb = res['xyz'].cpu().numpy(), res['rgb'].cpu().numpy()
    points.write_ply(a.out, xyz, points.mean_rgb_to_u8(rgb))
    print('fused %d voxels of %g from %d frames of %dx%d into %s in %.2f s' % (xyz.shape[0], voxel, ex.N, ex.H, ex.W, a.out,
                                                                              time.perf_counter() - t0))
    return res


if __name__ == '__main__':
    main()
