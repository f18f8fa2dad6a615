"""TEST INFRASTRUCTURE — CPU oracle, not product code.

numpy fp64 restatement of the point-cloud export (dvd_b200/points.py, csrc/points.cu): oracle/geometry.py's unprojection,
then the pixel selection (depth finite and > 1e-2, no flying pixel), the voxel keys, the colours, and the per-voxel reduction
in (key, pixel index) order with one fp64 rounding per addition.
"""
import numpy as np
import torch

from . import geometry

KEY_BITS = 21


def world_points(depth, K, c2w):
    """depth [N,H,W], K [N,3,3] (column form), c2w [N,3|4,4] -> P [N,3,H,W] fp64 with K^-1 = inv(K) in fp64."""
    d = torch.from_numpy(np.asarray(depth, dtype=np.float64))[:, None]
    K = np.asarray(K, dtype=np.float64).reshape(-1, 3, 3)
    c2w = np.asarray(c2w, dtype=np.float64)
    c2w = c2w.reshape(K.shape[0], -1, 4)
    kinv = torch.from_numpy(np.linalg.inv(K))
    R, t = torch.from_numpy(c2w[:, :3, :3].copy()), torch.from_numpy(c2w[:, :3, 3].copy())
    return geometry.unproject(d, R, t, kinv).numpy()


def select_mask(depth, edge_tol):
    """[N,H,W] bool: finite, > 1e-2 (fp32) and max_n |d - d_n| / d <= edge_tol (fp64) over the in-image 4-neighbours."""
    d = np.asarray(depth, dtype=np.float32)
    ok = np.isfinite(d) & (d > np.float32(1e-2))
    dd = d.astype(np.float64)
    with np.errstate(all='ignore'):
        for axis in (1, 2):
            for s in (1, -1):
                n = np.roll(dd, s, axis=axis)
                good = np.abs(dd - n) / dd <= edge_tol
                border = [slice(None)] * 3
                border[axis] = 0 if s == 1 else -1    # the rolled-in value is not a neighbour
                good[tuple(border)] = True
                ok &= good
    return ok


def colours(img):
    """floor(255 clip(img, 0, 1)) in fp32, NaN -> 0; img [..., 3] -> uint8"""
    v = np.asarray(img, dtype=np.float32)
    v = np.where(np.isnan(v), np.float32(0), v)
    return (np.clip(v, np.float32(0), np.float32(1)) * np.float32(255)).astype(np.uint8)


def keys(xyz, voxel, origin):
    """xyz [M,3] -> int64 keys (kx << 42 | ky << 21 | kz), k = floor(xyz / voxel) - origin; ValueError when out of range."""
    q = np.floor(np.asarray(xyz, dtype=np.float32).astype(np.float64) / voxel)
    o = np.asarray(origin, dtype=np.float64)
    if not ((q >= o) & (q < o + 2 ** KEY_BITS)).all():
        raise ValueError('voxel key out of range')
    k = q.astype(np.int64) - np.asarray(origin, dtype=np.int64)
    return (k[:, 0] << (2 * KEY_BITS)) | (k[:, 1] << KEY_BITS) | k[:, 2]


def select(depth, img, P, edge_tol, voxel=None, origin=(0, 0, 0), base=0):
    """The dict ops.points_select returns, from host arrays (P [N,3,H,W] fp32 or fp64)."""
    mask = select_mask(depth, edge_tol)
    N, H, W = mask.shape
    idx = np.flatnonzero(mask.reshape(-1))
    f, r = idx // (H * W), idx % (H * W)
    xyz = np.asarray(P).reshape(N, 3, H * W)[f, :, r]
    out = {'mask': mask.astype(np.uint8), 'index': base + idx.astype(np.int64), 'xyz': xyz,
           'rgb': colours(np.asarray(img).reshape(N, 3, H * W)[f, :, r])}
    if voxel is not None:
        out['key'] = keys(xyz, voxel, origin)
    return out


def reduce(key, index, xyz, rgb, hw, min_views):
    """Per-voxel fp64 means (sequential sums in (key, index) order), counts and distinct frames of the runs seen in at least
    min_views frames, in key order."""
    order = np.lexsort((index, key))
    k = key[order]
    M = k.shape[0]
    if M == 0:
        return {'xyz': np.zeros((0, 3)), 'rgb': np.zeros((0, 3)), 'count': np.zeros(0, np.int32), 'views': np.zeros(0, np.int32)}
    starts = np.flatnonzero(np.r_[True, k[1:] != k[:-1]])
    lens = np.diff(np.r_[starts, M])
    frame = index[order] // hw
    new_frame = np.r_[True, frame[1:] != frame[:-1]]
    new_frame[starts] = True
    views = np.add.reduceat(new_frame.astype(np.int64), starts)
    vals = np.concatenate([np.asarray(xyz, dtype=np.float32), np.asarray(rgb).astype(np.float32)], 1)[order].astype(np.float64)
    acc = np.zeros((starts.shape[0], 6))
    for j in range(int(lens.max())):           # one addition per step and run, in sorted order
        live = lens > j
        acc[live] += vals[starts[live] + j]
    mean = acc / lens[:, None]
    keep = views >= min_views
    return {'xyz': mean[keep, :3], 'rgb': mean[keep, 3:], 'count': lens[keep].astype(np.int32), 'views': views[keep].astype(np.int32)}


def fuse(depth, img, P, voxel, origin, edge_tol=0.05, min_views=2):
    """Fused cloud of one sequence of frames (P from the unprojection of depth)."""
    N, H, W = np.asarray(depth).shape
    s = select(depth, img, P, edge_tol, voxel, origin)
    return reduce(s['key'], s['index'], s['xyz'], s['rgb'], H * W, min_views)
