"""TEST INFRASTRUCTURE — the frame stage of scripts/preprocess/shutterstock/generate_frame_midas.py restated as functions
(numpy, CPU), from the full-resolution MiDaS depth on, and the synthetic ShutterStock tracks its fixture is written from.

The arithmetic is the script's line for line, in numpy's dtypes: with fp32 MVS maps the ratios, the medians and their mean
are fp32. skimage.transform.resize is oracle.frames.sk_resize, as in the DAVIS fixture.
"""
import numpy as np

from .frames import sk_resize

# (name, H, W, files in the track directory, MVS dtype, K / T_1_G dtype). Sorted by name, so a track's id is its index:
# id 0 and id 3 are trimmed by the script ([14:] and [:134]); id 2's K has two rows, so the script skips it.
TRACKS = (('a_landscape', 160, 448, 17, np.float32, np.float64),    # W > 384: 128x384, a shrink on both axes
          ('b_portrait', 448, 160, 3, np.float64, np.float32),      # H > 384: 384x128
          ('c_short_k', 64, 96, 2, np.float32, np.float64),
          ('d_small', 64, 96, 136, np.float32, np.float64),         # W <= 384: floor(96/32)*32 = 96.0, not resized
          ('e_square', 96, 96, 3, np.float32, np.float32))          # square: the portrait branch, H <= 384
F32_THRESHOLD = np.float32(1e-3)


def timestamps(n, t):
    """n distinct integer timestamps whose numeric order differs from the lexicographic order of their decimal strings."""
    return [7 + 13 * i ** 2 + t for i in range(n)]


def synthetic_frame(t, f):
    """-> {'prediction/img', 'prediction/mvs_depth', 'prediction/K', 'prediction/T_1_G'} of frame f (numeric order) of track t."""
    name, H, W, _, mdt, kdt = TRACKS[t]
    g = np.random.default_rng(1000 * t + f)
    yy, xx = np.mgrid[0:H, 0:W]
    img = np.stack([0.5 + 0.35 * np.sin(xx / (9.0 + 2 * c) + f * 0.4 + t) * np.cos(yy / (7.0 + c)) for c in range(3)], -1)
    img = np.clip(img + g.normal(0, 0.04, img.shape), 0, 1).astype(np.float32)
    mvs = (2.0 + 0.8 * np.sin(xx / 23.0 + f * 0.2) * np.cos(yy / 17.0 + t) + g.uniform(0, 0.05, (H, W))).astype(mdt)
    # holes at and below the threshold: zeros, negatives, values exactly at 1e-3 (fp32 and fp64) and just above it; their
    # count alternates in parity so that odd and even numbers of valid pixels occur
    flat = mvs.reshape(-1)
    idx = g.permutation(H * W)[:40 + f % 2]
    flat[idx[:10]] = 0
    flat[idx[10:14]] = -1.5
    flat[idx[14:20]] = 1e-3
    flat[idx[20:26]] = F32_THRESHOLD
    flat[idx[26:30]] = np.nextafter(F32_THRESHOLD, np.float32(1))
    flat[idx[30:]] = g.uniform(0, 1e-3, len(idx) - 30)
    mvs[H // 4:H // 4 + 6, W // 3:W // 3 + 9] = 0
    K = np.array([[0.9 * W + t, 0, W / 2 - 0.25], [0, 0.9 * W + 1.5, H / 2 + 0.5], [0, 0, 1]], dtype=kdt)
    if name == 'c_short_k':
        K = K[:2]
    a = 0.03 * f + 0.1 * t
    T = np.eye(4)
    T[:3, :3] = [[np.cos(a), -np.sin(a) * 0.6, np.sin(a) * 0.8], [np.sin(a), np.cos(a) * 0.6, -np.cos(a) * 0.8], [0, 0.8, 0.6]]
    T[:3, 3] = [0.3 * f - 0.1, 0.05 * t + 0.02 * f, 1.5 - 0.1 * f]
    return {'prediction/img': img, 'prediction/mvs_depth': mvs, 'prediction/K': K, 'prediction/T_1_G': T.astype(kdt)}


def track_files(t):
    """-> [(file name, numeric frame index)] of track t, in the glob's (lexicographic) order."""
    name, _, _, n, _, _ = TRACKS[t]
    return sorted(('%s_%d.h5' % (name, s), f) for f, s in enumerate(timestamps(n, t)))


def kept_frames(t):
    """numeric frame indices the script prepares for track t (TRIM_BAD_FRAMES)."""
    n = TRACKS[t][3]
    return list(range(n))[{0: slice(14, None), 3: slice(None, 134)}.get(t, slice(None))]


def get_im_size(im, dim_max=384, multiple=32):
    H, W, _ = im.shape
    if W > H:
        if W > dim_max:
            sc = dim_max / W
            target_W = dim_max
        else:
            target_W = np.floor(W / multiple) * multiple
            sc = target_W / W
        target_H = int(np.round((H * sc) / multiple) * multiple)
        return [target_H, target_W]
    if H > dim_max:
        sc = dim_max / H
        target_H = dim_max
    else:
        target_H = np.floor(H / multiple) * multiple
        sc = target_H / H
    target_W = int(np.round((W * sc) / multiple) * multiple)
    return [target_H, target_W]


def frame_scale(nn_depth, mvs_depth):
    """One frame's median of nn / mvs over the pixels where mvs > 1e-3 (generate_frame_midas.py:167-172)."""
    idx, idy = np.where(mvs_depth > 1e-3)
    return np.median(nn_depth[idx, idy] / mvs_depth[idx, idy])


def calibrate(depths, mvs_depths):
    """-> (scales, s) of the script's scale loop."""
    scales = [frame_scale(d, m) for d, m in zip(depths, mvs_depths)]
    return scales, np.mean(scales)


def frame_outputs(img_orig, depth, mvs_depth, K, T_1_G, s):
    """The arrays the script writes for one frame (generate_frame_midas.py:177-213)."""
    H, W, _ = img_orig.shape
    target_H, target_W = get_im_size(img_orig)
    img = sk_resize(img_orig, (target_H, target_W)).astype(np.float32)
    T_G_1 = np.array(T_1_G)
    T_G_1[:3, 3] *= s
    T_G_1 = np.linalg.inv(T_G_1).astype(np.float32)
    depth_mvs = (mvs_depth * s).astype(np.float32)
    depth_mvs = sk_resize(depth_mvs, [target_H, target_W]).astype(np.float32)
    in_1 = np.array(K)
    in_1[0, 0] /= W / target_W
    in_1[1, 1] /= H / target_H
    in_1[0, 2] = (target_W - 1) / 2
    in_1[1, 2] = (target_H - 1) / 2
    in_1 = in_1.astype(np.float32)
    depth = sk_resize(depth.astype(np.float32), [target_H, target_W]).astype(np.float32)
    return dict(img=img, pose_c2w=T_G_1, depth_mvs=depth_mvs, intrinsics=in_1, depth_pred=depth, img_orig=img_orig,
                motion_seg=None)
