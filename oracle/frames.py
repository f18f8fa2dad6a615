"""TEST INFRASTRUCTURE — the frame stage of scripts/preprocess/davis/generate_frame_midas.py restated as functions (numpy /
scipy, CPU), from the full-resolution MiDaS depth on.

`sk_resize` is skimage.transform.resize(x, shape, preserve_range=True) as skimage >= 0.19 computes it for a float32 input:
ndimage.gaussian_filter with sigma = max(0, (in / out - 1) / 2) and mode 'mirror' (skimage's 'reflect'), then
ndimage.zoom(order=1, mode='mirror', grid_mode=True), then a clip to the input's min and max. skimage is not installed where
this project runs, so this is the one link of the chain that is not checked against the library itself; the fixture's run of
the reference script uses this function in place of skimage's.
"""
import numpy as np
from scipy import ndimage as ndi


def sk_resize(image, output_shape):
    image = np.asarray(image)
    output_shape = tuple(output_shape) + tuple(image.shape[len(output_shape):])
    factors = np.divide(image.shape, output_shape)
    lo, hi = image.min(), image.max()
    if any(o < i for o, i in zip(output_shape, image.shape)):
        image = ndi.gaussian_filter(image, np.maximum(0, (factors - 1) / 2), cval=0, mode='mirror')
    out = ndi.zoom(image, [1 / f for f in factors], order=1, mode='mirror', cval=0, grid_mode=True)
    np.clip(out, lo, hi, out=out)
    return out


def select_points(w2c, intrinsics, h_pt, mask, depth_map=None):
    """One frame's point selection (generate_frame_midas.py:81-101): -> (pts [3,n], mvs depth [n], nn [n] fp32 or None)."""
    H, W = mask.shape
    out = w2c @ h_pt
    im_pt = intrinsics @ out[:3, :]
    depth = im_pt[2, :].copy()
    im_pt = im_pt / im_pt[2:, :]
    sel = np.where((im_pt[0, :] >= 0) * (im_pt[0, :] < W) * (im_pt[1, :] >= 0) * (im_pt[1, :] < H))[0]
    pts, depth = im_pt[:, sel], depth[sel]
    sel = np.where(ndi.map_coordinates(mask, [pts[1, :], pts[0, :]]) < 0.1)[0]
    pts, depth = pts[:, sel], depth[sel]
    sel = np.where(depth > 1e-3)[0]
    pts, depth = pts[:, sel], depth[sel]
    nn = None if depth_map is None else ndi.map_coordinates(depth_map, [pts[1, :], pts[0, :]])
    return pts, depth, nn


def calibrate(extrinsics, intrinsics, h_pt, masks, full_pred_depths):
    """-> (pts_list, mvs_depths, pred_depths, medians, s) of the script's scale loop."""
    pts_list, mvs, pred, med = [], [], [], []
    for f, (mask, d) in enumerate(zip(masks, full_pred_depths)):
        pts, depth, nn = select_points(extrinsics[f], intrinsics, h_pt, mask, d)
        pts_list.append(pts)
        mvs.append(depth)
        pred.append(nn)
        med.append(np.median(nn / depth))
    return pts_list, mvs, pred, med, np.mean(med)


def working_size(H, W, max_W=384, multiple=64):
    sc = max_W / W
    return int(np.round((H * sc) / multiple) * multiple), max_W


def frame_outputs(img_orig, mask, full_pred_depth, w2c, intrinsics, s):
    """The arrays the script writes for one frame (generate_frame_midas.py:110-148)."""
    H, W, _ = img_orig.shape
    th, tw = working_size(H, W)
    img = sk_resize(img_orig, [th, tw]).astype(np.float32)
    T = w2c.copy()
    T[:3, 3] *= s
    pose = np.linalg.inv(T).astype(np.float32)
    depth = sk_resize(full_pred_depth.astype(np.float32), [th, tw]).astype(np.float32)
    in_1 = intrinsics.copy()
    in_1[0, 0] /= W / tw
    in_1[1, 1] /= H / th
    in_1[0, 2] = (tw - 1) / 2
    in_1[1, 2] = (th - 1) / 2
    motion = np.where(sk_resize(mask, [th, tw]) > 1e-3, 1, 0)
    return dict(img=img, pose_c2w=pose, depth_mvs=depth, intrinsics=in_1.astype(np.float32), depth_pred=depth,
                img_orig=img_orig, motion_seg=motion)
