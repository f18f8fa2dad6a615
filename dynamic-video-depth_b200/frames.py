"""A video's frame files, built from its images and its camera reconstruction: scripts/preprocess/davis/generate_frame_midas.py
on the GPU.

  input   <davis_root>/JPEGImages/1080p/<track>/*.jpg, Annotations/1080p/<track>/*.png (motion masks, red channel),
          triangulation/<track>.intrinsics.txt (row 0: id fx fy cx cy), .matrices.txt (id + 16 camera-to-world entries per
          frame), .obj (the world points, its `v` lines)
  output  frame_%05d.npz per frame with the reference's keys, shapes and dtypes: img [h,384,3], img_orig [H,W,3], depth_pred and
          depth_mvs [h,384] (the same array, as the reference writes it), intrinsics [3,3], pose_c2w [4,4] (fp32) and
          motion_seg [h,384] (int64), h = round(H·384/W / 64)·64

Per chunk of frames, the images go to the device once: MiDaS runs on them between two bicubic resizes (ops.resize_bicubic_ac
around MidasEngine.forward, the resize of MidasNet(resize=[256, 512])); the full-resolution depth and mask maps stay on the
device for the scale calibration (ops.spline_prefilter, ops.calib_ratios) and the working-size resize (ops.aa_resize). The
per-frame medians of nn / depth (ops.row_medians) are read back once; the metric scale is their mean, s, and every camera's
translation is multiplied by it before the pose is inverted. PIL decodes the JPEG and PNG files on the host, in a thread
pool, so the pixels are exactly the reference's.

Deliberate deviations from the reference script:
  * W <= 384 raises ValueError (the script fails there with a NameError: its scale factor is only set for W > 384);
  * a frame with no selected point raises ValueError naming the frames (the script gives s = NaN and NaN poses);
  * the .obj reader keeps every `v` line in file order, where the script's trimesh.load may merge repeated vertices;
  * skimage.transform.resize is computed as the scipy calls skimage >= 0.19 makes (gaussian_filter, zoom(order=1,
    mode='mirror', grid_mode=True), clip); MiDaS resizes the raw image and lets its stem normalise, where the script
    normalises first (bicubic weights sum to one: the difference is rounding only).
"""
import glob
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from PIL import Image

from . import ops
from .flow_pairs import FRAME_FMT

MAX_W = 384
MULTIPLE = 64
MIDAS_SIZE = (256, 512)
# world-to-camera of the reconstruction (OpenGL axes) -> the camera convention the projection uses
_FLIP = np.asarray([[1, 0, 0, 0], [0, -1, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]])


def read_obj_vertices(path):
    """The `v x y z` lines of a Wavefront .obj, in file order -> [V,3] fp64."""
    pts = []
    with open(path) as f:
        for line in f:
            parts = line.split()
            if parts and parts[0] == 'v':
                pts.append([float(x) for x in parts[1:4]])
    if not pts:
        raise ValueError('%s has no vertices' % path)
    return np.asarray(pts, dtype=np.float64)


def read_cameras(davis_root, track):
    """-> (intrinsics [3,3], extrinsics [N,4,4] world-to-camera, h_pt [4,V]) as generate_frame_midas.py:51-63 builds them."""
    base = os.path.join(davis_root, 'triangulation', track)
    fx, fy, cx, cy = np.loadtxt(base + '.intrinsics.txt')[0][1:]
    extrinsics = np.loadtxt(base + '.matrices.txt')[:, 1:]
    extrinsics = _FLIP[None, ...] @ np.linalg.inv(np.reshape(extrinsics, [-1, 4, 4]))
    points = read_obj_vertices(base + '.obj')
    h_pt = np.ones([points.shape[0], 4])
    h_pt[:, :3] = points
    intrinsics = np.zeros([3, 3])
    intrinsics[[0, 0, 1, 1, 2], [0, 2, 1, 2, 2]] = [fx, cx, fy, cy, 1]
    return intrinsics, extrinsics, h_pt.T


def working_size(H, W):
    """(target_H, target_W): width 384, height rounded to a multiple of 64 (generate_frame_midas.py:112-121)."""
    if W <= MAX_W:
        raise ValueError('frames %dx%d: the frame stage needs W > %d (the reference defines no working size below)' % (H, W, MAX_W))
    target_H = int(np.round((H * (MAX_W / W)) / MULTIPLE) * MULTIPLE)
    if target_H < 1:
        raise ValueError('frames %dx%d give a working height of 0' % (H, W))
    return target_H, MAX_W


def frame_intrinsics(intrinsics, H, W, target_H, target_W):
    in_1 = intrinsics.copy()
    in_1[0, 0] /= W / target_W
    in_1[1, 1] /= H / target_H
    in_1[0, 2] = (target_W - 1) / 2
    in_1[1, 2] = (target_H - 1) / 2
    return in_1.astype(np.float32)


def frame_pose(w2c, s):
    """cam-to-world of a world-to-camera matrix whose translation is scaled by s, fp32."""
    T = w2c.copy()
    T[:3, 3] *= s
    return np.linalg.inv(T).astype(np.float32)


def decode_image(path):
    return np.asarray(Image.open(path)).astype(np.float32) / 255


def decode_mask(path):
    return np.asarray(Image.open(path).convert('RGB')).astype(np.float32)[:, :, 0] / 255


class FrameBuilder:
    """Prepares the frames of `track` under `davis_root` with `midas_net` (a MidasNet on CUDA, eval mode), `chunk` frames per
    device pass. After construction: `scale` (s), `medians` [N], `n_frames`, and `frame(i)` / `write(out_dir)` for the outputs."""

    def __init__(self, davis_root, track, midas_net, chunk=8, workers=8):
        if chunk < 1:
            raise ValueError('chunk must be >= 1, got %d' % chunk)
        self.frames = sorted(glob.glob(os.path.join(davis_root, 'JPEGImages', '1080p', track, '*.jpg')))
        self.masks = sorted(glob.glob(os.path.join(davis_root, 'Annotations', '1080p', track, '*.png')))
        if not self.frames or len(self.frames) != len(self.masks):
            raise FileNotFoundError('track %s under %s: %d images and %d masks' % (track, davis_root, len(self.frames),
                                                                                  len(self.masks)))
        self.intrinsics, self.extrinsics, h_pt = read_cameras(davis_root, track)
        if self.extrinsics.shape[0] < len(self.frames):
            raise ValueError('%d cameras for %d frames' % (self.extrinsics.shape[0], len(self.frames)))
        self.n_frames = len(self.frames)
        self.workers = workers
        dev = next(midas_net.parameters()).device
        if dev.type != 'cuda' or midas_net.training:
            raise ValueError('midas_net must live on a CUDA device, in eval mode')
        self._run(midas_net, h_pt, chunk, dev)

    def _run(self, net, h_pt, chunk, dev):
        N = self.n_frames
        points = torch.from_numpy(np.ascontiguousarray(h_pt[:3].T)).to(dev)
        w2c = torch.from_numpy(np.ascontiguousarray(self.extrinsics[:N])).to(dev)
        fx, fy, cx, cy = (float(self.intrinsics[i, j]) for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
        ratio = torch.empty(N, points.shape[0], dtype=torch.float64, device=dev)
        eng = net.engine()
        self._img, self._depth, self._mask = [], [], []
        weights = None
        with ThreadPoolExecutor(self.workers) as pool:
            for a in range(0, N, chunk):
                b = min(a + chunk, N)
                imgs = np.stack(list(pool.map(decode_image, self.frames[a:b])))
                masks = np.stack(list(pool.map(decode_mask, self.masks[a:b])))
                n, H, W, _ = imgs.shape
                if a == 0:
                    self.size = (H, W)
                    self.target = working_size(H, W)
                    weights = [torch.from_numpy(ops.gaussian_weights(i, o)[1]).to(dev) for i, o in zip(self.size, self.target)]
                if (H, W) != self.size or masks.shape[1:] != self.size:
                    raise ValueError('frame %d is %dx%d, frame 0 %dx%d' % ((a, H, W) + self.size))
                img = torch.from_numpy(imgs).to(dev)                               # [n,H,W,3]
                mask = torch.from_numpy(masks).to(dev)                             # [n,H,W]
                x = ops.resize_bicubic_ac(img.permute(0, 3, 1, 2).contiguous(), *MIDAS_SIZE)
                with torch.no_grad():
                    d = eng.forward(x, train=False)
                full = ops.resize_bicubic_ac(d.contiguous(), H, W).reshape(n, H, W)
                ops.calib_ratios(ops.spline_prefilter(full), ops.spline_prefilter(mask), w2c[a:b], points, fx, fy, cx, cy,
                                 out=ratio[a:b])
                th, tw = self.target
                self._img.append(ops.aa_resize(img, th, tw, weights))
                self._depth.append(ops.aa_resize(full.reshape(n, H, W, 1), th, tw, weights))
                self._mask.append(ops.aa_resize(mask.reshape(n, H, W, 1), th, tw, weights))
        self._img, self._depth, self._mask = (torch.cat(t) for t in (self._img, self._depth, self._mask))
        med, cnt = ops.row_medians(ratio)
        med, cnt = med.cpu().numpy(), cnt.cpu().numpy()
        empty = np.nonzero(cnt == 0)[0]
        if empty.size:
            raise ValueError('no reconstructed point passes the selection in frame(s) %s: the scale is undefined' % empty.tolist())
        self.medians = med
        self.counts = cnt
        self.scale = np.mean(med)

    def frame(self, i):
        """The arrays frame_%05d.npz of frame i holds (img_orig is decoded again, as the reference does)."""
        H, W = self.size
        th, tw = self.target
        img = self._img[i].cpu().numpy()
        depth = self._depth[i, ..., 0].cpu().numpy()
        mask = self._mask[i, ..., 0].cpu().numpy()
        return dict(img=img, pose_c2w=frame_pose(self.extrinsics[i], self.scale), depth_mvs=depth,
                    intrinsics=frame_intrinsics(self.intrinsics, H, W, th, tw), depth_pred=depth,
                    img_orig=decode_image(self.frames[i]), motion_seg=np.where(mask > 1e-3, 1, 0))

    def write(self, out_dir):
        os.makedirs(out_dir, exist_ok=True)
        for i in range(self.n_frames):
            np.savez(os.path.join(out_dir, FRAME_FMT % i), **self.frame(i))
        return self.n_frames
