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

ShutterStock (scripts/preprocess/shutterstock/generate_frame_midas.py): ShutterstockFrameBuilder
  input   the per-frame HDF5 files of a track, <root>/triangulation/<track>/*_<timestamp>.h5, read by
          read_shutterstock_track (tracks: sorted(glob(<root>/triangulation/*)), a track's id its index there; frames sorted by
          the integer timestamp; track 0 keeps frames [14:] and track 3 [:134]; a track whose frame 0 prediction/K has fewer
          than 3 rows is skipped). Per frame: prediction/img [H,W,3] fp32 in [0,1], prediction/mvs_depth [H,W] (fp32 or fp64),
          prediction/K [3,3], prediction/T_1_G [4,4] (world-to-camera)
  output  frame_%05d.npz per frame: img [th,tw,3], depth_pred and depth_mvs [th,tw] (two different arrays), intrinsics [3,3]
          and pose_c2w [4,4] (fp32), img_orig as stored and motion_seg=None, with (th, tw) = get_im_size(H, W) (multiples of 32,
          384 along the longer side)

MiDaS runs at the stored size (MidasEngine.forward, the reference's MidasNet(resize=None)). The calibration is dense: per frame
the median of nn / mvs over every pixel where mvs > 1e-3 (ops.dense_ratios, then ops.row_medians), in the MVS map's dtype as
numpy computes it (fp32 threshold, quotient and median for fp32 maps), and s = np.mean of the medians on the host. The
reference's `if not img:` fallback to attrs['image_path'] is unreachable with h5py (a Dataset's truth value is the validity
of its id, and a missing key raises KeyError), so it is not built: a frame without prediction/img raises KeyError.

Deliberate deviations from the ShutterStock script, all ValueError:
  * a frame with no pixel where mvs > 1e-3 (the script gives s = NaN and NaN poses);
  * frames of one track with different stored sizes or MVS dtypes (the training data needs one working size);
  * a stored size that is not a multiple of 32, which the MiDaS engine cannot run (MidasEngine.forward raises ValueError for
    it; the reference fails inside its decoder for most such sizes and otherwise predicts depth at a larger size than the image);
  * a working size of 0 (a side under 32 where the script rounds down);
  * a prediction/img that is not fp32 [H,W,3].

COLMAP: ColmapFrameBuilder, the DAVIS computation on a COLMAP reconstruction of any posed video
  input   a sparse model read by read_colmap_model (cameras, images, points3D as .bin, or as .txt when the .bin files are not
          all there; one PINHOLE or SIMPLE_PINHOLE camera shared by every registered image), the registered images at
          <images_dir>/<name>, and optionally masks at <masks_dir>/<name without its extension>.png (red channel, as DAVIS)
  output  the DAVIS frame files, one per registered image in the sorted order of the names: the same keys, dtypes, working
          size and intrinsics; motion_seg is all 0 without masks

The model becomes what read_cameras returns for a DAVIS track, and FrameBuilder's device passes and frame() run unchanged on
it. COLMAP's world-to-camera [R | t], R = qvec2rotmat(q), is already in the projection's camera axes (x right, y down, z
forward), so no axis flip is applied. Deliberate deviations from what a DAVIS track of the same scene would hold:
  * COLMAP puts the centre of the top-left pixel at (0.5, 0.5), the reference's projection and spline sampling at (0, 0):
    the intrinsics carry cx - 0.5 and cy - 0.5;
  * every point of points3D, in the order of the ids, goes to the calibration, as every .obj vertex does; the visibility
    tracks are not used, so the in-image, mask and depth tests alone select the points;
  * an image file in images_dir that the model did not register raises ValueError: dropping it would shift the time stamps
    (idx / n_frames) of every later frame. So do a camera model other than PINHOLE or SIMPLE_PINHOLE, more than one camera,
    a decoded image whose size is not the camera's, and a model without points or registered images.
"""
import glob
import os
import struct
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from PIL import Image

from . import ops
from .flow_pairs import FRAME_FMT

MAX_W = 384
MULTIPLE = 64
MIDAS_SIZE = (256, 512)
SS_MAX_DIM = 384
SS_MULTIPLE = 32
SS_TRIMS = {0: slice(14, None), 3: slice(None, 134)}    # TRIM_BAD_FRAMES, by track id
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


def _net_device(net):
    dev = next(net.parameters()).device
    if dev.type != 'cuda' or net.training:
        raise ValueError('midas_net must live on a CUDA device, in eval mode')
    return dev


def decode_image(path):
    return np.asarray(Image.open(path)).astype(np.float32) / 255


def decode_mask(path):
    return np.asarray(Image.open(path).convert('RGB')).astype(np.float32)[:, :, 0] / 255


class _FrameFiles:
    """The writer both builders share: frame_%05d.npz of frame(i) for every frame."""

    def write(self, out_dir):
        os.makedirs(out_dir, exist_ok=True)
        for i in range(self.n_frames):
            np.savez(os.path.join(out_dir, FRAME_FMT % i), **self.frame(i))
        return self.n_frames


class FrameBuilder(_FrameFiles):
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
        self._run(midas_net, h_pt, chunk, _net_device(midas_net))

    def _run(self, net, h_pt, chunk, dev):
        """The device passes over self.frames and self.masks (mask paths, or None for all-zero masks) with the cameras
        self.intrinsics, self.extrinsics and the points h_pt [4,V]."""
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
                n, H, W, _ = imgs.shape
                if self.masks is None:                                             # every point passes the mask test
                    masks = np.zeros((n, H, W), np.float32)
                else:
                    masks = np.stack(list(pool.map(decode_mask, self.masks[a:b])))
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


# ---- COLMAP -------------------------------------------------------------------------------------------------------------------
# model id -> (name, parameter count), as COLMAP's read_write_model.py lists them; the count is what skips a camera's record
COLMAP_CAMERA_MODELS = {0: ('SIMPLE_PINHOLE', 3), 1: ('PINHOLE', 4), 2: ('SIMPLE_RADIAL', 4), 3: ('RADIAL', 5), 4: ('OPENCV', 8),
                        5: ('OPENCV_FISHEYE', 8), 6: ('FULL_OPENCV', 12), 7: ('FOV', 5), 8: ('SIMPLE_RADIAL_FISHEYE', 4),
                        9: ('RADIAL_FISHEYE', 5), 10: ('THIN_PRISM_FISHEYE', 12)}
IMAGE_EXTS = ('.jpg', '.jpeg', '.png')


def qvec2rotmat(q):
    """COLMAP's rotation of a stored quaternion (w, x, y, z), [..., 4] -> [..., 3, 3] fp64, with its expressions as written
    (the quaternion is not normalised)."""
    q = np.asarray(q, dtype=np.float64)
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    R = [[1 - 2 * y ** 2 - 2 * z ** 2, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
         [2 * x * y + 2 * w * z, 1 - 2 * x ** 2 - 2 * z ** 2, 2 * y * z - 2 * w * x],
         [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x ** 2 - 2 * y ** 2]]
    return np.stack([np.stack(r, -1) for r in R], -2)


class _Reader:
    """Little-endian fields of a COLMAP .bin file, read in order."""

    def __init__(self, path):
        self.path = path
        with open(path, 'rb') as f:
            self.data = f.read()
        self.pos = 0

    def read(self, fmt):
        try:
            v = struct.unpack_from('<' + fmt, self.data, self.pos)
        except struct.error:
            raise ValueError('%s ends inside a record' % self.path) from None
        self.pos += struct.calcsize('<' + fmt)
        return v

    def name(self):
        end = self.data.find(b'\0', self.pos)
        if end < 0:
            raise ValueError('%s ends inside an image name' % self.path)
        s = self.data[self.pos:end].decode('utf-8')
        self.pos = end + 1
        return s

    def done(self):
        if self.pos > len(self.data):
            raise ValueError('%s ends inside a record' % self.path)
        if self.pos < len(self.data):
            raise ValueError('%s has %d bytes after its last record' % (self.path, len(self.data) - self.pos))


def _text_lines(path):
    with open(path) as f:
        return [ln.rstrip('\r\n') for ln in f]


def _cameras_bin(path):
    r = _Reader(path)
    cams = {}
    for _ in range(r.read('Q')[0]):
        cid, model, w, h = r.read('iiQQ')
        if model not in COLMAP_CAMERA_MODELS:
            raise ValueError('%s: camera %d has the unknown model id %d, whose parameters cannot be skipped' % (path, cid, model))
        name, k = COLMAP_CAMERA_MODELS[model]
        cams[cid] = (name, w, h, r.read('%dd' % k))
    r.done()
    return cams


def _cameras_txt(path):
    cams = {}
    for ln in _text_lines(path):
        e = ln.split()
        if e and not e[0].startswith('#'):
            cams[int(e[0])] = (e[1], int(e[2]), int(e[3]), tuple(float(v) for v in e[4:]))
    return cams


def _images_bin(path):
    """-> {image id: (qvec, tvec, camera id, name)}"""
    r = _Reader(path)
    imgs = {}
    for _ in range(r.read('Q')[0]):
        iid, *qt, cid = r.read('i7di')
        name = r.name()
        n2d = r.read('Q')[0]
        r.pos += 24 * n2d                                    # (x, y, point3D id) per 2-D point: not used
        imgs[iid] = (qt[:4], qt[4:], cid, name)
    r.done()
    return imgs


def _images_txt(path):
    imgs = {}
    lines = iter(_text_lines(path))
    for ln in lines:
        if not ln.strip() or ln.lstrip().startswith('#'):
            continue
        e = ln.split(None, 9)
        if len(e) < 10:
            raise ValueError('%s: image line %r has no name' % (path, ln))
        imgs[int(e[0])] = (tuple(float(v) for v in e[1:5]), tuple(float(v) for v in e[5:8]), int(e[8]), e[9].strip())
        next(lines, None)                                    # its 2-D points, possibly an empty line
    return imgs


def _points_bin(path):
    """-> (ids [V] uint64, xyz [V,3] fp64). A record is 51 bytes (u64 id, 3 f64, 3 u8, f64 error, u64 track length) followed
    by 8 bytes (i32 image id, i32 point2D index) per track element, which are skipped."""
    r = _Reader(path)
    n = r.read('Q')[0]
    data, pos, unpack = r.data, r.pos, struct.Struct('<Q3d3BdQ').unpack_from
    ids, xyz = [], []
    try:
        for _ in range(n):
            rec = unpack(data, pos)
            ids.append(rec[0])
            xyz.append(rec[1:4])
            pos += 51 + 8 * rec[8]
    except struct.error:
        raise ValueError('%s ends inside a record' % path) from None
    r.pos = pos
    r.done()
    return np.asarray(ids, np.uint64), np.asarray(xyz, np.float64).reshape(-1, 3)


def _points_txt(path):
    ids, xyz = [], []
    for ln in _text_lines(path):
        e = ln.split(None, 4)
        if e and not e[0].startswith('#'):
            ids.append(int(e[0]))
            xyz.append([float(v) for v in e[1:4]])
    return np.asarray(ids, np.uint64), np.asarray(xyz, np.float64).reshape(-1, 3)


def _colmap_model(model_dir):
    """read_colmap_model's values, and the camera's (height, width)."""
    parts = ('cameras', 'images', 'points3D')
    if all(os.path.isfile(os.path.join(model_dir, p + '.bin')) for p in parts):
        readers, ext = (_cameras_bin, _images_bin, _points_bin), '.bin'
    elif all(os.path.isfile(os.path.join(model_dir, p + '.txt')) for p in parts):
        readers, ext = (_cameras_txt, _images_txt, _points_txt), '.txt'
    else:
        raise FileNotFoundError('%s holds neither cameras, images and points3D .bin nor the three .txt files' % model_dir)
    cams, imgs, (ids, xyz) = (read(os.path.join(model_dir, p + ext)) for read, p in zip(readers, parts))
    if not imgs:
        raise ValueError('the model in %s has no registered image' % model_dir)
    if not len(ids):
        raise ValueError('the model in %s has no 3-D point' % model_dir)
    used = sorted({im[2] for im in imgs.values()})
    if len(used) != 1:
        raise ValueError('the registered images use %d cameras (%s); the frame files need one camera for the whole video'
                         % (len(used), used))
    if used[0] not in cams:
        raise ValueError('the registered images use camera %d, which the model does not hold' % used[0])
    model, w, h, params = cams[used[0]]
    if model == 'PINHOLE' and len(params) == 4:
        fx, fy, cx, cy = params
    elif model == 'SIMPLE_PINHOLE' and len(params) == 3:
        fx, cx, cy = params
        fy = fx
    else:
        raise ValueError('camera %d is %s with %d parameters; only PINHOLE and SIMPLE_PINHOLE are supported: undistort first: '
                         '`colmap image_undistorter`' % (used[0], model, len(params)))
    order = sorted(imgs.values(), key=lambda im: im[3])
    names = [im[3] for im in order]
    extrinsics = np.zeros([len(order), 4, 4])
    extrinsics[:, :3, :3] = qvec2rotmat([im[0] for im in order])
    extrinsics[:, :3, 3] = [im[1] for im in order]
    extrinsics[:, 3, 3] = 1
    h_pt = np.ones([len(ids), 4])
    h_pt[:, :3] = xyz[np.argsort(ids, kind='stable')]
    intrinsics = np.zeros([3, 3])
    intrinsics[[0, 0, 1, 1, 2], [0, 2, 1, 2, 2]] = [fx, cx - 0.5, fy, cy - 0.5, 1]       # pixel centres at integers
    return intrinsics, names, extrinsics, h_pt.T, (int(h), int(w))


def read_colmap_model(model_dir):
    """A COLMAP sparse model (cameras, images and points3D as .bin, or as .txt when the three .bin files are not all present)
    -> (intrinsics [3,3] fp64 with cx - 0.5 and cy - 0.5, the registered image names sorted, extrinsics [N,4,4] fp64
    world-to-camera [[qvec2rotmat(q), t], [0, 1]] in the order of the names, h_pt [4,V] fp64 of every point in the order of
    the ids): what read_cameras returns for a DAVIS track. ValueError when the registered images do not share one PINHOLE or
    SIMPLE_PINHOLE camera, or the model has no registered image or no point."""
    return _colmap_model(model_dir)[:4]


def colmap_frame_paths(images_dir, names, size):
    """<images_dir>/<name> of each registered image. ValueError for an image file (.jpg, .jpeg, .png) under images_dir that is
    not registered, or a registered image whose size is not size = (height, width); FileNotFoundError for a missing one."""
    registered = set(names)
    extra = []
    for d, _, files in os.walk(images_dir):
        for f in files:
            rel = os.path.relpath(os.path.join(d, f), images_dir).replace(os.sep, '/')
            if os.path.splitext(f)[1].lower() in IMAGE_EXTS and rel not in registered:
                extra.append(rel)
    if extra:
        raise ValueError('%d image(s) under %s are not registered in the model; dropping them would shift the time of every '
                         'later frame, so remove them or register them: %s' % (len(extra), images_dir, sorted(extra)))
    paths = [os.path.join(images_dir, n) for n in names]
    missing = [n for n, p in zip(names, paths) if not os.path.isfile(p)]
    if missing:
        raise FileNotFoundError('registered image(s) missing under %s: %s' % (images_dir, missing))
    for n, p in zip(names, paths):
        with Image.open(p) as im:
            if (im.height, im.width) != tuple(size):
                raise ValueError('image %s is %dx%d, its camera %dx%d (height x width)' % ((n, im.height, im.width) + tuple(size)))
    return paths


class ColmapFrameBuilder(FrameBuilder):
    """Prepares the frames of a COLMAP reconstruction: the images registered in the sparse model under `model_dir`
    (read_colmap_model), sorted by name, read from `images_dir`, with masks `<masks_dir>/<name without extension>.png` or, when
    `masks_dir` is None, all-zero masks. FrameBuilder's device passes and outputs, on `midas_net` (a MidasNet on CUDA, eval
    mode), `chunk` frames per pass. After construction: `names`, `scale` (s), `medians` [N], `counts` [N], `n_frames`, and
    `frame(i)` / `write(out_dir)`.

    Device memory: the ratios of every point in every frame, [N, V] fp64 (8·N·V bytes: 0.8 GB at N = 200, V = 5·10^5), stay
    on the device until the per-frame medians, whose sort of all N rows at once takes about five times as much again (4.0 GB
    at N = 200, V = 5·10^5, tools/bench_prepare_colmap.py); beside them, one chunk's full-resolution images and maps and the
    working-size outputs of every frame. The points are never subsampled: that would change the medians."""

    def __init__(self, images_dir, model_dir, midas_net, masks_dir=None, chunk=8, workers=8):
        if chunk < 1:
            raise ValueError('chunk must be >= 1, got %d' % chunk)
        self.intrinsics, self.names, self.extrinsics, h_pt, size = _colmap_model(model_dir)
        self.frames = colmap_frame_paths(images_dir, self.names, size)
        self.masks = None
        if masks_dir is not None:
            self.masks = [os.path.join(masks_dir, os.path.splitext(n)[0] + '.png') for n in self.names]
            missing = [p for p in self.masks if not os.path.isfile(p)]
            if missing:
                raise FileNotFoundError('%d mask(s) missing: %s' % (len(missing), missing))
        self.n_frames = len(self.frames)
        self.workers = workers
        self._run(midas_net, h_pt, chunk, _net_device(midas_net))


# ---- ShutterStock -------------------------------------------------------------------------------------------------------------
def get_im_size(H, W, dim_max=SS_MAX_DIM, multiple=SS_MULTIPLE):
    """[target_H, target_W] of the ShutterStock script (generate_frame_midas.py:87-106): the longer side (the height when
    H >= W) becomes dim_max, or is rounded down to a multiple when it is not longer than dim_max, which yields a numpy float;
    the other side keeps the aspect ratio, rounded to a multiple. The values are the script's, types included, because the
    intrinsics are computed from them."""
    if W > H:
        if W > dim_max:
            sc = dim_max / W
            target_W = dim_max
        else:
            target_W = np.floor(W / multiple) * multiple
            sc = target_W / W
        return [int(np.round((H * sc) / multiple) * multiple), target_W]
    if H > dim_max:
        sc = dim_max / H
        target_H = dim_max
    else:
        target_H = np.floor(H / multiple) * multiple
        sc = target_H / H
    return [target_H, int(np.round((W * sc) / multiple) * multiple)]


def shutterstock_tracks(root):
    """The script's track list: sorted(glob(<root>/triangulation/*)); a track's id is its index here."""
    return sorted(glob.glob(os.path.join(root, 'triangulation', '*')))


def read_shutterstock_track(root, track_index, open_file=None):
    """-> (track name, handles) of track `track_index` under <root>/triangulation: one open handle per frame, ordered by the
    integer timestamp after the last '_' of the file name, trimmed as TRIM_BAD_FRAMES does for track ids 0 and 3. handles is
    None when frame 0's prediction/K has fewer than 3 rows (the script skips such a track). open_file(path) opens one file;
    the default is h5py.File(path, 'r'), imported here only."""
    tracks = shutterstock_tracks(root)
    if not 0 <= track_index < len(tracks):
        raise ValueError('track id %d: %s holds %d tracks' % (track_index, os.path.join(root, 'triangulation'), len(tracks)))
    path = tracks[track_index]
    files = sorted(glob.glob(os.path.join(path, '*.h5')))
    ts = [int(os.path.basename(f).split('_')[-1].split('.')[0]) for f in files]
    files = [files[i] for i in np.argsort(ts)]
    files = files[SS_TRIMS.get(track_index, slice(None))]
    if not files:
        raise FileNotFoundError('track %d (%s) has no frame file left to read' % (track_index, path))
    if open_file is None:
        import h5py
        open_file = lambda p: h5py.File(p, 'r')                                 # noqa: E731
    handles = [open_file(f) for f in files]
    if len(np.array(handles[0]['prediction/K'])) < 3:
        for h in handles:
            getattr(h, 'close', lambda: None)()
        return os.path.basename(path), None
    return os.path.basename(path), handles


def _item(h, key, f):
    try:
        return h[key]
    except KeyError:
        raise KeyError('frame %d has no %s (the image_path fallback of the reference is not supported)' % (f, key)) from None


class ShutterstockFrameBuilder(_FrameFiles):
    """Prepares the frames of one ShutterStock track from `handles` (read_shutterstock_track's, or any objects with
    ['prediction/...'] item access) with `midas_net` (a MidasNet on CUDA, eval mode), `chunk` frames per device pass. After
    construction: `scale` (s), `medians` [N] and `counts` [N] (valid pixels per frame), `n_frames`, `size` (H, W), `target`
    (th, tw), and `frame(i)` / `write(out_dir)` for the outputs."""

    def __init__(self, handles, midas_net, chunk=8):
        if chunk < 1:
            raise ValueError('chunk must be >= 1, got %d' % chunk)
        self.handles = list(handles)
        if not self.handles:
            raise ValueError('a track needs at least one frame')
        self.n_frames = len(self.handles)
        self.K = [np.array(h['prediction/K']) for h in self.handles]
        self.T_1_G = [np.array(h['prediction/T_1_G']) for h in self.handles]
        dev = next(midas_net.parameters()).device
        if dev.type != 'cuda' or midas_net.training:
            raise ValueError('midas_net must live on a CUDA device, in eval mode')
        self._run(midas_net, chunk, dev)

    def _image(self, f):
        img = np.asarray(_item(self.handles[f], 'prediction/img', f))
        if img.dtype != np.float32 or img.ndim != 3 or img.shape[2] != 3:
            raise ValueError('frame %d: prediction/img must be float32 [H,W,3], got %s %s' % (f, img.dtype, img.shape))
        return img

    def _set_size(self, H, W, mvs_dtype):
        if H % SS_MULTIPLE or W % SS_MULTIPLE:
            raise ValueError('frames %dx%d: MiDaS runs at the stored size, which must be a multiple of %d' % (H, W, SS_MULTIPLE))
        if mvs_dtype not in (np.float32, np.float64):
            raise ValueError('prediction/mvs_depth must be float32 or float64, got %s' % mvs_dtype)
        self.size, self.mvs_dtype = (H, W), mvs_dtype
        self.target_raw = get_im_size(H, W)
        self.target = tuple(int(t) for t in self.target_raw)
        if min(self.target) < 1:
            raise ValueError('frames %dx%d give a working size of %dx%d' % ((H, W) + self.target))

    def _run(self, net, chunk, dev):
        N = self.n_frames
        eng = net.engine()
        img_out, pred_out, mvs_full, meds, cnts = [], [], [], [], []
        weights = None
        for a in range(0, N, chunk):
            b = min(a + chunk, N)
            imgs = [self._image(f) for f in range(a, b)]
            mvs = [np.asarray(self.handles[f]['prediction/mvs_depth']) for f in range(a, b)]
            if a == 0:
                self._set_size(*imgs[0].shape[:2], mvs[0].dtype)
                weights = [torch.from_numpy(ops.gaussian_weights(i, o)[1]).to(dev) for i, o in zip(self.size, self.target)]
            for f, (im, m) in enumerate(zip(imgs, mvs), a):
                if im.shape[:2] != self.size or m.shape != self.size or m.dtype != self.mvs_dtype:
                    raise ValueError('frame %d: image %s and MVS map %s %s, frame 0 %s with %s' % (
                        f, im.shape[:2], m.shape, m.dtype, self.size, np.dtype(self.mvs_dtype)))
            n = b - a
            H, W = self.size
            th, tw = self.target
            img = torch.from_numpy(np.stack(imgs)).to(dev)                                     # [n,H,W,3]
            mvs_d = torch.from_numpy(np.stack(mvs)).to(dev)                                    # [n,H,W], stored dtype
            with torch.no_grad():
                nn = eng.forward(img.permute(0, 3, 1, 2).contiguous(), train=False).reshape(n, H, W)
            med, cnt = ops.row_medians(ops.dense_ratios(nn, mvs_d))
            meds.append(med)
            cnts.append(cnt)
            img_out.append(ops.aa_resize(img, th, tw, weights))
            pred_out.append(ops.aa_resize(nn.reshape(n, H, W, 1), th, tw, weights))
            mvs_full.append(mvs_d)
        med, cnt = torch.cat(meds).cpu().numpy(), torch.cat(cnts).cpu().numpy()
        empty = np.nonzero(cnt == 0)[0]
        if empty.size:
            raise ValueError('no pixel with mvs_depth > 1e-3 in frame(s) %s: the scale is undefined' % empty.tolist())
        self.medians, self.counts = med, cnt
        self.scale = np.mean(med)                          # numpy's mean of the medians' dtype, as the script takes it
        s = float(self.scale)
        th, tw = self.target
        # depth_mvs = (mvs * s).astype(float32), then the resize: a product of the stored dtype rounded once to fp32
        mvs_out = [ops.aa_resize((m * s).float().unsqueeze(-1).contiguous(), th, tw, weights) for m in mvs_full]
        self._img, self._pred, self._mvs = (torch.cat(t) for t in (img_out, pred_out, mvs_out))

    def frame(self, i):
        """The arrays frame_%05d.npz of frame i holds (img_orig is read again from the handle, as the reference does)."""
        H, W = self.size
        return dict(img=self._img[i].cpu().numpy(), pose_c2w=frame_pose(self.T_1_G[i], self.scale),
                    depth_mvs=self._mvs[i, ..., 0].cpu().numpy(), intrinsics=frame_intrinsics(self.K[i], H, W, *self.target_raw),
                    depth_pred=self._pred[i, ..., 0].cpu().numpy(), img_orig=self._image(i), motion_seg=None)
