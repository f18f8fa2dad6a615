"""The one reader of a test export and the one writer of what the commands render from it.

A test export is the directory of `batch%04d.npz` files `Model.test_on_batch` (models/scene_flow_motion_field.py) writes;
a file may hold several frames. Frames checks every file before it returns, so a command that reads its export first
fails on a bad file before it touches the device or writes anything.
"""
import glob
import os
import re
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np
import torch

DEPTHS = ('depth', 'depth_nn', 'depth_gt')


def frame_range(frames):
    """`frames` when it looks like a:b (a Python slice of the frames in file order), else ValueError; an argparse type"""
    if not re.fullmatch(r'-?\d*:-?\d*', frames):
        raise ValueError('--frames must look like a:b, got %r' % frames)
    return frames


def chunk_size(chunk):
    """int(chunk), the frames per device chunk, when it is >= 1, else ValueError; an argparse type"""
    if int(chunk) < 1:
        raise ValueError('chunk must be >= 1, got %r' % chunk)
    return int(chunk)


def cuda_device(device=None):
    """CUDA device `device` (default: the current one), made the current device"""
    dev = torch.device('cuda', torch.cuda.current_device() if device is None else device)
    torch.cuda.set_device(dev)
    return dev


def _npy_shape(z, key):
    """the shape of member `key` of the open npz file `z`, read from its .npy header alone"""
    with z.zip.open(key + '.npy') as fp:
        version = np.lib.format.read_magic(fp)
        read = np.lib.format.read_array_header_1_0 if version == (1, 0) else np.lib.format.read_array_header_2_0
        return read(fp)[0]


def list_files(test_dir):
    """The `batch%04d.npz` files in `test_dir` in index order; ValueError when there are none."""
    found = glob.glob(os.path.join(test_dir, 'batch*.npz'))
    files = sorted((int(m.group(1)), f) for f in found for m in [re.fullmatch(r'batch(\d+)\.npz', os.path.basename(f))] if m)
    if not files:
        raise ValueError('no batch%%04d.npz files in %s' % test_dir)
    return [f for _, f in files]


class Frames:
    """The frames of the export `files` (list_files), flattened in file order and selected by `sel` ('a:b', see frame_range).
    Each file must hold `keys` (`depth` among them) and may hold `optional` keys. Every file is opened once and every key
    checked here: depth-like keys are [B,1,H,W] with one H x W in all files, `img_1` [B,3,H,W] (from its .npy header), `K`
    holds 9 B values and `cam_c2w` 12 B or 16 B, B the frames of the file's `depth`. An optional depth-like key is in all
    files or none; an optional `pair_path` counts for a file when it holds one path per frame. ValueError otherwise.

    Per selected frame: a depth-like key is an [N,H,W] fp32 attribute of its name (None for an optional one no file holds),
    `K` [N,3,3] fp32 in column form (the files hold K^T), `c2w` [N,3,4] fp32 and `pair_path` a list of str or None. `ids` are
    the frame numbers (positions in the whole export), `file_of` the file of each frame, and `images(s, e)` reads `img_1`."""

    def __init__(self, files, sel=None, keys=('depth', 'img_1', 'K', 'cam_c2w'), optional=()):
        lo, hi = frame_range(sel).split(':') if sel is not None else ('', '')
        sl = slice(int(lo) if lo else None, int(hi) if hi else None)
        parts = {k: [] for k in tuple(keys) + tuple(optional) if k != 'img_1'}
        where, HW = [], None
        for f in files:
            with np.load(f) as z:
                missing = [k for k in keys if k not in z.files]
                if missing:
                    raise ValueError('%s lacks %s' % (f, ', '.join(missing)))
                d = z['depth']
                if d.ndim != 4 or d.shape[1] != 1:
                    raise ValueError('%s: depth must be [B,1,H,W], got %s' % (f, d.shape))
                B = d.shape[0]
                HW = HW or d.shape[2:]
                if d.shape[2:] != HW:
                    raise ValueError('%s: frames of %dx%d, the first file has %dx%d' % (f, *d.shape[2:], *HW))
                if 'img_1' in keys:
                    shape = _npy_shape(z, 'img_1')
                    if shape != (B, 3, *HW):
                        raise ValueError('%s: img_1 %s does not match depth %s' % (f, shape, d.shape))
                for k in parts:
                    if k not in z.files:                                # an optional key
                        if k == 'pair_path':
                            parts[k] += [None] * B
                        continue
                    a = d if k == 'depth' else z[k]
                    if k in DEPTHS:
                        if a.shape != (B, 1, *HW):
                            raise ValueError('%s: %s must be [%d,1,%d,%d], got %s' % (f, k, B, *HW, a.shape))
                        parts[k].append(np.asarray(a, dtype=np.float32)[:, 0])
                    elif k == 'K':
                        if a.size != 9 * B:
                            raise ValueError('%s: K %s does not hold %d frames' % (f, a.shape, B))
                        parts[k].append(np.asarray(a, dtype=np.float32).reshape(B, 3, 3).transpose(0, 2, 1))
                    elif k == 'cam_c2w':
                        if a.size not in (12 * B, 16 * B):
                            raise ValueError('%s: cam_c2w %s does not hold %d frames' % (f, a.shape, B))
                        parts[k].append(np.asarray(a, dtype=np.float32).reshape(B, -1, 4)[:, :3])
                    elif k == 'pair_path':
                        pp = [str(p) for p in np.asarray(a).reshape(-1)]
                        parts[k] += pp if len(pp) == B else [None] * B
            where += [(f, b) for b in range(B)]
        for k in optional:
            if k in DEPTHS and 0 < len(parts[k]) < len(files):
                raise ValueError('%s is in %d of the %d files of %s; it must be in all or none'
                                 % (k, len(parts[k]), len(files), os.path.dirname(files[0])))
        self.files, self.ids = files, np.arange(len(where))[sl]
        if len(self.ids) == 0:
            raise ValueError('the frame selection %r is empty (%d frames)' % (sel, len(where)))
        for k, v in parts.items():
            if k == 'pair_path':
                v = v[sl]
            else:
                v = np.concatenate(v)[sl] if v else None
            setattr(self, 'c2w' if k == 'cam_c2w' else k, v)
        self._where = where[sl]
        self.file_of = [f for f, _ in self._where]
        self.N, (self.H, self.W) = len(self.ids), HW

    def images(self, s, e):
        """img_1 of frames s..e-1 as [e-s,3,H,W] fp32, each file read once per call"""
        out = np.empty((e - s, 3, self.H, self.W), dtype=np.float32)
        cache = {}
        for j, (f, b) in enumerate(self._where[s:e]):
            if f not in cache:
                with np.load(f) as z:
                    cache[f] = np.asarray(z['img_1'], dtype=np.float32)
            out[j] = cache[f][b]
        return out


def to_device(dev, *arrays):
    """The host arrays in one fp32 buffer sent to device `dev` in one copy: device views with the arrays' shapes."""
    g = torch.from_numpy(np.concatenate([np.asarray(a, dtype=np.float32).reshape(-1) for a in arrays])).to(dev)
    out, o = [], 0
    for a in arrays:
        n = int(np.prod(np.shape(a)))
        out.append(g[o:o + n].view(np.shape(a)))
        o += n
    return out


class _Video:
    def __init__(self, path, fps, shape):
        h, w = shape[0] + shape[0] % 2, shape[1] + shape[1] % 2
        self.w = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*'mp4v'), fps, (w, h))
        if not self.w.isOpened():
            raise RuntimeError('cv2.VideoWriter could not open %s (mp4v, %dx%d)' % (path, w, h))

    def write(self, frame):
        h, w = frame.shape[:2]
        self.w.write(np.pad(frame, ((0, h % 2), (0, w % 2), (0, 0))) if h % 2 or w % 2 else frame)


class Writer:
    """A context that writes PNG files from a pool of min(8, CPUs) threads (cv2 releases the GIL) and mp4v videos. On exit it
    releases the videos and waits for every PNG file; one that cv2 could not write is a RuntimeError naming it."""

    def __init__(self):
        self._pool = ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1))
        self._pngs, self._videos = [], []

    def __enter__(self):
        return self

    def png(self, path, img):
        """queues the write of the BGR uint8 image `img` [h,w,3] to `path`"""
        self._pngs.append((path, self._pool.submit(cv2.imwrite, path, img)))

    def video(self, path, fps, shape):
        """a video of frames of `shape` (h, w) at `fps`; its .write(frame) takes BGR uint8 [h,w,3] frames, and a frame of odd
        height or width is padded to even sizes at the bottom and right with black"""
        self._videos.append(_Video(path, fps, shape))
        return self._videos[-1]

    def __exit__(self, exc_type, exc, tb):
        for v in self._videos:
            v.w.release()
        self._pool.shutdown(wait=True)
        if exc_type is None:
            for path, f in self._pngs:
                if not f.result():
                    raise RuntimeError('cv2.imwrite could not write %s' % path)
