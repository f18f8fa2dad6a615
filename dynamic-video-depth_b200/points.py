"""World-space point clouds of a video's refined depth maps: one cloud per frame, and a fused cloud of the voxels seen in
several frames (what stays put; a moving object occupies different voxels in each frame and drops out).

Conventions (those of the test export's `batch%04d.npz` files and of the model's own `global_p1`):
  K      [N,3,3] intrinsics, column form (the files store K^T); K^-1 is np.linalg.inv(K) in fp64, transposed, rounded to
         fp32, as the datasets build it, and the points come from the library's unprojection P = R (d K^-1 (x, y, 1)) + t
  c2w    [N,3,4] or [N,4,4] camera-to-world (R | t)
  depth  [N,H,W] fp32; img [N,3,H,W] fp32 in [0, 1]

A pixel is kept when its depth is finite and > 1e-2 (depth2disp's validity) and it is no flying pixel: |d - d_n| / d <=
edge_tol for each in-image 4-neighbour n. Voxel keys are floor(P / voxel) per axis in fp64, offset by a grid origin, 21 bits
per axis. The fused cloud holds, per voxel seen in at least `min_views` frames, the fp64 means of position and colour,
summed in (key, pixel index) order, so it is bitwise reproducible and independent of how the frames are chunked.
"""
import numpy as np
import torch

from . import ops

EDGE_TOL = 0.05
KEY_BITS = 21
VOXEL_DEPTH_FRACTION = 0.002


def camera_block(K, c2w):
    """Host K [N,3,3] (column form) and c2w [N,3,4] / [N,4,4] -> fp32 [N,30]: K^T | (K^-1)^T | R | t, the pose inputs of
    ops.pack_poses in the datasets' storage (K^-1 inverted in fp64 from the fp32 K)."""
    K = np.asarray(K, dtype=np.float32).reshape(-1, 3, 3)
    c2w = np.asarray(c2w, dtype=np.float32)
    N = K.shape[0]
    if c2w.shape[-2:] not in ((3, 4), (4, 4)) or c2w.reshape(-1, *c2w.shape[-2:]).shape[0] != N:
        raise ValueError('c2w must be [%d,3,4] or [%d,4,4], got %s' % (N, N, c2w.shape))
    c2w = c2w.reshape(N, c2w.shape[-2], 4)
    kinv_t = np.linalg.inv(K.astype(np.float64)).transpose(0, 2, 1).astype(np.float32)
    return np.concatenate([K.transpose(0, 2, 1).reshape(N, 9), kinv_t.reshape(N, 9), c2w[:, :3, :3].reshape(N, 9),
                           c2w[:, :3, 3]], 1)


def world_points(depth, cam):
    """depth [N,H,W] fp32 and the device camera_block [N,30] -> P [N,3,H,W] fp32 (dvd_unproject_fwd)."""
    N, H, W = depth.shape
    R = cam[:, 18:27]
    poses = ops.pack_poses(cam[:, 0:9], cam[:, 9:18], R, R, cam[:, 27:30], cam[:, 27:30])
    return ops.unproject_fwd(depth.reshape(N, 1, H, W), poses, 1)


def default_voxel(depth):
    """VOXEL_DEPTH_FRACTION x the median of the valid (finite, > 1e-2) depths of a host array."""
    d = np.asarray(depth, dtype=np.float32)
    valid = d[np.isfinite(d) & (d > np.float32(1e-2))]
    if valid.size == 0:
        raise ValueError('no valid depth (finite and > 1e-2) to derive a voxel size from')
    return VOXEL_DEPTH_FRACTION * float(np.median(valid))


def default_origin(c2w, voxel):
    """Voxel grid origin that centres the 2^21-voxel range of each axis on the mean camera centre."""
    c = np.asarray(c2w, dtype=np.float64)
    c = c.reshape(-1, c.shape[-2], 4)[:, :3, 3].mean(0)
    return tuple(int(v) for v in (np.floor(c / voxel) - 2 ** (KEY_BITS - 1)))


def _to_device_block(K, c2w, device):
    return torch.from_numpy(camera_block(_host(K), _host(c2w))).to(device)


def _host(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _split_frames(sel, n_frames, hw, base):
    """per-frame (xyz, rgb) views of a selection in pixel order"""
    bounds = base + hw * torch.arange(n_frames + 1, device=sel['index'].device, dtype=torch.int64)
    cuts = torch.searchsorted(sel['index'], bounds).cpu().tolist()
    return [(sel['xyz'][a:b], sel['rgb'][a:b]) for a, b in zip(cuts[:-1], cuts[1:])]


def frame_points(depth, img, K, c2w, edge_tol=EDGE_TOL):
    """Per-frame clouds of device depth [N,H,W] and img [N,3,H,W]: a list of N (xyz [n,3] fp32, rgb [n,3] uint8) device tensors
    of the kept pixels in pixel order."""
    N, H, W = depth.shape
    P = world_points(depth, _to_device_block(K, c2w, depth.device))
    return _split_frames(ops.points_select(depth, img, P, edge_tol), N, H * W, 0)


class Fuser:
    """Accumulates the kept points of consecutive chunks of frames and reduces them per voxel."""

    def __init__(self, H, W, voxel, origin, edge_tol=EDGE_TOL, min_views=2):
        if not voxel > 0:
            raise ValueError('voxel must be positive, got %r' % voxel)
        if int(min_views) < 1:
            raise ValueError('min_views must be >= 1, got %r' % min_views)
        self.H, self.W, self.voxel, self.origin = H, W, float(voxel), tuple(int(o) for o in origin)
        self.edge_tol, self.min_views = float(edge_tol), int(min_views)
        self.frames = 0
        self.parts = []

    def add(self, depth, img, cam):
        """One chunk: device depth [n,H,W], img [n,3,H,W], camera_block [n,30]. Returns the chunk's per-frame clouds."""
        n, H, W = depth.shape
        if (H, W) != (self.H, self.W):
            raise ValueError('frame size %dx%d, expected %dx%d' % (H, W, self.H, self.W))
        P = world_points(depth, cam)
        try:
            sel = ops.points_select(depth, img, P, self.edge_tol, self.voxel, self.origin, base=self.frames * H * W)
        except ops.KeyRangeError as e:
            raise ValueError('the scene spans more than 2^%d voxels of %g along an axis (or reaches more than 2^%d voxels from '
                             'the mean camera centre); use a larger voxel (%s)' % (KEY_BITS, self.voxel, KEY_BITS - 1, e)) from None
        self.parts.append({k: sel[k] for k in ('key', 'index', 'xyz', 'rgb')})
        frames = _split_frames(sel, n, H * W, self.frames * H * W)
        self.frames += n
        return frames

    def result(self):
        """Fused cloud: dict of device tensors xyz, rgb [R,3] fp64 means, count, views [R] int32, in key order."""
        cat = {k: torch.cat([p[k] for p in self.parts]) if self.parts else None for k in ('key', 'index', 'xyz', 'rgb')}
        if cat['key'] is None:
            raise ValueError('no frames were added')
        skey, order = torch.sort(cat['key'], stable=True)
        return ops.voxel_reduce(skey.contiguous(), order.contiguous(), cat['index'], cat['xyz'], cat['rgb'], self.H * self.W,
                                self.min_views)


def fuse_points(depth, img, K, c2w, voxel=None, edge_tol=EDGE_TOL, min_views=2, origin=None, chunk=None):
    """Fused cloud of device depth [N,H,W] and img [N,3,H,W] (see Fuser.result). voxel defaults to default_voxel(depth),
    origin to default_origin(c2w, voxel); `chunk` frames are selected at a time (all at once by default)."""
    N, H, W = depth.shape
    voxel = default_voxel(_host(depth)) if voxel is None else float(voxel)
    origin = default_origin(_host(c2w), voxel) if origin is None else origin
    cam = _to_device_block(K, c2w, depth.device)
    fz = Fuser(H, W, voxel, origin, edge_tol, min_views)
    step = N if not chunk else int(chunk)
    for s in range(0, N, step):
        fz.add(depth[s:s + step].contiguous(), img[s:s + step].contiguous(), cam[s:s + step].contiguous())
    return fz.result()


# ---- PLY (binary little-endian: float x, y, z; uchar red, green, blue) -------------------------------------------------------
PLY_DTYPE = np.dtype([('x', '<f4'), ('y', '<f4'), ('z', '<f4'), ('red', 'u1'), ('green', 'u1'), ('blue', 'u1')])


def mean_rgb_to_u8(rgb):
    """fp64 mean colours in [0, 255] -> uint8, rounded half up"""
    return np.clip(np.floor(np.asarray(rgb, dtype=np.float64) + 0.5), 0, 255).astype(np.uint8)


def write_ply(path, xyz, rgb):
    xyz = np.asarray(xyz, dtype=np.float32).reshape(-1, 3)
    rgb = np.asarray(rgb, dtype=np.uint8).reshape(-1, 3)
    if xyz.shape[0] != rgb.shape[0]:
        raise ValueError('xyz has %d rows, rgb %d' % (xyz.shape[0], rgb.shape[0]))
    v = np.empty(xyz.shape[0], dtype=PLY_DTYPE)
    for i, c in enumerate('xyz'):
        v[c] = xyz[:, i]
    for i, c in enumerate(('red', 'green', 'blue')):
        v[c] = rgb[:, i]
    head = ('ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n'
            'property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n' % v.shape[0])
    with open(path, 'wb') as f:
        f.write(head.encode('ascii'))
        f.write(v.tobytes())


def read_ply(path):
    """The vertices write_ply wrote -> (xyz [n,3] fp32, rgb [n,3] uint8)."""
    with open(path, 'rb') as f:
        data = f.read()
    end = data.index(b'end_header\n') + len(b'end_header\n')
    head = data[:end].decode('ascii').split('\n')
    if head[0] != 'ply' or head[1] != 'format binary_little_endian 1.0':
        raise ValueError('%s is not a binary little-endian PLY file' % path)
    n = int(next(line for line in head if line.startswith('element vertex')).split()[2])
    v = np.frombuffer(data, dtype=PLY_DTYPE, count=n, offset=end)
    return np.stack([v['x'], v['y'], v['z']], 1), np.stack([v['red'], v['green'], v['blue']], 1)
