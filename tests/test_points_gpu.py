"""GPU: the point-cloud export (csrc/points.cu, dvd_b200/points.py, dvd_b200/export_points.py) against the numpy oracle
(oracle/points.py): world points, selection, keys, colours, the voxel reduction, reproducibility across runs and chunk sizes,
a ray-cast static scene with exact depths, and train -> test -> export_points end to end."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cameras(N, H, W):
    from dvd_b200 import synthetic
    K, c2w = [], []
    for i in range(N):
        R, t, k = synthetic.camera(3 * i, H, W)
        k = k.clone()
        k[1, 1] *= 0.9                     # fx != fy, cx != cy: a transposed K shows
        m = torch.eye(4, dtype=torch.float64)
        m[:3, :3], m[:3, 3] = R, t + torch.tensor([0.0, 0.1 * i, -0.05 * i], dtype=torch.float64)
        K.append(k), c2w.append(m)
    return torch.stack(K).float().numpy(), torch.stack(c2w).float().numpy()


def _inputs(N, H, W, seed=0, plant=True):
    from dvd_b200 import synthetic
    depth = synthetic.make_depths(N, H, W, seed=seed, lo=2.0, hi=6.0)[:, 0].clone()
    g = torch.Generator().manual_seed(seed + 1)
    img = torch.rand(N, 3, H, W, generator=g) * 1.2 - 0.1
    if plant:
        t = np.float32(1e-2)
        flat = depth.view(-1)
        for i, v in enumerate([t, np.nextafter(t, np.float32(1)), np.nextafter(t, np.float32(0)), 0.0, -1.0, np.nan, np.inf,
                               20.0]):
            flat[(i * 131 + 7)::(997 + i)] = float(v)
        depth[:, H // 3, :] *= 1.3         # a depth edge: flying pixels on both sides at edge_tol 0.05
        img.view(-1)[5::211] = float('nan')
    K, c2w = _cameras(N, H, W)
    return depth.contiguous(), img.contiguous(), K, c2w


def _dev(*ts):
    return [torch.as_tensor(t).cuda().contiguous() for t in ts]


@pytest.mark.parametrize('N,H,W', [(2, 37, 53), (3, 64, 96)])
def test_world_points_are_the_unprojection_and_match_the_oracle(N, H, W):
    from dvd_b200 import ops, points
    from oracle import points as op
    depth, _, K, c2w = _inputs(N, H, W, plant=False)
    d, = _dev(depth)
    P = points.world_points(d, torch.from_numpy(points.camera_block(K, c2w)).cuda())
    # the model's own convention: K^T, (K^-1)^T from the fp64 inverse, R_c2w, t
    Kt = torch.from_numpy(K.transpose(0, 2, 1).copy()).cuda()
    Ki = torch.from_numpy(np.linalg.inv(K.astype(np.float64)).transpose(0, 2, 1).astype(np.float32)).cuda()
    R, t = torch.from_numpy(c2w[:, :3, :3].copy()).cuda(), torch.from_numpy(c2w[:, :3, 3].copy()).cuda()
    ref = ops.unproject_fwd(d[:, None].contiguous(), ops.pack_poses(Kt, Ki, R, R, t, t), 1)
    assert torch.equal(P.view(torch.int32), ref.view(torch.int32))
    assert rel_err(P, torch.from_numpy(op.world_points(depth.numpy(), K, c2w))) < 1e-6


def _check_select(depth, img, K, c2w, edge_tol, voxel, base=0):
    from dvd_b200 import ops, points
    from oracle import points as op
    d, im = _dev(depth, img)
    P = points.world_points(d, torch.from_numpy(points.camera_block(K, c2w)).cuda())
    origin = points.default_origin(c2w, voxel)
    got = ops.points_select(d, im, P, edge_tol, voxel, origin, base=base)
    ref = op.select(depth.numpy(), img.numpy(), P.cpu().numpy(), edge_tol, voxel, origin, base=base)
    for k in ('mask', 'index', 'key', 'rgb', 'xyz'):
        a = got[k].cpu().numpy()
        assert a.dtype == ref[k].dtype and np.array_equal(a, ref[k]), k
    return got, P


@pytest.mark.parametrize('N,H,W,tol', [(1, 5, 7, 0.05), (2, 37, 53, 0.05), (3, 64, 96, 0.0625), (5, 288, 512, 0.05)])
def test_selection_matches_the_oracle_exactly(N, H, W, tol):
    depth, img, K, c2w = _inputs(N, H, W, seed=N)
    got, _ = _check_select(depth, img, K, c2w, tol, 0.01, base=N * 1000)
    m = got['mask'].sum().item()
    assert 0 < m < N * H * W and got['index'].numel() == m


def test_edge_tol_equality_and_borders_on_the_device():
    # the CPU test's planted cases, through the kernel
    depth = torch.full((2, 3, 4), 2.0)
    depth[0, 1, 1] = 4.0
    depth[1, 0, 1] = 1.0625
    depth[1, 0, 0] = 1.0
    img = torch.rand(2, 3, 3, 4)
    K, c2w = _cameras(2, 3, 4)
    for tol in (0.5, 0.0625, float(np.nextafter(0.0625, 0)), 0.0):
        _check_select(depth, img, K, c2w, tol, 0.125)


def test_key_range_and_argument_errors():
    import ctypes
    from dvd_b200 import _lib, ops, points
    depth, img, K, c2w = _inputs(1, 16, 24, plant=False)
    d, im = _dev(depth, img)
    P = points.world_points(d, torch.from_numpy(points.camera_block(K, c2w)).cuda())
    with pytest.raises(ops.KeyRangeError):
        ops.points_select(d, im, P, 0.05, 1e-7, (0, 0, 0))
    fz = points.Fuser(16, 24, 1e-7, (0, 0, 0))
    with pytest.raises(ValueError, match='larger voxel'):
        fz.add(d, im, torch.from_numpy(points.camera_block(K, c2w)).cuda())
    with pytest.raises(ValueError):
        ops.points_select(d, im[:, :2].contiguous(), P, 0.05)
    with pytest.raises(ValueError):
        ops.points_select(d.cpu(), im.cpu(), P.cpu(), 0.05)
    lib = _lib.load()
    n = ctypes.c_longlong(0)
    assert lib.dvd_points_select(None, None, None, 1, 4, 4, 0.05, 1.0, 0, 0, 0, 0, None, None, None, None, None, None, 0,
                                 ctypes.byref(n), None) == -2
    assert b'null pointer' in lib.dvd_last_error()
    assert lib.dvd_points_select_scratch_bytes(0, 4, 4) == -1 and lib.dvd_voxel_reduce_scratch_bytes(0) == -1


def _fuse_ref(depth, img, P, voxel, origin, tol, min_views):
    from oracle import points as op
    return op.fuse(depth.numpy(), img.numpy(), P.cpu().numpy(), voxel, origin, tol, min_views)


@pytest.mark.parametrize('min_views', [1, 2, 3])
def test_voxel_reduction_matches_the_oracle(min_views):
    from dvd_b200 import points
    N, H, W = 7, 64, 96
    depth, img, K, c2w = _inputs(N, H, W, seed=3)
    d, im = _dev(depth, img)
    voxel = 0.05
    origin = points.default_origin(c2w, voxel)
    got = points.fuse_points(d, im, K, c2w, voxel=voxel, min_views=min_views)
    P = points.world_points(d, torch.from_numpy(points.camera_block(K, c2w)).cuda())
    ref = _fuse_ref(depth, img, P, voxel, origin, 0.05, min_views)
    for k in ('count', 'views'):
        assert np.array_equal(got[k].cpu().numpy(), ref[k]), k
    # the same sequential fp64 sums in the same order: equal, where the bound would be count * eps * sum |x|
    for k in ('xyz', 'rgb'):
        assert np.array_equal(got[k].cpu().numpy(), ref[k]), k
    assert ref['count'].shape[0] > (100 if min_views == 1 else 10) and (ref['views'] >= min_views).all()
    if min_views == 1:
        assert int(got['count'].sum()) == int(points.ops.points_select(d, im, P, 0.05)['index'].numel())


def test_fused_cloud_is_reproducible_and_independent_of_the_chunking():
    from dvd_b200 import points
    N, H, W = 12, 72, 128
    depth, img, K, c2w = _inputs(N, H, W, seed=5)
    d, im = _dev(depth, img)
    runs = [points.fuse_points(d, im, K, c2w, chunk=c) for c in (None, None, 1, 7, N)]
    a = runs[0]
    assert a['count'].numel() > 0
    for b in runs[1:]:
        for k in ('xyz', 'rgb', 'count', 'views'):
            assert torch.equal(a[k], b[k]), k
    # the per-frame clouds: the selection split by frame
    per = points.frame_points(d, im, K, c2w)
    P = points.world_points(d, torch.from_numpy(points.camera_block(K, c2w)).cuda())
    full = points.ops.points_select(d, im, P, 0.05)
    assert len(per) == N and sum(x.shape[0] for x, _ in per) == full['xyz'].shape[0]
    assert torch.equal(torch.cat([x for x, _ in per]), full['xyz']) and torch.equal(torch.cat([c for _, c in per]), full['rgb'])


# ---- a static scene with exact depths --------------------------------------------------------------------------------------
Z_GROUND, Z_TOP, HALF = 0.05, 1.05, 1.0       # ground plane, and a box [-1, 1]^2 x [Z_GROUND, Z_TOP] standing on it


def _look(centre, theta):
    fwd = np.array([-0.15 * centre[0], -0.15 * centre[1], -1.0])
    fwd /= np.linalg.norm(fwd)
    ref = np.array([math.cos(theta + 0.3), math.sin(theta + 0.3), 0.0])
    right = np.cross(fwd, ref)
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    return np.stack([right, down, fwd], 1)    # columns: camera x, y, z in the world


def _scene(n_cam=12, H=72, W=96):
    """ray-cast depth and a checker texture for n_cam cameras above the box (inside its footprint, so its sides are hidden)"""
    K = np.array([[70.0, 0.0, 47.3], [0.0, 66.0, 35.8], [0.0, 0.0, 1.0]])
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
    rays = np.einsum('ij,jhw->ihw', np.linalg.inv(K), np.stack([xs, ys, np.ones_like(xs)]))
    depth, img, c2w = [], [], []
    for i in range(n_cam):
        th = 2 * math.pi * i / n_cam
        C = np.array([0.5 * math.cos(th), 0.45 * math.sin(th), 3.0 + 0.1 * math.sin(2 * th)])
        R = _look(C, th)
        dw = np.einsum('ij,jhw->ihw', R, rays)                   # world direction per unit camera depth
        t_top = (Z_TOP - C[2]) / dw[2]
        hit = np.stack([C[a] + t_top * dw[a] for a in range(3)])
        on_top = (np.abs(hit[0]) <= HALF) & (np.abs(hit[1]) <= HALF)
        t = np.where(on_top, t_top, (Z_GROUND - C[2]) / dw[2])
        p = np.stack([C[a] + t * dw[a] for a in range(3)])
        chk = (np.floor(p[0] * 4) + np.floor(p[1] * 4)) % 2
        img.append(np.stack([0.2 + 0.6 * chk, 0.5 + 0.3 * on_top, 0.9 - 0.7 * chk]))
        depth.append(t)
        m = np.eye(4)
        m[:3, :3], m[:3, 3] = R, C
        c2w.append(m)
    K = np.repeat(K[None], n_cam, 0)
    return (np.stack(depth).astype(np.float32), np.stack(img).astype(np.float32), K.astype(np.float32),
            np.stack(c2w).astype(np.float32))


def _surface_distance(p):
    ground = np.abs(p[:, 2] - Z_GROUND)
    dx = np.maximum(np.abs(p[:, 0]) - HALF, 0)
    dy = np.maximum(np.abs(p[:, 1]) - HALF, 0)
    top = np.sqrt(dx ** 2 + dy ** 2 + (p[:, 2] - Z_TOP) ** 2)
    return np.minimum(ground, top)


def test_static_scene_fuses_onto_its_surfaces():
    from dvd_b200 import points
    depth, img, K, c2w = _scene()
    d, im = _dev(depth, img)
    res = points.fuse_points(d, im, K, c2w, voxel=0.1, min_views=2)
    xyz, views = res['xyz'].cpu().numpy(), res['views'].cpu().numpy()
    assert xyz.shape[0] > 500
    size = float(np.linalg.norm(xyz.max(0) - xyz.min(0)))
    dist = _surface_distance(xyz)
    assert dist.max() <= 1e-5 * size, (dist.max(), size)
    top = np.abs(xyz[:, 2] - Z_TOP) < 0.05
    assert top.sum() > 100 and (~top).sum() > 50                 # both surfaces are there
    centre = top & (np.abs(xyz[:, 0]) < 0.4) & (np.abs(xyz[:, 1]) < 0.4)
    assert centre.sum() >= 40 and (views[centre] == 12).all(), np.unique(views[centre])
    assert views.max() == 12
    # the per-frame clouds lie on the surfaces too
    for x, _ in points.frame_points(d, im, K, c2w):
        x = x.cpu().numpy()
        assert x.shape[0] > 0 and _surface_distance(x).max() <= 1e-5 * size


def test_a_transposed_camera_is_off_the_surfaces():
    """the scene test's sensitivity: the same files with R^T for R (or K^T for K) do not fuse onto the surfaces"""
    from dvd_b200 import points
    depth, img, K, c2w = _scene()
    d, im = _dev(depth, img)
    bad = c2w.copy()
    bad[:, :3, :3] = c2w[:, :3, :3].transpose(0, 2, 1)
    for k, c in ((K, bad), (K.transpose(0, 2, 1).copy(), c2w)):
        try:
            res = points.fuse_points(d, im, k, c, voxel=0.1, min_views=1)
        except ValueError:
            continue
        assert _surface_distance(res['xyz'].cpu().numpy()).max() > 1e-2


# ---- train -> test -> export_points ------------------------------------------------------------------------------------------
BASE = ('--net scene_flow_motion_field --dataset synthetic_sequence --gaps 1,2 --n_frames 8 --height 64 --width 96 --epoch_batches 4 '
        '--lr 1e-6 --batch_size 1 --optim adam --gpu 0 --workers 0 --save_net 1 --save_net_opt --one_way --loss_type l1 --l1_mul 0 '
        '--acc_mul 1 --disp_mul 1 --warm_sf 1 --scene_lr_mul 1000 --repeat 1 --flow_mul 1 --sf_mag_div 100 --time_dependent --midas '
        '--use_disp --vis_batches_train 0 --manual_seed 1').split()


def _run(module, args):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', module] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    return r.stdout


@pytest.mark.timeout(1800)
def test_train_test_export_points_equals_the_oracle(tmp_path):
    from dvd_b200 import ops, points
    from oracle import points as op
    logdir = str(tmp_path / 'log')
    _run('dvd_b200.train', BASE + ['--logdir', logdir, '--epoch', '1'])
    full = os.path.join(logdir, 'scene_flow_motion_field_synthetic_sequence', '0')
    out_root = str(tmp_path / 'test') + '/'
    _run('dvd_b200.test', ['--net', 'scene_flow_motion_field', '--dataset', 'synthetic_sequence', '--checkpoint_path', full,
                           '--epoch', '1', '--batch_size', '1', '--output_dir', out_root, '--gpu', '0', '--workers', '0'])
    test_dir = os.path.join(out_root + 'scene_flow_motion_field_synthetic_sequence_epoch_1', 'epoch0001_test')
    ply, per_dir = str(tmp_path / 'scene.ply'), str(tmp_path / 'frames')
    _run('dvd_b200.export_points', ['--test_dir', test_dir, '--out', ply, '--per_frame', per_dir, '--chunk', '3',
                                    '--min_views', '2', '--frames', '1:'])
    # the oracle on the same files, fed the library's unprojection of them
    zs = [np.load(os.path.join(test_dir, 'batch%04d.npz' % i)) for i in range(1, 8)]
    depth = np.concatenate([z['depth'][:, 0] for z in zs])
    img = np.concatenate([z['img_1'] for z in zs])
    Kt = np.concatenate([z['K'].reshape(-1, 3, 3) for z in zs])
    c2w = np.concatenate([z['cam_c2w'] for z in zs])
    Ki = np.linalg.inv(Kt.transpose(0, 2, 1).astype(np.float64)).transpose(0, 2, 1).astype(np.float32)
    R, t = c2w[:, :3, :3].copy(), c2w[:, :3, 3].copy()
    dv, Ktd, Kid, Rd, td = _dev(depth[:, None], Kt, Ki, R, t)
    P = ops.unproject_fwd(dv, ops.pack_poses(Ktd, Kid, Rd, Rd, td, td), 1).cpu().numpy()
    voxel = points.default_voxel(depth)
    ref = op.fuse(depth, img, P, voxel, points.default_origin(c2w, voxel), 0.05, 2)
    assert ref['count'].shape[0] > 100
    want = str(tmp_path / 'want.ply')
    points.write_ply(want, ref['xyz'], points.mean_rgb_to_u8(ref['rgb']))
    assert open(ply, 'rb').read() == open(want, 'rb').read()
    sel = op.select(depth, img, P, 0.05)
    HW = depth.shape[1] * depth.shape[2]
    f = sel['index'] // HW
    assert sorted(os.listdir(per_dir)) == ['frame_%05d.ply' % i for i in range(1, 8)]
    for j in range(7):
        x, c = points.read_ply(os.path.join(per_dir, 'frame_%05d.ply' % (j + 1)))
        assert np.array_equal(x, sel['xyz'][f == j]) and np.array_equal(c, sel['rgb'][f == j])
