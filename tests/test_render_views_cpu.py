"""CPU: the novel-view oracle (oracle/render_views.py) against facts that need no oracle (identity, an analytic shift,
occlusion, ties), and the host side of dvd_b200/render_views.py that runs before the device is touched: camera paths, the
world-to-camera blocks, the camera file, render.json and every ValueError."""
import json
import os

import numpy as np
import pytest

from oracle import points as opoints
from oracle import render_views as orv

F32 = np.float32


def _cams(N, f=64.0, cx=32.0, cy=24.0):
    K = np.tile(np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]], F32), (N, 1, 1))
    c2w = np.tile(np.eye(4, dtype=F32)[:3], (N, 1, 1))
    return K, c2w


def _scene(N, H, W, seed=0):
    """smooth depth with a few invalid pixels and a depth step, random colours, cameras turning and moving a little"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    depth = np.stack([3 + 0.4 * np.sin(x / 9 + i) * np.cos(y / 7) for i in range(N)]).astype(F32)
    depth[:, H // 2:, W // 3:W // 2] *= F32(0.6)
    depth[:, 2, 3], depth[:, 5, 7] = np.nan, -1
    img = rng.uniform(-0.1, 1.1, (N, 3, H, W)).astype(F32)
    K = np.tile(np.array([[60, 0, (W - 1) / 2], [0, 55, (H - 1) / 2], [0, 0, 1]], F32), (N, 1, 1))
    c2w = np.zeros((N, 3, 4), F32)
    for i in range(N):
        a = 0.02 * i
        c2w[i, :, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
        c2w[i, :, 3] = [0.05 * i, 0.01 * i, -0.02 * i]
    return depth, img, K, c2w


def _P(depth, K, c2w):
    return opoints.world_points(depth, K, c2w).astype(F32)


def _bgr(img_t):
    return opoints.colours(np.moveaxis(img_t, 0, -1))[..., ::-1]


def test_lock_at_the_reference_frame_reproduces_that_frame():
    N, H, W, k = 3, 24, 40, 1
    depth, img, K, c2w = _scene(N, H, W)
    vK, vc = orv.lock_path(K, c2w, k)
    views, cov = orv.render(depth, img, _P(depth, K, c2w), vK, vc, 1, None)
    kept = opoints.select_mask(depth, 0.05)[k]
    assert 0 < kept.sum() < H * W
    assert np.array_equal(views[k][kept], _bgr(img[k])[kept])       # bitwise, every kept pixel
    assert not views[k][~kept].any()                                  # holes exactly at the dropped pixels
    assert cov[k] == kept.sum()


@pytest.mark.parametrize('b,Z,shift', [(0.25, 2.0, 8), (0.5, 4.0, 8), (-0.125, 2.0, -4)])
def test_fronto_parallel_plane_shifts_by_f_b_over_Z(b, Z, shift):
    N, H, W = 1, 48, 64
    K, c2w = _cams(N)
    depth = np.full((N, H, W), Z, F32)
    img = np.random.default_rng(1).uniform(0, 1, (N, 3, H, W)).astype(F32)
    vc = c2w.copy()
    vc[:, 0, 3] = b                                                   # camera moved by b along x: the image moves by -f b / Z
    views, cov = orv.render(depth, img, _P(depth, K, c2w), K, vc, 1, None)
    src = _bgr(img[0])
    if shift > 0:
        assert np.array_equal(views[0][:, :W - shift], src[:, shift:])
        assert not views[0][:, W - shift:].any()
    else:
        assert np.array_equal(views[0][:, -shift:], src[:, :W + shift])
        assert not views[0][:, :-shift].any()
    assert cov[0] == H * (W - abs(shift))


def test_near_square_occludes_the_far_plane():
    N, H, W = 1, 48, 64
    K, c2w = _cams(N)
    depth = np.full((N, H, W), 4.0, F32)
    depth[:, 16:32, 24:40] = 2.0
    img = np.random.default_rng(2).uniform(0, 1, (N, 3, H, W)).astype(F32)
    vc = c2w.copy()
    vc[:, 0, 3] = 0.25                                                # near square shifts 8 px, the plane 4 px
    views, _ = orv.render(depth, img, _P(depth, K, c2w), K, vc, 1, None, edge_tol=10.0)
    src = _bgr(img[0])
    assert np.array_equal(views[0][16:32, 16:32], src[16:32, 24:40])  # the square wins where both land
    assert np.array_equal(views[0][:16, :60], src[:16, 4:64])         # the plane above it moved by 4


def test_at_equal_depth_the_frames_own_point_wins_and_the_static_cloud_fills_holes():
    N, H, W = 1, 24, 32
    K, c2w = _cams(N, cx=16, cy=12)
    depth = np.full((N, H, W), 2.0, F32)
    img = np.random.default_rng(3).uniform(0, 1, (N, 3, H, W)).astype(F32)
    P = _P(depth, K, c2w)
    full = np.moveaxis(P[0], 0, -1).reshape(-1, 3)                    # the same points as a static cloud, all green
    green = np.tile(np.array([[0, 255, 0]], np.uint8), (H * W, 1))
    depth_h = depth.copy()
    depth_h[0, 10:14, 5:9] = np.nan                                   # a hole in the frame (and its flying-pixel ring)
    views, cov = orv.render(depth_h, img, P, K, c2w, 1, (full, green))
    kept = opoints.select_mask(depth_h, 0.05)[0]
    assert np.array_equal(views[0][kept], _bgr(img[0])[kept])
    assert (views[0][~kept] == [0, 255, 0]).all()
    assert cov[0] == H * W


@pytest.mark.parametrize('s', [2, 3, 4])
def test_footprint_covers_s_by_s_pixels_from_the_rounded_centre(s):
    H, W = 16, 16
    K = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]], F32)
    Wc = np.eye(4, dtype=F32)[:3]
    keys = np.full(H * W, orv.EMPTY, np.uint64)
    orv.splat(keys, np.array([[7.5, 3.49, 1.0]], F32), np.array([5], np.uint64), Wc, K, H, W, s)
    x0, y0 = 8 - (s - 1) // 2, 3 - (s - 1) // 2
    hit = np.flatnonzero(keys != orv.EMPTY)
    assert sorted(hit) == sorted((y0 + dy) * W + x0 + dx for dy in range(s) for dx in range(s))
    assert (keys[hit] == (np.uint64(np.float32(1).view(np.uint32)) << np.uint64(32)) | np.uint64(5)).all()


def test_near_plane_and_non_finite_points_are_dropped():
    K = np.eye(3, dtype=F32)
    Wc = np.eye(4, dtype=F32)[:3]
    xyz = np.array([[0, 0, 1e-2], [0, 0, np.nextafter(F32(1e-2), F32(1))], [np.nan, 0, 1], [np.inf, 0, 1], [0, 0, -1]], F32)
    assert orv.project(xyz, Wc, K)[3].tolist() == [False, True, False, False, False]


# ---- dvd_b200/render_views.py host side ----------------------------------------------------------------------------------------
def test_wiggle_and_lock_paths():
    from dvd_b200 import render_views as rv
    N, H, W = 5, 12, 16
    depth, _, K, c2w = _scene(N, H, W)
    ids = np.arange(3, 3 + N)
    m = rv.median_depth(depth)
    assert m == orv.median_depth(depth)
    gK, gc = rv.camera_path(K, c2w, ids, 'wiggle', amplitude=0.03, period=60, median=m)
    oK, oc = orv.wiggle_path(K, c2w, ids, 0.03, 60, m)
    assert gc.dtype == np.float32 and np.array_equal(gc, oc) and np.array_equal(gK, K)
    assert np.array_equal(gc[:, :, :3], c2w[:, :, :3])
    off = gc[:, :, 3].astype(np.float64) - c2w[:, :, 3]
    assert np.allclose(np.linalg.norm(off, axis=1), 0.03 * m, rtol=1e-5)
    gK, gc = rv.camera_path(K, c2w, ids, 'lock')                     # default: the middle selected frame
    assert np.array_equal(gc, np.repeat(c2w[2:3], N, 0)) and np.array_equal(gK, np.repeat(K[2:3], N, 0))
    gK, gc = rv.camera_path(K, c2w, ids, 'lock', ref_frame=6)
    assert np.array_equal(gc, orv.lock_path(K, c2w, 3)[1])
    with pytest.raises(ValueError):
        rv.camera_path(K, c2w, ids, 'lock', ref_frame=2)
    with pytest.raises(ValueError):
        rv.camera_path(K, c2w, ids, 'orbit')


def test_view_blocks_are_the_fp64_inverse_rounded_once():
    from dvd_b200 import render_views as rv
    _, _, K, c2w = _scene(4, 8, 8)
    cams = rv.view_cams(K, c2w)
    assert cams.shape == (4, 21) and cams.dtype == np.float32
    for i in range(4):
        assert np.array_equal(cams[i, :12].reshape(3, 4), orv.w2c(c2w[i]))
        assert np.array_equal(cams[i, 12:].reshape(3, 3), K[i])


def test_camera_file(tmp_path):
    from dvd_b200 import render_views as rv
    _, _, _, c2w = _scene(3, 8, 8)
    full = np.concatenate([c2w, np.tile([[[0, 0, 0, 1]]], (3, 1, 1)).astype(F32)], 1)
    for arr in (c2w, full, full.astype(np.float64)):
        p = str(tmp_path / 'c.npy')
        np.save(p, arr)
        assert np.array_equal(rv.load_cameras(p, 3), c2w)
    for bad in (c2w[:2], c2w[:, :2], np.zeros((3, 3, 3), F32), np.zeros((3, 12), F32), np.zeros((3, 3, 4), np.int32)):
        np.save(str(tmp_path / 'b.npy'), bad)
        with pytest.raises(ValueError):
            rv.load_cameras(str(tmp_path / 'b.npy'), 3)
    with pytest.raises(ValueError):
        rv.load_cameras(str(tmp_path / 'missing.npy'), 3)
    K = np.tile(np.eye(3, dtype=F32), (3, 1, 1))
    gK, gc = rv.camera_path(K, c2w, np.arange(3), 'wiggle', cameras=c2w[::-1])   # overrides the path, keeps K(t)
    assert np.array_equal(gc, c2w[::-1]) and np.array_equal(gK, K)


def test_index_range():
    from dvd_b200 import render_views as rv
    rv.check_index_range(224, 384, 2 ** 32 - 224 * 384 - 1)
    with pytest.raises(ValueError):
        rv.check_index_range(224, 384, 2 ** 32 - 224 * 384)
    depth, img, K, c2w = _scene(1, 8, 8)
    huge = np.broadcast_to(np.zeros((1, 3), F32), (2 ** 32 - 64, 3))    # no memory behind it: the check comes first
    with pytest.raises(ValueError):
        orv.render(depth, img, _P(depth, K, c2w), K, c2w, 1, (huge, np.broadcast_to(np.zeros((1, 3), np.uint8), huge.shape)))


def _export(d, N, H, W):
    depth, img, K, c2w = _scene(N, H, W)
    os.makedirs(d, exist_ok=True)
    full = np.concatenate([c2w, np.tile([[[0, 0, 0, 1]]], (N, 1, 1)).astype(F32)], 1)
    np.savez(os.path.join(d, 'batch0000.npz'), depth=depth[:, None], img_1=img, K=K.transpose(0, 2, 1), cam_c2w=full)
    return str(d)


def test_arguments_and_files_are_checked_before_the_device(tmp_path):
    from dvd_b200 import render_views as rv
    d = _export(tmp_path / 'exp', 3, 8, 12)
    out = str(tmp_path / 'out')
    for kw in (dict(splat=0), dict(splat=5), dict(chunk=0), dict(edge_tol=-1.0), dict(min_views=0), dict(voxel=-1.0),
               dict(static=str(tmp_path / 'nope.ply')), dict(cameras=np.zeros((2, 3, 4), F32)), dict(path='orbit'),
               dict(ref_frame=7), dict(frames='5:9')):
        with pytest.raises(ValueError):
            rv.render_views(d, out, **kw)
    np.save(str(tmp_path / 'c.npy'), np.zeros((4, 3, 4), F32))
    with pytest.raises(ValueError):
        rv.render_views(d, out, cameras=str(tmp_path / 'c.npy'))
    with pytest.raises(ValueError):
        rv.render_views(str(tmp_path / 'empty'), out)
    assert not os.path.exists(out)


def test_record_and_cli_defaults(tmp_path):
    from dvd_b200 import render_views as rv
    a = rv.parse_args(['--test_dir', 'x', '--out', 'y'])
    assert (a.path, a.ref_frame, a.amplitude, a.period, a.cameras, a.static, a.voxel, a.min_views, a.edge_tol, a.splat, a.frames,
            a.chunk) == ('lock', None, 0.03, 60, None, 'auto', None, 2, 0.05, 1, None, 16)
    with pytest.raises(SystemExit):
        rv.parse_args(['--test_dir', 'x', '--out', 'y', '--path', 'orbit'])
    _, _, K, c2w = _scene(2, 8, 8)
    rec = rv.record('x', [4, 5], K, c2w, [64, 16], {'splat': 1}, 8, 8, 10)
    rec = json.loads(json.dumps(rec))
    assert (rec['height'], rec['width'], rec['static_points'], rec['options']) == (8, 8, 10, {'splat': 1})
    assert [v['frame'] for v in rec['views']] == [4, 5] and [v['coverage'] for v in rec['views']] == [1.0, 0.25]
    assert np.array_equal(np.array([v['c2w'] for v in rec['views']], F32), c2w)
    assert np.array_equal(np.array([v['K'] for v in rec['views']], F32), K)
