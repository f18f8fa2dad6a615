"""CPU: the depth-of-field oracle (oracle/refocus.py) against facts that need no oracle (identity without blur, an
independent fp64 disc blur, a sharp foreground that takes nothing from the background, a blurred foreground that spreads
over a sharp background, invalid depths as infinitely far), and the host side of dvd_b200/refocus.py that runs before the
device is touched: the focal disparities of the three focus modes, the depth_nn reader, refocus.json and argument checks."""
import json
import os

import numpy as np
import pytest

from oracle import refocus as orf

F32 = np.float32


def _bgr(img_t):
    """floor(255 clip(img)) with NaN -> 0, BGR: the colour rule of points.cu, test_videos and render_views"""
    c = np.clip(np.nan_to_num(np.asarray(img_t, F32), nan=0.0), 0, 1)
    return (c * F32(255)).astype(np.uint8).transpose(1, 2, 0)[..., ::-1]


def _frame(H, W, seed=0):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    depth = (2 + 3 * x / W + np.sin(y / 5)).astype(F32)
    depth[1, 2], depth[3, 4], depth[5, 6], depth[7, 8] = np.nan, -1, 0, np.inf
    img = rng.uniform(-0.2, 1.2, (3, H, W)).astype(F32)
    img[:, 0, :3] = np.nan
    return depth, img


@pytest.mark.parametrize('scale,R', [(0.0, 16), (40.0, 0), (0.0, 0)])
def test_no_blur_reproduces_the_frame(scale, R):
    depth, img = _frame(20, 28)
    out = orf.render_frame(depth, img, F32(0.3), scale, R)
    assert np.array_equal(out, _bgr(img))


def test_everything_in_focus_reproduces_the_frame():
    H, W = 16, 24
    _, img = _frame(H, W, 1)
    depth = np.full((H, W), 2.5, F32)
    assert np.array_equal(orf.render_frame(depth, img, F32(1) / F32(2.5), 30.0, 8), _bgr(img))


def _disc_blur_fp64(img, c0, R):
    """an independent fp64 restatement for a uniform blur radius c0: weights clamp(c0 - r + 1/2, 0, 1) over the R disc,
    normalised over the taps inside the image"""
    _, H, W = img.shape
    col = np.clip(np.nan_to_num(img.astype(np.float64), nan=0.0), 0, 1)
    S, Wt = np.zeros((3, H, W)), np.zeros((H, W))
    for dy in range(-R, R + 1):
        for dx in range(-R, R + 1):
            if dx * dx + dy * dy > R * R:
                continue
            w = min(max(c0 - np.hypot(dx, dy) + 0.5, 0.0), 1.0)
            if w == 0:
                continue
            ys, yd = slice(max(dy, 0), H + min(dy, 0)), slice(max(-dy, 0), H + min(-dy, 0))
            xs, xd = slice(max(dx, 0), W + min(dx, 0)), slice(max(-dx, 0), W + min(-dx, 0))
            S[:, yd, xd] += w * col[:, ys, xs]
            Wt[yd, xd] += w
    return S / Wt


@pytest.mark.parametrize('z,R', [(4.0, 8), (1.5, 5), (8.0, 16)])
def test_uniform_plane_out_of_focus_is_a_disc_blur(z, R):
    H, W = 30, 41
    _, img = _frame(H, W, 2)
    depth = np.full((H, W), z, F32)
    phi, scale = F32(1 / 2.0), F32(24.0)
    c0 = float(min(F32(R), scale * abs(F32(1) / F32(z) - phi)))
    assert 1 < c0 <= R
    out = orf.render_frame(depth, img, phi, scale, R).astype(np.int64)
    ref = np.floor(255 * _disc_blur_fp64(img, c0, R)).astype(np.int64)[::-1].transpose(1, 2, 0)
    assert np.abs(out - ref).max() <= 1
    assert not np.array_equal(out, _bgr(img))


def _square_scene(H=48, W=64):
    depth = np.full((H, W), 8.0, F32)
    depth[16:32, 24:40] = 2.0
    img = np.random.default_rng(3).uniform(0, 1, (3, H, W)).astype(F32)
    return depth, img


def test_sharp_foreground_takes_nothing_from_the_blurred_background():
    depth, img = _square_scene()
    out = orf.render_frame(depth, img, F32(0.5), 40.0, 12)          # focus on the near square, the background at c = 12
    src = _bgr(img)
    assert np.array_equal(out[16:32, 24:40], src[16:32, 24:40])
    assert (out[:8] != src[:8]).any()                                 # the background is blurred


def test_blurred_foreground_spreads_over_the_sharp_background():
    R = 6
    depth, img = _square_scene()
    out = orf.render_frame(depth, img, F32(0.125), 40.0, R)         # focus on the background, the square at c = 6 (= R)
    src = _bgr(img)
    H, W = depth.shape
    y, x = np.mgrid[0:H, 0:W]
    cheb = np.maximum(np.maximum(16 - y, y - 31), np.maximum(24 - x, x - 39))   # > 0 outside the square
    far = cheb > R + 1
    assert np.array_equal(out[far], src[far])
    ring = (cheb >= 1) & (cheb <= 2)
    assert (out[ring] != src[ring]).any(axis=-1).mean() > 0.9        # the square's colour lands past its edge


def test_invalid_depths_render_as_infinitely_far():
    H, W = 20, 24
    depth, img = _frame(H, W, 4)
    bad = np.zeros((H, W), bool)
    bad[6:12, 8:14] = True
    outs = []
    for v in (np.nan, -1.0, 0.0, np.inf, 1e-2):
        d = depth.copy()
        d[bad] = v
        assert (orf.disparity(d)[bad] == 0).all()
        outs.append(orf.render_frame(d, img, F32(0.25), 30.0, 8))
    assert all(np.array_equal(outs[0], o) for o in outs[1:])
    c = orf.blur_radius(orf.disparity(np.where(bad, np.nan, depth)), F32(0.25), F32(30.0), 8)
    assert (c[bad] == np.fmin(F32(8), F32(30.0) * F32(0.25))).all()


def test_tap_order():
    t = orf.taps(2)
    assert len(t) == 13 and t[0] == (-2, 0) and t[-1] == (2, 0) and t == sorted(t)
    assert len(orf.taps(32)) == sum(1 for dy in range(-32, 33) for dx in range(-32, 33) if dx * dx + dy * dy <= 1024)


# ---- focus ---------------------------------------------------------------------------------------------------------------------
def test_focus_depth_and_pull():
    from dvd_b200 import refocus as rf
    depth = np.full((5, 8, 8), 3.0, F32)
    m = rf.source_median(depth, 'x')
    assert m == 3.0
    assert np.array_equal(rf.focus_disparities(depth, m, focus_depth=2.0), np.full(5, F32(1 / 6.0)))
    phi = rf.focus_disparities(depth, m, focus_pull=(0.5, 2.0))
    hand = [F32(1 / 1.5 + (1 / 6.0 - 1 / 1.5) * (t / 4)) for t in range(5)]
    assert phi.dtype == F32 and phi.tolist() == hand
    assert np.array_equal(phi, orf.focus_pull(5, 0.5, 2.0, m)) and np.array_equal(rf.focus_disparities(depth, m, focus_depth=2.0),
                                                                                   orf.focus_depth(5, 2.0, m))
    assert rf.focus_disparities(depth[:1], m, focus_pull=(0.5, 2.0)).tolist() == [F32(1 / 1.5)]


def test_focus_point_window_and_fallbacks():
    from dvd_b200 import refocus as rf
    N, H, W = 4, 10, 12
    depth = np.full((N, H, W), 5.0, F32)
    depth[0, 3:6, 6:9] = np.nan                                      # frame 0: no valid depth in the window -> 1/m
    depth[1, 3:6, 6:9] = [[1, 2, 3], [4, 5, 6], [7, 8, 9]]          # frame 1: median 5 of nine values
    depth[1, 3, 6] = -1                                               # ... with one invalid: median of 2..9 = 5.5
    depth[2, 3:6, 6:9] = 0                                            # frame 2: none valid -> keeps frame 1's
    depth[3, 3:6, 6:9] = 2.0
    m = 4.0
    phi = rf.focus_disparities(depth, m, focus_point=(7, 4), focus_window=1)
    assert phi.tolist() == [F32(1 / 4.0), F32(1 / 5.5), F32(1 / 5.5), F32(0.5)]
    assert np.array_equal(phi, orf.focus_point(depth, 7, 4, 1, m))
    # the window is clipped to the image; the default point is the centre (W // 2, H // 2)
    depth[:, 0, 0] = 1.25
    assert rf.focus_disparities(depth[3:], m, focus_point=(0, 0), focus_window=0).tolist() == [F32(0.8)]
    assert rf.focus_disparities(depth[3:], m, focus_point=(0, 0), focus_window=1).tolist() == [F32(1 / 5.0)]
    assert np.array_equal(rf.focus_disparities(depth, m, focus_window=3), orf.focus_point(depth, W // 2, H // 2, 3, m))
    for bad in ((12, 0), (0, 10), (-1, 3)):
        with pytest.raises(ValueError):
            rf.focus_disparities(depth, m, focus_point=bad)


def test_mean_blur_is_the_mean_of_the_kernels_radius():
    from dvd_b200 import refocus as rf
    depth, _ = _frame(12, 16, 5)
    phi = np.array([0.2, 0.4], F32)
    got = rf.mean_blur(np.stack([depth, depth]), phi, F32(30.0), 8)
    for t in range(2):
        c = orf.blur_radius(orf.disparity(depth), phi[t], F32(30.0), 8)
        assert got[t] == pytest.approx(c.astype(np.float64).mean(), rel=1e-12)


# ---- files, record, arguments --------------------------------------------------------------------------------------------------
def _export(d, N, H, W, nn=True, per_file=2, nn_files=None):
    rng = np.random.default_rng(0)
    os.makedirs(d, exist_ok=True)
    depth = rng.uniform(1, 4, (N, 1, H, W)).astype(F32)
    for b, s in enumerate(range(0, N, per_file)):
        e = min(s + per_file, N)
        z = dict(depth=depth[s:e], img_1=rng.uniform(0, 1, (e - s, 3, H, W)).astype(F32),
                 K=np.tile(np.eye(3, dtype=F32), (e - s, 1, 1)), cam_c2w=np.tile(np.eye(4, dtype=F32), (e - s, 1, 1)))
        if nn and (nn_files is None or b in nn_files):
            z['depth_nn'] = depth[s:e] * F32(1.5)
        np.savez(os.path.join(d, 'batch%04d.npz' % b), **z)
    return str(d), depth[:, 0]


def test_depth_nn_is_read_with_the_frames(tmp_path):
    from dvd_b200.export_io import Frames, list_files
    d, depth = _export(tmp_path / 'a', 5, 6, 7)
    nn = Frames(list_files(d), '1:4', optional=('depth_nn',)).depth_nn
    assert np.array_equal(nn, depth[1:4] * F32(1.5))
    d, _ = _export(tmp_path / 'b', 5, 6, 7, nn=False)
    assert Frames(list_files(d), optional=('depth_nn',)).depth_nn is None
    d, _ = _export(tmp_path / 'c', 5, 6, 7, nn_files=(0, 2))
    with pytest.raises(ValueError, match='depth_nn'):
        Frames(list_files(d), optional=('depth_nn',))


def test_errors_once_the_files_are_read(tmp_path):
    from dvd_b200 import refocus as rf
    d, _ = _export(tmp_path / 'exp', 3, 8, 12)
    out = str(tmp_path / 'out')
    for kw in (dict(focus_point=(12, 0)), dict(focus_point=(0, 8)), dict(frames='5:9')):
        with pytest.raises(ValueError):
            rf.refocus(d, out, **kw)
    z = dict(np.load(os.path.join(d, 'batch0000.npz')))
    z['depth_nn'][:] = np.nan
    np.savez(os.path.join(d, 'batch0000.npz'), **z)
    with pytest.raises(ValueError, match='initial depth'):
        rf.refocus(d, out, frames='0:2')
    with pytest.raises(ValueError):
        rf.refocus(str(tmp_path / 'empty'), out)
    assert not os.path.exists(out)


def test_argument_checks(tmp_path):
    from dvd_b200 import refocus as rf
    base = ['--test_dir', 'x', '--out', 'y']
    a = rf.parse_args(base)
    assert (a.aperture, a.max_blur, a.focus_point, a.focus_depth, a.focus_pull, a.focus_window, a.frames, a.chunk) == \
        (8.0, 16, None, None, None, 2, None, 16)
    a = rf.parse_args(base + ['--focus_point', '3,4', '--max_blur', '32', '--aperture', '0'])
    assert a.focus_point == (3, 4) and a.max_blur == 32 and a.aperture == 0
    assert rf.parse_args(base + ['--focus_pull', '0.5:2']).focus_pull == (0.5, 2.0)
    for bad in (['--aperture', 'nan'], ['--aperture', 'inf'], ['--aperture', '-1'], ['--max_blur', '33'], ['--max_blur', '-1'],
                ['--focus_depth', '2', '--focus_pull', '1:2'], ['--focus_point', '1,2', '--focus_depth', '2'],
                ['--focus_point', '1'], ['--focus_point', 'a,b'], ['--focus_pull', '1:0'], ['--focus_pull', '1:nan'],
                ['--focus_depth', '0'], ['--focus_depth', '-2'], ['--focus_window', '-1'], ['--chunk', '0'], ['--frames', '3']):
        with pytest.raises(SystemExit):
            rf.parse_args(base + bad)
    d, _ = _export(tmp_path / 'exp', 3, 8, 12)
    out = str(tmp_path / 'out')
    for kw in (dict(aperture=float('nan')), dict(aperture=-1.0), dict(max_blur=33), dict(max_blur=2.5), dict(chunk=0),
               dict(focus_depth=2.0, focus_pull=(1.0, 2.0)), dict(focus_point=(1, 1), focus_depth=2.0), dict(focus_depth=0.0),
               dict(focus_pull=(1.0, -1.0)), dict(focus_window=-1)):
        with pytest.raises(ValueError):
            rf.refocus(d, out, **kw)
    assert not os.path.exists(out)


def test_record():
    from dvd_b200 import refocus as rf
    med, scale = {'refined': 2.0, 'initial': 3.0}, {'refined': 16.0, 'initial': 24.0}
    phi = {'refined': np.array([0.5, 0.25], F32), 'initial': np.array([0.1, 0.2], F32)}
    mc = {'refined': np.array([1.5, 2.0]), 'initial': np.array([3.0, 4.0])}
    rec = json.loads(json.dumps(rf.record('x', [4, 5], {'max_blur': 16}, 8, 9, med, scale, phi, mc, True)))
    assert (rec['m'], rec['m_nn'], rec['compare_written'], rec['height'], rec['width']) == (2.0, 3.0, True, 8, 9)
    assert rec['frames'][1] == {'frame': 5, 'focus_disp': 0.25, 'mean_blur': 2.0, 'focus_disp_nn': float(F32(0.2)),
                                'mean_blur_nn': 4.0}
    rec = rf.record('x', [4], {}, 8, 9, {'refined': 2.0}, {'refined': 16.0}, phi, mc, False)
    assert rec['m_nn'] is None and rec['initial'] is None and set(rec['frames'][0]) == {'frame', 'focus_disp', 'mean_blur'}
