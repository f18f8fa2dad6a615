"""GPU: `dvd_splat_views` / `dvd_resolve_views` (csrc/render_views.cu) and `dvd_b200.render_views` against the numpy
restatement of the renderer (oracle/render_views.py): written views and coverage bitwise for every camera path, footprint and
static-cloud source, independence of the chunking, run-to-run reproducibility, and the command line with its videos."""
import json
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from oracle import points as opoints
from oracle import render_views as orv

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _export(d, N, H, W, seed=0, per_file=2):
    """batch%04d.npz files of a sloped background plane seen by N nearly still cameras, a near square that moves across it
    (a moving object: one frame's voxels each), invalid depths (NaN, -1) and out-of-range / NaN colours"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    depth = np.empty((N, 1, H, W), F32)
    for i in range(N):
        dep = 3.0 + 0.5 * x / W + 0.2 * y / H
        x0 = (3 * i) % max(W - W // 4, 1)
        dep[H // 3:H // 3 + H // 4, x0:x0 + W // 4] = 1.5
        depth[i, 0] = dep
    depth[:, 0, 2, 3], depth[:, 0, 5, 7] = np.nan, -1.0
    img = rng.uniform(-0.1, 1.1, (N, 3, H, W)).astype(F32)
    img[:, :, 0, :2] = np.nan
    f = 0.8 * W
    K = np.tile(np.array([[f, 0, (W - 1) / 2], [0, 0.9 * f, (H - 1) / 2], [0, 0, 1]], F32), (N, 1, 1))
    c2w = np.tile(np.eye(4, dtype=F32), (N, 1, 1))
    for i in range(N):
        a = 0.002 * i
        c2w[i, :3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
        c2w[i, :3, 3] = [1e-3 * i, 0, 0]
    os.makedirs(d, exist_ok=True)
    for b, s in enumerate(range(0, N, per_file)):
        e = min(s + per_file, N)
        np.savez(os.path.join(d, 'batch%04d.npz' % b), depth=depth[s:e], img_1=img[s:e], K=K[s:e].transpose(0, 2, 1),
                 cam_c2w=c2w[s:e])
    return str(d)


def _camera_file(d, N):
    """[N,4,4] cameras moved sideways and turned a little from frame 0's"""
    c = np.tile(np.eye(4, dtype=F32), (N, 1, 1))
    for i in range(N):
        a = -0.01 * i
        c[i, :3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
        c[i, :3, 3] = [0.04 * i - 0.1, 0.02, -0.05]
    p = os.path.join(d, 'cams.npy')
    np.save(p, c)
    return p


def _oracle(test_dir, path, splat, static, ply=None, cameras=None, min_views=2):
    from dvd_b200 import points
    from dvd_b200.export_points import Frames, list_files
    fr = Frames(list_files(test_dir))
    N, H, W = fr.N, fr.H, fr.W
    img = fr.images(0, N)
    dev = torch.device('cuda')
    P = points.world_points(torch.from_numpy(fr.depth).to(dev), torch.from_numpy(points.camera_block(fr.K, fr.c2w)).to(dev))
    P = P.cpu().numpy()                                     # the library's own points, as the renderer sees them
    if cameras is not None:
        vK, vc = fr.K, np.load(cameras)[:, :3].astype(F32)
    elif path == 'lock':
        vK, vc = orv.lock_path(fr.K, fr.c2w, N // 2)
    else:
        vK, vc = orv.wiggle_path(fr.K, fr.c2w, fr.ids, 0.03, 60, orv.median_depth(fr.depth))
    cloud = None
    if static == 'auto':
        voxel = points.default_voxel(fr.depth)
        cloud = orv.static_cloud(opoints.fuse(fr.depth, img, P, voxel, points.default_origin(fr.c2w, voxel), 0.05, min_views))
    elif static == 'ply':
        cloud = points.read_ply(ply)
    return orv.render(fr.depth, img, P, vK, vc, splat, cloud)


def _render(test_dir, out, path, splat, static, ply=None, cameras=None, chunk=16, min_views=2):
    from dvd_b200 import render_views as rv
    res = rv.render_views(test_dir, out, path=path, splat=splat, static=ply if static == 'ply' else static, cameras=cameras,
                          chunk=chunk, min_views=min_views)
    views = np.stack([cv2.imread(p, cv2.IMREAD_COLOR) for p in res['views']])
    return res, views


CASES = [  # N, H, W, splat, static, path
    (1, 64, 96, 1, 'none', 'lock'),
    (1, 224, 384, 1, 'auto', 'wiggle'),
    (3, 64, 96, 2, 'auto', 'wiggle'),
    (3, 224, 384, 3, 'ply', 'cameras'),
    (3, 40, 101, 2, 'none', 'cameras'),
    (17, 64, 96, 3, 'auto', 'lock'),
    (17, 40, 101, 1, 'ply', 'wiggle'),
    (17, 224, 384, 2, 'auto', 'cameras'),
]


@pytest.mark.parametrize('N,H,W,splat,static,path', CASES)
def test_views_and_coverage_match_the_oracle_bitwise(tmp_path, N, H, W, splat, static, path):
    from dvd_b200 import export_points
    d = _export(tmp_path / 'exp', N, H, W, seed=N + W)
    ply = None
    if static == 'ply':
        ply = str(tmp_path / 'scene.ply')
        export_points.main(['--test_dir', d, '--out', ply, '--min_views', '1'])
    cams = _camera_file(str(tmp_path), N) if path == 'cameras' else None
    min_views = 1 if N == 1 else 2
    res, views = _render(d, str(tmp_path / 'out'), 'lock' if path == 'cameras' else path, splat, static, ply, cams,
                         min_views=min_views)
    ref, cov = _oracle(d, path, splat, static, ply, cams, min_views)
    assert views.shape == (N, H, W, 3)
    assert np.array_equal(views, ref)
    assert np.array_equal(res['coverage'], cov)
    assert (cov > 0).all()
    if static != 'none':
        assert res['record']['static_points'] > 0
    rec = json.load(open(res['json']))
    assert [v['coverage'] for v in rec['views']] == [float(c) / (H * W) for c in cov]


def test_lock_render_of_the_reference_frame_is_that_frame(tmp_path):
    from dvd_b200 import ops
    from dvd_b200.export_points import Frames, list_files
    N, H, W = 5, 64, 96
    d = _export(tmp_path / 'exp', N, H, W)
    res, views = _render(d, str(tmp_path / 'out'), 'lock', 1, 'none')
    fr = Frames(list_files(d))
    k = N // 2
    kept = opoints.select_mask(fr.depth, 0.05)[k]
    colours = opoints.colours(np.moveaxis(fr.images(k, k + 1)[0], 0, -1))[..., ::-1]
    assert np.array_equal(views[k][kept], colours[kept]) and not views[k][~kept].any()
    assert res['coverage'][k] == kept.sum()
    assert ops.LAUNCHES['n'] > 0


def test_chunking_and_repeated_runs_give_identical_files(tmp_path):
    N, H, W = 17, 64, 96
    d = _export(tmp_path / 'exp', N, H, W, seed=5)
    outs = []
    for i, chunk in enumerate((1, 7, N, 7)):
        res, _ = _render(d, str(tmp_path / ('out%d' % i)), 'wiggle', 2, 'auto', chunk=chunk)
        outs.append([open(p, 'rb').read() for p in res['views']])
        assert len(outs[-1]) == N
    assert outs[0] == outs[1] == outs[2] == outs[3]


def test_kernels_reject_what_they_cannot_index():
    from dvd_b200 import ops
    dev = torch.device('cuda')
    keys = ops.view_keys(2, 8, 8, dev)
    cams = torch.zeros(2, 21, device=dev)
    xyz = torch.zeros(4, 3, device=dev)
    with pytest.raises(ValueError):
        ops.splat_views(keys, xyz, cams, 5)
    with pytest.raises(ValueError):
        ops.splat_views(keys, xyz, cams, 1, index=torch.tensor([0, 1, 2, 128], device=dev))
    with pytest.raises(ValueError):
        ops.splat_views(keys, xyz, torch.zeros(3, 21, device=dev))
    ops.splat_views(keys, xyz, cams, 1)                      # all behind the near plane: nothing lands
    out, cov = ops.resolve_views(keys, torch.zeros(2, 3, 8, 8, device=dev))
    assert not out.any() and cov.tolist() == [0, 0]


def test_command_line_writes_views_and_videos(tmp_path):
    N, H, W = 5, 48, 72
    d = _export(tmp_path / 'exp', N, H, W, seed=9)
    out = str(tmp_path / 'out')
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', 'dvd_b200.render_views', '--test_dir', d, '--out', out, '--path', 'wiggle',
                        '--splat', '2', '--chunk', '2'], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    pngs = sorted(f for f in os.listdir(out) if f.endswith('.png'))
    assert pngs == ['view_%05d.png' % i for i in range(N)]
    for name, w in (('views.mp4', W), ('compare.mp4', 2 * W)):
        cap = cv2.VideoCapture(os.path.join(out, name))
        assert cap.isOpened(), name
        assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == N and cap.get(cv2.CAP_PROP_FPS) == 30, name
        assert (int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT)), int(cap.get(cv2.CAP_PROP_FRAME_WIDTH))) == (H, w), name
        cap.release()
    rec = json.load(open(os.path.join(out, 'render.json')))
    assert rec['options']['path'] == 'wiggle' and rec['options']['splat'] == 2 and len(rec['views']) == N
    assert rec['static_points'] > 0 and all(0 < v['coverage'] <= 1 for v in rec['views'])
