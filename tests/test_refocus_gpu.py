"""GPU: `dvd_refocus` (csrc/refocus.cu) and `dvd_b200.refocus` against the numpy restatement of the depth of field
(oracle/refocus.py): frames bitwise for every blur radius and focus mode, planted invalid depths and colours, independence
of the chunking, run-to-run reproducibility, and the command line with its videos and refocus.json."""
import json
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from oracle import refocus as orf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _scene(N, H, W, seed=0):
    """a sloped plane with a near square moving across it; invalid depths (NaN, -1, 0, +inf), NaN and out-of-range colours,
    and from 3 frames on an all-invalid frame 1"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    depth = np.empty((N, H, W), F32)
    for i in range(N):
        dep = 1.5 + 4.0 * x / W + 0.5 * y / H
        x0 = (3 * i) % max(W - W // 4, 1)
        dep[H // 3:H // 3 + H // 4, x0:x0 + W // 4] = 1.0
        depth[i] = dep
    depth[:, 2, 3], depth[:, 5, 7], depth[:, 6, 1], depth[:, H - 1, W - 1] = np.nan, -1.0, 0.0, np.inf
    if N >= 3:
        depth[1] = np.where(rng.uniform(size=(H, W)) < 0.5, np.nan, -1.0)
        depth[1, ::3, ::2] = 0.0
    img = rng.uniform(-0.1, 1.1, (N, 3, H, W)).astype(F32)
    img[:, :, 0, :2] = np.nan
    return depth, img


def _phi(depth, mode, m):
    N, H, W = depth.shape
    if mode == 'point':
        return orf.focus_point(depth, W // 3, H // 2, 2, m)
    if mode == 'depth':
        return orf.focus_depth(N, 0.7, m)
    return orf.focus_pull(N, 0.3, 3.0, m)


CASES = [  # N, H, W, R, focus mode, aperture
    (1, 64, 96, 32, 'pull', 20.0),
    (1, 224, 384, 16, 'point', 20.0),
    (3, 64, 96, 8, 'depth', 8.0),
    (3, 224, 384, 1, 'point', 8.0),
    (3, 40, 101, 32, 'point', 40.0),
    (17, 64, 96, 16, 'pull', 8.0),
    (17, 40, 101, 8, 'depth', 20.0),
    (17, 224, 384, 0, 'pull', 8.0),
]


@pytest.mark.parametrize('N,H,W,R,mode,aperture', CASES)
def test_kernel_matches_the_oracle_bitwise(N, H, W, R, mode, aperture):
    from dvd_b200 import ops
    depth, img = _scene(N, H, W, seed=N + W + R)
    m = orf.median_valid(depth)
    phi = _phi(depth, mode, m)
    s = F32(aperture * m)
    dev = torch.device('cuda')
    got = ops.refocus(torch.from_numpy(depth).to(dev), torch.from_numpy(img).to(dev), torch.from_numpy(phi).to(dev), s, R)
    ref = orf.render(depth, img, phi, s, R)
    assert got.shape == (N, H, W, 3)
    assert np.array_equal(got.cpu().numpy(), ref)
    if R >= 8:
        assert (ref != np.stack([orf.render_frame(depth[t], img[t], phi[t], 0.0, 0) for t in range(N)])).any()


def test_no_blur_is_the_frame_and_arguments_are_checked():
    from dvd_b200 import ops
    N, H, W = 3, 33, 70
    depth, img = _scene(N, H, W, seed=1)
    dev = torch.device('cuda')
    d, i, p = (torch.from_numpy(a).to(dev) for a in (depth, img, np.full(N, 0.4, F32)))
    col = np.clip(np.nan_to_num(img, nan=0.0), 0, 1)
    frame = (col * F32(255)).astype(np.uint8).transpose(0, 2, 3, 1)[..., ::-1]
    for s, R in ((0.0, 32), (50.0, 0)):
        assert np.array_equal(ops.refocus(d, i, p, s, R).cpu().numpy(), frame)
    for kw in (dict(max_radius=33), dict(max_radius=-1), dict(scale=float('nan')), dict(scale=-1.0), dict(scale=float('inf'))):
        a = dict(scale=1.0, max_radius=4)
        a.update(kw)
        with pytest.raises(ValueError):
            ops.refocus(d, i, p, **a)
    with pytest.raises(ValueError):
        ops.refocus(d, i[:2], p, 1.0, 4)
    with pytest.raises(ValueError):
        ops.refocus(d, i, p[:2], 1.0, 4)
    with pytest.raises(ValueError):
        ops.refocus(d.cpu(), i, p, 1.0, 4)


def _export(d, N, H, W, seed=0, per_file=3, nn=True):
    """batch%04d.npz files of _scene with a flickering depth_nn (each frame's depth scaled and warped a little)"""
    depth, img = _scene(N, H, W, seed)
    rng = np.random.default_rng(seed + 100)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    nnd = np.stack([depth[t] * (1 + 0.2 * rng.uniform(-1, 1)) * (1 + 0.1 * np.sin(x / 7 + t)) for t in range(N)]).astype(F32)
    os.makedirs(d, exist_ok=True)
    for b, s in enumerate(range(0, N, per_file)):
        e = min(s + per_file, N)
        z = dict(depth=depth[s:e, None], img_1=img[s:e], K=np.tile(np.eye(3, dtype=F32), (e - s, 1, 1)),
                 cam_c2w=np.tile(np.eye(4, dtype=F32), (e - s, 1, 1)))
        if nn:
            z['depth_nn'] = nnd[s:e, None]
        np.savez(os.path.join(d, 'batch%04d.npz' % b), **z)
    return str(d)


def _oracle_of_files(d, frames, aperture, R, mode):
    """the oracle of the npz files: the refined render of every selected frame and the focal disparities of both sources"""
    from dvd_b200.export_points import Frames, list_files
    fr = Frames(list_files(d), frames)
    nn = np.concatenate([np.load(f)['depth_nn'][:, 0] for f in list_files(d)])[fr.ids]
    out = {}
    for name, dep in (('refined', fr.depth), ('initial', nn)):
        m = orf.median_valid(dep)
        phi = {'point': lambda: orf.focus_point(dep, fr.W // 2, fr.H // 2, 2, m),
               'depth': lambda: orf.focus_depth(fr.N, 1.5, m), 'pull': lambda: orf.focus_pull(fr.N, 0.5, 2.0, m)}[mode]()
        out[name] = (m, phi, F32(aperture * m))
    m, phi, s = out['refined']
    return orf.render(fr.depth, fr.images(0, fr.N), phi, s, R), out


@pytest.mark.parametrize('mode,R,frames', [('point', 16, None), ('depth', 8, '2:9'), ('pull', 32, '1:')])
def test_written_frames_equal_the_oracle_of_the_files(tmp_path, mode, R, frames):
    from dvd_b200 import refocus as rf
    N, H, W = 10, 48, 72
    d = _export(tmp_path / 'exp', N, H, W, seed=R)
    kw = {'point': {}, 'depth': dict(focus_depth=1.5), 'pull': dict(focus_pull=(0.5, 2.0))}[mode]
    res = rf.refocus(d, str(tmp_path / 'out'), aperture=12.0, max_blur=R, frames=frames, chunk=4, **kw)
    ref, src = _oracle_of_files(d, frames, 12.0, R, mode)
    got = np.stack([cv2.imread(p, cv2.IMREAD_COLOR) for p in res['frames_written']])
    assert np.array_equal(got, ref)
    rec = json.load(open(res['json']))
    assert rec['m'] == src['refined'][0] and rec['m_nn'] == src['initial'][0] and rec['compare_written']
    assert [f['focus_disp'] for f in rec['frames']] == src['refined'][1].astype(np.float64).tolist()
    assert [f['focus_disp_nn'] for f in rec['frames']] == src['initial'][1].astype(np.float64).tolist()
    assert rec['refined']['scale'] == float(src['refined'][2]) and rec['initial']['scale'] == float(src['initial'][2])
    assert all(0 <= f['mean_blur'] <= R and 0 <= f['mean_blur_nn'] <= R for f in rec['frames'])


def test_chunking_and_repeated_runs_give_identical_files(tmp_path):
    from dvd_b200 import refocus as rf
    N = 17
    d = _export(tmp_path / 'exp', N, 40, 101, seed=5)
    outs = []
    for i, chunk in enumerate((1, 7, N, 7)):
        res = rf.refocus(d, str(tmp_path / ('out%d' % i)), max_blur=16, focus_pull=(0.4, 2.5), chunk=chunk)
        outs.append([open(p, 'rb').read() for p in res['frames_written']])
        assert len(outs[-1]) == N
    assert outs[0] == outs[1] == outs[2] == outs[3]


def test_command_line_writes_frames_videos_and_json(tmp_path):
    N, H, W = 7, 45, 70
    d = _export(tmp_path / 'exp', N, H, W, seed=9)
    out = str(tmp_path / 'out')
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', 'dvd_b200.refocus', '--test_dir', d, '--out', out, '--max_blur', '12',
                        '--chunk', '3'], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    pngs = sorted(f for f in os.listdir(out) if f.endswith('.png'))
    assert pngs == ['dof_%05d.png' % i for i in range(N)]
    ref, _ = _oracle_of_files(d, None, 8.0, 12, 'point')
    for i, p in enumerate(pngs):
        assert np.array_equal(cv2.imread(os.path.join(out, p), cv2.IMREAD_COLOR), ref[i]), p
    for name, w in (('dof.mp4', W), ('compare.mp4', 3 * W)):
        cap = cv2.VideoCapture(os.path.join(out, name))
        assert cap.isOpened(), name
        assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == N and cap.get(cv2.CAP_PROP_FPS) == 30, name
        assert (int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT)), int(cap.get(cv2.CAP_PROP_FRAME_WIDTH))) == (H + H % 2, w + w % 2), name
        cap.release()
    rec = json.load(open(os.path.join(out, 'refocus.json')))
    assert rec['options']['max_blur'] == 12 and rec['options']['focus_point'] == [W // 2, H // 2] and len(rec['frames']) == N
    assert rec['compare_written'] and rec['m_nn'] is not None


def test_without_depth_nn_no_comparison_is_written(tmp_path):
    from dvd_b200 import refocus as rf
    d = _export(tmp_path / 'exp', 4, 32, 48, nn=False)
    res = rf.refocus(d, str(tmp_path / 'out'), focus_depth=1.0)
    assert sorted(os.listdir(str(tmp_path / 'out'))) == ['dof.mp4', 'dof_00000.png', 'dof_00001.png', 'dof_00002.png',
                                                        'dof_00003.png', 'refocus.json']
    rec = res['record']
    assert not rec['compare_written'] and rec['m_nn'] is None and 'compare' not in res['videos']
