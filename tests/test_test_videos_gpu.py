"""GPU: `dvd_vis_panels` (csrc/test_videos.cu) and `dvd_b200.test_videos` against the numpy restatement of the canvases
(oracle/test_videos.py): comparison, RGB and temporal-slice canvases bitwise, chunking, and the end-to-end `train` -> `test
--videos` run with its videos and page."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from oracle import test_videos as ov

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_struct_size_matches_ctypes():
    from dvd_b200 import _lib
    lib = _lib.load()
    assert lib.dvd_struct_size(4) == ctypes.sizeof(_lib.VisPanel)
    assert lib.dvd_struct_size(99) == -1


def _export(d, N, H, W, seed, per_file=2):
    """batch%04d.npz files of N frames with planted cases: NaN, zero and negative initial depth, zero / 1e-8 / NaN / negative GT,
    NaN and out-of-range colours, and a slice row whose initial depth is constant over every frame."""
    rng = np.random.default_rng(seed)
    depth = rng.uniform(0.5, 6.0, (N, 1, H, W)).astype(np.float32)
    nn = rng.uniform(0.5, 6.0, (N, 1, H, W)).astype(np.float32)
    gt = rng.uniform(0.0, 6.0, (N, 1, H, W)).astype(np.float32)
    img = rng.uniform(-0.1, 1.1, (N, 3, H, W)).astype(np.float32)
    nn[:, 0, 1, :3] = [np.nan, 0.0, -2.0]
    gt[:, 0, 2, :5] = [0.0, np.float32(1e-8), np.nextafter(np.float32(1e-8), np.float32(1)), np.nan, -np.float32(1e-8)]
    gt[:, 0, 3, :2] = -1.0
    img[:, :, 0, :2] = np.nan
    img[:, 1, 1, :4] = [0.0, 1.0, np.float32(128) / np.float32(255), np.inf]
    r = ov.default_slice_rows(H)[0]
    nn[:, 0, r, :] = 3.0                                        # a constant slice: vmin == vmax
    os.makedirs(d, exist_ok=True)
    for i, s in enumerate(range(0, N, per_file)):
        e = min(s + per_file, N)
        np.savez(os.path.join(d, 'batch%04d.npz' % i), depth=depth[s:e], depth_nn=nn[s:e], depth_gt=gt[s:e], img_1=img[s:e],
                 K=np.eye(3, dtype=np.float32))
    return dict(depth=depth, depth_nn=nn, depth_gt=gt, img_1=img)


def _read(d, kind, n):
    return np.stack([cv2.imread(os.path.join(d, '%s_%04d.png' % (kind, i)), cv2.IMREAD_UNCHANGED) for i in range(n)])


@pytest.mark.parametrize('N,H,W', [(1, 64, 96), (3, 224, 384), (17, 36, 101)])
def test_canvases_equal_the_oracle(tmp_path, N, H, W):
    from dvd_b200 import test_videos
    d = str(tmp_path / 'run' / 'epochbest_test')
    ex = _export(d, N, H, W, seed=N)
    res = test_videos.render_test_videos(d, chunk=2)
    lut = ov.turbo_lut()
    a, b = ov.default_slice_rows(H)
    assert res['slice_rows'] == (a, b) and res['frames'] == N
    assert len(os.listdir(d)) == len(res['compare']) + len(res['rgb']) + len(res['temporal_slice']) + (N + 1) // 2
    cmp_ref = ov.compare_canvases(ex['depth'], ex['depth_nn'], ex['depth_gt'], lut)
    assert np.array_equal(_read(d, 'compare', N), cmp_ref)
    assert np.array_equal(_read(d, 'rgb', N), ov.rgb_canvases(ex['img_1']))
    sl_ref = ov.slice_canvases(ex['depth'], ex['depth_nn'], (a, b), lut)
    assert np.array_equal(_read(d, 'temporal_slice', b - a), sl_ref)
    # the planted cases reach the canvases: NaN initial depth and 0 / 0 GT are black, the constant slice is the first colour
    _, _, pos = ov.layout(3, H, W)
    (y0, x0), (y1, x1), (y2, x2) = pos
    assert cmp_ref[0, y1 + 1, x1].tolist() == [0, 0, 0] and cmp_ref[0, y2 + 2, x2 + 4].tolist() == [0, 0, 0]
    _, _, spos = ov.layout(2, N, W)
    assert (sl_ref[0, spos[1][0]:spos[1][0] + N, spos[1][1]:spos[1][1] + W] == lut[0]).all()


def test_template_pixels_outside_the_panels_are_kept():
    """random template bytes, two panels with gaps between them, odd canvas widths (byte stores) and a multiple of 4 (word stores)"""
    from dvd_b200 import ops
    dev = torch.device('cuda')
    g = torch.Generator().manual_seed(0)
    lut = torch.from_numpy(ov.turbo_lut()).to(dev)
    for CH, CW in ((40, 61), (40, 64), (33, 203)):
        n, h, w = 3, 17, 23
        tmpl = torch.randint(0, 256, (n, CH, CW, 3), dtype=torch.uint8, generator=g)
        src = torch.rand(n, h, w, generator=g) * 4 + 0.5
        img = torch.rand(n, 3, h, w, generator=g)
        vmin = torch.full((n,), 0.25, dtype=torch.float64, device=dev)
        vmax = torch.tensor([2.0, 1.0, 0.25], dtype=torch.float64, device=dev)
        out = torch.empty(n, CH, CW, 3, dtype=torch.uint8, device=dev)
        sd, idv = src.to(dev), img.to(dev)
        ops.vis_panels(tmpl.to(dev), [ops.vis_panel(sd, 'disp', h, w, 3, 5, (h * w, w, 1, 0), vmin=vmin, vmax=vmax),
                                      ops.vis_panel(idv, 'rgb', h, w, 9, 5 + w + 3, (3 * h * w, w, 1, h * w))],
                       lut, out, tmpl_stride=CH * CW * 3)
        o = out.cpu().numpy()
        ref = tmpl.numpy().copy()
        for c in range(n):
            ref[c, 3:3 + h, 5:5 + w] = ov.colour(ov.disp(src[c].numpy()), vmin[c].item(), vmax[c].item(), ov.turbo_lut())
        ref[:, 9:9 + h, 8 + w:8 + 2 * w] = ov.rgb_canvases(img.numpy())
        assert np.array_equal(o, ref), (CH, CW)
    with pytest.raises(RuntimeError, match='overlap'):
        ops.vis_panels(tmpl.to(dev), [ops.vis_panel(idv, 'rgb', h, w, 0, 0, (3 * h * w, w, 1, h * w)),
                                      ops.vis_panel(idv, 'rgb', h, w, h - 1, w - 1, (3 * h * w, w, 1, h * w))], None, out)
    with pytest.raises(ValueError, match='reads element'):
        ops.vis_panels(tmpl.to(dev), [ops.vis_panel(idv, 'rgb', h + 1, w, 0, 0, (3 * h * w, w, 1, h * w))], None, out)


def test_chunk_sizes_give_byte_identical_files(tmp_path):
    from dvd_b200 import test_videos
    N = 17
    src = str(tmp_path / 'src' / 'epochbest_test')
    _export(src, N, 64, 96, seed=5, per_file=3)
    pngs = {}
    for chunk in (1, 7, N):
        d = str(tmp_path / ('c%d' % chunk) / 'epochbest_test')
        shutil.copytree(src, d)
        res = test_videos.render_test_videos(d, chunk=chunk)
        pngs[chunk] = {os.path.basename(p): open(p, 'rb').read() for k in ('compare', 'rgb', 'temporal_slice') for p in res[k]}
    assert len(pngs[1]) == 2 * N + 20
    assert pngs[1] == pngs[7] == pngs[N]


BASE = ('--net scene_flow_motion_field --dataset synthetic_sequence --gaps 1,2 --n_frames 8 --height 64 --width 96 --epoch_batches 4 '
        '--lr 1e-6 --batch_size 1 --optim adam --gpu 0 --workers 0 --save_net 1 --save_net_opt --one_way --loss_type l1 --l1_mul 0 '
        '--acc_mul 1 --disp_mul 1 --warm_sf 1 --scene_lr_mul 1000 --repeat 1 --flow_mul 1 --sf_mag_div 100 --time_dependent --midas '
        '--use_disp --vis_batches_train 0 --manual_seed 1').split()


def _run(module, args):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', module] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    return r.stdout


def _check_outputs(outdir, n, n_slices):
    from dvd_b200 import ops
    parent, es = os.path.dirname(outdir), os.path.basename(outdir)
    names = sorted(os.listdir(outdir))
    assert names == sorted(['batch%04d.npz' % i for i in range(n)] + ['compare_%04d.png' % i for i in range(n)]
                           + ['rgb_%04d.png' % i for i in range(n)] + ['temporal_slice_%04d.png' % i for i in range(n_slices)])
    for video, frames, fps, like in ((es + '.mp4', n, 30, 'compare_0000.png'), (es + '_rgb.mp4', n, 30, 'rgb_0000.png'),
                                     (es + '_temporal.mp4', n_slices, 2, 'temporal_slice_0000.png')):
        cap = cv2.VideoCapture(os.path.join(parent, video))
        assert cap.isOpened(), video
        h, w = cv2.imread(os.path.join(outdir, like)).shape[:2]
        assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == frames and cap.get(cv2.CAP_PROP_FPS) == fps, video
        vw, vh = int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
        assert (vh, vw) == (h + h % 2, w + w % 2) and vw % 2 == 0 and vh % 2 == 0, video
        cap.release()
    page = open(os.path.join(parent, es + '.html')).read()
    assert sorted(re.findall(r'src="([^"]+)"', page)) == sorted([es + '.mp4', es + '_rgb.mp4', es + '_temporal.mp4'])
    zs = [np.load(os.path.join(outdir, 'batch%04d.npz' % i)) for i in range(n)]
    d = torch.from_numpy(np.concatenate([z['depth'] for z in zs])).cuda()
    g = torch.from_numpy(np.concatenate([z['depth_gt'] for z in zs]).astype(np.float32)).cuda()
    loss = float((ops.disp_vali(d, g).double() / (d.shape[2] * d.shape[3])).mean())
    assert 'Disparity loss %.6g' % loss in page, (loss, page)


@pytest.mark.timeout(2400)
def test_train_test_videos_end_to_end(tmp_path):
    logdir = str(tmp_path / 'log')
    _run('dvd_b200.train', BASE + ['--logdir', logdir, '--epoch', '1', '--validate'])
    full = os.path.join(logdir, 'scene_flow_motion_field_synthetic_sequence', '0')
    out_root = str(tmp_path / 'test') + '/'
    _run('dvd_b200.test', ['--net', 'scene_flow_motion_field', '--dataset', 'synthetic_sequence', '--checkpoint_path', full,
                           '--epoch', '-1', '--batch_size', '1', '--output_dir', out_root, '--gpu', '0', '--workers', '0',
                           '--videos', '--slice_rows', '8:12'])
    outdir = os.path.join(out_root + 'scene_flow_motion_field_synthetic_sequence_epoch_-1', 'epochbest_test')
    _check_outputs(outdir, 8, 4)
    # the standalone entry point on a copy of the npz files alone
    other = str(tmp_path / 'again' / 'epochbest_test')
    os.makedirs(other)
    for i in range(8):
        shutil.copy(os.path.join(outdir, 'batch%04d.npz' % i), other)
    _run('dvd_b200.test_videos', ['--test_dir', other, '--slice_rows', '8:12', '--gpu', '0'])
    _check_outputs(other, 8, 4)
    for f in os.listdir(outdir):
        if f.endswith('.png'):
            assert open(os.path.join(outdir, f), 'rb').read() == open(os.path.join(other, f), 'rb').read(), f
