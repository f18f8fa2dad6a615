"""CPU: dvd_b200/export_io.py, the one reader of a test export and the one writer of what the commands render from it: each
file is opened once, a bad img_1 stops every command before the device, and the writer's and the upload's contracts."""
import os

import cv2
import numpy as np
import pytest
import torch

F32 = np.float32


def _export(d, N=5, H=6, W=8, per_file=2, bad_img_file=None, no_pair_path_file=None):
    """batch%04d.npz files as the test driver writes them (K stored as K^T, cam_c2w 4x4); frames, K"""
    rng = np.random.default_rng(0)
    os.makedirs(d, exist_ok=True)
    depth = rng.uniform(1, 4, (N, 1, H, W)).astype(F32)
    K = np.tile(np.array([[40.0, 0, W / 2], [0, 41.0, H / 2], [0, 0, 1]], F32), (N, 1, 1))
    c2w = np.tile(np.eye(4, dtype=F32), (N, 1, 1))
    c2w[:, 0, 3] = np.arange(N)
    for fi, s in enumerate(range(0, N, per_file)):
        e = min(s + per_file, N)
        z = dict(depth=depth[s:e], depth_nn=depth[s:e] * F32(2), depth_gt=depth[s:e] * F32(3),
                 img_1=rng.uniform(0, 1, (e - s, 3, H, W + (fi == bad_img_file))).astype(F32),
                 K=K[s:e].transpose(0, 2, 1)[:, None, None], cam_c2w=c2w[s:e],
                 pair_path=np.asarray(['/v/frame_%05d.npz' % (10 + i) for i in range(s, e)]))
        if fi == no_pair_path_file:
            del z['pair_path']
        np.savez(os.path.join(d, 'batch%04d.npz' % fi), **z)
    return str(d), depth[:, 0], K, c2w[:, :3]


def test_reader_opens_each_file_once(tmp_path, monkeypatch):
    from dvd_b200.export_io import Frames, list_files
    d, depth, K, c2w = _export(tmp_path / 'exp', no_pair_path_file=1)
    opened = []
    load = np.load

    def counting_load(f, *args, **kw):
        opened.append(os.path.basename(f))
        return load(f, *args, **kw)

    monkeypatch.setattr(np, 'load', counting_load)
    ex = Frames(list_files(d), '1:', ('depth', 'depth_nn', 'depth_gt', 'img_1', 'K', 'cam_c2w'), ('pair_path',))
    assert sorted(opened) == ['batch0000.npz', 'batch0001.npz', 'batch0002.npz']
    assert (ex.N, ex.H, ex.W) == (4, 6, 8) and ex.ids.tolist() == [1, 2, 3, 4]
    assert ex.depth.shape == (4, 6, 8) and ex.depth.dtype == F32
    for k, f in (('depth', 1), ('depth_nn', 2), ('depth_gt', 3)):
        assert np.array_equal(getattr(ex, k), depth[1:] * F32(f))
    assert np.array_equal(ex.K, K[1:]) and np.array_equal(ex.c2w, c2w[1:])
    assert ex.pair_path == ['/v/frame_00011.npz', None, None, '/v/frame_00014.npz']
    assert [os.path.basename(f) for f in ex.file_of] == ['batch0000.npz', 'batch0001.npz', 'batch0001.npz', 'batch0002.npz']
    assert ex.images(0, 4).shape == (4, 3, 6, 8)


def test_a_bad_img_1_stops_every_command_before_the_device(tmp_path, monkeypatch):
    from dvd_b200 import evaluate, export_points, refocus, render_views

    def no_device(*args, **kw):
        raise AssertionError('the device was touched')

    monkeypatch.setattr(torch.cuda, 'set_device', no_device)
    monkeypatch.setattr(torch.cuda, 'current_device', no_device)
    d, _, _, _ = _export(tmp_path / 'exp', bad_img_file=1)
    out = str(tmp_path / 'out')
    with pytest.raises(ValueError, match='batch0001.npz: img_1'):
        export_points.main(['--test_dir', d, '--out', os.path.join(out, 'scene.ply'), '--per_frame', out, '--chunk', '2'])
    with pytest.raises(ValueError, match='batch0001.npz: img_1'):
        refocus.refocus(d, out, chunk=2)
    with pytest.raises(ValueError, match='batch0001.npz: img_1'):
        render_views.render_views(d, out, chunk=2)
    with pytest.raises(ValueError, match='batch0001.npz: img_1'):
        evaluate.evaluate_export(d, str(tmp_path / 'frames'), flows_dir=str(tmp_path / 'flows'), out=out)
    assert not os.path.exists(out)


def test_writer_and_upload(tmp_path):
    from dvd_b200.export_io import Writer, to_device
    img = np.random.default_rng(1).integers(0, 256, (5, 7, 3), dtype=np.uint8)
    with Writer() as w:
        w.png(str(tmp_path / 'a.png'), img)
        v = w.video(str(tmp_path / 'a.mp4'), 30, (5, 7))
        v.write(img)
    assert np.array_equal(cv2.imread(str(tmp_path / 'a.png')), img)
    cap = cv2.VideoCapture(str(tmp_path / 'a.mp4'))
    ok, frame = cap.read()
    cap.release()
    assert ok and frame.shape == (6, 8, 3)                        # odd sizes padded to even
    missing = str(tmp_path / 'no_such_dir' / 'b.png')
    with pytest.raises(RuntimeError, match='no_such_dir'):
        with Writer() as w:
            w.png(missing, img)
    a, b = np.arange(6, dtype=F32).reshape(2, 3), np.arange(4, dtype=F32).reshape(1, 2, 2) + 10
    ga, gb = to_device(torch.device('cpu'), a, b)
    assert ga.shape == (2, 3) and gb.shape == (1, 2, 2) and ga.untyped_storage().data_ptr() == gb.untyped_storage().data_ptr()
    assert np.array_equal(ga.numpy(), a) and np.array_equal(gb.numpy(), b)
