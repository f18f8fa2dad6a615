"""CPU: the frame stage's restatement (oracle/frames.py) and readers (dvd_b200.frames) against the fixture written by the
unmodified generate_frame_midas.py (tests/golden/frames_golden.pt, oracle/gen_golden_frames.py), and the argument checks of
the frame-preparation ops."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import frames as oracle_frames
from oracle import golden_io

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.fixture(scope='module')
def gold():
    return golden_io.load_golden(GOLDEN, 'frames_golden')


@pytest.fixture(scope='module')
def layout(gold, tmp_path_factory):
    root = str(tmp_path_factory.mktemp('davis'))
    for rel, data in gold['inputs'].items():
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, 'wb') as f:
            f.write(data.numpy().tobytes())
    return root


def dog_inputs(gold):
    def dec(k):
        return Image.open(io.BytesIO(gold['inputs'][k].numpy().tobytes()))
    jpgs = sorted(k for k in gold['inputs'] if k.startswith('JPEGImages/1080p/dog/'))
    pngs = sorted(k for k in gold['inputs'] if k.startswith('Annotations/1080p/dog/'))
    return ([np.asarray(dec(k)).astype(np.float32) / 255 for k in jpgs],
            [np.asarray(dec(k).convert('RGB')).astype(np.float32)[:, :, 0] / 255 for k in pngs])


def test_readers_return_the_scripts_cameras(gold, layout):
    from dvd_b200 import frames as fr
    G = gold['globals']
    K, E, h_pt = fr.read_cameras(layout, 'dog')
    assert np.array_equal(K, G['intrinsics'].numpy())
    assert np.array_equal(h_pt, G['h_pt'].numpy())
    # the script's save loop scales its extrinsics in place (T_G_1 is a view)
    scaled = E.copy()
    scaled[:, :3, 3] *= G['s']
    assert np.array_equal(scaled, G['extrinsics'].numpy())


def test_oracle_reproduces_the_calibration_bitwise(gold, layout):
    from dvd_b200 import frames as fr
    G = gold['globals']
    K, E, h_pt = fr.read_cameras(layout, 'dog')
    _, masks = dog_inputs(gold)
    pts, mvs, pred, med, s = oracle_frames.calibrate(E, K, h_pt, masks, [d.numpy() for d in G['full_pred_depths']])
    for f in range(len(masks)):
        assert np.array_equal(pts[f], G['pts_list'][f].numpy())
        assert np.array_equal(mvs[f], G['mvs_depths'][f].numpy())
        assert np.array_equal(pred[f], G['pred_depths'][f].numpy())
        assert med[f] == G['scales'][f]
        assert 0 < pts[f].shape[1] < h_pt.shape[1]
    assert s == G['s']


def test_oracle_reproduces_the_written_arrays_bitwise(gold, layout):
    from dvd_b200 import frames as fr
    G = gold['globals']
    K, E, _ = fr.read_cameras(layout, 'dog')
    imgs, masks = dog_inputs(gold)
    for f, ref in enumerate(gold['outputs']['dog']):
        out = oracle_frames.frame_outputs(imgs[f], masks[f], G['full_pred_depths'][f].numpy(), E[f], K, G['s'])
        assert {k: (tuple(v.shape), str(v.dtype)) for k, v in out.items()} == ref['meta']
        for k in ('img', 'pose_c2w', 'intrinsics', 'depth_pred'):
            assert np.array_equal(out[k], ref[k].numpy()), k
        assert np.array_equal(out['depth_mvs'], ref['depth_pred'].numpy())
        assert np.array_equal(out['motion_seg'], ref['motion_seg'].numpy().astype(np.int64))
        assert float(out['img_orig'].astype(np.float64).sum()) == ref['img_orig_checksum']
        assert 0 < ref['motion_seg'].sum() < ref['motion_seg'].numel()
        # the product's host-side pieces are the same arithmetic
        H, W = imgs[f].shape[:2]
        assert np.array_equal(fr.frame_intrinsics(K, H, W, *fr.working_size(H, W)), ref['intrinsics'].numpy())
        assert np.array_equal(fr.frame_pose(E[f], G['s']), ref['pose_c2w'].numpy())


def test_fixture_weights_checksum(gold):
    from dvd_b200 import synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    net = synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True), gold['weight_seed'], gold['head_bias'])
    cs = float(sum(v.double().abs().sum() for v in net.state_dict().values()))
    assert abs(cs - gold['weight_checksum']) <= 1e-9 * gold['weight_checksum']


def test_working_size_and_gaussian_weights():
    from scipy.ndimage import gaussian_filter1d
    from dvd_b200 import frames as fr, ops
    assert fr.working_size(1080, 1920) == (192, 384)
    assert fr.working_size(480, 854) == (192, 384)
    with pytest.raises(ValueError):
        fr.working_size(360, 384)
    for n_in, n_out in ((1080, 192), (1920, 384), (160, 128), (400, 384)):
        r, w = ops.gaussian_weights(n_in, n_out)
        assert len(w) == 2 * r + 1
        imp = np.zeros(2 * r + 41)
        imp[r + 20] = 1.0
        sigma = max(0.0, (n_in / n_out - 1) / 2)
        if sigma > 1e-15:
            assert np.array_equal(gaussian_filter1d(imp, sigma)[20:20 + 2 * r + 1], w[::-1])


def test_ops_reject_cpu_tensors_and_bad_shapes():
    from dvd_b200 import ops
    with pytest.raises(ValueError):
        ops.resize_bicubic_ac(torch.zeros(1, 3, 8, 8), 4, 4)
    with pytest.raises(ValueError):
        ops.spline_prefilter(torch.zeros(1, 8, 8))
    with pytest.raises(ValueError):
        ops.spline_sample(torch.zeros(1, 8, 8, dtype=torch.float64), torch.zeros(1, 4, 2, dtype=torch.float64))
    with pytest.raises(ValueError):
        ops.calib_ratios(*(torch.zeros(1, 8, 8, dtype=torch.float64),) * 2, torch.zeros(1, 4, 4, dtype=torch.float64),
                         torch.zeros(5, 3, dtype=torch.float64), 1, 1, 0, 0)
    with pytest.raises(ValueError):
        ops.row_medians(torch.zeros(2, 5, dtype=torch.float64))
    with pytest.raises(ValueError):
        ops.aa_resize(torch.zeros(1, 8, 8, 3), 4, 4)
