"""CPU: the ShutterStock frame stage's restatement (oracle/shutterstock_frames.py) and host pieces (dvd_b200.frames) against
the fixture written by the unmodified shutterstock/generate_frame_midas.py (tests/golden/shutterstock_frames_golden.pt,
oracle/gen_golden_shutterstock.py), the track reader on fake handles, PairBuilder on frame files whose motion_seg is None,
and the argument checks of the new ops."""
import os

import numpy as np
import pytest
import torch

from oracle import golden_io
from oracle import shutterstock_frames as ssf

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
NAMES = [t[0] for t in ssf.TRACKS]


@pytest.fixture(scope='module')
def gold():
    return golden_io.load_golden(GOLDEN, 'shutterstock_frames_golden')


def test_synthetic_inputs_are_the_fixtures(gold):
    for t, name in enumerate(NAMES):
        rec = gold['tracks'][name]
        assert rec['skipped'] == (name == 'c_short_k')
        if rec['skipped']:
            continue
        assert rec['order'] == ssf.kept_frames(t)
        for i, f in enumerate(rec['order']):
            img = ssf.synthetic_frame(t, f)['prediction/img']
            assert float(img.astype(np.float64).sum()) == rec['frames'][i]['checksums']['img_orig'], (name, i)


def test_oracle_reproduces_the_scale_and_the_written_arrays_bitwise(gold):
    from dvd_b200 import frames as fr
    for t, name in enumerate(NAMES):
        rec = gold['tracks'][name]
        if rec['skipped']:
            continue
        scales, s = rec['scales'].numpy(), rec['s'].numpy()[()]
        mdt = ssf.TRACKS[t][4]
        assert scales.dtype == mdt and s.dtype == mdt
        assert np.mean(list(scales)) == s and np.mean(list(scales)).dtype == s.dtype
        for i, f in enumerate(rec['order']):
            inp = ssf.synthetic_frame(t, f)
            ref = rec['frames'][i]
            img, mvs, K, T = (inp['prediction/' + k] for k in ('img', 'mvs_depth', 'K', 'T_1_G'))
            H, W = img.shape[:2]
            # the product's host pieces: working size, intrinsics and pose are the script's arithmetic
            raw = fr.get_im_size(H, W)
            assert raw == ssf.get_im_size(img) and [type(x) for x in raw] == [type(x) for x in ssf.get_im_size(img)]
            assert np.array_equal(fr.frame_intrinsics(K, H, W, *raw), ref['intrinsics'].numpy())
            assert np.array_equal(fr.frame_pose(T, s), ref['pose_c2w'].numpy())
            if i not in rec['depths']:
                continue
            nn = rec['depths'][i].numpy()
            sc = ssf.frame_scale(nn, mvs)
            assert sc == scales[i] and sc.dtype == mdt, (name, i)
            out = ssf.frame_outputs(img, nn, mvs, K, T, s)
            assert {k: (tuple(np.asarray(v).shape), str(np.asarray(v).dtype)) for k, v in out.items()} == ref['meta']
            for k in ('depth_pred', 'depth_mvs', 'img'):
                if k in ref:
                    assert np.array_equal(out[k], ref[k].numpy()), (name, i, k)
                assert float(out[k].astype(np.float64).sum()) == ref['checksums'][k], (name, i, k)
            assert np.array_equal(out['intrinsics'], ref['intrinsics'].numpy())
            assert np.array_equal(out['pose_c2w'], ref['pose_c2w'].numpy())


def test_fixture_weights_checksum(gold):
    from dvd_b200 import synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    net = synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True), gold['weight_seed'], gold['head_bias'])
    cs = float(sum(v.double().abs().sum() for v in net.state_dict().values()))
    assert abs(cs - gold['weight_checksum']) <= 1e-9 * gold['weight_checksum']


@pytest.mark.parametrize('H,W', [(1080, 1920), (416, 736), (736, 416), (160, 448), (448, 160), (192, 352), (352, 192), (64, 96),
                                 (96, 96), (384, 384), (480, 480), (1080, 1080), (20, 40), (40, 20), (31, 31), (200, 370)])
def test_get_im_size_is_the_scripts(H, W):
    from dvd_b200 import frames as fr
    mine, ref = fr.get_im_size(H, W), ssf.get_im_size(np.zeros((H, W, 3)))
    assert mine == ref and [type(x) for x in mine] == [type(x) for x in ref]


def test_get_im_size_cases():
    from dvd_b200 import frames as fr
    assert fr.get_im_size(416, 736) == [224, 384]
    assert fr.get_im_size(736, 416) == [384, 224]
    th, tw = fr.get_im_size(192, 352)
    assert (th, tw) == (192, 352) and isinstance(tw, np.floating)
    th, tw = fr.get_im_size(96, 96)                          # square frames take the portrait branch
    assert (th, tw) == (96, 96) and isinstance(th, np.floating) and isinstance(tw, int)
    assert fr.get_im_size(1080, 1080) == [384, 384]
    assert fr.get_im_size(20, 40) == [0, 32]                 # a working size of 0: round(0.5) is 0
    assert fr.get_im_size(31, 31) == [0, 0]


class _Fake(dict):
    attrs = {}

    def __init__(self, path):
        super().__init__()
        self.path = path
        track = os.path.basename(os.path.dirname(path))
        t = NAMES.index(track)
        f = dict(ssf.track_files(t))[os.path.basename(path)]
        self.frame = f
        self.update(ssf.synthetic_frame(t, f) if t != 3 else {'prediction/K': np.eye(3)})
        self.closed = False

    def close(self):
        self.closed = True


def write_empty_layout(root):
    for t, name in enumerate(NAMES):
        d = os.path.join(root, 'triangulation', name)
        os.makedirs(d)
        for fn, _ in ssf.track_files(t):
            open(os.path.join(d, fn), 'wb').close()


def test_read_shutterstock_track_orders_trims_and_skips(tmp_path):
    from dvd_b200 import frames as fr
    root = str(tmp_path)
    write_empty_layout(root)
    assert [os.path.basename(p) for p in fr.shutterstock_tracks(root)] == NAMES
    for t, name in enumerate(NAMES):
        got, handles = fr.read_shutterstock_track(root, t, open_file=_Fake)
        assert got == name
        if name == 'c_short_k':
            assert handles is None
            continue
        assert [h.frame for h in handles] == ssf.kept_frames(t)
        # numeric, not lexicographic, timestamp order (the two differ on the file lists of tracks 0, 1 and 3)
        stamps = [int(os.path.basename(h.path).split('_')[-1].split('.')[0]) for h in handles]
        assert stamps == sorted(stamps)
        if t in (0, 1, 3):
            assert [f for _, f in ssf.track_files(t)] != sorted(f for _, f in ssf.track_files(t))
    _, h0 = fr.read_shutterstock_track(root, 0, open_file=_Fake)
    _, h3 = fr.read_shutterstock_track(root, 3, open_file=_Fake)
    assert len(h0) == 17 - 14 and len(h3) == 134
    with pytest.raises(ValueError):
        fr.read_shutterstock_track(root, 5, open_file=_Fake)


def test_pair_builder_reads_motion_seg_none_as_absent(tmp_path):
    """frame files as the ShutterStock script writes them (motion_seg=None), with finished flow files: no device needed"""
    from dvd_b200.flow_pairs import FLOW_FMT, FRAME_FMT, PairBuilder, read_npz
    frames, flows = tmp_path / 'frames', tmp_path / 'flows'
    frames.mkdir()
    flows.mkdir()
    g = np.random.default_rng(0)
    H, W, n = 32, 48, 4
    for f in range(n):
        K = np.array([[40.0, 0, 23.5], [0, 40.0, 15.5], [0, 0, 1]], np.float32)
        pose = np.eye(4, dtype=np.float32)
        pose[:3, 3] = [0.1 * f, 0, 0]
        np.savez(str(frames / (FRAME_FMT % f)), img=g.random((H, W, 3)).astype(np.float32), pose_c2w=pose,
                 depth_mvs=(1 + g.random((H, W))).astype(np.float32), intrinsics=K,
                 depth_pred=(1 + g.random((H, W))).astype(np.float32), img_orig=g.random((H, W, 3)).astype(np.float32),
                 motion_seg=None)
    for a in range(n):
        for b in range(a + 1, n):
            np.savez(str(flows / (FLOW_FMT % (a, b))), flow_1_2=g.normal(size=(H, W, 2)).astype(np.float32),
                     flow_2_1=g.normal(size=(H, W, 2)).astype(np.float32), mask_1=(g.random((H, W)) < 0.3).astype(np.uint8),
                     mask_2=(g.random((H, W)) < 0.3).astype(np.uint8), frame_id_1=a, frame_id_2=b)
    assert 'motion_seg' not in read_npz(str(frames / (FRAME_FMT % 0)))
    b = PairBuilder(str(frames), str(flows), [1, 2], device='cpu')
    assert b.raw_pairs == 0 and len(b) == 3
    for i in range(len(b)):
        it = b[i]
        assert torch.equal(it['motion_seg_1'], it['mask_2'])
        assert 0 < float(it['mask_2'].sum()) < it['mask_2'].numel()


def test_ops_reject_cpu_tensors_and_bad_arguments():
    from dvd_b200 import ops
    with pytest.raises(ValueError):
        ops.dense_ratios(torch.zeros(1, 8, 8), torch.ones(1, 8, 8))
    with pytest.raises(ValueError):
        ops.row_medians(torch.zeros(2, 5, dtype=torch.float32))
    with pytest.raises(ValueError):
        ops.row_medians(torch.zeros(2, 5, dtype=torch.float16))
