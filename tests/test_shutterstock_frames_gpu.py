"""GPU: the ShutterStock calibration kernels (csrc/frame_prep.cu: dvd_dense_ratios, dvd_sorted_median_f32) against numpy, and
dvd_b200.frames.ShutterstockFrameBuilder against the fixture written by the unmodified shutterstock/generate_frame_midas.py
(tests/golden/shutterstock_frames_golden.pt, oracle/gen_golden_shutterstock.py), then the written frames through PairBuilder,
the shutterstock dataset and, when h5py is installed, the prepare_frames CLI on real .h5 files."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import golden_io
from oracle import shutterstock_frames as ssf

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
NAMES = [t[0] for t in ssf.TRACKS]


@pytest.fixture(scope='module')
def gold():
    return golden_io.load_golden(GOLDEN, 'shutterstock_frames_golden')


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from dvd_b200 import ops
    return ops


def edge_maps(N, H, W, dtype, seed):
    g = np.random.default_rng(seed)
    nn = (g.random((N, H, W)) * 8).astype(np.float32)
    mvs = (g.random((N, H, W)) * 4 - 0.5).astype(dtype)
    f = mvs.reshape(-1)
    k = f.size
    f[:k // 10] = np.float32(1e-3)                                       # the fp32 threshold: rejected for fp32 maps
    f[k // 10:k // 5] = 1e-3                                             # the fp64 threshold
    f[k // 5:k // 4] = np.nextafter(np.float32(1e-3), np.float32(1))
    f[k // 4:k // 4 + 7] = [0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 1e-40]
    g.shuffle(f)
    n = nn.reshape(-1)
    n[:11] = [0.0, -0.0, -0.0, 0.0, np.inf, 1e-42, -1e-42, 3.0, -2.0, np.float32(7e37), 1e-38]
    return nn, mvs


def check_ratios(ops, nn, mvs, offset=0):
    """dense_ratios on (optionally 4-byte offset) device copies against numpy's nn[sel] / mvs[sel], bitwise"""
    N, H, W = nn.shape
    def dev(a):
        t = torch.from_numpy(a.reshape(-1)).cuda()
        if offset:
            buf = torch.empty(a.size + offset, dtype=t.dtype, device='cuda')
            buf[offset:] = t
            t = buf[offset:]
        return t.view(N, H, W)
    out = ops.dense_ratios(dev(nn), dev(mvs)).cpu().numpy().reshape(N, H, W)
    assert out.dtype == (np.float32 if mvs.dtype == np.float32 else np.float64)
    sel = mvs > 1e-3
    ref = nn[sel] / mvs[sel]
    assert ref.dtype == out.dtype
    itype = np.int32 if out.dtype == np.float32 else np.int64
    assert np.array_equal(out[sel].view(itype), ref.view(itype))                   # bitwise: signed zeros, inf, subnormals
    rej = out[~sel]
    assert np.isnan(rej).all() and not np.signbit(rej).any()                       # positive NaN: sorted last
    return int(sel.sum())


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_dense_ratios_match_numpy_bitwise(ops, dtype):
    for (N, H, W), seed in (((3, 64, 96), 0), ((2, 37, 53), 1), ((1, 1, 3), 2)):
        if H * W < 20:
            nn = np.array([[[-0.0, 2.0, 5.0]]], np.float32)
            mvs = np.array([[[1.0, np.float32(1e-3), 1e-3]]], dtype)
        else:
            nn, mvs = edge_maps(N, H, W, dtype, seed)
        for offset in (0, 1):                                                      # vector path, then scalar path
            check_ratios(ops, nn, mvs, offset)


def test_fp32_medians_match_numpy_bitwise(ops):
    g = np.random.default_rng(3)
    V = 1001
    counts = [0, 1, 2, 3, 4, 999, 1000, 1001, 64, 65]
    rows = np.full((len(counts), V), np.nan, np.float32)
    for r, c in enumerate(counts):
        v = (g.random(c) * 10 ** g.uniform(-3, 3, c)).astype(np.float32)
        v[: c // 3] = np.round(v[: c // 3], 1)                                  # ties
        rows[r, :c] = v
        g.shuffle(rows[r])                                                      # NaN anywhere: the device sort puts it last
    rows = np.abs(rows)                                                         # positive NaN
    med, cnt = ops.row_medians(torch.from_numpy(rows).cuda())
    med, cnt = med.cpu().numpy(), cnt.cpu().numpy()
    assert med.dtype == np.float32 and cnt.tolist() == counts
    for r, c in enumerate(counts):
        if c == 0:
            assert np.isnan(med[r])
            continue
        ref = np.median(rows[r][~np.isnan(rows[r])])
        assert ref.dtype == np.float32 and med[r].view(np.int32) == ref.view(np.int32), (c, med[r], ref)
    # the even case is the fp32 (a + b) / 2: a sum that is not exact in fp32
    a, b = np.float32(1.0), np.nextafter(np.float32(1.0), np.float32(2))
    m, _ = ops.row_medians(torch.tensor([[a, b, np.float32(16777216.0), np.float32(0.5)]]).cuda())
    assert m.cpu().numpy()[0] == np.median(np.array([a, b, 16777216.0, 0.5], np.float32))


@pytest.mark.parametrize('dtype', [np.float32, np.float64])
def test_scale_matches_numpy_on_the_device_medians(ops, dtype):
    nn, mvs = edge_maps(5, 48, 64, dtype, 7)
    nn = np.abs(nn)
    ratio = ops.dense_ratios(torch.from_numpy(nn).cuda(), torch.from_numpy(mvs).cuda())
    med, cnt = ops.row_medians(ratio)
    med = med.cpu().numpy()
    scales, s = ssf.calibrate(list(nn), list(mvs))
    itype = np.int32 if dtype == np.float32 else np.int64
    assert np.array_equal(med.view(itype), np.asarray(scales).view(itype))
    assert np.mean(med).dtype == s.dtype and np.mean(med) == s
    assert cnt.cpu().numpy().tolist() == [int((m > 1e-3).sum()) for m in mvs]


def seeded_net(gold):
    from dvd_b200 import synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    net = synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True, resize=None), gold['weight_seed'], gold['head_bias'])
    assert abs(float(sum(v.double().abs().sum() for v in net.state_dict().values())) - gold['weight_checksum']) < 1e-6 * gold[
        'weight_checksum']
    return net.cuda().eval()


def handles(t, frames):
    return [ssf.synthetic_frame(t, f) for f in frames]


def rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / np.abs(b).max())


def eager_scale(net, hs):
    """the reference's path on a GPU: eager PyTorch MiDaS with TF32 at the stored size, then the script's calibration"""
    from oracle import depth_nets
    sd = {k: v.cuda() for k, v in net.state_dict().items()}
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
    try:
        with torch.no_grad():
            nn = [depth_nets.midas_forward(sd, torch.from_numpy(h['prediction/img']).permute(2, 0, 1)[None].cuda(), True)[0, 0]
                  .cpu().numpy() for h in hs]
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return ssf.calibrate(nn, [h['prediction/mvs_depth'] for h in hs])[1]


@pytest.mark.parametrize('name', ['a_landscape', 'b_portrait', 'd_small', 'e_square'])
def test_builder_matches_the_fixture(ops, gold, name):
    from dvd_b200 import frames as fr
    t = NAMES.index(name)
    rec = gold['tracks'][name]
    net = seeded_net(gold)
    hs = handles(t, rec['order'])
    b = fr.ShutterstockFrameBuilder(hs, net, chunk=2 if len(hs) < 10 else 16)
    s_ref = rec['s'].numpy()[()]
    assert type(b.scale) is type(s_ref)
    e_eager = abs(float(eager_scale(net, hs)) - float(s_ref)) / float(s_ref)
    e_mine = abs(float(b.scale) - float(s_ref)) / float(s_ref)
    print('%s: s native %.3g, eager TF32 %.3g (relative)' % (name, e_mine, e_eager))
    assert e_mine <= 3 * e_eager + 1e-6
    for i, ref in enumerate(rec['frames']):
        out = b.frame(i)
        assert {k: (tuple(np.asarray(v).shape), str(np.asarray(v).dtype)) for k, v in out.items()} == ref['meta']
        assert out['motion_seg'] is None
        assert np.array_equal(out['intrinsics'], ref['intrinsics'].numpy())
        assert np.array_equal(out['img_orig'], hs[i]['prediction/img'])
        p, pr = out['pose_c2w'], ref['pose_c2w'].numpy()
        # the rotation does not depend on s: fp32 rounding of the inverse; the translation moves with s
        assert np.abs(p[:3, :3] - pr[:3, :3]).max() <= 4 * 2 ** -24 * np.abs(pr[:3, :3]).max()
        assert rel(p[:3, 3], pr[:3, 3]) <= 3 * e_eager + 1e-6
        for k in ('img', 'depth_pred', 'depth_mvs'):
            if k in ref:
                err = rel(out[k], ref[k].numpy())
                assert err <= 1e-3, (i, k, err)
            cs = float(out[k].astype(np.float64).sum())
            assert abs(cs - ref['checksums'][k]) <= 1e-3 * abs(ref['checksums'][k]), (i, k)
    b2 = fr.ShutterstockFrameBuilder(hs, net, chunk=2 if len(hs) < 10 else 16)
    assert b2.scale == b.scale and np.array_equal(b2.medians, b.medians)
    for k in ('img', 'depth_pred', 'depth_mvs'):
        assert np.array_equal(b2.frame(0)[k], b.frame(0)[k])                    # two runs are bitwise equal


def test_builder_rejects_what_the_script_cannot_prepare(ops, gold):
    from dvd_b200 import frames as fr
    net = seeded_net(gold)
    hs = handles(4, [0, 1])
    hs[1] = dict(hs[1], **{'prediction/mvs_depth': np.zeros_like(hs[1]['prediction/mvs_depth'])})
    with pytest.raises(ValueError, match=r'frame\(s\) \[1\]'):
        fr.ShutterstockFrameBuilder(hs, net)
    with pytest.raises(ValueError, match='frame 1'):
        fr.ShutterstockFrameBuilder(handles(4, [0]) + handles(0, [0]), net)          # two stored sizes
    odd = {'prediction/img': np.zeros((70, 96, 3), np.float32), 'prediction/mvs_depth': np.ones((70, 96), np.float32),
           'prediction/K': np.eye(3), 'prediction/T_1_G': np.eye(4)}
    with pytest.raises(ValueError, match='multiple of 32'):
        fr.ShutterstockFrameBuilder([odd], net)
    wide = {'prediction/img': np.zeros((32, 1024, 3), np.float32), 'prediction/mvs_depth': np.ones((32, 1024), np.float32),
            'prediction/K': np.eye(3), 'prediction/T_1_G': np.eye(4)}
    with pytest.raises(ValueError, match='working size'):
        fr.ShutterstockFrameBuilder([wide], net)                                   # get_im_size gives 0 x 384
    with pytest.raises(KeyError, match='prediction/img'):
        fr.ShutterstockFrameBuilder([{k: v for k, v in handles(4, [0])[0].items() if k != 'prediction/img'}], net)


def test_written_frames_go_through_pairs_and_the_shutterstock_dataset(ops, gold, tmp_path):
    from dvd_b200 import frames as fr
    from dvd_b200.datasets import get_dataset
    from dvd_b200.flow_pairs import FLOW_FMT, PairBuilder, pair_list, read_npz
    root = tmp_path / 'shutterstock'
    net = seeded_net(gold)
    b = fr.ShutterstockFrameBuilder(handles(0, gold['tracks']['a_landscape']['order']), net)
    assert b.write(str(root / 'frames_midas' / 'a_landscape')) == 3
    b = fr.ShutterstockFrameBuilder(handles(3, range(6)), net)
    assert b.write(str(root / 'frames_midas' / 'd_small')) == 6
    d = read_npz(str(root / 'frames_midas' / 'a_landscape' / 'frame_00000.npz'))
    assert 'motion_seg' not in d and d['img'].shape == (128, 384, 3)
    # raw flows at a lower resolution: resized and masked on the GPU
    g = np.random.default_rng(0)
    flows = root / 'flow_pairs' / 'd_small'
    flows.mkdir(parents=True)
    for a, c in pair_list(6, [1, 2]):
        np.savez(str(flows / (FLOW_FMT % (a, c))), flow_1_2=g.normal(0, 1, (32, 48, 2)).astype(np.float32),
                 flow_2_1=g.normal(0, 1, (32, 48, 2)).astype(np.float32))
    pb = PairBuilder(str(root / 'frames_midas' / 'd_small'), str(flows), [1, 2])
    assert pb.raw_pairs == len(pb) == 7
    for i in range(len(pb)):
        it = pb[i]
        assert torch.equal(it['motion_seg_1'], it['mask_2'])
        assert 0 < float(it['mask_2'].sum()) < it['mask_2'].numel()
    assert pb.write(str(root / 'sequences_select_pairs_midas' / 'd_small' / '001')) == 7
    opt = types.SimpleNamespace(subsample=False, overfit=False, repeat=1, cache=False, select=False, gaps='1,2',
                                data_root=str(root), track_id=1)
    ds = get_dataset('shutterstock')(opt, mode='train')
    assert len(ds) == 7 and ds.frame_dir.endswith('d_small')
    for i in range(7):
        assert torch.equal(ds[i]['motion_seg_1'], ds[i]['mask_2']) and torch.equal(ds[i]['img_1'], pb[i]['img_1'])
    vali = get_dataset('shutterstock')(opt, mode='vali')
    assert len(vali) == 6 and vali[0]['img'].shape == (3, 64, 96)


class _NpzH5:
    """h5py.File stand-in for the CLI test where h5py is not installed: the '.h5' files hold the frame's arrays as .npz"""

    def __init__(self, path, mode='r'):
        with np.load(path) as z:
            self.items = {k.replace('.', '/'): z[k] for k in z.keys()}
        self.attrs = {}

    def __getitem__(self, key):
        return self.items[key]

    def close(self):
        pass


def test_prepare_frames_pairs_and_train_clis_on_a_shutterstock_layout(ops, gold, tmp_path, monkeypatch):
    import subprocess
    import sys
    from dvd_b200 import prepare_frames, prepare_pairs, synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    from oracle import raft as oracle_raft
    monkeypatch.setitem(sys.modules, 'h5py', types.SimpleNamespace(File=_NpzH5))
    root = tmp_path / 'ss'
    for name, n in (('clip', 20), ('other', 2)):                                   # clip is track 0: frames [14:] kept
        d = root / 'triangulation' / name
        d.mkdir(parents=True)
        for f in range(n):
            arrs = ssf.synthetic_frame(3, f)
            if name == 'other':
                arrs['prediction/K'] = arrs['prediction/K'][:2]                     # skipped
            with open(str(d / ('%s_%d.h5' % (name, 5 + 10 * f))), 'wb') as fh:
                np.savez(fh, **{k.replace('/', '.'): v for k, v in arrs.items()})
    ckpt = str(tmp_path / 'midas_cpkt.pt')
    torch.save(synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True), gold['weight_seed'],
                                   gold['head_bias']).state_dict(), ckpt)
    prepare_frames.main(['--shutterstock_root', str(root), '--midas_ckpt', ckpt, '--out', str(root / 'frames_midas')])
    assert sorted(os.listdir(str(root / 'frames_midas'))) == ['clip']
    assert len(os.listdir(str(root / 'frames_midas' / 'clip'))) == 6
    with np.load(str(root / 'frames_midas' / 'clip' / 'frame_00000.npz'), allow_pickle=True) as z:
        # frame 14 by the numeric order of the timestamps (5, 15, ..., 195: lexicographically 105 would come first)
        assert np.array_equal(z['img_orig'], ssf.synthetic_frame(3, 14)['prediction/img'])
        assert z['motion_seg'].item() is None
    raft_ckpt = str(tmp_path / 'raft.pth')
    torch.save({'module.' + k: v for k, v in oracle_raft.seeded_state_dict(0, 0.7).items()}, raft_ckpt)
    prepare_pairs.main(['--frames', str(root / 'frames_midas' / 'clip'), '--raft_ckpt', raft_ckpt, '--raft_iters', '2',
                        '--out', str(root / 'sequences_select_pairs_midas' / 'clip' / '001'), '--gaps', '1,2'])
    assert len(os.listdir(str(root / 'sequences_select_pairs_midas' / 'clip' / '001'))) == 4 + 3
    args = ('--net scene_flow_motion_field --dataset shutterstock --track_id 0 --gaps 1,2 --epoch 1 --epoch_batches 2 '
            '--lr 1e-6 --batch_size 1 --optim adam --gpu 0 --workers 0 --one_way --loss_type l1 --l1_mul 0 --acc_mul 1 '
            '--disp_mul 1 --warm_sf 1 --scene_lr_mul 1000 --flow_mul 1 --sf_mag_div 100 --time_dependent --midas --use_disp '
            '--vis_batches_train 0 --manual_seed 1').split()
    args += ['--data_root', str(root), '--logdir', str(tmp_path / 'log')]
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=repo + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', 'dvd_b200.train'] + args, cwd=repo, env=env, capture_output=True, text=True,
                       timeout=1100)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith('epoch 1:')]
    assert lines, r.stdout[-2000:]
    log = eval(lines[0].split(':', 1)[1])
    assert all(v == v and abs(v) != float('inf') for v in log.values()), log


def test_prepare_frames_cli_on_h5_files(ops, gold, tmp_path):
    h5py = pytest.importorskip('h5py')
    from dvd_b200 import frames as fr, prepare_frames, synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    root = tmp_path / 'ss'
    for t, name in enumerate(NAMES):                                            # every track: the ids decide the trims
        d = root / 'triangulation' / name
        d.mkdir(parents=True)
        for fn, f in ssf.track_files(t):
            with h5py.File(str(d / fn), 'w') as h:
                for k, v in ssf.synthetic_frame(t, f).items():
                    h[k] = v
    ckpt = str(tmp_path / 'midas_cpkt.pt')
    torch.save(synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True), gold['weight_seed'],
                                   gold['head_bias']).state_dict(), ckpt)
    out = tmp_path / 'frames_midas'
    prepare_frames.main(['--shutterstock_root', str(root), '--midas_ckpt', ckpt, '--out', str(out), '--chunk', '2'])
    assert sorted(os.listdir(str(out))) == ['a_landscape', 'b_portrait', 'd_small', 'e_square']     # c_short_k is skipped
    assert len(os.listdir(str(out / 'd_small'))) == 134
    net = seeded_net(gold)
    for name in ('b_portrait', 'e_square'):
        tid = [os.path.basename(p) for p in fr.shutterstock_tracks(str(root))].index(name)
        _, hs = fr.read_shutterstock_track(str(root), tid)
        try:
            b = fr.ShutterstockFrameBuilder(hs, net, chunk=2)
            for i in range(b.n_frames):
                with np.load(str(out / name / ('frame_%05d.npz' % i)), allow_pickle=True) as z:
                    got = {k: z[k] for k in z.keys()}
                exp = b.frame(i)
                assert got['motion_seg'].item() is None
                for k in ('img', 'depth_pred', 'depth_mvs', 'intrinsics', 'pose_c2w', 'img_orig'):
                    assert np.array_equal(got[k], exp[k]), (name, i, k)
        finally:
            for h in hs:
                h.close()
    # with h5py a missing prediction/img raises KeyError: the reference's image_path fallback is unreachable
    p = tmp_path / 'noimg.h5'
    with h5py.File(str(p), 'w') as h:
        for k, v in ssf.synthetic_frame(4, 0).items():
            if k != 'prediction/img':
                h[k] = v
    with h5py.File(str(p), 'r') as h:
        with pytest.raises(KeyError):
            h['prediction/img']
        with pytest.raises(KeyError, match='prediction/img'):
            fr.ShutterstockFrameBuilder([h], net)
