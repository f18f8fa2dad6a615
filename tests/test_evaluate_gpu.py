"""GPU: the export evaluation kernels (csrc/depth_metrics.cu) and `dvd_b200.evaluate` against the numpy restatement
(oracle/evaluate.py) on a seeded scene: exact selection, sums to 1e-9, exact counts, bitwise reproducibility across runs and
chunkings, the command line, and RAFT flows against the flows PairBuilder wrote."""
import filecmp
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import evaluate as oev

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
EXPORTED = [0, 1, 2, 3, 5, 6, 7]          # frame 4 is not in the export
N_FILES, H, W = 8, 40, 56


def _rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def make_scene(root, seed=0, n=N_FILES, h=H, w=W):
    """frame files with motion_seg, finished flowpair files for gaps 1..3, and a test export of the frames EXPORTED: a sloped
    plane with a near square moving across it; refined depth = truth with 1 % noise, initial = 1.1 x truth with 5 % noise,
    depth_gt = truth; planted invalid depths (NaN, -1, 0, +inf), an all-invalid refined and initial frame 2, and frame 6's
    camera moved 2.5 forward so that part of the scene lies behind it"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    truth = np.empty((n, h, w), F32)
    seg = np.zeros((n, h, w), F32)
    for i in range(n):
        dep = 2.0 + 1.5 * x / w + 0.3 * y / h
        x0 = 3 * i
        dep[h // 3:h // 3 + h // 4, x0:x0 + w // 4] = 1.2
        seg[i, h // 3:h // 3 + h // 4, x0:x0 + w // 4] = 1
        truth[i] = dep
    K = np.array([[40.0, 0, w / 2], [0, 40.0, h / 2], [0, 0, 1]])
    poses = np.tile(np.eye(4), (n, 1, 1))
    for i in range(n):
        poses[i, :3, :3] = _rot_y(0.01 * i)
        poses[i, :3, 3] = [0.05 * i, 0.01 * i, 2.5 if i == 6 else 0.0]
    refined = (truth * (1 + 0.01 * rng.standard_normal(truth.shape))).astype(F32)
    initial = (truth * (1.1 + 0.05 * rng.standard_normal(truth.shape))).astype(F32)
    gt = truth.copy()
    for d in (refined, initial, gt):
        d[:, 2, 3], d[:, 5, 7], d[:, 6, 1], d[:, h - 1, w - 1] = np.nan, -1.0, 0.0, np.inf
    refined[2] = np.nan
    initial[2] = -1.0
    gt[:, 0, :5] = 0.0
    fdir, pdir, tdir = (os.path.join(root, k) for k in ('frames', 'flows', 'export'))
    for d in (fdir, pdir, tdir):
        os.makedirs(d)
    for i in range(n):
        img = rng.random((h, w, 3)).astype(F32)
        np.savez(os.path.join(fdir, 'frame_%05d.npz' % i), img=img, img_orig=img, pose_c2w=poses[i], intrinsics=K,
                 depth_mvs=gt[i], depth_pred=initial[i], motion_seg=seg[i])
    for g in (1, 2, 3):
        for a in range(n - 1 - g):
            f12 = np.zeros((h, w, 2), F32)
            f12[..., 0] = -40.0 * 0.05 * g / truth[a] + 0.3 * rng.standard_normal((h, w))
            f12[..., 1] = -0.2 * g + 0.3 * rng.standard_normal((h, w))
            f12[0, 0] = np.nan
            m2 = (rng.random((h, w)) < 0.1).astype(np.uint8)
            np.savez(os.path.join(pdir, 'flowpair_%05d_%05d.npz' % (a, a + g)), flow_1_2=f12, flow_2_1=-f12, mask_1=m2, mask_2=m2,
                     frame_id_1=a, frame_id_2=a + g)
    ids = np.asarray(EXPORTED)
    for fi, s in enumerate(range(0, len(ids), 2)):
        sel = ids[s:s + 2]
        B = len(sel)
        np.savez(os.path.join(tdir, 'batch%04d.npz' % fi), depth=refined[sel, None], depth_nn=initial[sel, None],
                 depth_gt=gt[sel, None], img_1=np.zeros((B, 3, h, w), F32),
                 K=np.broadcast_to(K.T, (B, 1, 1, 3, 3)).astype(F32), cam_c2w=poses[sel].astype(F32),
                 pair_path=np.asarray([os.path.join(fdir, 'frame_%05d.npz' % f) for f in sel]))
    return {'frames': fdir, 'flows': pdir, 'export': tdir, 'refined': refined[ids], 'initial': initial[ids], 'gt': gt[ids],
            'seg': (seg[ids] != 0).astype(np.uint8)}


@pytest.fixture(scope='module')
def scene(tmp_path_factory):
    return make_scene(str(tmp_path_factory.mktemp('evaluate')))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ---- kernels ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N,h,w,levels', [(1, 1, 1, 0), (1, 7, 9, 3), (3, 40, 56, 0), (5, 33, 101, 4), (17, 64, 96, 0),
                                          (2, 224, 384, 6)])
def test_selection_is_exact(N, h, w, levels):
    from dvd_b200 import ops
    rng = np.random.default_rng(N * h + w)
    v = rng.uniform(-0.5, 5, (N, h, w)).astype(F32)
    if levels:
        v = np.round(v * levels) / levels                # many ties
    other = rng.uniform(0, 3, (N, h, w)).astype(F32)
    v.reshape(-1)[rng.choice(v.size, v.size // 7)] = np.nan
    v.reshape(-1)[rng.choice(v.size, v.size // 11)] = np.inf
    other.reshape(-1)[rng.choice(v.size, v.size // 13)] = -np.inf
    if N >= 3:
        v[1] = np.nan                                    # an empty frame
    for o in (None, other):
        med, cnt = ops.masked_select_median(_cuda(v), None if o is None else _cuda(o))
        rm, rc = oev.masked_select_median(v, o)
        assert np.array_equal(cnt.cpu().numpy(), rc)
        assert np.array_equal(med.cpu().numpy().view(np.uint32), rm.view(np.uint32)), (med, rm)


def _near(x, thresholds, tol=1e-9):
    x = np.asarray(x, np.float64)
    return sum(int((np.abs(x - t) <= tol * abs(t)).sum()) for t in thresholds)


def _assert_sums(got, ref, count_slots, near):
    """fp64 sums within 1e-9 relative; count slots exact up to the pixels within 1e-9 of a threshold"""
    sums = np.ones(got.shape[-1], bool)
    sums[list(count_slots)] = False
    np.testing.assert_allclose(got[..., sums], ref[..., sums], rtol=1e-9, atol=1e-300)
    assert (np.abs(got[..., ~sums] - ref[..., ~sums]) <= near).all()


def test_accuracy_sums_match_the_oracle(scene):
    from dvd_b200 import ops
    d, dn, g = scene['refined'], scene['initial'], scene['gt']
    N = d.shape[0]
    rng = np.random.default_rng(5)
    scales = np.ones((N, 2, 3))
    scales[:, :, 1] = rng.uniform(0.8, 1.25, (N, 2))
    scales[:, :, 2] = rng.uniform(0.8, 1.25, 2)
    got = ops.depth_metrics(_cuda(d), _cuda(dn), _cuda(g), _cuda(scales)).cpu().numpy()
    ref = oev.accuracy_sums(d, dn, g, scales)
    near = 0
    for n in range(N):
        for j, dd in enumerate((d, dn)):
            for a in range(3):
                near += _near(oev.accuracy_terms(dd[n], g[n], scales[n, j, a])['ratio'], oev.DELTAS)
    counts = [0] + [1 + 7 * a + k for a in range(3) for k in (4, 5, 6)]
    _assert_sums(got.reshape(N, 2, 22), ref, counts, near)
    assert got[2, 0, 0] == 0 and got[2, 1, 0] == 0 and got[0, 0, 0] > 0      # the all-invalid frame


def _pairs(gaps):
    from dvd_b200.evaluate import select_pairs
    sp = select_pairs(N_FILES, gaps, EXPORTED)
    slot = {f: i for i, f in enumerate(EXPORTED)}
    pairs = [p for g in gaps for p in sp[g]]
    return pairs, [slot[a] for a, _ in pairs], [slot[b] for _, b in pairs]


def _flows(scene, pairs):
    fl, mk = [], []
    for a, b in pairs:
        z = np.load(os.path.join(scene['flows'], 'flowpair_%05d_%05d.npz' % (a, b)))
        fl.append(z['flow_1_2'])
        mk.append(z['mask_2'])
    return np.stack(fl), np.stack(mk)


def test_pair_sums_match_the_oracle(scene):
    from dvd_b200 import evaluate as ev
    from dvd_b200.export_points import Frames, list_files
    from dvd_b200.points import camera_block
    fr = Frames(list_files(scene['export']))
    cam = camera_block(fr.K, fr.c2w)
    pairs, ia, ib = _pairs([1, 2, 3])
    fl, mk = _flows(scene, pairs)
    d, dn, seg = scene['refined'], scene['initial'], scene['seg']
    for chunk in (1, 4, 64):
        got = ev.pair_consistency(_cuda(d), _cuda(dn), _cuda(cam), ia, ib, fl, mk, _cuda(seg), chunk)
        if chunk == 1:
            first = got
        assert np.array_equal(got.view(np.uint64), first.view(np.uint64))
    ref = oev.pair_sums(d, dn, cam, ia, ib, fl, mk, seg)
    near = 0
    for p in range(len(pairs)):
        for D in (d, dn):
            t = oev.pair_terms(D[ia[p]], D[ib[p]], cam[ia[p]], cam[ib[p]], fl[p], mk[p])
            near += _near(t['e_r'][t['good']], (1.0, 3.0)) + _near(t['z'][t['eval']], (1e-3,))
    _assert_sums(got, ref, [0, 1, 4, 5], near)
    assert got[:, :, 0, 1].sum() > 0 and got[:, :, 0, 0].sum() > 0                  # behind pixels and evaluated ones
    assert (got[:, :, 1, 0] < got[:, :, 0, 0]).any() and got[:, :, 1, 0].sum() > 0   # the static region is a proper subset
    two = [i for i, (a, b) in enumerate(pairs) if 2 in (a, b)]
    assert two and (got[two, :, :, 0] == 0).all() and np.isnan(ev.consistency_from_sums(got[two[0], 0, 0])['e_r'])


# ---- the whole export ---------------------------------------------------------------------------------------------------------
def _read(d):
    return {k: open(os.path.join(d, k), 'rb').read() for k in ('metrics.json', 'frames.csv', 'pairs.csv')}


def test_export_is_bitwise_reproducible_and_chunk_independent(scene, tmp_path):
    from dvd_b200 import evaluate as ev
    outs = []
    for i, chunk in enumerate((16, 16, 1, 3)):
        res = ev.evaluate_export(scene['export'], scene['frames'], scene['flows'], gaps=[1, 2, 3], out=str(tmp_path / str(i)),
                                 chunk=chunk)
        outs.append(_read(str(tmp_path / str(i))))
    assert all(o == outs[0] for o in outs[1:])
    rec = res['record']
    assert rec['frames'] == EXPORTED and rec['static_region'] and not rec['depth_gt_is_depth_nn']
    assert rec['n_pairs'] == len(_pairs([1, 2, 3])[0]) == len(res['pairs'])
    # against the oracle: per-frame accuracy counts and pooled sums, pooled pair sums
    acc = rec['accuracy']['refined']
    d, g = scene['refined'], scene['gt']
    mg, cg = oev.masked_select_median(g, d)
    md, _ = oev.masked_select_median(d, g)
    assert acc['count'] == int(cg[-1]) and [r['refined_count'] for r in res['frames']] == cg[:-1].tolist()
    assert acc['median_gt'] == float(mg[-1]) and acc['median'] == float(md[-1])
    assert acc['scale_sequence'] == float(np.float64(mg[-1]) / np.float64(md[-1]))
    s = oev.accuracy_sums(d, d, g, np.ones((len(EXPORTED), 2, 3)))[:, 0].sum(0)
    assert abs(acc['none']['abs_rel'] - s[1] / s[0]) <= 1e-9 * s[1] / s[0]
    assert res['frames'][2]['refined_none_abs_rel'] == 'nan' and res['frames'][2]['refined_count'] == 0
    text = ev.summary(rec)
    assert 'static' in text and 'refined' in text


def test_command_line_writes_what_the_api_writes(scene, tmp_path):
    from dvd_b200 import evaluate as ev
    ev.evaluate_export(scene['export'], scene['frames'], scene['flows'], gaps=[1, 3], out=str(tmp_path / 'api'), chunk=5)
    r = subprocess.run([sys.executable, '-m', 'dvd_b200.evaluate', '--test_dir', scene['export'], '--frames', scene['frames'],
                        '--flows', scene['flows'], '--gaps', '1,3', '--out', str(tmp_path / 'cli')], cwd=ROOT,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert 'refined' in r.stdout and 'initial' in r.stdout and 'reading' in r.stdout
    assert _read(str(tmp_path / 'api')) == _read(str(tmp_path / 'cli'))


def test_raft_checkpoint_equals_the_flows_pair_builder_wrote(scene, tmp_path):
    from dvd_b200 import evaluate as ev
    from dvd_b200.flow_pairs import PairBuilder
    from dvd_b200.raft import RaftNet
    from oracle import raft as oracle_raft
    sd = oracle_raft.seeded_state_dict(0, 0.7)
    ckpt = str(tmp_path / 'raft.pth')
    torch.save(sd, ckpt)
    net = RaftNet()
    net.load_state_dict(sd)
    flows = str(tmp_path / 'raft_flows')
    # two iterations: the seeded network's flows stay small enough for most pixels to pass the forward-backward check
    PairBuilder(scene['frames'], None, [1, 2], raft=net.cuda(), raft_iters=2).write(str(tmp_path / 'seq'), flows_out=flows)
    a = ev.evaluate_export(scene['export'], scene['frames'], raft=ckpt, gaps=[1, 2], out=str(tmp_path / 'a'), raft_iters=2)['record']
    b = ev.evaluate_export(scene['export'], scene['frames'], flows, gaps=[1, 2], out=str(tmp_path / 'b'))['record']
    assert a['flows'] == 'raft' and b['flows'] == os.path.abspath(flows)
    assert a['consistency'] == b['consistency'] and a['accuracy'] == b['accuracy']
    assert filecmp.cmp(str(tmp_path / 'a' / 'pairs.csv'), str(tmp_path / 'b' / 'pairs.csv'), shallow=False)
    assert a['consistency']['refined']['all']['count'] > 0
