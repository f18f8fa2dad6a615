"""CPU: the numpy restatement of the export evaluation (oracle/evaluate.py) on closed-form scenes, the lower median, and the
host side of `dvd_b200.evaluate`: frame numbering, pair restriction, metrics from sums, the file schema and argument errors."""
import csv
import json
import os

import numpy as np
import pytest
import torch

from oracle import evaluate as oev

F32 = np.float32


# ---- closed-form scenes ---------------------------------------------------------------------------------------------------------
def _plane_scene(n, H, W, Z=2.0, f=64.0, bx=0.0625):
    """a fronto-parallel plane at depth Z seen by cameras translated by bx per frame along x: the flow from a to b = a + g is
    exactly -f g bx / Z pixels along x (2 px per frame with the defaults)"""
    from dvd_b200.points import camera_block
    K = np.tile(np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], F32), (n, 1, 1))
    c2w = np.tile(np.eye(4, dtype=F32)[:3], (n, 1, 1))
    c2w[:, 0, 3] = bx * np.arange(n)
    return np.full((n, H, W), Z, F32), camera_block(K, c2w), f * bx / Z


def _plane_flow(H, W, shift, g):
    flow = np.zeros((H, W, 2), F32)
    flow[..., 0] = -shift * g
    x = np.arange(W)[None, :] + flow[..., 0]
    mask = ((x < 0) | (x > W - 1)).astype(np.uint8)
    return flow, mask


def test_plane_with_analytic_flows_is_consistent():
    H, W, n = 32, 64, 4
    depth, cam, shift = _plane_scene(n, H, W)
    pairs = [(0, 1), (1, 3), (0, 2)]
    flows, masks = zip(*[_plane_flow(H, W, shift, b - a) for a, b in pairs])
    for a, b in pairs:
        t = oev.pair_terms(depth[a], depth[b], cam[a], cam[b], flows[pairs.index((a, b))], masks[pairs.index((a, b))])
        assert t['good'].sum() == H * (W - 2 * (b - a)) and not t['behind'].any()
        assert np.nanmax(t['e_r']) <= 1e-12 and np.nanmax(t['e_d']) == 0.0
    s = oev.pair_sums(depth, depth, cam, [a for a, _ in pairs], [b for _, b in pairs], flows, masks)
    assert s[:, :, 0, 2].max() <= 1e-9 and (s[:, :, 0, 3] == 0).all() and (s[:, :, 0, 4] == s[:, :, 0, 0]).all()
    assert (s[:, :, 1] == 0).all()                          # no motion_seg: no static region


@pytest.mark.parametrize('c', [0.5, 0.8, 1.25, 2.0])
def test_scaled_plane_shifts_by_the_analytic_amount(c):
    H, W, n, g = 32, 64, 3, 2
    depth, cam, shift = _plane_scene(n, H, W)
    flow, mask = _plane_flow(H, W, shift, g)
    d = (c * depth).astype(F32)
    cz = np.float64(d[0, 0, 0]) / 2.0                 # c as the fp32 depth holds it
    t = oev.pair_terms(d[0], d[g], cam[0], cam[g], flow, mask)
    want = shift * g * abs(1 - 1 / cz)                # the points at c Z move by f g bx / (c Z), the flow says f g bx / Z
    er = t['e_r'][t['good']]
    assert er.size > 0 and np.abs(er - want).max() <= 1e-9 * max(want, 1)
    assert np.nanmax(t['e_d']) <= 1e-12
    # accuracy of the scaled depth against the plane: AbsRel |c - 1| unaligned, 0 under the frame and sequence scales
    from dvd_b200 import evaluate as ev
    gt = depth
    mg, _ = oev.masked_select_median(gt, d)
    md, _ = oev.masked_select_median(d, gt)
    sc = np.float64(mg) / np.float64(md)
    scales = np.stack([np.stack([np.ones(n), sc[:n], np.full(n, sc[n])], 1)] * 2, 1)
    m = ev.accuracy_from_sums(oev.accuracy_sums(d, d, gt, scales)[:, 0].sum(0))
    assert abs(m['none']['abs_rel'] - abs(cz - 1)) <= 1e-12
    assert m['frame']['abs_rel'] == 0 and m['sequence']['abs_rel'] == 0 and m['frame']['d1'] == 1
    assert m['count'] == n * H * W


def test_behind_pixels_are_counted_apart():
    H, W = 16, 32
    depth, cam, _ = _plane_scene(2, H, W)
    cam[1, 18:27] = np.diag([-1, 1, -1]).astype(F32).reshape(9)     # camera b turned around: every point lies behind it
    flow, mask = np.zeros((H, W, 2), F32), np.zeros((H, W), np.uint8)
    s = oev.pair_sums(depth, depth, cam, [0], [1], [flow], [mask])
    assert s[0, 0, 0, 0] == 0 and s[0, 0, 0, 1] == H * W and s[0, 0, 0, 2] == 0


def test_taps_are_border_clamped_and_must_all_be_valid():
    H, W = 8, 10
    depth, cam, _ = _plane_scene(2, H, W)
    flow = np.zeros((H, W, 2), F32)
    flow[..., 0] = 0.5
    db = depth[1].copy()
    db[3, 5] = np.nan                                   # invalidates the pixels whose taps touch (5, 3)
    t = oev.pair_terms(depth[0], db, cam[0], cam[1], flow, np.zeros((H, W), np.uint8))
    assert not t['eval'][3, 4] and not t['eval'][3, 5] and not t['eval'][2, 4] and t['eval'][3, 6] and t['eval'][1, 4]
    assert t['eval'][:, W - 1].all()                    # q = W - 0.5 clamps to W - 1: both x taps are column W - 1


# ---- the lower median ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [0, 1, 2, 3, 4, 7, 1000, 1001])
def test_lower_median_is_rank_n_minus_1_over_2(n):
    rng = np.random.default_rng(n)
    x = rng.choice(np.asarray([0.5, 1.0, 1.0, 2.0, 3.5], F32), n) if n < 1000 else rng.uniform(0.1, 9, n).astype(F32)
    got = oev.lower_median(x)
    if n == 0:
        assert np.isnan(got)
    else:
        assert got == np.sort(x)[(n - 1) // 2] == np.partition(x, (n - 1) // 2)[(n - 1) // 2]


def test_masked_select_excludes_invalid_values():
    v = np.asarray([[[np.nan, np.inf, -np.inf, 1e-2, 0.5, 3.0, 2.0, 2.0]], [[np.nan] * 8], [[5.0, 0.0, -1, 7, np.nan, 1, 1, 1]]],
                   F32)
    other = np.ones_like(v)
    other[0, 0, 5] = np.nan                              # masks the 3.0 of frame 0
    med, cnt = oev.masked_select_median(v, other)
    assert cnt.tolist() == [3, 0, 5, 8]
    assert med[0] == F32(2.0) and np.isnan(med[1]) and med[2] == F32(1.0) and med[3] == F32(1.0)
    med, cnt = oev.masked_select_median(v)
    assert cnt.tolist() == [4, 0, 5, 9] and med[0] == F32(2.0) and med[3] == F32(2.0)
    assert F32(1e-2) == v[0, 0, 3] and not oev.valid(v[0, 0, 3])


# ---- host side of dvd_b200.evaluate -------------------------------------------------------------------------------------------
def test_frame_numbers_come_from_pair_path():
    from dvd_b200.evaluate import frame_number
    assert frame_number('/data/frames_midas/dog/frame_00017.npz', 3) == 17
    assert frame_number('frame_123456.npz', 0) == 123456
    assert frame_number('synthetic_frame_004', 9) == 9 and frame_number('frame_00017.png', 2) == 2


def test_pairs_follow_pair_list_restricted_to_exported_frames():
    from dvd_b200.evaluate import select_pairs
    from dvd_b200.flow_pairs import pair_list
    got = select_pairs(10, [1, 2], range(10))
    assert got[1] + got[2] == pair_list(10, [1, 2])
    got = select_pairs(10, [1, 4], [0, 1, 2, 4, 5, 6])
    assert got[1] == [(0, 1), (1, 2), (4, 5), (5, 6)] and got[4] == [(0, 4), (1, 5), (2, 6)]
    assert select_pairs(10, [8], range(10))[8] == [(0, 8)]     # pair_list(10, [8]) is (0, 8) alone
    with pytest.raises(ValueError, match='gap 8'):
        select_pairs(10, [1, 8], range(8))
    with pytest.raises(ValueError, match='gap 3'):
        select_pairs(10, [3], [0, 1, 2])


def test_metrics_from_sums_match_the_definitions():
    from dvd_b200.evaluate import accuracy_from_sums, consistency_from_sums
    rng = np.random.default_rng(0)
    d, g = rng.uniform(0.5, 4, (2, 6, 7)).astype(F32), rng.uniform(0.5, 4, (2, 6, 7)).astype(F32)
    g[1] = np.nan                                        # an empty frame: count 0, NaN metrics, nothing added to the pool
    scales = np.ones((2, 2, 3))
    scales[:, :, 1] = 1.3
    s = oev.accuracy_sums(d, d, g, scales)
    m = accuracy_from_sums(s[0, 0])
    dp, gg = 1.3 * d[0].astype(np.float64), g[0].astype(np.float64)
    assert m['count'] == 42 and abs(m['frame']['rmse'] - np.sqrt(((dp - gg) ** 2).mean())) <= 1e-12
    assert abs(m['frame']['rmse_log'] - np.sqrt(((np.log(dp) - np.log(gg)) ** 2).mean())) <= 1e-12
    assert m['frame']['d1'] == (np.maximum(dp / gg, gg / dp) < 1.25).mean()
    e = accuracy_from_sums(s[1, 0])
    assert e['count'] == 0 and all(np.isnan(e[a][k]) for a in ('none', 'frame', 'sequence') for k in e[a])
    pooled = accuracy_from_sums(s[:, 0].sum(0))
    assert pooled['none']['abs_rel'] == m['none']['abs_rel']
    c = consistency_from_sums(np.asarray([[4, 1, 2.0, 0.4, 3, 4], [0, 2, 0, 0, 0, 0]]))
    assert c['e_r'][0] == 0.5 and c['e_r_lt1'][0] == 0.75 and np.isnan(c['e_d'][1]) and c['behind'][1] == 2


def write_export(d, depth, depth_nn, depth_gt, cam_K, c2w, pair_paths, per_file=2):
    """batch%04d.npz files as the test driver writes them (K and cam_c2w in its storage: K^T)"""
    os.makedirs(d, exist_ok=True)
    N, H, W = depth.shape
    for fi, s in enumerate(range(0, N, per_file)):
        e = min(s + per_file, N)
        np.savez(os.path.join(d, 'batch%04d.npz' % fi), depth=depth[s:e, None], depth_nn=depth_nn[s:e, None],
                 depth_gt=depth_gt[s:e, None], img_1=np.zeros((e - s, 3, H, W), F32), K=cam_K[s:e].transpose(0, 2, 1)[:, None, None],
                 cam_c2w=c2w[s:e], pair_path=np.asarray(pair_paths[s:e]))


def write_frames(d, n, H, W, motion_seg=False):
    os.makedirs(d, exist_ok=True)
    K = np.array([[50.0, 0, W / 2], [0, 50.0, H / 2], [0, 0, 1]])
    for f in range(n):
        extra = {'motion_seg': np.zeros((H, W), np.float32)} if motion_seg else {}
        np.savez(os.path.join(d, 'frame_%05d.npz' % f), img=np.zeros((H, W, 3), F32), pose_c2w=np.eye(4), intrinsics=K,
                 depth_mvs=np.ones((H, W), F32), depth_pred=np.ones((H, W), F32), **extra)


def test_export_reader_numbers_and_checks(tmp_path):
    from dvd_b200.evaluate import Export
    N, H, W = 5, 6, 8
    rng = np.random.default_rng(1)
    dep = rng.uniform(1, 3, (N, H, W)).astype(F32)
    K = np.tile(np.array([[50.0, 0, 4], [0, 50.0, 3], [0, 0, 1]], F32), (N, 1, 1))
    c2w = np.tile(np.eye(4, dtype=F32), (N, 1, 1))
    paths = ['/x/frames_midas/t/frame_%05d.npz' % (2 * i + 1) for i in range(N)]
    write_export(str(tmp_path / 'a'), dep, dep, dep, K, c2w, paths)
    ex = Export(str(tmp_path / 'a'))
    assert ex.numbers.tolist() == [1, 3, 5, 7, 9] and ex.gt_is_nn() and ex.cam.shape == (N, 30)
    assert np.array_equal(ex.cam[:, :9].reshape(N, 3, 3), K.transpose(0, 2, 1))
    gt = dep.copy()
    gt[2, 1, 1] = np.nextafter(gt[2, 1, 1], F32(9))
    write_export(str(tmp_path / 'b'), dep, dep, gt, K, c2w, ['img_%d' % i for i in range(N)])
    ex = Export(str(tmp_path / 'b'))
    assert ex.numbers.tolist() == list(range(N)) and not ex.gt_is_nn()
    write_export(str(tmp_path / 'c'), dep, dep, dep, K, c2w, ['frame_00001.npz'] * N)
    with pytest.raises(ValueError, match='distinct'):
        Export(str(tmp_path / 'c'))


def test_evaluate_rejects_bad_arguments_before_the_device(tmp_path):
    from dvd_b200 import evaluate as ev
    N, H, W = 4, 6, 8
    dep = np.full((N, H, W), 2.0, F32)
    K = np.tile(np.array([[50.0, 0, 4], [0, 50.0, 3], [0, 0, 1]], F32), (N, 1, 1))
    c2w = np.tile(np.eye(4, dtype=F32), (N, 1, 1))
    test_dir = str(tmp_path / 'export')
    write_export(test_dir, dep, dep, dep, K, c2w, ['frame_%05d.npz' % i for i in range(N)])
    write_frames(str(tmp_path / 'frames_bad'), N, H + 2, W)
    with pytest.raises(ValueError, match='6x8'):
        ev.evaluate_export(test_dir, str(tmp_path / 'frames_bad'), flows_dir=str(tmp_path))
    write_frames(str(tmp_path / 'frames'), N, H, W)
    with pytest.raises(ValueError, match='gap 4'):
        ev.evaluate_export(test_dir, str(tmp_path / 'frames'), flows_dir=str(tmp_path), gaps=[1, 4])
    for kw in ({'gaps': [0]}, {'gaps': [1, 1]}, {'chunk': 0}, {'flows_dir': None}, {'raft': 'r.pth'}):
        args = dict(flows_dir=str(tmp_path), gaps=[1], chunk=4)
        args.update(kw)
        with pytest.raises(ValueError):
            ev.evaluate_export(test_dir, str(tmp_path / 'frames'), **args)
    with pytest.raises(FileNotFoundError):
        ev.evaluate_export(test_dir, str(tmp_path / 'nowhere'), flows_dir=str(tmp_path))


def test_command_line_errors():
    from dvd_b200.evaluate import parse_args
    base = ['--test_dir', 'T', '--frames', 'F']
    a = parse_args(base + ['--flows', 'D'])
    assert a.gaps == [1, 2, 4, 8] and a.chunk == 16 and a.out is None and a.raft_ckpt is None and a.raft_iters == 20
    assert parse_args(base + ['--raft_ckpt', 'r.pth', '--gaps', '3,1']).gaps == [3, 1]
    for bad in ([], ['--flows', 'D', '--raft_ckpt', 'r'], ['--flows', 'D', '--gaps', '1,x'], ['--flows', 'D', '--gaps', '0'],
                ['--flows', 'D', '--chunk', '0']):
        with pytest.raises(SystemExit):
            parse_args(base + bad)


def test_ops_reject_cpu_and_malformed_tensors():
    from dvd_b200 import ops
    x = torch.ones(2, 4, 5)
    with pytest.raises(ValueError):
        ops.masked_select_median(x)
    with pytest.raises(ValueError):
        ops.depth_metrics(x, x, x, torch.ones(2, 2, 3, dtype=torch.float64))
    with pytest.raises(ValueError):
        ops.pair_consistency(x, x, torch.ones(2, 30), torch.zeros(1, dtype=torch.int32), torch.ones(1, dtype=torch.int32),
                             torch.zeros(1, 4, 5, 2), torch.zeros(1, 4, 5, dtype=torch.uint8))


def test_files_have_the_documented_schema(tmp_path):
    """record / frame_table / pair_table on oracle sums, written and read back"""
    from dvd_b200 import evaluate as ev

    class Ex:
        N, H, W = 3, 4, 5
        numbers = np.asarray([4, 5, 6])
        depth_gt = np.ones((3, 4, 5), F32)
        depth_nn = np.ones((3, 4, 5), F32)

        def gt_is_nn(self):
            return True

    rng = np.random.default_rng(2)
    d = rng.uniform(0.5, 2, (3, 4, 5)).astype(F32)
    d[1] = 0                                           # an empty frame
    g = rng.uniform(0.5, 2, (3, 4, 5)).astype(F32)
    s = oev.accuracy_sums(d, d, g, np.ones((3, 2, 3)))
    acc = {name: {'sums': s[:, j], 'median_gt': np.ones(4, F32), 'median': np.ones(4, F32), 'scale': np.ones(4)}
           for j, name in enumerate(ev.SOURCES)}
    pairs = [(4, 5), (5, 6), (4, 6)]
    ps = rng.uniform(0, 1, (3, 2, 2, 6))
    ps[..., 0] = 10
    for static in (True, False):
        rec = ev.record('T', 'F', 'D', False, [1, 2], Ex(), acc, pairs, ps, static)
        paths = ev.write_outputs(str(tmp_path / str(static)), rec, ev.frame_table(Ex(), acc), ev.pair_table(pairs, ps, static))
        back = json.load(open(paths['metrics.json']))
        assert back['frames'] == [4, 5, 6] and back['n_pairs'] == 3 and back['depth_gt_is_depth_nn'] is True
        for name in ev.SOURCES:
            a = back['accuracy'][name]
            assert set(a) == {'count', 'none', 'frame', 'sequence', 'median_gt', 'median', 'scale_sequence'}
            assert a['count'] == 40 and set(a['none']) == set(ev.ACC_METRICS)
            c = back['consistency'][name]
            assert set(c['all']) == set(ev.PAIR_METRICS) | {'per_gap'} and set(c['all']['per_gap']) == {'1', '2'}
            assert c['all']['count'] == 30 and c['all']['per_gap']['2']['count'] == 10
            assert (c['static'] is None) == (not static)
        rows = list(csv.DictReader(open(paths['frames.csv'])))
        assert [r['frame'] for r in rows] == ['4', '5', '6'] and rows[1]['refined_count'] == '0'
        assert rows[1]['refined_none_abs_rel'] == 'nan' and len(rows[0]) == 1 + 2 * (2 + 3 * 7)
        rows = list(csv.DictReader(open(paths['pairs.csv'])))
        assert [(r['frame_a'], r['frame_b'], r['gap']) for r in rows] == [('4', '5', '1'), ('5', '6', '1'), ('4', '6', '2')]
        assert len(rows[0]) == 3 + 2 * (2 if static else 1) * 6 and rows[0]['initial_all_count'] == '10'
    assert 'refined' in ev.summary(rec) and 'not an independent' in ev.summary(rec)
