"""CPU: the numpy restatement of the scene-flow kernels (oracle/tracks.py) and the host rules of dvd_b200.tracks: consistency
with a zero scene flow equals oracle/evaluate.py's refined consistency, the drawing rule's invariants (order independence,
occlusion, tail), time stamps and Euler steps, argument errors and the output layout."""
import os

import numpy as np
import pytest
import torch

from oracle import evaluate as oev
from oracle import tracks as otr

F32 = np.float32


def _scene(seed=0, n=4, h=24, w=32):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    depth = (2.0 + x / w + 0.2 * rng.standard_normal((n, h, w))).astype(F32)
    depth[:, 3, 4], depth[:, 7, 9] = np.nan, 0.0
    K = np.array([[30.0, 0, w / 2], [0, 30.0, h / 2], [0, 0, 1]])
    c2w = np.tile(np.eye(4)[:3], (n, 1, 1))
    c2w[:, 0, 3] = 0.05 * np.arange(n)
    from dvd_b200.points import camera_block
    cam = camera_block(np.repeat(K[None], n, 0), c2w)
    flow = np.stack([np.stack([-1.5 + 0.3 * rng.standard_normal((h, w)), 0.3 * rng.standard_normal((h, w))], -1)
                     for _ in range(3)]).astype(F32)
    mask = (rng.random((3, h, w)) < 0.1).astype(np.uint8)
    seg = np.zeros((n, h, w), np.uint8)
    seg[:, 8:16, 10:20] = 1
    return depth, cam, flow, mask, seg, K, c2w


def test_zero_scene_flow_is_evaluate_refined_consistency():
    depth, cam, flow, mask, seg, _, _ = _scene()
    ia, ib = [0, 1, 0], [1, 2, 3]
    for p in range(3):
        a, b = oev.pair_terms(depth[ia[p]], depth[ib[p]], cam[ia[p]], cam[ib[p]], flow[p], mask[p]), \
            otr.pair_terms_sf(depth[ia[p]], depth[ib[p]], cam[ia[p]], cam[ib[p]], flow[p], mask[p], np.zeros((3,) + depth.shape[1:], F32))
        for k in ('eval', 'behind', 'good'):
            assert np.array_equal(a[k], b[k])
        for k in ('e_r', 'e_d', 'z'):
            assert np.array_equal(a[k].view(np.uint64), b[k].view(np.uint64)), k
    got = otr.pair_sums_sf(depth, cam, ia, ib, flow, mask, np.zeros((3, 3) + depth.shape[1:], F32), seg)
    ref = oev.pair_sums(depth, depth, cam, ia, ib, flow, mask, seg)[:, 0]
    np.testing.assert_allclose(got[:, :2], ref, rtol=1e-12)       # the oracles add in different orders
    assert np.array_equal(got[:, 1] + got[:, 2], got[:, 1] + got[:, 2])
    np.testing.assert_allclose(got[:, 1] + got[:, 2], got[:, 0], rtol=1e-12)   # static and moving partition all
    assert got[:, 2, 0].sum() > 0


def test_fixed_sum_follows_the_kernel_order():
    rng = np.random.default_rng(1)
    for hw in (1, 255, 2049, 40 * 56, 224 * 384):
        v = rng.standard_normal(hw) * 10.0 ** rng.integers(-8, 8, hw)
        s = otr.fixed_sum(v)
        assert abs(s - np.sum(v)) <= 1e-12 * np.abs(v).sum()
        P = otr.parts_for(hw)
        T = P * 256
        acc = [0.0] * T
        for i in range(hw):                                     # one thread's pixels, then the tree, in plain python
            acc[i % T] += float(v[i])
        if hw <= 2049:
            blocks = []
            for b in range(P):
                warps = []
                for w in range(8):
                    lanes = acc[b * 256 + w * 32:b * 256 + w * 32 + 32]
                    for o in (16, 8, 4, 2, 1):
                        lanes = [lanes[l] + lanes[l + o] for l in range(o)]
                    warps.append(lanes[0])
                t = 0.0
                for x in warps:
                    t += x
                blocks.append(t)
            t = 0.0
            for x in blocks:
                t += x
            assert t == s


def _tracks(seed=0, M=40, L1=7, F=5, h=24, w=32):
    rng = np.random.default_rng(seed)
    K = np.array([[30.0, 0, w / 2], [0, 30.0, h / 2], [0, 0, 1]], F32)
    c2w = np.tile(np.eye(4)[:3], (F, 1, 1)).astype(F32)
    c2w[:, 0, 3] = 0.05 * np.arange(F)
    from dvd_b200.render_views import view_cams
    cams = view_cams(np.repeat(K[None], F, 0), c2w)
    X = np.stack([rng.uniform(-1.2, 1.2, (M, L1)), rng.uniform(-0.9, 0.9, (M, L1)), rng.uniform(-0.5, 4.0, (M, L1))], -1).astype(F32)
    X[0, -1] = np.nan
    first = rng.integers(0, F, M).astype(np.int32)
    length = rng.integers(1, L1 + 1, M).astype(np.int32)
    rgb = rng.integers(0, 256, (M, 3)).astype(np.uint8)
    depth = rng.uniform(1.0, 3.0, (F, h, w)).astype(F32)
    depth[:, 0, :] = np.nan
    img = rng.uniform(-0.1, 1.1, (F, 3, h, w)).astype(F32)
    img[0, 0, 0, 0] = np.nan
    return X, first, length, rgb, cams, depth, img, np.arange(F, dtype=np.int32)


def test_drawing_is_order_independent():
    args = _tracks()
    ref = otr.draw(*args, tail=3)
    for seed in (1, 2):
        got = otr.draw(*args, tail=3, rng=np.random.default_rng(seed))
        for a, b in zip(ref, got):
            assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    assert (ref[2] == 1).any() and ((ref[2] == 0) & ~np.isnan(ref[1][..., 0])).any()   # visible and hidden or off-image heads


def test_a_track_behind_the_depth_is_hidden_and_in_front_it_shows():
    X, first, length, rgb, cams, depth, img, number = _tracks(M=1, L1=1, F=1)
    depth[:] = 2.0
    X[0, 0] = (0.0, 0.0, 1.0)
    out, proj, vis = otr.draw(X, first * 0, length * 0 + 1, rgb, cams, depth, img, number, tail=0)
    assert vis[0, 0] == 1 and np.array_equal(out[0, 12, 16], rgb[0, ::-1])
    X[0, 0] = (0.0, 0.0, 2.0 * 1.06)
    out2, proj2, vis2 = otr.draw(X, first * 0, length * 0 + 1, rgb, cams, depth, img, number, tail=0)
    assert vis2[0, 0] == 0 and not np.isnan(proj2[0, 0, 0])
    base = (np.minimum(np.fmax(img[0], 0), 1) * F32(255)).astype(np.uint8)
    assert np.array_equal(out2[0], base.transpose(1, 2, 0)[..., ::-1])             # the frame itself
    X[0, 0] = (0.0, 0.0, -1.0)                                                      # behind the camera: dropped
    _, proj3, vis3 = otr.draw(X, first * 0, length * 0 + 1, rgb, cams, depth, img, number, tail=0)
    assert vis3[0, 0] == 0 and np.isnan(proj3[0, 0]).all()


def test_tail_limits_the_segments_and_fades_them():
    X, first, length, rgb, cams, depth, img, number = _tracks(M=1, L1=6, F=6)
    depth[:] = np.nan
    X[0] = np.stack([np.linspace(-0.8, 0.8, 6), np.zeros(6), np.full(6, 2.0)], 1)
    first[:], length[:] = 0, 6
    img[:] = 0.0
    rgb[:] = 255
    outs = {}
    for tail in (0, 2, 5):
        outs[tail] = otr.draw(X, first, length, rgb, cams, depth, img, number, tail=tail)[0]
    lit = {t: int((outs[t][5].max(-1) > 0).sum()) for t in outs}
    assert lit[0] == 9 and lit[0] < lit[2] < lit[5]                                   # the 3x3 head, then longer tails
    row = outs[5][5, 12]
    # rank 1 next to the head is brighter than rank 5 at the far end
    xs = np.nonzero(row.max(-1))[0]
    assert row[xs[-1] - 2].max() > row[xs[0]].max() > 0


def test_time_stamps_and_euler_steps():
    from dvd_b200 import tracks
    assert tracks.time_stamps([0, 5, 199], 200).dtype == np.float32
    assert tracks.time_stamps([5], 200)[0] == np.float32(5 / 200)
    assert tracks.time_step(200) == 1 / 200
    for n in (7, 80, 200, 1000):
        for a, g in ((0, 1), (3, 2), (n - 9, 8)):
            assert tracks.euler_steps(a, a + g, n) == g
    assert tracks.euler_steps(10, 12, 200, unit=2.0) == 1 and tracks.euler_steps(10, 11, 200, unit=2.0) in (0, 1)


def test_subsample_checkpoints_are_refused(tmp_path):
    from dvd_b200 import tracks
    torch.save({'subsample': True, 'time_dependent': True, 'n_freq_xyz': 16, 'n_freq_t': 16, 'sf_mag_div': 100.0},
               str(tmp_path / 'opt.pt'))
    with pytest.raises(ValueError, match='subsample'):
        tracks.training_options(str(tmp_path))
    with pytest.raises(ValueError, match='subsample'):
        tracks.trace_export(str(tmp_path), str(tmp_path), str(tmp_path), flows_dir=str(tmp_path))
    torch.save({'subsample': False, 'time_dependent': False, 'n_freq_xyz': 16, 'n_freq_t': 16, 'sf_mag_div': 100.0},
               str(tmp_path / 'opt.pt'))
    assert tracks.training_options(str(tmp_path)).sf_mag_div == 100.0


@pytest.mark.parametrize('kw, match', [(dict(query_every=0), 'query_every'), (dict(stride=0), 'stride'),
                                       (dict(length=65), 'length'), (dict(length=0), 'length'), (dict(tail=65), 'tail'),
                                       (dict(tail=-1), 'tail'), (dict(gaps=[1, 1]), 'gaps'), (dict(chunk=0), 'chunk'),
                                       (dict(flows_dir=None), 'exactly one')])
def test_argument_errors(tmp_path, kw, match):
    from dvd_b200 import tracks
    args = dict(flows_dir=str(tmp_path))
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        tracks.trace_export(str(tmp_path), str(tmp_path), str(tmp_path), **args)


def test_command_line_errors():
    from dvd_b200 import tracks
    base = ['--test_dir', 'x', '--checkpoint_path', 'y', '--frames', 'z', '--flows', 'f']
    assert tracks.parse_args(base).length == 30
    for extra in (['--length', '65'], ['--stride', '0'], ['--gaps', '0'], ['--tail', '100']):
        with pytest.raises(SystemExit):
            tracks.parse_args(base + extra)
    with pytest.raises(SystemExit):
        tracks.parse_args(base[:6])                                                    # neither --flows nor --raft_ckpt


def test_query_pixels_colours_and_output_layout(tmp_path):
    from dvd_b200 import tracks
    d = np.full((20, 30), 2.0, F32)
    d[2, 2] = np.nan
    seg = np.zeros((20, 30), np.uint8)
    seg[10:, :] = 1
    idx = tracks.query_pixels(d, 20, 30, 4)
    assert 2 * 30 + 2 not in idx and (idx % 30 % 4 == 2).all() and (idx // 30 % 4 == 2).all()
    assert (tracks.query_pixels(d, 20, 30, 4, seg) // 30 >= 10).all()
    c = tracks.track_colours(np.array([29, 0, 15]), np.array([10, 10, 0]), 20, 30)
    assert c.dtype == np.uint8 and c.shape == (3, 3) and c[0, 0] == 255 and c[1, 1] == 255 and c[1, 0] < 128
    sums = np.zeros((2, 2, 3, 6))
    sums[:, :, :, 0], sums[:, :, :, 2] = 10, 5
    rows = tracks.pair_table([(0, 1), (1, 3)], [1, 2], sums, True)
    assert list(rows[0])[:4] == ['frame_a', 'frame_b', 'gap', 'steps']
    assert 'scene_flow_moving_e_r' in rows[0] and 'static_assumption_static_count' in rows[1] and rows[1]['steps'] == 2
    tracks.write_npz(str(tmp_path / 'a.npz'), x=np.arange(3), y=np.ones((2, 2), bool))
    tracks.write_npz(str(tmp_path / 'b.npz'), x=np.arange(3), y=np.ones((2, 2), bool))
    assert open(str(tmp_path / 'a.npz'), 'rb').read() == open(str(tmp_path / 'b.npz'), 'rb').read()
    assert np.load(str(tmp_path / 'a.npz'))['y'].all()
