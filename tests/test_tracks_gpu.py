"""GPU: the scene-flow kernels (csrc/tracks.cu) and `dvd_b200.tracks`: scene-flow consistency against dvd_pair_consistency and
oracle/tracks.py bit for bit, the drawing against the oracle bit for bit and for every chunking, the semantics on a scene with a
square moving at a known velocity and a field that outputs it, agreement with the export's sf_1_2 and the fp64 MLP oracle, and
bitwise-reproducible command output."""
import os
import subprocess
import sys
import types
from argparse import Namespace

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import tracks as otr
from test_evaluate_gpu import EXPORTED, N_FILES, make_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ---- consistency with the scene flow ------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def seeded(tmp_path_factory):
    return make_scene(str(tmp_path_factory.mktemp('tracks_eval')))


def _pairs_of(scene, gaps):
    from dvd_b200.evaluate import select_pairs
    from dvd_b200.export_io import Frames, list_files
    from dvd_b200.points import camera_block
    sp = select_pairs(N_FILES, gaps, EXPORTED)
    slot = {f: i for i, f in enumerate(EXPORTED)}
    pairs = [p for g in gaps for p in sp[g]]
    fl = np.stack([np.load(os.path.join(scene['flows'], 'flowpair_%05d_%05d.npz' % p))['flow_1_2'] for p in pairs])
    mk = np.stack([np.load(os.path.join(scene['flows'], 'flowpair_%05d_%05d.npz' % p))['mask_2'] for p in pairs])
    fr = Frames(list_files(scene['export']))
    return (np.asarray([slot[a] for a, _ in pairs], np.int32), np.asarray([slot[b] for _, b in pairs], np.int32), fl, mk,
            camera_block(fr.K, fr.c2w))


def test_zero_scene_flow_equals_pair_consistency_bitwise(seeded):
    from dvd_b200 import ops
    ia, ib, fl, mk, cam = _pairs_of(seeded, [1, 2, 3])
    d, dn, seg = (_cuda(seeded[k]) for k in ('refined', 'initial', 'seg'))
    args = (_cuda(cam), _cuda(ia), _cuda(ib), _cuda(fl), _cuda(mk))
    ref = ops.pair_consistency(d, dn, *args, seg).cpu().numpy()
    got = ops.pair_consistency_sf(d, *args, torch.zeros(len(ia), 3, *d.shape[1:], device='cuda'), seg).cpu().numpy()
    assert np.array_equal(got[:, :2].view(np.uint64), ref[:, 0].view(np.uint64))
    assert got[:, 2, 0].sum() > 0 and np.array_equal(got[:, 1] + got[:, 2], got[:, 1] + got[:, 2])
    got_none = ops.pair_consistency_sf(d, *args, torch.zeros(len(ia), 3, *d.shape[1:], device='cuda')).cpu().numpy()
    assert np.array_equal(got_none[:, 0].view(np.uint64), got[:, 0].view(np.uint64)) and (got_none[:, 1:] == 0).all()


def test_seeded_scene_flow_equals_the_oracle_bitwise(seeded):
    from dvd_b200 import ops
    ia, ib, fl, mk, cam = _pairs_of(seeded, [1, 2, 3])
    rng = np.random.default_rng(3)
    sf = (0.05 * rng.standard_normal((len(ia), 3) + seeded['refined'].shape[1:])).astype(F32)
    sf[0, :, 5, 5] = np.nan
    got = ops.pair_consistency_sf(_cuda(seeded['refined']), _cuda(cam), _cuda(ia), _cuda(ib), _cuda(fl), _cuda(mk), _cuda(sf),
                                  _cuda(seeded['seg'])).cpu().numpy()
    ref = otr.pair_sums_sf(seeded['refined'], cam, ia, ib, fl, mk, sf, seeded['seg'])
    assert np.array_equal(got.view(np.uint64), ref.view(np.uint64))
    assert got[:, 0, 1].sum() > 0 and got[:, 2, 0].sum() > 0


# ---- drawing ------------------------------------------------------------------------------------------------------------------
def _seeded_tracks(seed, M, L1, F, h, w):
    rng = np.random.default_rng(seed)
    from dvd_b200.render_views import view_cams
    K = np.array([[0.8 * w, 0, w / 2], [0, 0.8 * w, h / 2], [0, 0, 1]], F32)
    c2w = np.tile(np.eye(4)[:3], (F, 1, 1)).astype(F32)
    c2w[:, 0, 3] = 0.05 * np.arange(F)
    cams = view_cams(np.repeat(K[None], F, 0), c2w)
    # positions around the view frustum: some off the image, some behind the camera, some behind the depth map
    X = np.stack([rng.uniform(-1.5, 1.5, (M, L1)), rng.uniform(-1.0, 1.0, (M, L1)), rng.uniform(-0.5, 4.0, (M, L1))], -1)
    X = np.cumsum(0.3 * X, 1).astype(F32) / np.arange(1, L1 + 1, dtype=F32)[None, :, None] * 3
    X[-1, -1] = np.nan
    first = rng.integers(-2, F, M).astype(np.int32)
    length = rng.integers(1, L1 + 1, M).astype(np.int32)
    rgb = rng.integers(0, 256, (M, 3)).astype(np.uint8)
    depth = rng.uniform(1.0, 3.0, (F, h, w)).astype(F32)
    depth[:, :, :5] = np.nan
    img = rng.uniform(-0.1, 1.1, (F, 3, h, w)).astype(F32)
    img[0, 1, 2, 3] = np.nan
    return X, first, length, rgb, cams, depth, img, (np.arange(F) + 1).astype(np.int32)


@pytest.mark.parametrize('M,L1,F,h,w,tail', [(300, 9, 7, 40, 56, 4), (1000, 31, 5, 57, 101, 10), (1, 1, 3, 16, 16, 0),
                                             (0, 4, 2, 16, 16, 3)])
def test_drawing_equals_the_oracle_for_every_chunk(M, L1, F, h, w, tail):
    from dvd_b200 import ops
    X, first, length, rgb, cams, depth, img, number = _seeded_tracks(M + F, max(M, 1), L1, F, h, w)
    X, first, length, rgb = X[:M], first[:M], length[:M], rgb[:M]
    ref = otr.draw(X, first, length, rgb, cams, depth, img, number, tail)
    args = [_cuda(a) for a in (X.reshape(M, L1, 3), first, length, rgb)]
    for chunk in (1, 3, F):
        proj = torch.full((M, L1, 3), float('nan'), device='cuda')
        vis = torch.zeros(M, L1, dtype=torch.uint8, device='cuda')
        outs = []
        for s in range(0, F, chunk):
            e = min(s + chunk, F)
            outs.append(ops.draw_tracks(*args, _cuda(cams[s:e]), _cuda(depth[s:e]), _cuda(img[s:e]), _cuda(number[s:e]), tail,
                                        proj=proj, vis=vis).cpu().numpy())
        assert np.array_equal(np.concatenate(outs), ref[0]), chunk
        assert np.array_equal(proj.cpu().numpy().view(np.uint32), ref[1].view(np.uint32)) and np.array_equal(vis.cpu().numpy(), ref[2])
    if M >= 300:
        drawn = ~np.isnan(ref[1][..., 0])
        assert (ref[2] == 1).any() and ((ref[2] == 0) & drawn).any()       # visible heads and hidden / off-image ones
        assert (ref[0] != ref[0][:1]).any()


# ---- a scene with a known motion -----------------------------------------------------------------------------------------------
N, H, W, FOC = 12, 48, 64, 40.0
V = np.array([0.1, 0.0, 0.0])          # the square's velocity per frame (world units)
SQ = (-0.925, -0.325, 0.6)             # the square at depth 2: x0, y0 (frame 0) and side, edges between pixel centres


def _camera(i):
    c = np.eye(4)
    c[0, 3] = 0.05 * i
    return c


def _depth_seg(i):
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    X, Y = (x - W / 2) * 2.0 / FOC + 0.05 * i, (y - H / 2) * 2.0 / FOC
    on = (X >= SQ[0] + V[0] * i) & (X < SQ[0] + V[0] * i + SQ[2]) & (Y >= SQ[1]) & (Y < SQ[1] + SQ[2])
    return np.where(on, 2.0, 4.0).astype(F32), on.astype(F32)


def make_moving_scene(root, n=N, exported=None):
    """frame files, analytic flowpair files for gaps 1..4, a test export and a checkpoint whose field outputs V per step"""
    from dvd_b200.networks.sceneflow_field import SceneFlowFieldNet
    from oracle import sf_mlp
    exported = list(range(n)) if exported is None else exported
    K = np.array([[FOC, 0, W / 2], [0, FOC, H / 2], [0, 0, 1]])
    fdir, pdir, tdir, cdir = (os.path.join(root, k) for k in ('frames', 'flows', 'export', 'ckpt'))
    for d in (fdir, pdir, tdir, cdir):
        os.makedirs(d)
    ds = [_depth_seg(i) for i in range(n)]
    rng = np.random.default_rng(0)
    for i in range(n):
        img = rng.random((H, W, 3)).astype(F32)
        np.savez(os.path.join(fdir, 'frame_%05d.npz' % i), img=img, img_orig=img, pose_c2w=_camera(i), intrinsics=K,
                 depth_mvs=ds[i][0], depth_pred=ds[i][0], motion_seg=ds[i][1])
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    for g in (1, 2, 3, 4):
        for a in range(n - 1 - g):
            d, on = ds[a][0].astype(np.float64), ds[a][1] != 0
            X = (x - W / 2) * d / FOC + 0.05 * a + np.where(on, V[0] * g, 0.0)
            Y = (y - H / 2) * d / FOC + np.where(on, V[1] * g, 0.0)
            f12 = np.stack([FOC * (X - 0.05 * (a + g)) / d + W / 2 - x, FOC * Y / d + H / 2 - y], -1).astype(F32)
            tx, ty = np.rint(x + f12[..., 0]).astype(int), np.rint(y + f12[..., 1]).astype(int)
            inside = (tx >= 0) & (tx < W) & (ty >= 0) & (ty < H)
            m2 = (~inside).astype(np.uint8)
            m2[inside] |= (ds[a + g][1][ty[inside], tx[inside]] != ds[a][1][inside]).astype(np.uint8)
            np.savez(os.path.join(pdir, 'flowpair_%05d_%05d.npz' % (a, a + g)), flow_1_2=f12, flow_2_1=-f12, mask_1=m2, mask_2=m2)
    for fi, f in enumerate(exported):
        np.savez(os.path.join(tdir, 'batch%04d.npz' % fi), depth=ds[f][0][None, None], depth_nn=ds[f][0][None, None],
                 depth_gt=ds[f][0][None, None], img_1=np.load(os.path.join(fdir, 'frame_%05d.npz' % f))['img'].transpose(2, 0, 1)[None],
                 K=K.T[None].astype(F32), cam_c2w=_camera(f)[None].astype(F32),
                 pair_path=np.asarray([os.path.join(fdir, 'frame_%05d.npz' % f)]))
    layers = sf_mlp.init_layers(seed=5)
    net = SceneFlowFieldNet(net_width=256, n_layers=4, time_dependent=True, N_freq_xyz=16, N_freq_t=16)
    sd = net.state_dict()
    for l, (w_, b_) in enumerate(layers):
        sd['convs.%d.conv.weight' % l] = w_.reshape(sd['convs.%d.conv.weight' % l].shape).clone()
        sd['convs.%d.conv.bias' % l] = b_.clone()
    sd['convs.5.conv.weight'].zero_()
    sd['convs.5.conv.bias'] = torch.tensor(V * 100.0, dtype=torch.float32)
    torch.save({'time_dependent': True, 'n_freq_xyz': 16, 'n_freq_t': 16, 'sf_mag_div': 100.0, 'use_motion_seg': False},
               os.path.join(cdir, 'opt.pt'))
    torch.save({'nets': [{}, sd]}, os.path.join(cdir, 'best.pt'))
    torch.save({'nets': [{}, {k: (v if k != 'convs.5.conv.weight' else v + 1e-3) for k, v in sd.items()}]},
               os.path.join(cdir, 'random.pt'))
    return {'frames': fdir, 'flows': pdir, 'export': tdir, 'ckpt': cdir, 'ds': ds, 'K': K, 'layers': layers}


@pytest.fixture(scope='module')
def moving(tmp_path_factory):
    return make_moving_scene(str(tmp_path_factory.mktemp('tracks_moving')))


def test_scene_flow_compensates_the_moving_square(moving, tmp_path):
    from dvd_b200 import tracks
    res = tracks.trace_export(moving['export'], moving['ckpt'], moving['frames'], moving['flows'], gaps=[1, 2, 4],
                              query_every=3, stride=4, length=6, tail=3, moving_only=True, out=str(tmp_path), chunk=5)
    rec = res['record']
    con = rec['consistency']
    assert rec['moving_region'] and rec['steps_per_gap'] == {'1': 1, '2': 2, '4': 4}
    for g in (1, 2, 4):
        without, with_ = con['static_assumption']['moving']['per_gap'][str(g)], con['scene_flow']['moving']['per_gap'][str(g)]
        assert without['count'] > 50 and with_['count'] == without['count']
        # uncompensated: the square's displacement f |v| g / z = 2 g pixels; compensated: fp32 noise
        assert abs(without['e_r'] - FOC * V[0] * g / 2.0) < 1e-3, (g, without['e_r'])
        assert with_['e_r'] < 1e-3, (g, with_['e_r'])
    assert rec['headline']['moving_e_r_scene_flow'] < 1e-3 < rec['headline']['moving_e_r_static_assumption']
    # tracks seeded on the square stay on it in every exported frame
    tr, proj, vis = res['tracks'], res['proj'], res['visible']
    assert tr['X'].shape[0] > 20
    for i in range(tr['X'].shape[0]):
        for k in range(int(tr['alive'][i])):
            f = int(tr['first'][i]) + k
            u, v = proj[i, k, :2]
            x, y = int(np.floor(u + F32(0.5))), int(np.floor(v + F32(0.5)))
            assert vis[i, k] == 1 and moving['ds'][f][1][y, x] == 1, (i, k)
            np.testing.assert_allclose(tr['X'][i, k] - tr['X'][i, 0], V * k, atol=1e-5)


def test_first_step_is_the_export_sf_and_steps_follow_the_fp64_mlp(moving):
    """The export's sf_1_2 comes from Model._predict_on_batch on the test pass's items; a track's first step from the same
    frame is the same chain evaluation for the same pixel, so X[1] = X[0] + sf_1_2 bit for bit."""
    from dvd_b200 import tracks
    from dvd_b200.datasets.davis_sequence import Dataset
    from dvd_b200.models.scene_flow_motion_field import Model
    from dvd_b200.points import camera_block
    from oracle import sf_mlp
    root = os.path.dirname(moving['frames'])
    os.makedirs(os.path.join(root, 'frames_midas'), exist_ok=True)
    link = os.path.join(root, 'frames_midas', 'track')
    if not os.path.exists(link):
        os.symlink(moving['frames'], link)
    ds = Dataset(Namespace(track_id='track', data_root=root, subsample=False, overfit=False), mode='vali')
    field = tracks.Field(moving['ckpt'], epoch=-1, device=torch.device('cuda'))
    field.net.load_state_dict(torch.load(os.path.join(moving['ckpt'], 'random.pt'))['nets'][1])   # a field that varies
    field.packed = field.net.packed(field.sf_mag_div)
    layers = [(c.conv.weight.detach().reshape(c.conv.weight.shape[0], -1).double().cpu(), c.conv.bias.detach().double().cpu())
              for c in field.net.convs]
    depth = np.stack([d for d, _ in moving['ds']])
    for a in (0, 5):
        b = torch.utils.data.default_collate([ds[a]])
        inp = Namespace(**{k: (v.cuda() if torch.is_tensor(v) else v) for k, v in b.items()})
        stub = types.SimpleNamespace(_input=inp, net_depth=lambda img: _cuda(depth[a][None, None]),
                                     opt=Namespace(midas=True, time_dependent=True, sf_mag_div=100.0), net_sceneflow=field.net)
        sf_export = Model._predict_on_batch(stub, is_train=False)['sf_1_2'][0].reshape(3, -1).cpu().numpy()
        cam = _cuda(camera_block(moving['K'][None].astype(F32), _camera(a)[None].astype(F32)))
        ts = torch.from_numpy(tracks.time_stamps([a], N)).cuda()
        tr = tracks.integrate(field, _cuda(depth[a:a + 1]), cam, ts, tracks.time_step(N), depth[a:a + 1], np.array([a]), 1, 3, 5,
                               last=N - 1)
        X, idx = tr['X'], tr['pixel']
        assert (tr['alive'] == 6).all()
        assert np.array_equal((X[:, 0] + sf_export[:, idx].T).view(np.uint32), X[:, 1].view(np.uint32)), a
        for n in (1, 3, 5):
            ref = sf_mlp.sf_multi_step(torch.from_numpy(X[:, 0].T.reshape(1, 3, 1, -1)).double(),
                                       torch.full((1, 1, 1, X.shape[0]), float(ts[0]), dtype=torch.float64), tracks.time_step(N), n,
                                       layers)
            mine = torch.from_numpy(X[:, n] - X[:, 0]).T.reshape(1, 3, 1, -1)
            assert rel_err(mine, ref) < 1e-4, (a, n, rel_err(mine, ref))


def _files(d):
    return {k: open(os.path.join(d, k), 'rb').read() for k in ('tracks.json', 'pairs.csv', 'tracks.npz')}


def test_command_writes_every_file_bitwise_reproducibly(moving, tmp_path):
    from dvd_b200 import tracks
    outs = []
    for i, chunk in enumerate((16, 16, 1, 3)):
        res = tracks.trace_export(moving['export'], moving['ckpt'], moving['frames'], moving['flows'], gaps=[1, 2],
                                  query_every=4, stride=6, length=5, tail=2, out=str(tmp_path / str(i)), chunk=chunk)
        outs.append(_files(str(tmp_path / str(i))))
    assert all(o == outs[0] for o in outs[1:])
    names = set(os.listdir(str(tmp_path / '0')))
    assert {'tracks.json', 'pairs.csv', 'tracks.npz', 'tracks.mp4'} <= names
    assert sorted(n for n in names if n.startswith('tracks_')) == ['tracks_%05d.png' % f for f in range(N)]
    z = np.load(str(tmp_path / '0' / 'tracks.npz'))
    M = z['positions'].shape[0]
    assert z['positions'].shape == (M, 6, 3) and z['proj'].shape == (M, 6, 3) and z['visible'].shape == (M, 6)
    assert z['query_pixel'].shape == (M, 2) and set(z['query_frame'].tolist()) == {0, 4, 8}
    assert (z['alive'][z['query_frame'] == 8] == 4).all()
    r = subprocess.run([sys.executable, '-m', 'dvd_b200.tracks', '--test_dir', moving['export'], '--checkpoint_path', moving['ckpt'],
                        '--frames', moving['frames'], '--flows', moving['flows'], '--gaps', '1,2', '--query_every', '4',
                        '--stride', '6', '--length', '5', '--tail', '2', '--out', str(tmp_path / 'cli')], cwd=ROOT,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert 'scene flow' in r.stdout and _files(str(tmp_path / 'cli')) == outs[0]
