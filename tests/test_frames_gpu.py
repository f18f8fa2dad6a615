"""GPU: the frame-preparation kernels (csrc/frame_prep.cu) and dvd_b200.frames.FrameBuilder against the library calls of
generate_frame_midas.py (torch's bicubic interpolate, scipy's map_coordinates, the scipy restatement of skimage's resize) and
against the fixture written by the unmodified script (tests/golden/frames_golden.pt, oracle/gen_golden_frames.py)."""
import io
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image
from scipy import ndimage as ndi

from oracle import frames as oracle_frames
from oracle import golden_io

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.fixture(scope='module')
def gold():
    return golden_io.load_golden(GOLDEN, 'frames_golden')


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from dvd_b200 import ops
    return ops


def ulps32(a, b):
    """|a - b| in units of the fp32 spacing at b (elementwise, fp64)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float32)
    return np.abs(a - b.astype(np.float64)) / np.spacing(np.abs(b)).astype(np.float64)


def inputs(gold, track):
    pre = 'JPEGImages/1080p/%s/' % track
    jpgs = sorted(k for k in gold['inputs'] if k.startswith(pre))
    masks = sorted(k for k in gold['inputs'] if k.startswith('Annotations/1080p/%s/' % track))
    dec = lambda k, **kw: Image.open(io.BytesIO(gold['inputs'][k].numpy().tobytes()))     # noqa: E731
    imgs = [np.asarray(dec(k)).astype(np.float32) / 255 for k in jpgs]
    ms = [np.asarray(dec(k).convert('RGB')).astype(np.float32)[:, :, 0] / 255 for k in masks]
    return imgs, ms


def write_layout(gold, root):
    for rel, data in gold['inputs'].items():
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, 'wb') as f:
            f.write(data.numpy().tobytes())


@pytest.mark.parametrize('shape', [((2, 3, 1080, 1920), (256, 512)), ((2, 1, 256, 512), (1080, 1920)), ((2, 3, 37, 53), (64, 96))])
def test_bicubic_matches_torch(ops, shape):
    (N, C, h, w), (H, W) = shape
    x = torch.rand(N, C, h, w, generator=torch.Generator().manual_seed(h)).cuda() * 3 - 1
    ref = F.interpolate(x, size=(H, W), mode='bicubic', align_corners=True)
    out = ops.resize_bicubic_ac(x, H, W)
    err = float((out - ref).abs().max() / ref.abs().max())
    print('bicubic %s: %.3g of max (bound 4 * 2^-24 = %.3g), %.4f differ' % (shape, err, 4 * 2 ** -24,
                                                                            float((out != ref).float().mean())))
    assert err <= 4 * 2 ** -24


def spline_case(H, W, P, seed):
    g = np.random.default_rng(seed)
    m = g.random((2, H, W)).astype(np.float32) * 5
    cols = [g.uniform(0, H - 1, (2, P)), g.uniform(0, W - 1, (2, P))]
    v, u = cols
    v[:, :20], u[:, 20:40] = np.arange(20) % H, np.arange(20) % W                     # integers
    v[:, 40:60], u[:, 60:80] = g.uniform(0, 1, 20), g.uniform(W - 2, W - 1, 20)          # within a pixel of the borders
    v[:, 80], u[:, 81], v[:, 82], u[:, 82] = H - 1, W - 1, H - 1, W - 1
    v[:, 83], u[:, 84], v[:, 85], u[:, 86] = np.nan, np.inf, -np.inf, np.nan
    v[:, 87], u[:, 88], v[:, 89], u[:, 90] = -0.3, W - 0.5, H - 0.2, -1e-9             # just outside
    return m, v, u


def test_spline_sampling_matches_scipy(ops):
    for (H, W, P, seed) in ((37, 53, 4000, 0), (160, 400, 20000, 1)):
        m, v, u = spline_case(H, W, P, seed)
        ref = np.stack([ndi.map_coordinates(m[i], [v[i], u[i]]) for i in range(2)])
        coef = ops.spline_prefilter(torch.from_numpy(m).cuda())
        vu = torch.from_numpy(np.stack([v, u], -1)).cuda().contiguous()
        out = ops.spline_sample(coef, vu).cpu().numpy()
        d = ulps32(out, ref)
        print('spline %dx%d: %.4f of values differ, max %.1f ulp' % (H, W, float((out != ref).mean()), float(d.max())))
        assert d.max() <= 1.0
        assert np.array_equal(out[:, 83:91], ref[:, 83:91])                             # NaN / inf / outside -> 0


def calib_inputs(gold, track='dog'):
    from dvd_b200 import frames as fr
    import tempfile
    with tempfile.TemporaryDirectory() as root:
        write_layout(gold, root)
        K, E, h_pt = fr.read_cameras(root, track)
    _, masks = inputs(gold, track)
    return K, E, h_pt, masks, [d.numpy() for d in gold['globals']['full_pred_depths']]


def device_calibration(ops, K, E, h_pt, masks, depths):
    dc = ops.spline_prefilter(torch.from_numpy(np.stack(depths)).cuda())
    mc = ops.spline_prefilter(torch.from_numpy(np.stack(masks)).cuda())
    ratio = ops.calib_ratios(dc, mc, torch.from_numpy(E[:len(depths)].copy()).cuda(), torch.from_numpy(h_pt[:3].T.copy()).cuda(),
                             K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    med, cnt = ops.row_medians(ratio)
    return ratio.cpu().numpy(), med.cpu().numpy(), cnt.cpu().numpy()


def test_calibration_teacher_forced(ops, gold):
    K, E, h_pt, masks, depths = calib_inputs(gold)
    G = gold['globals']
    ratio, med, cnt = device_calibration(ops, K, E, h_pt, masks, depths)
    H, W = masks[0].shape
    exact = []
    for f in range(len(depths)):
        # the reference's selection, and every point's distance to a bound or threshold
        out = E[f] @ h_pt
        im = K @ out[:3]
        z = im[2].copy()
        u, v = im[0] / im[2], im[1] / im[2]
        inb = (u >= 0) & (u < W) & (v >= 0) & (v < H)
        mval = np.full(u.shape, np.inf)
        mval[inb] = ndi.map_coordinates(masks[f], [v[inb], u[inb]])
        near = np.minimum.reduce([np.abs(u), np.abs(u - W), np.abs(v), np.abs(v - H), np.abs(mval - 0.1), np.abs(z - 1e-3)]) < 1e-9
        mine = ~np.isnan(ratio[f])
        sel = np.zeros_like(mine)
        sel[inb] = (mval[inb] < np.float32(0.1))
        sel &= z > 1e-3
        assert np.array_equal(mine[~near], sel[~near]), f
        assert cnt[f] == G['pts_list'][f].shape[1]
        ref_ratio = G['pred_depths'][f].numpy() / G['mvs_depths'][f].numpy()
        # nn is rounded to fp32 before the division, as scipy returns it: what remains is the fp64 projection's last bits
        exact.append(float(np.max(np.abs(np.sort(ratio[f][mine]) - np.sort(ref_ratio))) / np.max(np.abs(ref_ratio))))
        rel = abs(med[f] - G['scales'][f]) / abs(G['scales'][f])
        print('frame %d: %d points, median rel. err %.3g, ratios max rel. err %.3g' % (f, cnt[f], rel, exact[-1]))
        assert rel <= 2 ** -24 * 1.0 + 1e-15
    s = np.mean(med)
    print('s rel. err %.3g' % (abs(s - G['s']) / abs(G['s'])))
    assert abs(s - G['s']) <= 2 ** -23 * abs(G['s'])
    assert max(exact) <= 1e-13


def test_row_medians_even_odd(ops):
    r = torch.tensor([[3.0, float('nan'), 1.0, 2.0, 10.0], [float('nan')] * 5, [5.0, 1.0, 4.0, float('nan'), float('nan')]],
                     dtype=torch.float64).cuda()
    med, cnt = ops.row_medians(r)
    assert cnt.cpu().tolist() == [4, 0, 3]
    m = med.cpu().numpy()
    assert m[0] == 2.5 and np.isnan(m[1]) and m[2] == 4.0


@pytest.mark.parametrize('case', ['fixture', '1080p', '480p'])
def test_aa_resize_matches_scipy_restatement(ops, gold, case):
    if case == 'fixture':
        imgs, masks = inputs(gold, 'dog')
        img, mask, depth = imgs[0], masks[0], gold['globals']['full_pred_depths'][0].numpy()
    else:
        H, W = (1080, 1920) if case == '1080p' else (480, 854)
        g = np.random.default_rng(H)
        img = g.random((H, W, 3)).astype(np.float32)
        mask = (g.random((H, W)) < 0.02).astype(np.float32)
        depth = (3 + g.random((H, W))).astype(np.float32)
    th, tw = oracle_frames.working_size(*img.shape[:2])
    for name, x in (('img', img), ('depth', depth[..., None]), ('mask', mask[..., None])):
        ref = oracle_frames.sk_resize(x if name == 'img' else x[..., 0], [th, tw])
        out = ops.aa_resize(torch.from_numpy(np.ascontiguousarray(x))[None].cuda(), th, tw)[0].cpu().numpy()
        out = out if name == 'img' else out[..., 0]
        d = ulps32(out, ref)
        print('aa_resize %s %s: max %.1f ulp, %.4f differ' % (case, name, float(d.max()), float((out != ref).mean())))
        assert d.max() <= 1.0
        if name == 'mask':
            band = np.abs(ref - 1e-3) <= 1e-6
            assert np.array_equal((out > 1e-3)[~band], (ref > 1e-3)[~band])


def seeded_net():
    from dvd_b200 import synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    return synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True, resize=[256, 512]), 0, 2000.0)


def test_frame_builder_end_to_end(ops, gold, tmp_path):
    from dvd_b200 import frames as fr
    from dvd_b200.flow_pairs import pose_tensors, read_npz
    from oracle import depth_nets
    root = str(tmp_path / 'davis')
    write_layout(gold, root)
    net = seeded_net()
    assert abs(float(sum(v.double().abs().sum() for v in net.state_dict().values())) - gold['weight_checksum']) < 1e-6 * gold[
        'weight_checksum']
    net = net.cuda().eval()
    b = fr.FrameBuilder(root, 'dog', net, chunk=2)
    b2 = fr.FrameBuilder(root, 'dog', net, chunk=2)
    G = gold['globals']
    # eager PyTorch MiDaS with TF32 (the reference's path on a GPU) against the fixture, for the bound on s and the poses
    sd = {k: v.cuda() for k, v in net.state_dict().items()}
    imgs, masks = inputs(gold, 'dog')
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
    with torch.no_grad():
        eager = [depth_nets.midas_forward(sd, torch.from_numpy(i).permute(2, 0, 1)[None].cuda(), True, [256, 512])[0, 0].cpu().numpy()
                 for i in imgs]
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    K, E, h_pt, _, _ = calib_inputs(gold)
    s_eager = oracle_frames.calibrate(E, K, h_pt, masks, eager)[4]
    e_eager, e_mine = abs(s_eager - G['s']) / G['s'], abs(b.scale - G['s']) / G['s']
    print('s: native %.3g, eager TF32 %.3g (relative)' % (e_mine, e_eager))
    assert e_mine <= 3 * e_eager + 1e-6
    for i in range(b.n_frames):
        ref = gold['outputs']['dog'][i]
        out, out2 = b.frame(i), b2.frame(i)
        assert {k: (tuple(v.shape), str(v.dtype)) for k, v in out.items()} == ref['meta']
        for k in out:
            assert np.array_equal(out[k], out2[k]), k                           # two runs are bitwise equal
        assert np.array_equal(out['intrinsics'], ref['intrinsics'].numpy())
        assert ulps32(out['img'], ref['img'].numpy()).max() <= 1.0
        dp = ref['depth_pred'].numpy()
        derr = float(np.abs(out['depth_pred'] - dp).max() / np.abs(dp).max())
        terr = float(np.abs(out['pose_c2w'][:3, 3] - ref['pose_c2w'][:3, 3].numpy()).max() / np.abs(ref['pose_c2w'][:3, 3].numpy()).max())
        print('frame %d: depth %.3g (bound 1e-3), translation %.3g' % (i, derr, terr))
        assert derr <= 1e-3
        assert terr <= 3 * e_eager + 1e-6
        assert float(out['img_orig'].astype(np.float64).sum()) == ref['img_orig_checksum']
    out_dir = str(tmp_path / 'frames_midas' / 'dog')
    assert b.write(out_dir) == 3
    for i in range(3):
        got = read_npz(os.path.join(out_dir, 'frame_%05d.npz' % i))
        nxt = read_npz(os.path.join(out_dir, 'frame_%05d.npz' % ((i + 1) % 3)))
        pt = pose_tensors(got, nxt)
        exp = pose_tensors(b.frame(i), b.frame((i + 1) % 3))
        assert all(torch.equal(pt[k], exp[k]) for k in pt)


def test_frame_builder_rejects_frames_without_points(ops, gold, tmp_path):
    from dvd_b200 import frames as fr
    root = str(tmp_path / 'davis')
    write_layout(gold, root)
    with open(os.path.join(root, 'triangulation', 'dog.obj'), 'w') as f:
        f.write('v 0 0 10\n')                                                   # behind every camera
    with pytest.raises(ValueError, match='frame'):
        fr.FrameBuilder(root, 'dog', seeded_net().cuda().eval())
