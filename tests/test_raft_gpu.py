"""GPU: the RAFT forward of dvd_b200/raft.py (csrc/raft_ops.cu + the tensor-core convolutions) against the fixture written from the
reference's RAFT (tests/golden/raft_golden.pt, oracle/gen_golden_raft.py) and against oracle/raft.py in fp64.

Every stage is fed the fixture's inputs (teacher-forced) before the whole forward is run freely. Errors are tensor-normalised,
max|a - b| / max|b|. Parameters and images are rebuilt from the fixture's seeds and checked against its checksums."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')

pytestmark = pytest.mark.gpu


def rel(a, b, scale=None):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / (scale if scale is not None else max(float(b.abs().max()), 1e-30)))


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2)


def epe(a, b):
    """mean end-point error in pixels of two [B,2,H,W] flows"""
    return float((a.double().cpu() - b.double().cpu()).norm(dim=1).mean())


@pytest.fixture(scope='module')
def gold():
    from oracle.golden_io import load_golden
    return load_golden(GOLDEN, 'raft_golden')


@pytest.fixture(scope='module')
def sd(gold):
    from oracle import raft as oracle_raft
    sd = oracle_raft.seeded_state_dict(gold['weight_seed'], gold['gain'])
    chk = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(chk - gold['weight_checksum']) <= 1e-9 * gold['weight_checksum'], 'seeded parameters differ from the fixture\'s'
    return sd


@pytest.fixture(scope='module')
def net(sd):
    from dvd_b200.raft import RaftNet
    n = RaftNet()
    n.load_state_dict(sd)
    return n.cuda()


def images(case):
    from oracle import raft as oracle_raft
    im1, im2 = oracle_raft.seeded_pair(case['H'], case['W'], case['seed'])
    chk = float(im1.double().sum() + im2.double().sum())
    assert abs(chk - case['image_checksum']) <= 1e-9 * abs(case['image_checksum']), 'seeded images differ from the fixture\'s'
    return im1, im2


def eager_tf32(fn):
    """fn() in eager PyTorch with cuDNN's TF32 convolutions on: what the reference's own GPU path computes"""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        with torch.no_grad():
            return fn()
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def tf32_bound(eager_err):
    """TF32 stages are held to 1e-3 or, where a chain of TF32 layers is deeper than that allows, to three times the error eager
    PyTorch's TF32 convolutions make on the same stage in the same run"""
    return max(1e-3, 3 * eager_err)


def flat_pyramid(levels):
    return torch.cat([l.reshape(-1) for l in levels]).cuda().contiguous()


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('C', [64, 96, 128])
def test_instance_norm_against_fp64(C):
    from dvd_b200 import raft
    g = torch.Generator().manual_seed(C)
    x = (torch.randn(2, 20, 28, C, generator=g) * 3 + torch.randn(1, 1, 1, C, generator=g) * 5)
    res = torch.randn(2, 20, 28, C, generator=g)
    xd = x.double()
    mean, var = xd.mean((1, 2), keepdim=True), xd.var((1, 2), unbiased=False, keepdim=True)
    ref = torch.relu(torch.relu((xd - mean) / torch.sqrt(var + 1e-5)) + res.double())
    xg = x.cuda()
    stats = raft.instnorm_stats(xg)
    y = raft.norm_act(xg, stats, res.cuda(), relu_inner=True, relu_outer=True, round_out=False)
    assert rel(stats[..., 0], mean.reshape(2, C)) < 1e-5
    assert rel(y, ref) < 1e-5, rel(y, ref)
    # a fixed reduction order: a second launch gives the same bits
    assert torch.equal(raft.instnorm_stats(xg), stats)
    # the rounded output is the TF32 rounding of the same values
    from dvd_b200 import conv_ops
    yr = raft.norm_act(xg, stats, res.cuda(), relu_inner=True, relu_outer=True, round_out=True)
    assert torch.equal(yr, conv_ops.round_tf32(y.reshape(-1)).reshape(y.shape))


def test_stems_against_fp64(gold, sd, net):
    from dvd_b200 import conv_ops, raft
    from oracle import raft as oracle_raft
    case = gold['cases'][0]
    im1, _ = images(case)
    sd64 = oracle_raft.cast(sd, torch.float64)
    ref_f = oracle_raft.stem(sd64, 'fnet', im1.double(), 'instance')
    s = raft.raft_stem(im1.cuda(), net.fnet.conv1.weight.detach().contiguous(), net.fnet.conv1.bias.detach())
    y = raft.norm_act(s, raft.instnorm_stats(s), relu_inner=True, round_out=False)
    assert rel(nchw(y), ref_f) < 1e-5, rel(nchw(y), ref_f)
    ref_c = oracle_raft.stem(sd64, 'cnet', im1.double(), 'batch')
    c, n = net.cnet.conv1, net.cnet.norm1
    yc = conv_ops.stem_fwd(im1.cuda(), c, raft._Norm(n.weight.detach(), n.bias.detach(), net.plan().c_stem_mean, n.running_var, n.eps),
                           norm_mean=(127.5,) * 3, norm_std=(127.5,) * 3, round_out=False)
    assert rel(yc, ref_c) < 1e-5, rel(yc, ref_c)


def test_encoders_against_fixture(gold, sd, net):
    from oracle import raft as oracle_raft
    case = gold['cases'][0]
    im1, im2 = images(case)
    sdg = oracle_raft.cast(sd, torch.float32, 'cuda')
    ref = {'fmap1': rel(eager_tf32(lambda: oracle_raft.encoder(sdg, 'fnet', im1.cuda(), 'instance')), case['fmap1']),
           'net0': rel(eager_tf32(lambda: oracle_raft.context(sdg, im1.cuda())[0]), case['net0'])}
    f = net.encode(torch.cat([im1, im2]).cuda())
    e = {'fmap1': rel(nchw(f.fmap[0:1]), case['fmap1']), 'fmap2': rel(nchw(f.fmap[1:2]), case['fmap2']),
         'net0': rel(torch.tanh(nchw(f.cnet[0:1, ..., :128])), case['net0']),
         'inp': rel(torch.relu(nchw(f.cnet[0:1, ..., 128:])), case['inp'])}
    print('encoder errors (TF32 convolutions):', e, 'eager PyTorch TF32:', ref)
    assert max(e['fmap1'], e['fmap2']) <= tf32_bound(ref['fmap1']) and max(e['net0'], e['inp']) <= tf32_bound(ref['net0']), (e, ref)


def test_correlation_pyramid_is_fp32_grade(gold):
    from dvd_b200 import raft
    from oracle import raft as oracle_raft
    case = gold['cases'][0]
    f1, f2 = nhwc(case['fmap1']).cuda(), nhwc(case['fmap2']).cuda()
    B, h, w, _ = f1.shape
    levels = raft.pyramid_levels(raft.corr_pyramid(f1, f2), B, h, w)
    for l, (mine, ref) in enumerate(zip(levels, case['pyramid'])):
        assert mine.shape == ref[:, 0].shape
        assert rel(mine, ref[:, 0]) < 1e-5, (l, rel(mine, ref[:, 0]))
    # an odd grid (17 x 24: the pooling drops a row) and two pairs, against fp64
    g = torch.Generator().manual_seed(5)
    a, b = torch.randn(2, 17, 24, 256, generator=g), torch.randn(2, 17, 24, 256, generator=g)
    ref = oracle_raft.corr_pyramid(nchw(a).double(), nchw(b).double())
    levels = raft.pyramid_levels(raft.corr_pyramid(a.cuda(), b.cuda()), 2, 17, 24)
    for l, (mine, r) in enumerate(zip(levels, ref)):
        assert rel(mine, r[:, 0]) < 1e-5, (l, rel(mine, r[:, 0]))


@pytest.mark.parametrize('ci', [0, 1])
def test_lookup_against_fixture_and_fp64(gold, ci):
    from dvd_b200 import raft
    from oracle import raft as oracle_raft
    case = gold['cases'][ci]
    pyr = flat_pyramid(case['pyramid'])
    pmax = float(case['pyramid'][0].abs().max())
    pyr64 = [l.double() for l in case['pyramid']]
    left = 0
    for it in (0, 3, 19):
        c1 = case['coords1'][it:it + 1]
        out = raft.lookup(pyr, nhwc(c1).cuda(), round_out=False)
        assert float(out[..., 324:].abs().max()) == 0.0
        ref = oracle_raft.lookup(pyr64, c1.double())
        assert rel(nchw(out[..., :324]), ref, pmax) < 1e-5, (it, rel(nchw(out[..., :324]), ref, pmax))
        if it in case['steps']:
            assert rel(nchw(out[..., :324]), case['steps'][it]['corr'], pmax) < 1e-5
        h, w = c1.shape[-2:]
        left += int(((c1[:, 0] < 4) | (c1[:, 0] > w - 5) | (c1[:, 1] < 4) | (c1[:, 1] > h - 5)).sum())
    assert left > 0, 'no window left the image: the zero padding was not exercised'
    # centres far outside sample nothing
    far = torch.full_like(case['coords1'][0:1], -1000.0)
    assert float(raft.lookup(pyr, nhwc(far).cuda()).abs().max()) == 0.0


def test_lookup_channel_order_on_an_impulse():
    """a single non-zero entry of level 0 at q = (y 9, x 12): from a centre at (x 10, y 10) it is the offset (+2, -1), channel
    (2 + 4) * 9 + (-1 + 4): the window's slow index moves along x"""
    from dvd_b200 import raft
    B, h, w = 1, 16, 20
    levels = [torch.zeros(h * w, h >> l, w >> l) for l in range(4)]
    levels[0][:, 9, 12] = 1.0
    coords = torch.zeros(1, h, w, 2)
    coords[..., 0], coords[..., 1] = 10.0, 10.0
    out = raft.lookup(flat_pyramid(levels), coords.cuda(), round_out=False)
    assert int(out[0, 0, 0].argmax()) == 6 * 9 + 3 and float(out[0, 0, 0].sum()) == 1.0


def gru_state(net_in, inp):
    """the two GRU operands and the hidden state as RaftNet.init_state leaves them, from the fixture's tensors"""
    from dvd_b200 import conv_ops
    B, _, h, w = net_in.shape
    net = nhwc(net_in).cuda()
    X = torch.zeros(B, h, w, 384, device='cuda')
    X[..., :128] = conv_ops.round_tf32(net.reshape(-1)).reshape(net.shape)
    i_r = nhwc(inp).cuda()
    X[..., 128:256] = conv_ops.round_tf32(i_r.reshape(-1)).reshape(i_r.shape)
    return net, X, X.clone(), torch.empty_like(net)


@pytest.mark.parametrize('it', [0, 3])
def test_update_step_alone_from_the_fixture_state(gold, sd, net, it):
    from oracle import raft as oracle_raft
    case = gold['cases'][0]
    sdg = oracle_raft.cast(sd, torch.float32, 'cuda')
    st = case['steps'][it]
    pyr = flat_pyramid(case['pyramid'])
    hidden, X, XR, net_r = gru_state(st['net_in'], case['inp'])
    coords1 = nhwc(case['coords1'][it:it + 1]).cuda()
    before = coords1.clone()
    _, delta = net.update_step(net.plan(), pyr, coords1, hidden, X, XR, net_r, want_delta=True)
    e = {'net': rel(nchw(hidden), st['net']), 'delta_flow': rel(nchw(delta), case['delta_flow'][it:it + 1])}
    flow = case['coords1'][it:it + 1] - oracle_raft.coords_grid(1, *case['coords1'].shape[-2:], torch.float32, 'cpu')
    r_net, r_delta = eager_tf32(lambda: oracle_raft.update(sdg, st['net_in'].cuda(), case['inp'].cuda(), st['corr'].cuda(), flow.cuda()))
    ref = {'net': rel(r_net, st['net']), 'delta_flow': rel(r_delta, case['delta_flow'][it:it + 1])}
    print('update iteration %d errors:' % it, e, 'eager PyTorch TF32:', ref)
    assert e['net'] <= tf32_bound(ref['net']) and e['delta_flow'] <= tf32_bound(ref['delta_flow']), (e, ref)
    assert torch.equal(coords1, before + delta)


def test_init_state_splits_the_context(gold, net):
    case = gold['cases'][0]
    im1, _ = images(case)
    f = net.encode(im1.cuda())
    hidden, X, XR, _ = net.init_state(f.cnet)
    # the values test_encoders_against_fixture bounds, split and (for the convolution operand) TF32-rounded: 2^-11 on top
    assert torch.equal(hidden, torch.tanh(f.cnet[..., :128]))
    assert rel(X[..., 128:256], torch.relu(f.cnet[..., 128:])) < 5e-4 and rel(X[..., :128], hidden) < 5e-4
    assert torch.equal(X[..., 128:256], XR[..., 128:256])


def test_convex_upsampling_from_the_fixture(gold):
    from dvd_b200 import raft
    case = gold['cases'][0]
    fin = case['final'][1]
    low, mask = fin['flow_low'], nhwc(fin['up_mask'])
    B, _, h, w = low.shape
    coords1 = (nhwc(low) + raft.coords_grid(B, h, w, 'cpu')).cuda()
    parts = [mask[..., i * 192:(i + 1) * 192].contiguous().cuda() for i in range(3)]
    up = raft.upsample(parts, coords1, mask_scale=1.0)
    assert rel(nchw(up), fin['flow_up']) < 1e-5, rel(nchw(up), fin['flow_up'])


# ------------------------------------------------------------------------------------------------
def test_forward_is_deterministic(gold, net):
    im1, im2 = (t.cuda() for t in images(gold['cases'][0]))
    a = net(im1, im2, iters=4)
    b = net(im1, im2, iters=4)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def tf32_spread(sd, im1, im2, iters):
    """end-point spread of eager fp32 PyTorch on this GPU between TF32 convolutions on and off"""
    from oracle import raft as oracle_raft
    sdg = oracle_raft.cast(sd, torch.float32, 'cuda')
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    out = []
    try:
        for on in (True, False):
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = on, False
            with torch.no_grad():
                out.append(oracle_raft.raft_forward(sdg, im1, im2, iters)[1])
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return epe(out[0], out[1])


@pytest.mark.parametrize('ci', [0, 1])
@pytest.mark.parametrize('iters', [1, 4, 20])
def test_free_running_flow_against_fixture(gold, sd, net, ci, iters):
    case = gold['cases'][ci]
    im1, im2 = (t.cuda() for t in images(case))
    low, up = net(im1, im2, iters=iters)
    fin = case['final'][iters]
    err, s = epe(up, fin['flow_up']), tf32_spread(sd, im1, im2, iters)
    bound = max(4 * s, 1e-3)
    msg = '%dx%d iters=%d: mean EPE %.3e px (eager TF32 on/off spread %.3e px, bound %.3e, fixture floor %.1e, mean |flow| %.2f px) on %s' % (
        case['H'], case['W'], iters, err, s, bound, case['floor_epe'][iters], float(fin['flow_up'].norm(dim=1).mean()),
        torch.cuda.get_device_name(0))
    print(msg)
    assert err <= bound, msg
    assert low.shape == fin['flow_low'].shape and up.shape == fin['flow_up'].shape


def test_cached_features_and_batches_change_nothing(gold, net):
    from oracle import raft as oracle_raft
    case = gold['cases'][0]
    im1, im2 = (t.cuda() for t in images(case))
    im3 = oracle_raft.seeded_pair(case['H'], case['W'], 9)[1].cuda()
    fresh = net(im1, im2, iters=3)[1]
    feats = net.encode(torch.cat([im1, im2, im3]))
    one = net.flow(feats.index([0]), feats.index([1]), iters=3)
    assert torch.equal(nchw(one), fresh), 'features cached from a batch of frames give a different flow'
    a_idx, b_idx = [0, 1, 2, 1], [1, 0, 0, 2]
    batch = net.flow(feats.index(a_idx), feats.index(b_idx), iters=3)
    for k, (a, b) in enumerate(zip(a_idx, b_idx)):
        single = net.flow(feats.index([a]), feats.index([b]), iters=3)
        assert torch.equal(batch[k:k + 1], single), 'pair %d of the batch differs from the same pair run alone' % k


def test_rejected_requests(net):
    from dvd_b200.raft import RaftNet
    with pytest.raises(ValueError):
        RaftNet(small=True)
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 132, 160, device='cuda'), torch.zeros(1, 3, 132, 160, device='cuda'))
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 64, 96, device='cuda'), torch.zeros(1, 3, 64, 96, device='cuda'))
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 128, 160), torch.zeros(1, 3, 128, 160))
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 128, 160, device='cuda'), torch.zeros(1, 3, 128, 160, device='cuda'), flow_init=torch.zeros(1))


# ------------------------------------------------------------------------------------------------
def write_track(root, track, n, H, W):
    """a seeded synthetic track with frame files only: frames_midas/<track>/frame_%05d.npz with smooth moving images"""
    import numpy as np
    from oracle import raft as oracle_raft
    d = os.path.join(root, 'frames_midas', track)
    os.makedirs(d)
    rng = np.random.RandomState(0)
    base, _ = oracle_raft.seeded_pair(H + 32, W + 32, 3)
    K = np.array([[W, 0, W / 2], [0, W, H / 2], [0, 0, 1]], np.float64)
    for f in range(n):
        img = (base[0, :, f:f + H, 2 * f:2 * f + W] / 255).permute(1, 2, 0).numpy().astype(np.float32)
        pose = np.eye(4)
        pose[0, 3] = 0.01 * f
        depth = (2 + rng.rand(H, W)).astype(np.float32)
        np.savez(os.path.join(d, 'frame_%05d.npz' % f), img=img, img_orig=img, pose_c2w=pose, intrinsics=K, depth_mvs=depth,
                 depth_pred=depth)
    return d


def test_pairs_from_frames_alone_equal_pairs_from_saved_flows(tmp_path, net):
    from dvd_b200.flow_pairs import PairBuilder
    H, W, n, gaps = 128, 160, 12, [1, 2]
    frames = write_track(str(tmp_path), 'clip', n, H, W)
    direct = PairBuilder(frames, None, gaps, raft=net, raft_iters=2, raft_chunk=5)
    assert direct.raw_pairs == len(direct) == sum(n - 1 - g for g in gaps)
    flows = str(tmp_path / 'flow_pairs' / 'clip')
    direct.write(str(tmp_path / 'seq'), flows_out=flows)
    saved = PairBuilder(frames, flows, gaps)
    assert saved.raw_pairs == 0
    for i in range(len(direct)):
        a, b = direct[i], saved[i]
        assert a.keys() == b.keys()
        for k in a:
            if torch.is_tensor(a[k]):
                assert a[k].shape == b[k].shape and a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k
    f = direct.flows[0][0]
    assert torch.isfinite(f).all() and float(f.abs().max()) > 0


def test_train_cli_estimates_flows_from_a_raft_checkpoint(tmp_path, sd):
    import subprocess
    write_track(str(tmp_path), 'clip', 12, 128, 160)
    ckpt = str(tmp_path / 'raft.pth')
    torch.save({'module.' + k: v for k, v in sd.items()}, ckpt)
    args = ('--net scene_flow_motion_field --dataset video_frames --track_id clip --gaps 1,2 --epoch 1 --epoch_batches 2 '
            '--resident --lr 1e-6 --batch_size 1 --optim adam --gpu 0 --workers 0 --one_way --loss_type l1 --l1_mul 0 '
            '--acc_mul 1 --disp_mul 1 --warm_sf 1 --scene_lr_mul 1000 --flow_mul 1 --sf_mag_div 100 --time_dependent --use_disp '
            '--vis_batches_train 0 --manual_seed 1 --raft_iters 2').split()
    args += ['--data_root', str(tmp_path), '--logdir', str(tmp_path / 'log'), '--raft_ckpt', ckpt]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', 'dvd_b200.train'] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1100)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    lines = [l for l in r.stdout.splitlines() if l.startswith('epoch 1:')]
    assert lines, r.stdout[-2000:]
    log = eval(lines[0].split(':', 1)[1])       # the driver prints a plain dict of floats
    assert all(v == v and abs(v) != float('inf') for v in log.values()), log
