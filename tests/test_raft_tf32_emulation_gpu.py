"""GPU: the RAFT forward of dvd_b200/raft.py against oracle/raft_tf32.py, an fp64 emulation of its own precision model (the
reference's structure, RaftNet's TF32 rounding points). What is left between the two is fp32 accumulation order and the
occasional one-step TF32 rounding flip, so the bounds below are far tighter than test_raft_gpu.py's comparison with the
reference (3 x the eager-TF32 error, about 4e-3 to 1.3e-2): a producer that stops rounding, a swapped or shifted channel
slice, a merged layer in the wrong order or a wrong scale fails.

The emulation is teacher-forced at every tensor RaftNet.encode / RaftNet.flow trace: each stage is checked on RaftNet's own
inputs. The GRU operand buffers X and XR, written in place by four kernels, are checked slice by slice after each of them.
Cases: the fixture's 128x160 pair (all 20 iterations), its 136x192 pair (a 17 x 24 grid, odd in both directions; iterations
0-3), and 16 ordered pairs at 288x512, the production size and raft_chunk's default batch (iterations 0, 1, 9, 19).

Bounds: measured on an NVIDIA H100 80GB HBM3 (700 W power limit), set at about 3x the largest value observed over the cases
below. Every convolution the plan launches is also checked alone against fp64 on pre-rounded operands (CONV_CASES)."""
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, rel_err

pytestmark = pytest.mark.gpu

# TF32-rounded anchors: share of elements that differ from the emulation, share more than one TF32 step away, and the max-norm
# error of those far elements relative to the tensor's maximum. An element computed from anchored inputs is more than one step
# off only where it is a cancellation near zero. Observed maxima over the three cases: 9.7e-3 (convc2), 9.9e-4 (convc2),
# 3.0e-6 (convc2); a producer that stops rounding differs in about half of its elements
DIFF, FAR, FAR_REL = 0.03, 3e-3, 1e-5
# unrounded anchors: max-norm error relative to the tensor's maximum; observed 7.0e-6 (q of GRU half 0, K = 5 x 384)
UNROUNDED_REL = 2e-5
TOL = 2e-5          # single convolutions on pre-rounded operands against fp64 (test_conv2d_gpu.py)


def bits(t):
    return t.contiguous().view(torch.int32).long()


def tf32(t):
    from oracle.midas_tf32 import round_tf32
    return round_tf32(t.float())


def one_step(a, b):
    """every element of the fp32 tensors a and b equal or neighbouring TF32 values"""
    d = (bits(a) - bits(b)).abs()
    return bool(((d == 0) | (d == 0x2000)).all())


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def nchw(t):
    return t.permute(0, 3, 1, 2)


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


# ------------------------------------------------------------------------------------------------
# the plan's packed weights and each of its convolutions alone

def plan_layers(net):
    """(name, _TC, weight, bias) of every convolution the plan launches, weight and bias in the layout the plan must have
    built from the reference's parameters: zero input columns 324..351 of convc1, zero output rows 126/127 of the motion
    convolution split into its 192 correlation and 64 flow input channels, z before r, the mask head in slices of 192"""
    from dvd_b200.raft import BLOCK_NAMES
    P = net.plan()
    out = []
    for enc, blocks in (('fnet', P.f_blocks), ('cnet', P.c_blocks)):
        for name, m, (c1, c2, ds) in zip(BLOCK_NAMES, getattr(net, enc).blocks(), blocks):
            out += [('%s.%s.conv1' % (enc, name), c1, m.conv1.weight, m.conv1.bias),
                    ('%s.%s.conv2' % (enc, name), c2, m.conv2.weight, m.conv2.bias)]
            if ds is not None:
                out.append(('%s.%s.downsample' % (enc, name), ds, m.downsample[0].weight, m.downsample[0].bias))
    out += [('fnet.conv2', P.f_out, net.fnet.conv2.weight, net.fnet.conv2.bias),
            ('cnet.conv2', P.c_out, net.cnet.conv2.weight, net.cnet.conv2.bias)]
    u, e, g = net.update_block, net.update_block.encoder, net.update_block.gru
    out.append(('convc1', P.convc1, F.pad(e.convc1.weight, (0, 0, 0, 0, 0, 28)), e.convc1.bias))
    out += [('convc2', P.convc2, e.convc2.weight, e.convc2.bias), ('convf2', P.convf2, e.convf2.weight, e.convf2.bias)]
    w, b = F.pad(e.conv.weight, (0, 0, 0, 0, 0, 0, 0, 2)), F.pad(e.conv.bias, (0, 2))
    out += [('conv_flo', P.conv_flo, w[:, 192:], None), ('conv_cor', P.conv_cor, w[:, :192], b)]
    for tag, (zr, q) in zip('12', P.gru):
        cz, cr, cq = (getattr(g, 'conv%s%s' % (k, tag)) for k in 'zrq')
        out += [('gru.zr' + tag, zr, torch.cat([cz.weight, cr.weight]), torch.cat([cz.bias, cr.bias])),
                ('gru.q' + tag, q, cq.weight, cq.bias)]
    out += [('fh1', P.fh1, u.flow_head.conv1.weight, u.flow_head.conv1.bias), ('mask0', P.mask0, u.mask[0].weight, u.mask[0].bias)]
    out += [('mask2.%d' % i, c, u.mask[2].weight[192 * i:192 * (i + 1)], u.mask[2].bias[192 * i:192 * (i + 1)])
            for i, c in enumerate(P.mask2)]
    return [(n, tc, w.detach(), b.detach() if b is not None else None) for n, tc, w, b in out]


def test_plan_weight_images_are_the_rounded_weights(net):
    """_TC.image is [tap][Cout][Cin] with tap = ky * kw + kx: equal to round_tf32(W) bit for bit, the zero rows and columns
    included; the biases and the context stem's folded BatchNorm mean are the parameters' own"""
    layers = plan_layers(net)
    assert len(layers) == 2 * (12 + 2) + 2 + 5 + 4 + 2 + 3
    for name, tc, w, b in layers:
        co, ci, kh, kw = w.shape
        want = tf32(w).permute(2, 3, 0, 1).reshape(kh * kw, co, ci)
        assert (tc.cout, tc.cin, tc.k) == (co, ci, (kh, kw)), name
        assert same(tc.image, want), name
        assert (tc.bias is None) == (b is None) and (b is None or same(tc.bias, b)), name
    P = net.plan()
    assert same(P.c_stem_mean, (net.cnet.norm1.running_mean - net.cnet.conv1.bias).detach())


# name, Cin, Cout, (kh, kw), stride, bn, bias, relu, res, input side relative to the 1/8 grid
CONV_CASES = [
    ('fnet.layer1', 64, 64, (3, 3), 1, False, True, False, False, 4),
    ('fnet.layer2.0.conv1', 64, 96, (3, 3), 2, False, True, False, False, 4),
    ('fnet.layer2.0.downsample', 64, 96, (1, 1), 2, False, True, False, False, 4),
    ('fnet.layer2', 96, 96, (3, 3), 1, False, True, False, False, 2),
    ('fnet.layer3.0.conv1', 96, 128, (3, 3), 2, False, True, False, False, 2),
    ('fnet.layer3.0.downsample', 96, 128, (1, 1), 2, False, True, False, False, 2),
    ('fnet.layer3', 128, 128, (3, 3), 1, False, True, False, False, 1),
    ('conv2', 128, 256, (1, 1), 1, False, True, False, False, 1),
    ('cnet.layer1', 64, 64, (3, 3), 1, True, True, True, False, 4),
    ('cnet.layer2.0.conv1', 64, 96, (3, 3), 2, True, True, True, False, 4),
    ('cnet.layer2.0.downsample', 64, 96, (1, 1), 2, True, True, True, True, 4),
    ('cnet.layer2', 96, 96, (3, 3), 1, True, True, True, False, 2),
    ('cnet.layer3.0.conv1', 96, 128, (3, 3), 2, True, True, True, False, 2),
    ('cnet.layer3.0.downsample', 96, 128, (1, 1), 2, True, True, True, True, 2),
    ('cnet.layer3', 128, 128, (3, 3), 1, True, True, True, False, 1),
    ('convc1', 352, 256, (1, 1), 1, False, True, True, False, 1),
    ('convc2', 256, 192, (3, 3), 1, False, True, True, False, 1),
    ('convf2', 128, 64, (3, 3), 1, False, True, True, False, 1),
    ('conv_flo', 64, 128, (3, 3), 1, False, False, False, False, 1),
    ('conv_cor', 192, 128, (3, 3), 1, False, True, True, True, 1),
    ('gru.zr1', 384, 256, (1, 5), 1, False, True, False, False, 1),
    ('gru.q1', 384, 128, (1, 5), 1, False, True, False, False, 1),
    ('gru.zr2', 384, 256, (5, 1), 1, False, True, False, False, 1),
    ('gru.q2', 384, 128, (5, 1), 1, False, True, False, False, 1),
    ('fh1, mask0', 128, 256, (3, 3), 1, False, True, True, False, 1),
    ('mask2', 256, 192, (1, 1), 1, False, True, False, False, 1),
]


def _case_key(ci, co, k, stride, bn, bias, relu):
    return ci, co, tuple(k), stride, bool(bn), bool(bias), bool(relu)


def test_conv_cases_cover_every_launch_of_the_plan(net):
    keys = {_case_key(*c[1:8]) for c in CONV_CASES}
    for name, tc, _, _ in plan_layers(net):
        key = _case_key(tc.cin, tc.cout, tc.k, tc.stride, tc.bn is not None, tc.bias is not None, tc.relu)
        assert key in keys, (name, key)


@pytest.mark.parametrize('batch', [1, 16])
@pytest.mark.parametrize('grid', [(36, 64), (17, 24)], ids=['36x64', '17x24'])
@pytest.mark.parametrize('case', CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_raft_conv_launch_matches_fp64(case, grid, batch):
    from dvd_b200.raft import _TC
    name, ci, co, k, stride, use_bn, use_bias, relu, use_res, scale = case
    g = torch.Generator().manual_seed(ci * 7 + co + 13 * k[0] + k[1] + stride + 3 * scale)
    H, W = grid[0] * scale, grid[1] * scale
    pad = (k[0] // 2, k[1] // 2)
    OH, OW = (H + 2 * pad[0] - k[0]) // stride + 1, (W + 2 * pad[1] - k[1]) // stride + 1
    w = torch.randn(co, ci, *k, generator=g) / (ci * k[0] * k[1]) ** 0.5
    b = torch.randn(co, generator=g) if use_bias else None
    bn = None
    if use_bn:
        bn = torch.nn.BatchNorm2d(co).eval()
        with torch.no_grad():
            bn.weight.copy_(torch.rand(co, generator=g) + 0.5)
            bn.bias.copy_(torch.randn(co, generator=g))
            bn.running_mean.copy_(torch.randn(co, generator=g) * 0.1)
            bn.running_var.copy_(torch.rand(co, generator=g) + 0.5)
        bn = bn.cuda()
    x = tf32(torch.randn(batch, H, W, ci, generator=g)).cuda()
    res = torch.randn(batch, OH, OW, co, generator=g).cuda() if use_res else None
    ref = F.conv2d(nchw(x).double(), tf32(w).double().cuda(), b.double().cuda() if b is not None else None, stride=stride, padding=pad)
    if bn is not None:
        ref = F.batch_norm(ref, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(), bn.bias.double(), False, 0.0, bn.eps)
    if res is not None:
        ref = ref + nchw(res).double()
    if relu:
        ref = ref.relu()
    tc = _TC(w.cuda(), b.cuda() if b is not None else None, stride=stride, padding=pad, bn=bn, relu=relu, round_out=False)
    y = tc(x, res=res)
    assert y.shape == (batch, OH, OW, co)
    e = rel_err(nchw(y), ref)
    assert e < TOL, (name, e)
    tc.round_out = True
    assert same(tc(x, res=res), tf32(y)), name


# ------------------------------------------------------------------------------------------------
def test_trace_changes_nothing(gold, net):
    from oracle import raft as oracle_raft
    case = gold['cases'][0]
    frames = torch.cat(oracle_raft.seeded_pair(case['H'], case['W'], case['seed'])).cuda()
    f = net.encode(frames)
    tr = {}
    ft = net.encode(frames, trace=tr)
    assert same(f.fmap, ft.fmap) and same(f.cnet, ft.cnet) and tr
    a, b = f.index([0, 1]), f.index([1, 0])
    up, low = net.flow(a, b, iters=4, return_low=True)
    tr = {}
    up_t, low_t = net.flow(a, b, iters=4, return_low=True, trace=tr)
    assert same(up, up_t) and same(low, low_t) and len(tr['iters']) == 4
    assert same(tr['flow_up'], up)


# ------------------------------------------------------------------------------------------------
def _check_operands(tr, cnet, check_iters):
    """the GRU operand buffers slice by slice after each kernel that writes them, and the exact zeros"""
    from dvd_b200.raft import coords_grid
    B, h, w, _ = cnet.shape
    grid = coords_grid(B, h, w, cnet.device)
    X0, XR0 = tr['X'], tr['XR']
    # context_split: round(net) and round(relu(inp)); XR[:, :128] is written by gru_rh before q reads it
    assert same(X0[..., :128], tf32(tr['net'])), 'X[:, :128] after context_split is not round(net)'
    assert one_step(X0[..., :128], tf32(torch.tanh(cnet[..., :128].double()))), 'X[:, :128] after context_split: not tanh'
    assert same(X0[..., 128:256], tf32(torch.relu(cnet[..., 128:]))) and same(XR0[..., 128:256], X0[..., 128:256]), 'inp slice'
    for k in check_iters:
        it = tr['iters'][k]
        c_in = grid if k == 0 else tr['iters'][k - 1]['coords1']
        n_in = tr['net'] if k == 0 else tr['iters'][k - 1]['net.1']
        assert float(it['corr'][..., 324:].abs().max()) == 0.0, (k, 'the lookup\'s zero tail is not zero')
        assert float(it['motion'][..., 126:].abs().max()) == 0.0, (k, 'motion conv pad outputs 126/127 are not zero')
        flow = tf32(c_in - grid)
        for nm in ('X.pack', 'XR.pack'):
            buf = it[nm]
            assert same(buf[..., 256:382], it['motion'][..., :126]), (k, nm, 'channels 256..381 are not the motion output')
            assert same(buf[..., 382:384], flow), (k, nm, 'channels 382/383 are not tf32(coords1 - grid) as (x, y)')
            assert same(buf[..., 128:256], X0[..., 128:256]), (k, nm, 'inp slice changed')
        assert same(it['X.pack'][..., :128], tf32(n_in)), (k, 'X[:, :128] entering the iteration is not round(net)')
        nets = (n_in, it['net.0'])
        for i in (0, 1):
            XRr, Xg, zr = it['XR.rh.%d' % i], it['X.gru.%d' % i], it['zr.%d' % i]
            assert same(XRr[..., 128:], it['XR.pack'][..., 128:]), (k, i, 'gru_rh wrote outside XR[:, :128]')
            rh = tf32(torch.sigmoid(zr[..., 128:].double()) * nets[i].double())
            assert one_step(XRr[..., :128], rh), (k, i, 'XR[:, :128] is not round(sigmoid(r) net) within one TF32 step')
            assert same(Xg[..., :128], tf32(it['net.%d' % i])), (k, i, 'X[:, :128] after gru_update is not round(net)')
            assert same(Xg[..., 128:], it['X.pack'][..., 128:]), (k, i, 'gru_update wrote outside X[:, :128]')
        assert same(it['net_r'], tf32(it['net.1'])), (k, 'net_r is not round(net) after the second GRU half')


def _worst(rep, key):
    n, r = max(rep.items(), key=lambda kv: kv[1][key])
    return '%.2e (%s)' % (r[key], n)


def _check_report(rep, label):
    rounded = {n: r for n, r in rep.items() if r['rounded']}
    unrounded = {n: r for n, r in rep.items() if not r['rounded']}
    print('\n[%s] %d anchors | unrounded rel %s | rounded: differ %s, beyond one step %s, their error %s' % (
        label, len(rep), _worst(unrounded, 'rel_max'), _worst(rounded, 'diff'), _worst(rounded, 'far'), _worst(rounded, 'far_rel_max')))
    bad = [(n, r['rel_max']) for n, r in unrounded.items() if not r['rel_max'] <= UNROUNDED_REL]
    assert not bad, ('unrounded tensors beyond %.0e' % UNROUNDED_REL, bad)
    bad = [(n, r['diff'], r['far'], r['far_rel_max']) for n, r in rounded.items()
           if not (r['diff'] <= DIFF and r['far'] <= FAR and r['far_rel_max'] <= FAR_REL)]
    assert not bad, ('rounded tensors beyond (differ %.0e, far %.0e, far error %.0e)' % (DIFF, FAR, FAR_REL), bad)


def _check_against_emulation(net, sd, frames, a_idx, b_idx, iters, check_iters, label):
    from oracle import raft as oracle_raft
    from oracle.raft_tf32 import Anchors, RaftTF32, anchor_names, encoder_anchors, iteration_anchors, state_anchors
    sd64 = oracle_raft.cast(sd, torch.float64, 'cuda')
    t0 = torch.cuda.Event(enable_timing=True)
    t0.record()
    enc = {}
    feats = net.encode(frames, trace=enc)
    tr = {}
    net.flow(feats.index(a_idx), feats.index(b_idx), iters=iters, trace=tr)
    keep = set(check_iters) | {k - 1 for k in check_iters if k > 0}
    for k, it in enumerate(tr['iters']):
        if k not in keep:
            it.clear()
    fa, fb = feats.index(a_idx), feats.index(b_idx)
    B, h, w, _ = fa.fmap.shape
    with torch.no_grad():
        anc = Anchors(encoder_anchors(enc))
        RaftTF32(sd64, anchors=anc).encode(frames.double())
        assert sorted(anc.report) == sorted(anchor_names('encoder'))
        rep = dict(anc.report)
        del enc, anc
        A = state_anchors(tr, B, h, w)
        for k in check_iters:
            A.update(iteration_anchors(tr['iters'][k], 'it%d.' % k))
        anc = Anchors(A)
        emu = RaftTF32(sd64, anchors=anc)
        pyr = emu.pyramid(nchw(fa.fmap).double(), nchw(fb.fmap).double())
        net0, inp = emu.context_split(nchw(fa.cnet).double())
        coords0 = oracle_raft.coords_grid(B, h, w, torch.float64, 'cuda')
        for k in check_iters:
            c_in = coords0 if k == 0 else nchw(tr['iters'][k - 1]['coords1']).double()
            n_in = net0 if k == 0 else nchw(tr['iters'][k - 1]['net.1']).double()
            emu.update(pyr, n_in, inp, c_in, coords0, 'it%d.' % k)
        del pyr
        last = tr['iters'][iters - 1]
        emu.upsample(emu.up_mask(nchw(last['net_r']).double()), nchw(last['coords1']).double(), coords0)
    want = set(anchor_names('state')) | {'it%d.%s' % (k, n) for k in check_iters for n in anchor_names('iteration')}
    assert set(anc.report) == want, sorted(want ^ set(anc.report))
    rep.update(anc.report)
    t1 = torch.cuda.Event(enable_timing=True)
    t1.record()
    torch.cuda.synchronize()
    print('\n[%s] %d pairs, %dx%d grid, iterations %s: %.1f s, peak memory %.1f GB on %s' % (
        label, B, h, w, list(check_iters), t0.elapsed_time(t1) / 1e3, torch.cuda.max_memory_allocated() / 2 ** 30,
        torch.cuda.get_device_name(0)))
    _check_report(rep, label)
    _check_operands(tr, fa.cnet, check_iters)


def _fixture_frames(case):
    from oracle import raft as oracle_raft
    im1, im2 = oracle_raft.seeded_pair(case['H'], case['W'], case['seed'])
    chk = float(im1.double().sum() + im2.double().sum())
    assert abs(chk - case['image_checksum']) <= 1e-9 * abs(case['image_checksum']), 'seeded images differ from the fixture\'s'
    return torch.cat([im1, im2]).cuda()


def test_fixture_128x160_every_iteration_matches_tf32_emulation(gold, sd, net):
    _check_against_emulation(net, sd, _fixture_frames(gold['cases'][0]), [0], [1], 20, range(20), '128x160')


def test_fixture_136x192_odd_grid_matches_tf32_emulation(gold, sd, net):
    _check_against_emulation(net, sd, _fixture_frames(gold['cases'][1]), [0, 1], [1, 0], 4, range(4), '136x192')


@pytest.mark.timeout(1200)
def test_production_size_16_pairs_match_tf32_emulation(sd, net):
    """288 x 512 with 16 ordered pairs per launch (raft_chunk's default) among 8 frames: 4 seeded textures and a warped copy
    of each"""
    from oracle import raft as oracle_raft
    frames = torch.cat([torch.cat(oracle_raft.seeded_pair(288, 512, s, shift=6.0)) for s in range(4)]).cuda()
    a_idx = [0, 1, 2, 3, 4, 5, 6, 7, 0, 2, 4, 6, 1, 3, 5, 7]
    b_idx = [1, 0, 3, 2, 5, 4, 7, 6, 2, 4, 6, 0, 3, 5, 7, 1]
    _check_against_emulation(net, sd, frames, a_idx, b_idx, 20, (0, 1, 9, 19), '288x512 x16')
