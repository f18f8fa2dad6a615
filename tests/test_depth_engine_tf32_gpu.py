"""The MiDaS engine (dvd_b200.depth_engine) against an fp64 emulation of its own precision model (oracle/midas_tf32.py): the
reference's structure, the engine's TF32 rounding points and the engine's packed weight images. What is left between the two is
fp32 accumulation order and the occasional one-step TF32 rounding flip, so the bounds below are orders of magnitude tighter than
the fp32-oracle comparison of test_depth_engine_gpu.py (2-4 % of TF32 noise per tensor) and a wiring error of a few per cent —
a dropped term, a wrong align_corners, a missing skip gradient or ReLU mask — fails.

The emulation is teacher-forced at every tensor the engine saves for its backward: each layer is checked on the engine's own
inputs, and ReLU masks / max-pool argmaxes come from the engine, so flips at zero or near-ties cannot accumulate.

Bounds: measured on an H100 SXM (80 GB, 700 W), set at about 3x the largest value observed over all cases below."""
import pytest
import torch

from conftest import grad_agreement, rel_err

pytestmark = pytest.mark.gpu

# forward, TF32-rounded anchors: share of elements that differ from the emulation, share that differ by more than one TF32
# step, and the max-norm error of the latter relative to the tensor's maximum. An element computed from anchored inputs can only
# be more than one step off where its value is a cancellation near zero (the fp32 accumulation error exceeds a TF32 step of the
# small result). CHAINED tensors also read the fusion path x2-up-sampled from the fusion output `o`, which the engine does not
# save: a one-step flip in `o` is rounded once more on the way, so their far elements are up to a couple of steps of `o` off.
#   observed maxima over the cases below: 2.8e-2 (lr3), 3.4e-3 (lr3), 1.4e-5 (lr3), fusion path 6.8e-4 (p1)
FWD_DIFF, FWD_FAR, FWD_FAR_REL, FWD_FAR_REL_CHAINED = 0.08, 1e-2, 4e-5, 2e-3
CHAINED = ('refinenet3.t', 'refinenet2.t', 'refinenet1.t', 'p1')
POOL_FLIPS = 1e-4       # max-pool argmax of the emulated window (first maximum) vs the engine's index; observed 0
# forward, unrounded tensors (down-sample branch outputs, h2, depth): max-norm relative to the tensor's maximum; observed 3.1e-6
UNROUNDED_REL = 1e-5
# backward, every parameter tensor: |slope - 1|, relative L2, max-norm relative to the tensor's maximum;
#   observed maxima 3.3e-4 (layer2.0.bn2.weight), 1.07e-3 (layer3.3.bn2.weight), 1.8e-3 (layer3.4.bn1.weight); at the working
#   sizes 3.2e-4 (1x384x224), 1.41e-3 (2x64x384), 2.3e-3 (2x32x384, layer3.0.bn1.weight)
GRAD_SLOPE, GRAD_L2, GRAD_MAX = 1e-3, 3e-3, 5e-3
# data-gradient images: share of elements one TF32 step away from tf32(W * gamma * rsqrt(var + eps)) where rsqrtf and
# torch.rsqrt differ; observed 0 of 8.7e7
PACK_BWD_DIFF = 1e-3


def _net():
    from dvd_b200 import synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    return synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True), 0, 2000.0).eval().cuda()


def _conv_names(net):
    return {id(m): n for n, m in net.named_modules() if isinstance(m, torch.nn.Conv2d)}


def _shape(c):
    w = c.conv.weight
    return w.shape[0], w.shape[1] * c.groups, w.shape[2], c.groups


def _images(eng, names):
    from oracle.midas_tf32 import unpack_image
    out = {}
    for c in eng._all:
        Co, Ci, k, g = _shape(c)
        out[names[id(c.conv)]] = (unpack_image(c.w_fwd, Co, Ci, k, g, 0).double(), unpack_image(c.w_bwd, Co, Ci, k, g, 1).double())
    return out


def _bits(t):
    return t.contiguous().view(torch.int32).long()


def test_pack_images_are_the_weights():
    """forward image == tf32(W) bit for bit; data-gradient image == tf32(fp32(W * gamma * rsqrt(var + eps))) up to one TF32 step
    where rsqrtf and torch.rsqrt differ; zero outside the groups of a grouped layer"""
    from oracle.midas_tf32 import off_group_entries, round_tf32, unpack_image
    net = _net()
    eng = net.engine()
    eng.pack(need_bwd=True)
    torch.cuda.synchronize()
    names = _conv_names(net)
    assert len(eng._all) == len(names) - 4      # all but the stem, the head and refinenet4's unused first RCU (2 convs)
    n_diff = n_tot = 0
    for c in eng._all:
        Co, Ci, k, g = _shape(c)
        w = c.conv.weight.detach()
        f, b = unpack_image(c.w_fwd, Co, Ci, k, g, 0), unpack_image(c.w_bwd, Co, Ci, k, g, 1)
        assert torch.equal(_bits(f), _bits(round_tf32(w))), names[id(c.conv)]
        for img, mode in ((c.w_fwd, 0), (c.w_bwd, 1)):
            assert float(off_group_entries(img, Co, Ci, g, mode).abs().max()) == 0.0, (names[id(c.conv)], mode)
        if c.bn is None:
            assert torch.equal(_bits(b), _bits(round_tf32(w))), names[id(c.conv)]
            continue
        want = round_tf32(w * (c.bn.weight.detach() * torch.rsqrt(c.bn.running_var + c.bn.eps)).view(-1, 1, 1, 1))
        d = (_bits(b) - _bits(want)).abs()
        assert bool(((d == 0) | (d == 0x2000)).all()), names[id(c.conv)]
        n_diff += int((d != 0).sum())
        n_tot += d.numel()
    print('data-gradient images: %d of %d elements one TF32 step off (%.2e)' % (n_diff, n_tot, n_diff / n_tot))
    assert n_diff <= PACK_BWD_DIFF * n_tot


def _cotangent(kind, N, H, W):
    g = torch.Generator().manual_seed(4)
    if kind == 'white':
        return (torch.randn(N, 1, H, W, generator=g) * 1e-3).cuda()
    yy = torch.linspace(0, 1, H).view(1, 1, H, 1)
    xx = torch.linspace(0, 1, W).view(1, 1, 1, W)
    ph = torch.rand(N, 1, 1, 1, generator=g) * 6.28
    return (1e-3 * (1 + 0.5 * torch.sin(9.0 * yy + ph) * torch.cos(7.0 * xx - ph))).cuda()


def capture_engine(net):
    """What the emulation is teacher-forced with, read after a training forward of `net` and before anything re-packs its weights:
    the engine's saved tensors as anchors (plus the down-sample branch outputs, which the engine recomputes rather than saves)
    and its packed weight images in weight layout."""
    from oracle.midas_tf32 import engine_anchors
    eng = net.engine()
    A = engine_anchors(eng.saved)
    bi = 0
    for st in eng.stages:
        for b in st:
            if b.ds is not None:
                A['block%d.ds' % bi] = b.ds.fwd(A['block%d.cur' % bi], round_out=False)
            bi += 1
    return A, _images(eng, _conv_names(net))


def check_engine_against_emulation(sd, x, depth, cot, A, images, grads, tag):
    """The emulation of the forward that produced `depth` from images `x` (state dict `sd`, anchors and images from
    capture_engine), its backward from the cotangent `cot`, against the engine: every anchor and the depth map, then every
    parameter gradient in `grads` (name -> the engine's .grad)."""
    from oracle.midas_tf32 import Anchors, anchor_names, midas_tf32_forward
    sd = {k: (v.detach().cuda().double().clone().requires_grad_() if (v.dtype.is_floating_point and 'running' not in k)
              else v.cuda().double()) for k, v in sd.items()}
    anc = Anchors(A)
    torch.cuda.reset_peak_memory_stats()
    d_emu = midas_tf32_forward(sd, x.double(), images=images, anchors=anc)
    (d_emu * cot.double()).sum().backward()
    torch.cuda.synchronize()
    print('\n[%s] emulation peak memory %.1f GB' % (tag, torch.cuda.max_memory_allocated() / 2 ** 30))

    # ---- forward
    rep = anc.report
    missing = [n for n in anchor_names() if n not in rep]
    assert not missing, missing
    rounded = {n: r for n, r in rep.items() if r.get('rounded')}
    unrounded = {n: r for n, r in rep.items() if 'rounded' in r and not r['rounded']}
    assert len(unrounded) == 5, sorted(unrounded)       # 4 down-sample branches + h2
    direct = {n: r for n, r in rounded.items() if n not in CHAINED}

    def worst(d, key):
        n, r = max(d.items(), key=lambda kv: kv[1][key])
        return '%.2e (%s)' % (r[key], n)
    e_depth = rel_err(depth, d_emu)
    print('forward: depth %.2e | unrounded %s | rounded: differ %s, beyond one step %s, their error %s, in the fusion path %s | '
          'max-pool argmax flips %.2e' % (e_depth, worst(unrounded, 'rel_max'), worst(rounded, 'diff'), worst(rounded, 'far'),
                                          worst(direct, 'far_rel_max'), worst({n: rounded[n] for n in CHAINED}, 'far_rel_max'),
                                          rep['pool_idx']['flips']))
    assert e_depth < UNROUNDED_REL, e_depth
    bad = [(n, r['rel_max']) for n, r in unrounded.items() if r['rel_max'] > UNROUNDED_REL]
    assert not bad, bad
    bad = [(n, r['diff'], r['far'], r['far_rel_max']) for n, r in rounded.items()
           if r['diff'] > FWD_DIFF or r['far'] > FWD_FAR or r['far_rel_max'] > (FWD_FAR_REL_CHAINED if n in CHAINED else FWD_FAR_REL)]
    assert not bad, bad
    assert rep['pool_idx']['flips'] <= POOL_FLIPS, rep['pool_idx']

    # ---- backward: every parameter tensor
    report = []
    for k, g in grads.items():
        ref = sd[k].grad
        if ref is None:         # refinenet4.resConfUnit1 is not part of the net's graph
            assert float(g.abs().max()) == 0.0, k
            continue
        report.append((k,) + grad_agreement(g, ref))
    assert len(report) == len(grads) - 4
    for i, what in ((1, '|slope - 1|'), (2, 'rel L2'), (3, 'max-norm')):
        top = sorted(report, key=lambda r: -abs(r[i]))[:3]
        print('backward %s: ' % what + ', '.join('%s %.2e' % (r[0], abs(r[i])) for r in top))
    bad = [r for r in report if abs(r[1]) > GRAD_SLOPE or r[2] > GRAD_L2 or r[3] > GRAD_MAX]
    assert not bad, bad
    return report


def _check_engine_against_emulation(N, H, W, kind):
    net = _net()
    eng = net.engine()
    x = torch.rand(N, 3, H, W, generator=torch.Generator().manual_seed(3)).cuda()
    cot = _cotangent(kind, N, H, W)
    for p in net.parameters():
        p.grad = None
    depth = eng.forward(x, train=True)
    A, images = capture_engine(net)
    eng.backward(cot)
    torch.cuda.synchronize()
    check_engine_against_emulation(net.state_dict(), x, depth, cot, A, images,
                                   {k: p.grad for k, p in net.named_parameters()}, '%dx%dx%d %s' % (N, H, W, kind))


# The working sizes the frame builders produce (frames.working_size, frames.get_im_size), with their layer4 grids: 16:9 and 4:3
# videos (6 x 12, 8 x 12), a portrait phone video (22 x 12: the tallest activations the engine runs, 3.1x the pixels of
# 224 x 384 per image), a square one (12 x 12), a very wide COLMAP video (2 x 12), a ShutterStock portrait (12 x 7), very wide /
# very tall ShutterStock frames (1 x 12 / 12 x 1: one-row and one-column grids) and small ones (1 x 1). The emulation needs about
# 2.2 GB per 224 x 384 image, in proportion to the pixels: the large sizes carry a timeout like the bench-resolution test.
_LARGE = pytest.mark.timeout(1200)
ENGINE_CASES = [
    pytest.param((2, 64, 96), 'smooth', id='shape0-smooth'),
    pytest.param((2, 64, 96), 'white', id='shape0-white'),
    pytest.param((1, 224, 384), 'smooth', id='shape1-smooth'),
    pytest.param((1, 224, 384), 'white', id='shape1-white'),
    pytest.param((2, 192, 384), 'white', id='2x192x384-white', marks=_LARGE),
    pytest.param((2, 256, 384), 'white', id='2x256x384-white', marks=_LARGE),
    pytest.param((1, 704, 384), 'white', id='1x704x384-white', marks=_LARGE),
    pytest.param((1, 384, 384), 'white', id='1x384x384-white', marks=_LARGE),
    pytest.param((2, 64, 384), 'white', id='2x64x384-white'),
    pytest.param((1, 384, 224), 'white', id='1x384x224-white', marks=_LARGE),
    pytest.param((1, 384, 224), 'smooth', id='1x384x224-smooth', marks=_LARGE),
    pytest.param((2, 32, 384), 'white', id='2x32x384-white'),
    pytest.param((2, 384, 32), 'white', id='2x384x32-white'),
    pytest.param((4, 32, 32), 'white', id='4x32x32-white'),
]


@pytest.mark.parametrize('shape, kind', ENGINE_CASES)
def test_saved_tensors_match_tf32_emulation(shape, kind, monkeypatch):
    monkeypatch.delenv('DVD_BWD_OVERLAP', raising=False)
    _check_engine_against_emulation(*shape, kind)


def test_one_stream_backward_matches_tf32_emulation(monkeypatch):
    monkeypatch.setenv('DVD_BWD_OVERLAP', '0')
    _check_engine_against_emulation(4, 64, 96, 'white')


@pytest.mark.timeout(1200)
def test_saved_tensors_match_tf32_emulation_at_bench_resolution(monkeypatch):
    """the bench resolution at a bench-like batch, so the layers run the tile shapes and schedules (stream-K among them) of a
    training step. 8 images rather than the bench's 16: the fp64 emulation with its autograd graph needs about 2.2 GB per image at 224 x 384 (17-19 GB at 8)."""
    monkeypatch.delenv('DVD_BWD_OVERLAP', raising=False)
    _check_engine_against_emulation(8, 224, 384, 'white')
