"""The depth-net kernels at the one-row, one-column and single-pixel grids that wide, tall and small working sizes give layer4
(32 x 384, 384 x 32 and 32 x 32 images), writing into an output that is a view inside a larger buffer.

A kernel that computes a padded tile (128 x 1 or 8 x 16 pixels for a 12-pixel grid, 128 pixels for one) must skip every pixel
row outside the tensor; one that does not writes into whatever lies next to its output, which a freshly allocated output never
shows. Here each output sits 256 KB (a multiple of 128 bytes, so the 16-byte alignment the kernels need still holds; more than
one 128 x 256 fp32 tile) into a buffer filled with a NaN bit pattern no kernel computes, and that much follows it. After the
launch every sentinel must be intact and the output must match torch in fp64. The check is exact at both ends: the first and
the last element of every output are written, so moving either end of the checked range by one element fails it.

Also here: MidasEngine.forward rejects an image size that is not a multiple of 32 before it launches anything."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from test_conv2d_gpu import TOL, cl, gen, make_bn, make_conv, tf32

pytestmark = pytest.mark.gpu

PAD = 65536                         # elements of sentinel on either side of an output
SENTINELS = {torch.float32: 0x7FBADBAD, torch.uint8: 0xA5}     # a signalling-NaN pattern; 165 is no max-pool window index


class Guarded:
    """`n` elements of `dtype` at offset PAD of a buffer of PAD + n + PAD sentinels"""

    def __init__(self, n, dtype=torch.float32):
        self.n = n
        self.sentinel = SENTINELS[dtype]
        self.bits = torch.full((PAD + n + PAD,), self.sentinel, dtype=torch.int32 if dtype == torch.float32 else dtype, device='cuda')
        self.out = self.bits.view(dtype)[PAD:PAD + n]
        assert self.out.data_ptr() % 128 == 0

    def nhwc(self, N, C, H, W):
        """the output as a channels-last [N,C,H,W] tensor"""
        return self.out.view(N, H, W, C).permute(0, 3, 1, 2)

    def _intact(self, lo, hi):
        return bool((self.bits[:lo] == self.sentinel).all()) and bool((self.bits[hi:] == self.sentinel).all())

    def check(self, what):
        torch.cuda.synchronize()
        lo, hi = PAD, PAD + self.n
        assert self._intact(lo, hi), '%s wrote outside its output' % what
        # the check is tight: the first and the last output element were written, so a range one element shorter at
        # either end sees them
        assert not self._intact(lo + 1, hi) and not self._intact(lo, hi - 1), '%s left an end of its output unwritten' % what


class GuardedAlloc:
    """stands in for conv_ops.empty_cl: every output a wrapper allocates lands inside a guarded buffer"""

    def __init__(self):
        self.guards = []

    def __call__(self, N, C, H, W, device):
        g = Guarded(N * C * H * W)
        self.guards.append(g)
        return g.nhwc(N, C, H, W)

    def check(self, what):
        assert self.guards, 'no output was allocated'
        for g in self.guards:
            g.check(what)


def _guarded_grads(params):
    """.grad of every parameter as a zeroed view inside a guarded buffer"""
    guards = []
    for p in params:
        if p is None:
            continue
        g = Guarded(p.numel())
        g.out.zero_()
        p.grad = g.out.view(p.shape)
        guards.append(g)
    return guards


def _ws_reset():
    """the stream-K exchange area, its partial tiles zeroed (flags are zero between launches)"""
    from dvd_b200 import conv_ops as co
    ws = co.conv_workspace(torch.device('cuda'))
    ws[256:].zero_()
    return ws


def _ws_after(ws, expect_sk):
    torch.cuda.synchronize()
    assert int((ws[:256].view(torch.int32) != 0).sum()) == 0        # every raised flag lowered again
    if expect_sk:
        assert float(ws[256:].abs().max()) > 0, 'this launch is expected to take the stream-K schedule'


# N, H, W (input), Cin, Cout, k, stride, groups, bn, bias, the passes that take the stream-K schedule with a workspace
CONV_CASES = [
    (2, 1, 12, 2048, 256, 3, 1, 1, False, True, ('fwd',)),     # layer4_rn, 1 x 12: 2 tiles of 576 K-steps over 8 CTAs
    (2, 12, 1, 2048, 256, 3, 1, 1, False, True, ('fwd',)),     # 12 x 1 (an 8 x 16 tile)
    (1, 1, 1, 2048, 256, 3, 1, 1, False, True, ('fwd',)),      # 1 x 1: one tile over 4 CTAs
    (1, 1, 1, 256, 2048, 3, 1, 1, False, True, ('dgrad',)),    # data gradient with 2048 input channels: one tile over 4 CTAs
    (2, 1, 12, 1024, 2048, 1, 1, 1, True, False, ()),          # 1x1 1024 -> 2048: one GEMM over 24 pixels
    (4, 1, 1, 1024, 2048, 1, 1, 1, True, False, ()),
    (2, 2, 24, 1024, 1024, 3, 2, 32, True, False, ()),         # grouped stride 2, 32 ch / group -> 1 x 12
    (2, 24, 2, 2048, 2048, 3, 2, 32, True, False, ()),         # layer4.0.conv2, 64 ch / group -> 12 x 1
    (4, 2, 2, 1024, 1024, 3, 2, 32, True, False, ()),          # -> 1 x 1
    (2, 2, 24, 1024, 2048, 1, 2, 1, True, False, ()),          # layer4.0.downsample -> 1 x 12
    (4, 2, 2, 1024, 2048, 1, 2, 1, True, False, ()),           # -> 1 x 1
]


def _layer(case, seed):
    N, H, W, ci, co_, k, stride, groups, use_bn, bias, _ = case
    conv = make_conv(ci, co_, k, stride, groups, bias, seed)
    bn = make_bn(co_, seed + 1) if use_bn else None
    OH, OW = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    return conv, bn, OH, OW


@pytest.mark.parametrize('stream_k', [True, False])
@pytest.mark.parametrize('case', CONV_CASES)
def test_conv_forward_writes_only_its_output(case, stream_k, monkeypatch):
    N, H, W, ci, co_, k, stride, groups, use_bn, bias, sk = case
    from dvd_b200 import conv_ops as co
    conv, bn, OH, OW = _layer(case, 4000 + ci + H)
    g = gen(4100 + ci + H)
    x = tf32(torch.randn(N, ci, H, W, generator=g))
    res = torch.randn(N, co_, OH, OW, generator=g)
    ref = F.conv2d(x.double(), tf32(conv.weight.detach()).double(), conv.bias.double() if bias else None, stride=stride,
                   padding=k // 2, groups=groups)
    if bn is not None:
        ref = F.batch_norm(ref, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(), bn.bias.double(), False, 0.0, bn.eps)
    ref = (ref + res.double()).relu()
    c = co.Conv(conv.cuda(), bn.cuda() if bn is not None else None)
    c.pack(need_bwd=False)
    ws = _ws_reset()
    alloc = GuardedAlloc()
    with monkeypatch.context() as m:
        m.setattr(co, 'empty_cl', alloc)
        if not stream_k:
            m.setattr(co, 'conv_workspace', lambda device: None)
        y = c.fwd(cl(x), res=cl(res), relu=True, round_out=False)
    alloc.check('forward')
    _ws_after(ws, stream_k and 'fwd' in sk)
    assert rel_err(y, ref) < TOL


@pytest.mark.parametrize('stream_k', [True, False])
@pytest.mark.parametrize('case', CONV_CASES)
def test_conv_data_gradient_writes_only_its_output(case, stream_k, monkeypatch):
    N, H, W, ci, co_, k, stride, groups, use_bn, bias, sk = case
    from dvd_b200 import conv_ops as co
    conv, bn, OH, OW = _layer(case, 5000 + ci + H)
    from oracle.midas_tf32 import unpack_image
    gy = tf32(torch.randn(N, co_, OH, OW, generator=gen(5100 + ci + H)))
    c = co.Conv(conv.cuda(), bn.cuda() if bn is not None else None)
    c.pack()
    # the weights of the kernel's own data-gradient image (BatchNorm scale folded in with rsqrtf, then rounded; held to
    # tf32(W * gamma * rsqrt(var + eps)) by test_depth_engine_tf32_gpu), so that only the fp32 summation order is left
    w = unpack_image(c.w_bwd, co_, ci, k, groups, 1).double().cpu()
    ref = torch.nn.grad.conv2d_input((N, ci, H, W), w, gy.double(), stride=stride, padding=k // 2, groups=groups)
    ws = _ws_reset()
    alloc = GuardedAlloc()
    with monkeypatch.context() as m:
        m.setattr(co, 'empty_cl', alloc)
        if not stream_k:
            m.setattr(co, 'conv_workspace', lambda device: None)
        gx = c.dgrad(cl(gy), H, W, round_out=False)
    alloc.check('data gradient')
    _ws_after(ws, stream_k and 'dgrad' in sk)
    assert rel_err(gx, ref) < TOL


@pytest.mark.parametrize('ordered', [False, True])
@pytest.mark.parametrize('case', CONV_CASES)
def test_conv_weight_gradient_writes_only_its_output(case, ordered):
    """split-K partial sums added with atomics, or (deterministic mode) through a workspace in a fixed order; the weight, bias
    and BatchNorm gradients all accumulate into views inside guarded buffers"""
    from dvd_b200 import ops
    N, H, W, ci, co_, k, stride, groups, use_bn, bias, _ = case
    from dvd_b200 import conv_ops as co
    conv, bn, OH, OW = _layer(case, 6000 + ci + H)
    g = gen(6100 + ci + H)
    x = tf32(torch.randn(N, ci, H, W, generator=g))
    gm = tf32(torch.randn(N, co_, OH, OW, generator=g))
    ref = torch.nn.grad.conv2d_weight(x.double(), conv.weight.shape, gm.double(), stride=stride, padding=k // 2, groups=groups)
    ref_sum = gm.double().sum(dim=(0, 2, 3))
    if bn is not None:
        rstd = torch.rsqrt(bn.running_var.double() + bn.eps)
        ref_dgamma = ((ref * conv.weight.detach().double()).sum(dim=(1, 2, 3)) - bn.running_mean.double() * ref_sum) * rstd
        ref = ref * (bn.weight.detach().double() * rstd).view(-1, 1, 1, 1)
    conv, bn = conv.cuda(), (bn.cuda() if bn is not None else None)
    params = [conv.weight, conv.bias] + ([bn.weight, bn.bias] if bn is not None else [])
    guards = _guarded_grads(params)
    with ops.ordered_reductions(ordered):
        co.Conv(conv, bn).wgrad(cl(x), cl(gm), sums=True)
    for gd in guards:
        gd.check('weight gradient')
    assert rel_err(conv.weight.grad, ref) < TOL
    if bias:
        assert rel_err(conv.bias.grad, ref_sum) < 2e-5
    if bn is not None:
        assert rel_err(bn.weight.grad, ref_dgamma) < 5e-5
        assert rel_err(bn.bias.grad, ref_sum) < 2e-5


@pytest.mark.parametrize('align', [True, False])
@pytest.mark.parametrize('hw', [(12, 1), (1, 12), (1, 1)])
def test_upsample_writes_only_its_output(hw, align, monkeypatch):
    """x2 bilinear up-sampling from a one-column, one-row and single-pixel input (the decoder path from layer4_rn) and its
    adjoint, against torch in fp64"""
    from dvd_b200 import conv_ops as co
    H, W = hw
    N, C = 2, 256
    g0 = gen(12)
    x = torch.randn(N, C, H, W, generator=g0)
    gy = torch.randn(N, C, 2 * H, 2 * W, generator=g0)
    xd = x.double().requires_grad_()
    ref = F.interpolate(xd, scale_factor=2, mode='bilinear', align_corners=align)
    ref.backward(gy.double())
    alloc = GuardedAlloc()
    with monkeypatch.context() as m:
        m.setattr(co, 'empty_cl', alloc)
        y = co.upsample2x_fwd(cl(x), align, round_out=False)
        gx = co.upsample2x_bwd(cl(gy), align, round_out=False)
    alloc.check('upsample2x')
    assert rel_err(y, ref) < 1e-6
    assert rel_err(gx, xd.grad) < 1e-6


@pytest.mark.parametrize('hw', [(2, 2), (2, 1), (1, 2)])
def test_maxpool_writes_only_its_output(hw, monkeypatch):
    """3x3 stride-2 max-pool of a 2 x 2 / 2 x 1 / 1 x 2 input: one output pixel whose window is mostly padding; ReLU'd input,
    so exact zeros tie and the first maximum must win"""
    from dvd_b200 import _lib
    from dvd_b200 import conv_ops as co
    from dvd_b200.ops import _ptr, _stream
    H, W = hw
    N, C = 3, 64
    g0 = gen(13)
    x = torch.randn(N, C, H, W, generator=g0).relu()
    x[0, :8] = 0.0                                                  # whole windows of zeros
    xd = x.double().requires_grad_()
    ref = F.max_pool2d(xd, 3, 2, 1)
    gy = torch.randn(ref.shape, generator=g0)
    ref.backward(gy.double())
    OH, OW = ref.shape[2], ref.shape[3]
    yg, ig = Guarded(N * C * OH * OW), Guarded(N * OH * OW * C, torch.uint8)
    y, idx = yg.nhwc(N, C, OH, OW), ig.out.view(N, OH, OW, C)
    _lib.check(_lib.load().dvd_maxpool3x3s2_fwd(_ptr(cl(x)), _ptr(y), _ptr(idx), N, H, W, C, _stream()), 'dvd_maxpool3x3s2_fwd')
    yg.check('max-pool forward')
    ig.check('max-pool forward (indices)')
    assert torch.equal(y.cpu().double(), ref.detach())
    alloc = GuardedAlloc()
    with monkeypatch.context() as m:
        m.setattr(co, 'empty_cl', alloc)
        gx = co.maxpool_bwd(cl(gy), idx, H, W)
    alloc.check('max-pool backward')
    assert rel_err(gx, xd.grad) < 1e-6


def test_stem_writes_only_its_output(monkeypatch):
    """the stem of a 32 x 32 image (16 x 16 output) and its weight gradient, every gradient inside a guarded buffer"""
    from dvd_b200 import conv_ops as co
    N, H, W = 2, 32, 32
    g0 = gen(14)
    x = torch.rand(N, 3, H, W, generator=g0)
    conv = make_conv(3, 64, 7, 2, 1, False, 15)
    conv.padding = (3, 3)
    bn = make_bn(64, 16)
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    xd = ((x.double() - torch.tensor(mean).view(1, 3, 1, 1)) / torch.tensor(std).double().view(1, 3, 1, 1)).requires_grad_()
    wd = conv.weight.detach().double().requires_grad_()
    gd, bd = bn.weight.detach().double().requires_grad_(), bn.bias.detach().double().requires_grad_()
    ref = F.batch_norm(F.conv2d(xd, wd, None, 2, 3), bn.running_mean.double(), bn.running_var.double(), gd, bd, False, 0.0, bn.eps).relu()
    gy = torch.randn(ref.shape, generator=g0)
    ref.backward(gy.double())
    conv, bn = conv.cuda(), bn.cuda()
    alloc = GuardedAlloc()
    with monkeypatch.context() as m:
        m.setattr(co, 'empty_cl', alloc)
        y = co.stem_fwd(x.cuda(), conv, bn, mean, std, round_out=False)
    alloc.check('stem forward')
    assert rel_err(y, ref) < 1e-5
    guards = _guarded_grads([conv.weight, bn.weight, bn.bias])
    co.stem_wgrad(x.cuda(), cl(gy), y, conv, bn, mean, std)
    for g in guards:
        g.check('stem weight gradient')
    assert rel_err(conv.weight.grad, wd.grad) < 2e-5
    assert rel_err(bn.weight.grad, gd.grad) < 2e-5
    assert rel_err(bn.bias.grad, bd.grad) < 2e-5


# the clamp of the head in the reference's fp32: max(relu(o), 1e-2) with 1e-2 the fp32 number nearest to it
CLAMP = float(np.float32(1e-2))


def test_head_at_and_around_its_clamp():
    """depth = 10000 / max(relu(o), 1e-2) and its gradient with pre-activations o below 0, in [0, 1e-2), exactly at the fp32
    1e-2 (the clamp passes the gradient there: torch.clamp's backward takes self >= min) and above. Planted pixels hold one
    non-zero channel on a unit weight and a zero bias, so o is exact in fp32 and fp64 alike."""
    from dvd_b200 import _lib
    from dvd_b200.ops import _ptr, _stream
    N, H, W = 2, 16, 8
    P = N * H * W
    g0 = gen(17)
    xn = torch.randn(N, H, W, 32, generator=g0).relu()
    w = torch.randn(32, generator=g0) * 0.5
    w[0] = 1.0
    b = torch.zeros(1)
    planted = [CLAMP, CLAMP, float(np.nextafter(np.float32(CLAMP), np.float32(1))), float(np.nextafter(np.float32(CLAMP), np.float32(0))),
               5e-3, 1e-4, 0.0, 0.25]
    flat = xn.view(P, 32)
    # random pixels whose pre-activation lies in (5e-3, 0.1) are zeroed: near the clamp 1 / o^2 turns the fp32 rounding of a
    # cancelling 32-term sum into gradient errors of 1e-5 of the largest term
    o32 = flat @ w
    flat[(o32 > 5e-3) & (o32 < 0.1)] = 0.0
    for i, v in enumerate(planted):
        flat[7 * i] = 0.0
        flat[7 * i, 0] = v
    x = xn.permute(0, 3, 1, 2)                                      # channels-last [N,32,H,W]
    xd = x.double().requires_grad_()
    wd, bd = w.double().view(1, 32, 1, 1).requires_grad_(), b.double().requires_grad_()
    o = F.conv2d(xd, wd, bd)
    ref = 10000.0 / torch.clamp(o.relu(), min=CLAMP)
    gy = torch.randn(ref.shape, generator=g0)
    ref.backward(gy.double())
    o = o.detach().view(P)
    cats = {'below 0': o < 0, 'in [0, 1e-2)': (o >= 0) & (o < CLAMP), 'at 1e-2': o == CLAMP, 'above': o > CLAMP}
    assert all(int(m.sum()) >= 2 for m in cats.values()), {k: int(m.sum()) for k, m in cats.items()}

    dg = Guarded(P)
    depth = dg.out.view(N, 1, H, W)
    xc, wc, bc = cl(x), w.cuda(), b.cuda()
    _lib.check(_lib.load().dvd_head_fwd(_ptr(xc), _ptr(wc), _ptr(bc), _ptr(depth), P, _stream()), 'dvd_head_fwd')
    dg.check('head forward')
    assert rel_err(depth, ref) < 1e-5
    got, want = depth.detach().view(P).cpu().double(), ref.detach().view(P)
    pl = torch.tensor([7 * i for i in range(len(planted))])
    assert float(((got[pl] - want[pl]) / want[pl]).abs().max()) < 1e-6       # exact pre-activations: one fp32 division
    assert bool((got[o < CLAMP] == 1e6).all())

    gxg, gwg, gbg = Guarded(P * 32), Guarded(32), Guarded(1)
    gwg.out.zero_()
    gbg.out.zero_()
    gx = gxg.nhwc(N, 32, H, W)
    _lib.check(_lib.load().dvd_head_bwd(_ptr(xc), _ptr(wc), _ptr(bc), _ptr(gy.cuda()), _ptr(gx), _ptr(gwg.out), _ptr(gbg.out), P, 1, 0,
                                        _stream()), 'dvd_head_bwd')
    for gd, what in ((gxg, 'input'), (gwg, 'weight'), (gbg, 'bias')):
        gd.check('head backward (%s gradient)' % what)
    ref_gx = xd.grad * (x > 0)
    assert rel_err(gx, ref_gx) < 1e-5
    gxp = gx.detach().permute(0, 2, 3, 1).reshape(P, 32).cpu().double()
    rxp = ref_gx.permute(0, 2, 3, 1).reshape(P, 32)
    assert bool((gxp[o < CLAMP] == 0).all())                        # no gradient through the clamp or the ReLU
    at = cats['at 1e-2']
    assert float((gxp[at] - rxp[at]).abs().max() / rxp[at].abs().max()) < 1e-6
    assert rel_err(gwg.out, wd.grad.view(32)) < 1e-5 and rel_err(gbg.out, bd.grad) < 1e-5


def _engine_net():
    from dvd_b200 import synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    return synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True), 0, 2000.0).eval().cuda()


@pytest.mark.parametrize('shape', [(1, 100, 100), (1, 224, 370), (2, 48, 64), (1, 384, 16), (0, 32, 32)])
def test_engine_rejects_sizes_it_cannot_run(shape):
    """a size that is not a positive multiple of 32 is refused before the first launch: at 100 x 100 the up-sampled decoder path
    (8 x 8) would meet a 7 x 7 layer3_rn, which the convolution epilogue would read with the strides of its output"""
    from dvd_b200 import ops
    net = _engine_net()
    eng = net.engine()
    x = torch.rand(*shape[:1], 3, *shape[1:], device='cuda')
    n0 = ops.LAUNCHES['n']
    for train in (False, True):
        with pytest.raises(ValueError, match='multiples of 32'):
            eng.forward(x, train=train)
    with pytest.raises(ValueError, match='multiples of 32'):
        net(x)
    assert ops.LAUNCHES['n'] == n0
    # the smallest size it runs
    d = eng.forward(torch.rand(1, 3, 32, 32, device='cuda'), train=False)
    assert d.shape == (1, 1, 32, 32) and bool(torch.isfinite(d).all())
    assert ops.LAUNCHES['n'] > n0
