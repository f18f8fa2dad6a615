"""GPU parity of the general tensor-core convolution family (csrc/conv2d_tc.cu through the C ABI) and the CUDA-core depth-net
kernels (csrc/depth_ops.cu) against torch in fp64 on the same inputs.

Operands are rounded to TF32 on the host first (bit-exact emulation of cvt.rna, itself checked against dvd_round_tf32), the
weights through the same rounding the pack kernel applies, so that the only difference left is fp32 accumulation order:
the tolerances are 2e-5 of the tensor's maximum instead of the 1e-3 a TF32 comparison would need."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 2e-5


def tf32(t):
    """round-to-nearest (ties away) TF32, bit-exact emulation of cvt.rna.tf32.f32"""
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def gen(seed):
    return torch.Generator().manual_seed(seed)


def test_round_kernel_is_bit_exact():
    from dvd_b200 import conv_ops as co
    x = torch.randn(1, 64, 33, 17, generator=gen(0)) * 7.3
    y = co.round_tf32(x.cuda())
    assert torch.equal(y.cpu().view(torch.int32), tf32(x).view(torch.int32))


def make_conv(ci, co_, k, stride, groups, bias, seed):
    g = gen(seed)
    conv = torch.nn.Conv2d(ci, co_, k, stride=stride, padding=k // 2, groups=groups, bias=bias)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) / (ci // groups * k * k) ** 0.5)
        if bias:
            conv.bias.copy_(torch.randn(co_, generator=g))
    return conv


def make_bn(c, seed):
    g = gen(seed)
    bn = torch.nn.BatchNorm2d(c).eval()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(c, generator=g))
        bn.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn


FWD_CASES = [
    # N, H,  W,  Cin,  Cout, k, stride, groups, bn, bias, res, res2, relu, mask
    (2, 28, 48, 256, 512, 1, 1, 1, True, False, True, False, True, False),     # conv3 + bn3 + identity + relu
    (1, 56, 96, 64, 256, 1, 1, 1, True, False, False, False, False, False),    # layer1 downsample
    (3, 7, 12, 2048, 256, 1, 1, 1, False, False, False, False, False, False),  # ragged pixel count, K = 2048
    (2, 56, 96, 256, 256, 3, 1, 1, False, True, True, True, True, False),      # RCU conv2: bias + two residuals + relu
    (1, 28, 48, 256, 256, 3, 1, 1, False, True, False, False, True, True),     # with a mask
    (2, 14, 24, 512, 256, 3, 1, 1, False, False, False, False, True, False),   # layer2_rn + fused relu, ragged H
    (1, 112, 192, 256, 128, 3, 1, 1, False, True, False, False, False, False),  # head conv, Cout = 128
    (1, 30, 50, 128, 32, 3, 1, 1, False, True, False, False, True, False),     # ragged W, Cout = 32
    (1, 9, 13, 32, 16, 3, 1, 1, False, False, True, False, False, False),      # Cout = 16: direct-store epilogue
    (2, 56, 96, 256, 512, 1, 2, 1, True, False, False, False, False, False),   # downsample stride 2
    (1, 15, 25, 64, 128, 1, 2, 1, True, False, False, False, False, False),    # stride 2, odd sizes
    (2, 56, 96, 256, 256, 3, 1, 32, True, False, False, False, True, False),   # grouped, 8 ch / group
    (1, 28, 48, 512, 512, 3, 1, 32, True, False, False, False, True, False),   # 16 ch / group
    (2, 14, 24, 1024, 1024, 3, 1, 32, True, False, False, False, True, False),  # 32 ch / group
    (1, 7, 12, 2048, 2048, 3, 1, 32, True, False, False, False, True, False),  # 64 ch / group
    (2, 56, 96, 512, 512, 3, 2, 32, True, False, False, False, True, False),   # grouped + stride 2 (layer2.0.conv2)
    (1, 27, 45, 256, 256, 3, 2, 32, True, False, False, False, True, False),   # grouped + stride 2, odd sizes
    (16, 14, 24, 1024, 1024, 1, 1, 1, True, False, True, False, True, False),  # layer3 1x1 at the bench batch: 84 pair tiles on 74 pairs
    (16, 7, 12, 2048, 256, 3, 1, 1, False, True, False, False, True, False),   # layer4_rn at the bench batch: 6 pair tiles, 576 K-steps -> stream-K
    (16, 14, 24, 1024, 256, 3, 1, 1, False, True, True, True, True, False),    # layer3_rn class: 24 pair tiles, 288 K-steps -> stream-K, + residuals
    (2, 14, 24, 256, 256, 3, 1, 1, False, True, True, True, True, False),      # few tiles, 72 K-steps: tiles split four ways
    (1, 20, 36, 64, 64, 5, 1, 1, False, True, False, False, True, False),      # 5x5 (hourglass class): 25 taps
    (1, 24, 40, 32, 32, 11, 1, 1, False, True, False, False, True, False),     # 11x11: 121 taps
    # layer4 of the working sizes with a one-row, one-column or single-pixel layer4 grid (32 x 384, 384 x 32, 32 x 32 images):
    # a 128 x 1 or 8 x 16 pixel tile (TMA box wider or taller than the tensor) of which the epilogue keeps 12 pixels, or 1
    (2, 1, 12, 2048, 256, 3, 1, 1, False, True, False, False, True, False),    # layer4_rn, 1 x 12
    (2, 12, 1, 2048, 256, 3, 1, 1, False, True, False, False, True, False),    # layer4_rn, 12 x 1
    (4, 1, 1, 2048, 256, 3, 1, 1, False, True, False, False, True, False),     # layer4_rn, 1 x 1
    (2, 1, 12, 1024, 2048, 1, 1, 1, True, False, True, False, True, False),    # 1x1 1024 -> 2048 (one GEMM over 24 pixels)
    (2, 12, 1, 1024, 2048, 1, 1, 1, True, False, True, False, True, False),
    (4, 1, 1, 1024, 2048, 1, 1, 1, True, False, True, False, True, False),     # 4 pixels
    (2, 2, 24, 1024, 1024, 3, 2, 32, True, False, False, False, True, False),  # grouped stride 2, 32 ch / group -> 1 x 12
    (2, 24, 2, 1024, 1024, 3, 2, 32, True, False, False, False, True, False),  # -> 12 x 1
    (4, 2, 2, 1024, 1024, 3, 2, 32, True, False, False, False, True, False),   # -> 1 x 1
    (2, 2, 24, 2048, 2048, 3, 2, 32, True, False, False, False, True, False),  # layer4.0.conv2 (64 ch / group) -> 1 x 12
    (2, 24, 2, 2048, 2048, 3, 2, 32, True, False, False, False, True, False),  # -> 12 x 1
    (4, 2, 2, 2048, 2048, 3, 2, 32, True, False, False, False, True, False),   # -> 1 x 1
    (2, 2, 24, 1024, 2048, 1, 2, 1, True, False, False, False, False, False),  # layer4.0.downsample, 1x1 stride 2 -> 1 x 12
    (2, 24, 2, 1024, 2048, 1, 2, 1, True, False, False, False, False, False),  # -> 12 x 1
    (4, 2, 2, 1024, 2048, 1, 2, 1, True, False, False, False, False, False),   # -> 1 x 1
    (1, 1, 1, 2048, 256, 3, 1, 1, False, True, True, True, True, False),       # one tile of one pixel, 576 K-steps: stream-K over 4 CTAs
]


@pytest.mark.parametrize('case', FWD_CASES)
def test_conv_forward_matches_torch_fp64(case):
    from dvd_b200 import conv_ops as co
    N, H, W, ci, co_, k, stride, groups, use_bn, bias, has_res, has_res2, relu, has_mask = case
    seed = 1000 * k + ci + co_ + H + 7 * stride + groups
    g = gen(seed)
    conv = make_conv(ci, co_, k, stride, groups, bias, seed + 1)
    bn = make_bn(co_, seed + 2) if use_bn else None
    x = tf32(torch.randn(N, ci, H, W, generator=g))
    OH, OW = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    res = torch.randn(N, co_, OH, OW, generator=g) if has_res else None
    res2 = torch.randn(N, co_, OH, OW, generator=g) if has_res2 else None
    mask = torch.randn(N, co_, OH, OW, generator=g) if has_mask else None
    ref = F.conv2d(x.double(), tf32(conv.weight.detach()).double(), conv.bias.double() if bias else None, stride=stride,
                   padding=k // 2, groups=groups)
    if bn is not None:
        ref = F.batch_norm(ref, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(), bn.bias.double(), False, 0.0, bn.eps)
    for r in (res, res2):
        if r is not None:
            ref = ref + r.double()
    if relu:
        ref = ref.relu()
    if mask is not None:
        ref = ref * (mask > 0)
    conv, bn = conv.cuda(), (bn.cuda() if bn is not None else None)
    c = co.Conv(conv, bn)
    c.pack(need_bwd=False)
    y = c.fwd(cl(x), res=cl(res) if has_res else None, res2=cl(res2) if has_res2 else None, relu=relu, round_out=False) \
        if not has_mask else None
    if has_mask:
        d = co.make_desc(N, H, W, ci, OH, OW, co_, co.fwd_taps(k, k // 2), stride, c.kblock, relu=relu, round_out=False)
        y = co.conv2d_launch(d, cl(x), c.w_fwd, co.empty_cl(N, co_, OH, OW, 'cuda'), conv.bias, None, None, None, cl(mask),
                             workspace=co.conv_workspace(torch.device('cuda')))
    assert y.shape == ref.shape and y.is_contiguous(memory_format=torch.channels_last)
    e = rel_err(y, ref)
    assert e < TOL, e
    # rounded output is the RN rounding of the exact one
    if not has_mask:
        y2 = c.fwd(cl(x), res=cl(res) if has_res else None, res2=cl(res2) if has_res2 else None, relu=relu, round_out=True)
        assert torch.equal(y2, co.round_tf32(y))


def test_stream_k_matches_a_launch_without_workspace_and_leaves_flags_clear():
    """Same launch with and without the stream-K schedule (no exchange area = whole tiles): equal up to fp32 summation order;
    the flag words of the exchange area are back to zero afterwards (the next launch relies on it); launches of OTHER shapes in
    between (other tile widths, cluster counts) must not disturb it (stale lines of the exchange area in an SM's L1 did, once)."""
    from dvd_b200 import conv_ops as co
    g = gen(77)

    def layer(ci, co_, k, N, H, W, seed):
        conv = make_conv(ci, co_, k, 1, 1, True, seed).cuda()
        c = co.Conv(conv, None)
        c.pack(need_bwd=False)
        return c, cl(tf32(torch.randn(N, ci, H, W, generator=g)))

    layers = [layer(2048, 256, 3, 16, 7, 12, 78), layer(1024, 256, 3, 16, 14, 24, 79), layer(64, 64, 5, 1, 20, 36, 80),
              layer(512, 256, 3, 2, 14, 24, 81)]
    ws = co.conv_workspace(layers[0][1].device)
    assert ws is not None
    ws[256:].zero_()
    ref = []
    for c, x in layers:
        N, _, H, W = x.shape
        OH, OW = c.out_hw(H, W)
        d = co.make_desc(N, H, W, c.cin, OH, OW, c.cout, co.fwd_taps(c.k, c.pad), relu=True, round_out=False)
        ref.append(co.conv2d_launch(d, x, c.w_fwd, co.empty_cl(N, c.cout, OH, OW, 'cuda'), c.conv.bias, workspace=None))
    torch.cuda.synchronize()
    assert float(ws[256:].abs().max()) == 0.0
    first = None
    for rep in range(3):
        outs = [c.fwd(x, relu=True, round_out=False) for c, x in layers]
        torch.cuda.synchronize()
        assert int((ws[:256].view(torch.int32) != 0).sum()) == 0
        for y, r in zip(outs, ref):
            assert rel_err(y, r) < 4 * TOL       # two fp32 summation orders of up to 18 432 products against each other
        if first is None:
            first = outs
        else:
            assert all(torch.equal(a, b) for a, b in zip(outs, first))      # the schedule is deterministic
    assert float(ws[256:].abs().max()) > 0, 'these shapes are expected to take the stream-K schedule'


@pytest.mark.parametrize('nt', [160, 192, 224, 128])
def test_ragged_channel_tiles_match_torch_fp64(nt):
    """Cout = 1024 with channel tiles of `nt` (DVD_CONV_NT): the last tile is ragged in whole 32-channel blocks - its weight rows
    beyond Cout are zero-filled by the TMA unit and its epilogue skips them (BatchNorm + residual + ReLU + mask all indexed there)."""
    import os
    from dvd_b200 import conv_ops as co
    g = gen(300 + nt)
    N, H, W, ci, co_ = 3, 14, 24, 512, 1024
    conv = make_conv(ci, co_, 1, 1, 1, False, 301)
    bn = make_bn(co_, 302)
    x = tf32(torch.randn(N, ci, H, W, generator=g))
    res = torch.randn(N, co_, H, W, generator=g)
    mask = torch.randn(N, co_, H, W, generator=g)
    ref = F.conv2d(x.double(), tf32(conv.weight.detach()).double())
    ref = F.batch_norm(ref, bn.running_mean.double(), bn.running_var.double(), bn.weight.double(), bn.bias.double(), False, 0.0, bn.eps)
    ref = (ref + res.double()).relu() * (mask > 0)
    conv, bn = conv.cuda(), bn.cuda()
    c = co.Conv(conv, bn)
    c.pack(need_bwd=False)
    d = co.make_desc(N, H, W, ci, H, W, co_, co.fwd_taps(1, 0), 1, 0, relu=True, round_out=False, bn_eps=bn.eps)
    os.environ['DVD_CONV_NT'] = str(nt)
    try:
        y = co.conv2d_launch(d, cl(x), c.w_fwd, torch.full((N, co_, H, W), float('nan'), device='cuda').contiguous(memory_format=torch.channels_last),
                             None, c._bn_fwd(), cl(res), None, cl(mask))
    finally:
        del os.environ['DVD_CONV_NT']
    assert rel_err(y, ref) < TOL


@pytest.mark.parametrize('case', [(2, 30, 50, 128, 32, 3, 1), (1, 28, 48, 512, 512, 3, 32), (2, 20, 36, 64, 64, 5, 1), (1, 24, 40, 32, 32, 11, 1),
                                  (2, 56, 96, 256, 256, 3, 1)])
def test_wide_and_grouped_stencils_match_torch_fp64(case):
    """Wide, grouped and asymmetric-shape stencils (3x3 to 11x11, few or many output channels) with bias, residual and ReLU
    against torch fp64."""
    from dvd_b200 import conv_ops as co
    N, H, W, ci, co_, k, groups = case
    g = gen(500 + k + ci)
    conv = make_conv(ci, co_, k, 1, groups, True, 501 + k)
    x = tf32(torch.randn(N, ci, H, W, generator=g))
    res = torch.randn(N, co_, H, W, generator=g)
    ref = (F.conv2d(x.double(), tf32(conv.weight.detach()).double(), conv.bias.double(), padding=k // 2, groups=groups) + res.double()).relu()
    conv = conv.cuda()
    c = co.Conv(conv, None)
    c.pack(need_bwd=False)
    y = c.fwd(cl(x), res=cl(res), relu=True, round_out=False)
    assert rel_err(y, ref) < TOL


def test_batched_pack_is_bit_identical_to_single_layer_pack():
    """dvd_conv2d_pack_batch (one launch for a whole net: 32 x 32 transposed tiles, device-resident table) writes exactly the images
    dvd_conv2d_pack writes layer by layer: dense 1x1 / 3x3 with and without BatchNorm, Cin != Cout, grouped with 8 / 32 / 64
    channels per group."""
    from dvd_b200 import conv_ops as co
    specs = [(256, 512, 1, 1, True), (512, 256, 3, 1, False), (128, 32, 3, 1, False), (256, 256, 3, 32, True), (1024, 1024, 3, 32, True),
             (2048, 2048, 3, 32, True), (64, 256, 1, 1, True)]
    convs = []
    for i, (ci, co_, k, g, use_bn) in enumerate(specs):
        conv = make_conv(ci, co_, k, 1, g, not use_bn, 900 + i).cuda()
        bn = make_bn(co_, 950 + i).cuda() if use_bn else None
        # the flat parameter buffers of the engine hold convolution weights channels-last: same strides here
        conv.weight.data = conv.weight.data.contiguous(memory_format=torch.channels_last)
        convs.append(co.Conv(conv, bn))
    ref = []
    for c in convs:
        c.pack()
        ref.append((c.w_fwd.clone(), c.w_bwd.clone()))
        c.w_fwd.fill_(float('nan'))
        c.w_bwd.fill_(float('nan'))
    table = co.PackTable(convs)
    table.pack(need_bwd=True)
    torch.cuda.synchronize()
    for c, (f, b) in zip(convs, ref):
        assert torch.equal(c.w_fwd, f) and torch.equal(c.w_bwd, b)
    # forward images only (evaluation): the data-gradient images are left alone
    for c in convs:
        c.w_fwd.fill_(0.0)
        c.w_bwd.fill_(7.0)
    table.pack(need_bwd=False)
    torch.cuda.synchronize()
    for c, (f, b) in zip(convs, ref):
        assert torch.equal(c.w_fwd, f) and bool((c.w_bwd == 7.0).all())


DGRAD_CASES = [
    # N, H,  W,  Cin,  Cout, k, stride, groups, bn, res, mask
    (2, 28, 48, 64, 128, 3, 1, 1, False, True, True),
    (1, 56, 96, 256, 256, 1, 1, 1, True, True, True),
    (1, 28, 48, 128, 32, 3, 1, 1, False, False, False),      # head conv 128 -> 32: launch has Cin 32
    (2, 56, 96, 256, 512, 1, 2, 1, True, False, False),      # downsample stride 2: zero fill + one phase
    (1, 15, 25, 64, 128, 1, 2, 1, True, False, False),
    (2, 28, 48, 256, 256, 3, 1, 32, True, False, True),      # grouped
    (1, 14, 24, 2048, 2048, 3, 1, 32, True, False, True),
    (2, 56, 96, 512, 512, 3, 2, 32, True, False, True),      # grouped stride 2: four sub-pixel phases + mask
    (1, 27, 45, 256, 256, 3, 2, 32, True, True, False),      # odd sizes + residual
    (1, 20, 36, 64, 64, 7, 1, 1, False, False, False),       # 7x7
    # layer4 classes at the one-row, one-column and single-pixel grids (see FWD_CASES)
    (2, 1, 12, 2048, 256, 3, 1, 1, False, True, True),       # layer4_rn
    (2, 12, 1, 2048, 256, 3, 1, 1, False, True, True),
    (4, 1, 1, 2048, 256, 3, 1, 1, False, True, True),
    (2, 1, 12, 1024, 2048, 1, 1, 1, True, True, True),       # 1x1 1024 -> 2048
    (4, 1, 1, 1024, 2048, 1, 1, 1, True, True, True),
    (2, 2, 24, 1024, 1024, 3, 2, 32, True, False, True),     # grouped stride 2, 32 ch / group: 1 x 12 -> 2 x 24
    (2, 24, 2, 1024, 1024, 3, 2, 32, True, True, False),     # 12 x 1 -> 24 x 2
    (4, 2, 2, 1024, 1024, 3, 2, 32, True, False, True),      # 1 x 1 -> 2 x 2
    (2, 2, 24, 2048, 2048, 3, 2, 32, True, False, True),     # 64 ch / group
    (4, 2, 2, 2048, 2048, 3, 2, 32, True, True, False),
    (2, 2, 24, 1024, 2048, 1, 2, 1, True, False, False),     # 1x1 stride-2 downsample: zero fill + one phase
    (2, 24, 2, 1024, 2048, 1, 2, 1, True, False, False),
    (4, 2, 2, 1024, 2048, 1, 2, 1, True, False, False),
    (1, 1, 1, 2048, 256, 3, 1, 1, False, True, True),        # layer4_rn's data gradient at one pixel: 8 tiles of 72 K-steps
    (1, 1, 1, 256, 2048, 3, 1, 1, False, True, True),        # launch Cin 2048: one tile, 576 K-steps, stream-K over 4 CTAs
]


@pytest.mark.parametrize('case', DGRAD_CASES)
def test_conv_data_gradient_matches_torch_fp64(case):
    from dvd_b200 import conv_ops as co
    N, H, W, ci, co_, k, stride, groups, use_bn, has_res, has_mask = case
    seed = 2000 * k + ci + co_ + H + 7 * stride + groups
    g = gen(seed)
    conv = make_conv(ci, co_, k, stride, groups, False, seed + 1)
    bn = make_bn(co_, seed + 2) if use_bn else None
    OH, OW = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    gy = tf32(torch.randn(N, co_, OH, OW, generator=g))
    res = torch.randn(N, ci, H, W, generator=g) if has_res else None
    mask = torch.randn(N, ci, H, W, generator=g) if has_mask else None
    w = conv.weight.detach()
    if bn is not None:      # the scale of the BatchNorm behind the convolution is folded into the packed image, then rounded
        w = w * (bn.weight.detach() * torch.rsqrt(bn.running_var + bn.eps)).view(-1, 1, 1, 1)
    ref = torch.nn.grad.conv2d_input((N, ci, H, W), tf32(w).double(), gy.double(), stride=stride, padding=k // 2, groups=groups)
    if has_res:
        ref = ref + res.double()
    if has_mask:
        ref = ref * (mask > 0)
    conv, bn = conv.cuda(), (bn.cuda() if bn is not None else None)
    c = co.Conv(conv, bn)
    c.pack()
    gx = c.dgrad(cl(gy), H, W, res=cl(res) if has_res else None, mask=cl(mask) if has_mask else None, round_out=False)
    e = rel_err(gx, ref)
    # with a BatchNorm the kernel folds gamma * rsqrtf(var + eps) (2-ulp approximation) before rounding: a few weights land on
    # the other side of a TF32 rounding boundary than the host emulation
    assert e < (1e-4 if use_bn else TOL), e


WGRAD_CASES = [
    # N, H,  W,  Cin,  Cout, k, stride, groups, bn
    (2, 28, 48, 64, 128, 3, 1, 1, False),
    (1, 56, 96, 256, 256, 3, 1, 1, False),
    (3, 7, 12, 1024, 256, 1, 1, 1, True),        # 1x1, ragged K, four in-channel tiles, BatchNorm extras
    (1, 30, 50, 32, 128, 3, 1, 1, False),
    (1, 28, 48, 128, 32, 3, 1, 1, False),        # head conv 128 -> 32: swapped operands
    (2, 56, 96, 256, 512, 1, 2, 1, True),        # stride 2
    (1, 27, 45, 256, 256, 3, 2, 32, True),       # grouped + stride 2, odd sizes
    (2, 28, 48, 256, 256, 3, 1, 32, True),       # grouped 8 ch / group
    (1, 14, 24, 512, 512, 3, 1, 32, True),       # 16
    (1, 14, 24, 1024, 1024, 3, 1, 32, False),    # 32
    (1, 7, 12, 2048, 2048, 3, 1, 32, True),      # 64
    # layer4 classes at the one-row, one-column and single-pixel grids (see FWD_CASES)
    (2, 1, 12, 2048, 256, 3, 1, 1, False),       # layer4_rn
    (2, 12, 1, 2048, 256, 3, 1, 1, False),
    (4, 1, 1, 2048, 256, 3, 1, 1, False),
    (2, 1, 12, 1024, 2048, 1, 1, 1, True),       # 1x1 1024 -> 2048
    (4, 1, 1, 1024, 2048, 1, 1, 1, True),
    (2, 2, 24, 1024, 1024, 3, 2, 32, True),      # grouped stride 2, 32 ch / group
    (2, 24, 2, 1024, 1024, 3, 2, 32, True),
    (4, 2, 2, 1024, 1024, 3, 2, 32, True),
    (2, 2, 24, 2048, 2048, 3, 2, 32, True),      # 64 ch / group
    (4, 2, 2, 2048, 2048, 3, 2, 32, True),
    (2, 2, 24, 1024, 2048, 1, 2, 1, True),       # 1x1 stride-2 downsample
    (2, 24, 2, 1024, 2048, 1, 2, 1, True),
    (4, 2, 2, 1024, 2048, 1, 2, 1, True),
]


@pytest.mark.parametrize('channels_last_weight', [False, True])
@pytest.mark.parametrize('case', WGRAD_CASES)
def test_conv_weight_gradient_matches_torch_fp64(case, channels_last_weight):
    """dW = sc * sum gm x; with `sums` the same launch also yields the per-channel sums of gm (one extra MMA against a ones operand):
    d beta = sum gm and d gamma = rstd * (<W, sum gm x> - mean * sum gm); everything accumulates."""
    from dvd_b200 import conv_ops as co
    N, H, W, ci, co_, k, stride, groups, use_bn = case
    seed = 3000 * k + ci + co_ + H + 7 * stride + groups
    g = gen(seed)
    conv = make_conv(ci, co_, k, stride, groups, False, seed + 1)
    bn = make_bn(co_, seed + 2) if use_bn else None
    OH, OW = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    x = tf32(torch.randn(N, ci, H, W, generator=g))
    gm = tf32(torch.randn(N, co_, OH, OW, generator=g))
    ref = torch.nn.grad.conv2d_weight(x.double(), conv.weight.shape, gm.double(), stride=stride, padding=k // 2, groups=groups)
    ref_dgamma = None
    if bn is not None:
        rstd = torch.rsqrt(bn.running_var.double() + bn.eps)
        ref_dbeta = gm.double().sum(dim=(0, 2, 3))
        ref_dgamma = ((ref * conv.weight.detach().double()).sum(dim=(1, 2, 3)) - bn.running_mean.double() * ref_dbeta) * rstd
        ref = ref * (bn.weight.detach().double() * rstd).view(-1, 1, 1, 1)
    conv, bn = conv.cuda(), (bn.cuda() if bn is not None else None)
    if channels_last_weight and k > 1:
        conv.weight.data = conv.weight.data.contiguous(memory_format=torch.channels_last)
    conv.weight.grad = torch.zeros_like(conv.weight)
    if bn is not None:
        bn.weight.grad = torch.zeros_like(bn.weight)
        bn.bias.grad = torch.zeros_like(bn.bias)
    c = co.Conv(conv, bn)
    c.wgrad(cl(x), cl(gm), sums=True)
    e = rel_err(conv.weight.grad, ref)
    assert e < TOL, e
    if bn is not None:
        e = rel_err(bn.weight.grad, ref_dgamma)
        assert e < 5e-5, e
        e = rel_err(bn.bias.grad, ref_dbeta)
        assert e < 2e-5, e
    c.wgrad(cl(x), cl(gm), sums=True)          # accumulates
    assert rel_err(conv.weight.grad, 2 * ref) < TOL
    if bn is not None:
        assert rel_err(bn.bias.grad, 2 * ref_dbeta) < 2e-5


def test_conv_bias_gradient_rides_on_the_weight_gradient_launch():
    from dvd_b200 import conv_ops as co
    g = gen(77)
    conv = make_conv(256, 256, 3, 1, 1, True, 78).cuda()
    x = tf32(torch.randn(2, 256, 14, 24, generator=g))
    gm = tf32(torch.randn(2, 256, 14, 24, generator=g))
    conv.weight.grad, conv.bias.grad = torch.zeros_like(conv.weight), torch.zeros_like(conv.bias)
    co.Conv(conv).wgrad(cl(x), cl(gm), sums=True)
    assert rel_err(conv.bias.grad, gm.double().sum(dim=(0, 2, 3))) < 2e-5
    # swapped operands (Cout = 32): the sums come from the stand-alone kernel
    conv2 = make_conv(128, 32, 3, 1, 1, True, 79).cuda()
    x2 = tf32(torch.randn(1, 128, 20, 28, generator=g))
    gm2 = tf32(torch.randn(1, 32, 20, 28, generator=g))
    conv2.weight.grad, conv2.bias.grad = torch.zeros_like(conv2.weight), torch.zeros_like(conv2.bias)
    co.Conv(conv2).wgrad(cl(x2), cl(gm2), sums=True)
    assert rel_err(conv2.bias.grad, gm2.double().sum(dim=(0, 2, 3))) < 2e-5
    assert rel_err(conv2.weight.grad, torch.nn.grad.conv2d_weight(x2.double(), conv2.weight.shape, gm2.double(), padding=1)) < TOL


def test_relu_bwd_colsum():
    from dvd_b200 import conv_ops as co
    g0 = gen(5)
    g = torch.randn(2, 64, 9, 11, generator=g0)
    y = torch.randn(2, 64, 9, 11, generator=g0)
    mean, var = torch.randn(64, generator=g0), torch.rand(64, generator=g0) + 0.5
    gm = co.relu_bwd_colsum(cl(g), y=cl(y), gm=co.empty_cl(2, 64, 9, 11, 'cuda'), round_out=True)
    ref = tf32((g * (y > 0)).contiguous())
    assert torch.equal(gm.cpu(), ref)
    cs, dg = torch.zeros(64, device='cuda'), torch.zeros(64, device='cuda')
    co.relu_bwd_colsum(gm, colsum=cs, bn=(mean.cuda(), var.cuda(), 1e-5), dgamma=dg, round_out=False)
    s = ref.double().sum(dim=(0, 2, 3))
    assert rel_err(cs, s) < 1e-5
    assert rel_err(dg, -mean.double() * torch.rsqrt(var.double() + 1e-5) * s) < 1e-5


@pytest.mark.parametrize('shape', [(2, 64, 112, 192), (1, 8, 7, 9), (1, 4, 8, 8)])
def test_maxpool_matches_torch(shape):
    from dvd_b200 import conv_ops as co
    g0 = gen(6)
    x = torch.randn(*shape, generator=g0).relu()        # many exact zeros: ties
    xr = x.clone().requires_grad_()
    ref = F.max_pool2d(xr, 3, 2, 1)
    gy = torch.randn(ref.shape, generator=g0)
    ref.backward(gy)
    y, idx = co.maxpool_fwd(cl(x))
    assert torch.equal(y.cpu(), ref.detach())
    gx = co.maxpool_bwd(cl(gy), idx, shape[2], shape[3])
    assert rel_err(gx, xr.grad) < 1e-6


@pytest.mark.parametrize('shape', [(2, 64, 96), (1, 37, 51)])
def test_stem_matches_torch_fp64(shape):
    from dvd_b200 import conv_ops as co
    N, H, W = shape
    g0 = gen(7)
    x = torch.rand(N, 3, H, W, generator=g0)
    conv = make_conv(3, 64, 7, 2, 1, False, 8)
    conv.padding = (3, 3)
    bn = make_bn(64, 9)
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    xd = ((x.double() - torch.tensor(mean).view(1, 3, 1, 1)) / torch.tensor(std).double().view(1, 3, 1, 1)).requires_grad_()
    wd = conv.weight.detach().double().requires_grad_()
    gd, bd = bn.weight.detach().double().requires_grad_(), bn.bias.detach().double().requires_grad_()
    ref = F.batch_norm(F.conv2d(xd, wd, None, 2, 3), bn.running_mean.double(), bn.running_var.double(), gd, bd, False, 0.0, bn.eps).relu()
    gy = torch.randn(ref.shape, generator=g0)
    ref.backward(gy.double())
    conv, bn = conv.cuda(), bn.cuda()
    y = co.stem_fwd(x.cuda(), conv, bn, mean, std, round_out=False)
    assert rel_err(y, ref) < 1e-5
    for p in (conv.weight, bn.weight, bn.bias):
        p.grad = torch.zeros_like(p)
    co.stem_wgrad(x.cuda(), cl(gy), y, conv, bn, mean, std)
    assert rel_err(conv.weight.grad, wd.grad) < 2e-5
    assert rel_err(bn.weight.grad, gd.grad) < 2e-5
    assert rel_err(bn.bias.grad, bd.grad) < 2e-5


def test_head_matches_torch_fp64():
    from dvd_b200 import conv_ops as co
    g0 = gen(10)
    N, H, W = 2, 20, 36
    x = torch.randn(N, 32, H, W, generator=g0).relu()
    w = torch.randn(1, 32, 1, 1, generator=g0) * 40
    b = torch.tensor([2000.0])
    xd, wd, bd = x.double().requires_grad_(), w.double().requires_grad_(), b.double().requires_grad_()
    ref = 10000.0 / torch.clamp(F.conv2d(xd, wd, bd).relu(), min=1e-2)
    gy = torch.randn(ref.shape, generator=g0)
    ref.backward(gy.double())
    d = co.head_fwd(cl(x), w.cuda(), b.cuda())
    assert rel_err(d, ref) < 1e-5
    gw, gb = torch.zeros(1, 32, 1, 1, device='cuda'), torch.zeros(1, device='cuda')
    gx = co.head_bwd(cl(x), w.cuda(), b.cuda(), gy.cuda(), gw, gb, relu_mask=True, round_out=False)
    assert rel_err(gx, xd.grad * (x > 0)) < 1e-5
    assert rel_err(gw, wd.grad) < 1e-5 and rel_err(gb, bd.grad) < 1e-5


@pytest.mark.parametrize('align', [True, False])
def test_upsample_round_flag(align):
    from dvd_b200 import conv_ops as co
    x = torch.randn(1, 8, 5, 7, generator=gen(11))
    y0 = co.upsample2x_fwd(cl(x), align, round_out=False)
    assert rel_err(y0, F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=align)) < 1e-6
    assert torch.equal(co.upsample2x_fwd(cl(x), align, round_out=True), co.round_tf32(y0))
