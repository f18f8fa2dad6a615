"""GPU parity of the convolution weight gradient (csrc/conv2d_tc.cu, conv_wgrad_kernel) at the benchmark's batch: 16 images of
384x224, i.e. the layer classes of one 8-pair training step, against torch.nn.grad.conv2d_weight in fp64 on the same
TF32-rounded operands. At this size every CTA walks a long pixel range (split-K of 1 to 4 on the 14x24 layers), which the
small cases of test_conv2d_gpu.py never reach. BatchNorm extras (scale, dgamma, beta) or the conv-bias sum ride along, and a
second launch must accumulate.

The tensor cores add each 8-pixel group of products to the fp32 accumulator with a rounding that does not average out over
long sums: with 12k to 98k pixels per CTA (the 3x3 layers at 56x96 and above) the error reaches 3e-5 to 2.3e-4 of the
tensor's maximum. The warp-level mma.sync kernel this one replaced showed the same errors (to two digits) on these inputs,
on an H100 80GB HBM3. Those cases carry a `slack` factor on the tolerances, about 3x the error measured."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 2e-5

CASES = [
    # N, H, W, Cin, Cout, k, stride, groups, extra, slack
    (16, 14, 24, 1024, 1024, 1, 1, 1, 'bn', 1),       # layer3 conv1 / conv3
    (16, 56, 96, 256, 256, 3, 1, 1, 'bias', 5),       # refinenet residual conv units
    (16, 14, 24, 1024, 1024, 3, 1, 32, 'bn', 1),      # layer3 conv2, 32 channels per group
    (16, 112, 192, 256, 128, 3, 1, 1, 'bias', 10),    # output head conv 256 -> 128
    (16, 56, 96, 256, 256, 3, 1, 32, 'bn', 5),        # layer1 conv2, 8 channels per group
    (16, 224, 384, 128, 32, 3, 1, 1, 'bias', 35),     # output head conv 128 -> 32: swapped operands
    (16, 56, 96, 512, 512, 3, 2, 32, 'bn', 1),        # layer2.0 conv2: grouped, stride 2
    (16, 28, 48, 512, 1024, 1, 2, 1, 'bn', 1),        # layer3.0 downsample: 1x1 stride 2
]


def tf32(t):
    """round-to-nearest (ties away) TF32, bit-exact emulation of cvt.rna.tf32.f32"""
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


@pytest.mark.parametrize('case', CASES, ids=lambda c: '%dx%d_%d_%d_k%d_s%d_g%d_%s' % (c[1], c[2], c[3], c[4], c[5], c[6], c[7], c[8]))
def test_weight_gradient_at_bench_batch_matches_torch_fp64(case):
    from dvd_b200 import conv_ops as co
    N, H, W, ci, co_, k, stride, groups, extra, slack = case
    g = torch.Generator(device='cuda').manual_seed(ci + 3 * co_ + 7 * H + 11 * k + stride + groups)
    conv = torch.nn.Conv2d(ci, co_, k, stride=stride, padding=k // 2, groups=groups, bias=extra == 'bias').cuda()
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g, device='cuda') / (ci // groups * k * k) ** 0.5)
    bn = None
    if extra == 'bn':
        bn = torch.nn.BatchNorm2d(co_).eval().cuda()
        with torch.no_grad():
            bn.weight.copy_(torch.rand(co_, generator=g, device='cuda') + 0.5)
            bn.running_mean.copy_(torch.randn(co_, generator=g, device='cuda') * 0.1)
            bn.running_var.copy_(torch.rand(co_, generator=g, device='cuda') + 0.5)
    OH, OW = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    x = tf32(torch.randn(N, ci, H, W, generator=g, device='cuda')).contiguous(memory_format=torch.channels_last)
    gm = tf32(torch.randn(N, co_, OH, OW, generator=g, device='cuda')).contiguous(memory_format=torch.channels_last)

    ref = torch.nn.grad.conv2d_weight(x.double(), conv.weight.shape, gm.double(), stride=stride, padding=k // 2, groups=groups)
    ref_sum = gm.double().sum(dim=(0, 2, 3))
    if bn is not None:
        rstd = torch.rsqrt(bn.running_var.double() + bn.eps)
        ref_dgamma = ((ref * conv.weight.detach().double()).sum(dim=(1, 2, 3)) - bn.running_mean.double() * ref_sum) * rstd
        ref = ref * (bn.weight.detach().double() * rstd).view(-1, 1, 1, 1)
        bn.weight.grad, bn.bias.grad = torch.zeros_like(bn.weight), torch.zeros_like(bn.bias)
    else:
        conv.bias.grad = torch.zeros_like(conv.bias)
    conv.weight.grad = torch.zeros_like(conv.weight)
    c = co.Conv(conv, bn)
    for rep in (1, 2):                     # the second launch accumulates
        c.wgrad(x, gm, sums=True)
        torch.cuda.synchronize()
        e = rel_err(conv.weight.grad, rep * ref)
        assert e < TOL * slack, (rep, e)
        if bn is not None:
            assert rel_err(bn.weight.grad, rep * ref_dgamma) < 5e-5 * slack
            assert rel_err(bn.bias.grad, rep * ref_sum) < 2e-5
        else:
            assert rel_err(conv.bias.grad, rep * ref_sum) < 2e-5
