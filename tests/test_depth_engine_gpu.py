"""MiDaS on the repo's own kernels (dvd_b200.depth_engine: explicit forward / backward schedule over the wgmma convolutions)
against the CPU oracle (oracle/depth_nets.py, torch fp32 + autograd): depth maps within 1e-3 (TF32 convolutions), parameter
gradients by max-norm and by share of elements within tolerance."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


def _nets():
    from dvd_b200 import synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    return synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True), 0, 2000.0).eval()


@pytest.mark.parametrize('shape', [(2, 64, 96), (1, 224, 384)])
def test_midas_engine_forward_backward_vs_oracle(shape):
    from oracle import depth_nets
    N, H, W = shape
    net = _nets()
    x = torch.rand(N, 3, H, W, generator=torch.Generator().manual_seed(3))
    sd = {k: (v.detach().clone().requires_grad_() if (v.dtype.is_floating_point and 'running' not in k) else v)
          for k, v in net.state_dict().items()}
    ref = depth_nets.midas_forward(sd, x)
    cot = torch.randn(ref.shape, generator=torch.Generator().manual_seed(4)) * 1e-3
    (ref * cot).sum().backward()
    net = net.cuda()
    with torch.no_grad():
        d_inf = net(x.cuda())
    assert rel_err(d_inf, ref) < 1e-3, rel_err(d_inf, ref)
    d = net(x.cuda())
    assert d.requires_grad and torch.equal(d.detach(), d_inf)
    (d * cot.cuda()).sum().backward()
    # TF32 convolutions through a 101-layer net with random weights: the reference's own GPU path (cuDNN TF32) sits at a relative
    # L2 distance of 2-4 % per parameter tensor from the fp32 gradients, slope within 1e-2 (tools/debug_engine.py)
    # - and so does this engine. A wrong term (a missing skip gradient, a wrong mask) would show as
    # tens of per cent or a slope far from 1.
    report = []
    for k, p in net.named_parameters():
        gref = sd[k].grad
        if gref is None or float(gref.abs().max()) == 0.0:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, k
            continue
        g = p.grad.reshape(gref.shape).double().cpu()
        r = gref.double()
        slope = float((g * r).sum() / (r * r).sum()) - 1.0
        l2 = float(((g - r) ** 2).sum().sqrt() / (r * r).sum().sqrt())
        report.append((k, slope, l2, rel_err(p.grad.reshape(gref.shape), gref)))
    bad = [r for r in report if abs(r[1]) > 0.05 or r[2] > 0.15]
    assert not bad, bad[:10]
    num = sum(float(((p.grad.reshape(sd[k].grad.shape).double().cpu() - sd[k].grad.double()) ** 2).sum()) for k, p in net.named_parameters()
              if sd[k].grad is not None)
    den = sum(float((sd[k].grad.double() ** 2).sum()) for k, p in net.named_parameters() if sd[k].grad is not None)
    assert (num / den) ** 0.5 < 6e-2, (num / den) ** 0.5


def test_midas_engine_uses_no_library_kernels():
    """kineto trace of one training forward + backward: no cuDNN / cutlass / ATen convolution or batch-norm kernel."""
    from torch.profiler import ProfilerActivity, profile
    net = _nets().cuda()
    x = torch.rand(2, 3, 64, 96, device='cuda')
    net(x).sum().backward()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        net(x).sum().backward()
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    lib = [n for n in names if any(s in n.lower() for s in ('cudnn', 'cutlass', 'xmma', 'implicit_gemm', 'batch_norm', 'convolve'))]
    assert not lib, lib
    assert any('conv2d_tc_kernel' in n for n in names) and any('conv_wgrad_kernel' in n for n in names)


def test_stream_schedules_agree(monkeypatch):
    """The engine's stream schedules are pure re-orderings: single stream (DVD_BWD_OVERLAP=0) and two-stream backward (default)
    give the same depth map and the same parameter gradients up to fp32 summation order (atomics in the weight-gradient
    reductions)."""
    net = _nets().cuda()
    x = torch.rand(4, 3, 64, 96, device='cuda')
    w = torch.rand(4, 1, 64, 96, device='cuda')

    def run(env):
        monkeypatch.delenv('DVD_BWD_OVERLAP', raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        for p in net.parameters():
            p.grad = None
        d = net(x)
        (d * w).sum().backward()
        torch.cuda.synchronize()
        return d.detach().clone(), {k: p.grad.detach().clone() for k, p in net.named_parameters()}

    d0, g0 = run({'DVD_BWD_OVERLAP': '0'})
    # tolerances: the two-stream backward changes nothing but the order of fp32 atomics
    d1, g1 = run({})
    ed = float((d0 - d1).abs().max() / d0.abs().max())
    num = sum(float(((g1[k].double() - g0[k].double()) ** 2).sum()) for k in g0)
    den = sum(float((g0[k].double() ** 2).sum()) for k in g0)
    print('two-stream backward: depth', ed, 'grad L2', (num / den) ** 0.5)
    assert ed < 1e-6, ed
    assert (num / den) ** 0.5 < 1e-5, (num / den) ** 0.5
