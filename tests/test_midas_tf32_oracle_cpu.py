"""The TF32 emulation of the MiDaS engine (oracle/midas_tf32.py) has the reference's structure: with rounding switched off and the
packed images replaced by the plain weights it is oracle.depth_nets.midas_forward + autograd, in fp64, to rounding level — so it
cannot inherit a wiring error of the engine it is used to check (tests/test_depth_engine_tf32_gpu.py)."""
import torch

from conftest import rel_err


def _net():
    from dvd_b200 import synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    return synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True), 0, 2000.0).eval()


def _leaves(net):
    return {k: (v.detach().double().clone().requires_grad_() if (v.dtype.is_floating_point and 'running' not in k) else v.double())
            for k, v in net.state_dict().items()}


def test_unrounded_emulation_is_the_reference_structure():
    from oracle import depth_nets, midas_tf32
    net = _net()
    x = torch.rand(1, 3, 64, 96, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    sd_ref, sd_emu = _leaves(net), _leaves(net)
    # the random BatchNorm statistics of seed_net_ make the mean term of every gamma gradient count
    assert float(sd_ref['pretrained.layer3.5.bn2.running_mean'].abs().max()) > 0.05
    d_ref = depth_nets.midas_forward(sd_ref, x)
    d_emu = midas_tf32.midas_tf32_forward(sd_emu, x, images=None, rounding=False)
    assert rel_err(d_emu, d_ref) < 1e-12, rel_err(d_emu, d_ref)
    cot = torch.randn(d_ref.shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64) * 1e-3
    (d_ref * cot).sum().backward()
    (d_emu * cot).sum().backward()
    n = 0
    for k, p in sd_ref.items():
        if not (isinstance(p, torch.Tensor) and p.requires_grad):
            continue
        if p.grad is None:      # refinenet4.resConfUnit1: not part of the net's graph
            assert sd_emu[k].grad is None, k
            continue
        assert sd_emu[k].grad is not None and float(p.grad.abs().max()) > 0, k
        err = rel_err(sd_emu[k].grad, p.grad)
        assert err < 1e-12, (k, err)
        n += 1
    assert n == sum(1 for _ in net.parameters()) - 4


def test_tf32_rounding_matches_cvt_rna():
    """round to nearest, ties away from zero, on the 13 dropped mantissa bits"""
    from oracle.midas_tf32 import round_tf32
    one = 1.0
    ulp = 2.0 ** -10
    x = torch.tensor([one, one + ulp / 2, one + ulp / 2 - 2 ** -23, -(one + ulp / 2), one + 3 * ulp / 2, 0.0, -0.0],
                     dtype=torch.float64)
    want = torch.tensor([one, one + ulp, one, -(one + ulp), one + 2 * ulp, 0.0, -0.0], dtype=torch.float64)
    assert torch.equal(round_tf32(x), want)
    assert torch.equal(torch.signbit(round_tf32(x)), torch.signbit(want))


def test_image_layout_round_trip():
    """unpack_image inverts the documented pack layout ([t][co][c] forward, [t][ci][c] data gradient, GROUP_BLOCK-wide blocks for
    grouped layers), built here independently of it by scattering the weights element by element"""
    from oracle.midas_tf32 import GROUP_BLOCK, off_group_entries, unpack_image
    g = torch.Generator().manual_seed(0)
    for Cout, Cin, k, groups in ((64, 96, 3, 1), (256, 256, 3, 32), (128, 128, 1, 2), (64, 64, 3, 8)):
        w = torch.randn(Cout, Cin // groups, k, k, generator=g)
        cpg, opg = Cin // groups, Cout // groups
        kb = GROUP_BLOCK if groups > 1 else 0
        f = torch.zeros(k * k, Cout, kb or Cin)
        b = torch.zeros(k * k, Cin, kb or Cout)
        for co in range(Cout):
            for j in range(cpg):
                ci = (co // opg) * cpg + j
                for t in range(k * k):
                    f[t, co, ci - (co // kb) * kb if kb else ci] = w[co, j, t // k, t % k]
                    b[t, ci, co - (ci // kb) * kb if kb else co] = w[co, j, t // k, t % k]
        assert torch.equal(unpack_image(f, Cout, Cin, k, groups, 0), w)
        assert torch.equal(unpack_image(b, Cout, Cin, k, groups, 1), w)
        assert float(off_group_entries(f, Cout, Cin, groups, 0).abs().max()) == 0.0
        assert float(off_group_entries(b, Cout, Cin, groups, 1).abs().max()) == 0.0
