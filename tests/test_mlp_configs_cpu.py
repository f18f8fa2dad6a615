"""CPU: scene-flow MLP positional encodings other than the default 16 / 16. The CPU oracle (oracle/sf_mlp.py) against the
reference-generated fixture tests/golden/mlp_cfg_golden.pt (oracle/gen_golden_mlp_cfg.py), the state-dict layout of the
constructor, and the rejection of encodings wider than the kernels take (256 input features)."""
import pytest
import torch

from conftest import GOLDEN, rel_err
from test_oracle_step import frac_within


@pytest.fixture(scope='module')
def cfg_golden():
    from oracle.golden_io import load_golden
    return load_golden(GOLDEN, 'mlp_cfg_golden')


def _ids(g):
    return ['%d-%d-%s' % (c['n_freq_xyz'], c['n_freq_t'], 'T' if c['time_dependent'] else 'F') for c in g['configs']]


def layers_of(g, c, dtype=torch.float64):
    from oracle import sf_mlp
    sd = dict(g['hidden'])
    sd['convs.0.conv.weight'], sd['convs.0.conv.bias'] = c['w0'], c['b0']
    return sf_mlp.layers_from_state_dict(sd, dtype=dtype)


def test_fixture_covers_the_issue_configurations(cfg_golden):
    nin = {(c['n_freq_xyz'], c['n_freq_t'] if c['time_dependent'] else None): c['nin'] for c in cfg_golden['configs']}
    assert nin == {(8, 4): 60, (0, 0): 4, (0, 16): 36, (16, 0): 100, (10, None): 63, (1, 1): 12, (5, 3): 40,
                   (36, 16): 252, (42, None): 255, (0, 126): 256}


def test_oracle_matches_reference_for_every_configuration(cfg_golden):
    from oracle import sf_mlp
    g = cfg_golden
    for name, c in zip(_ids(g), g['configs']):
        kw = dict(n_freq_xyz=c['n_freq_xyz'], n_freq_t=c['n_freq_t'], time_dependent=c['time_dependent'])
        layers = layers_of(g, c)
        P1, ts = g['P1'].double(), g['ts'].double()
        raw = sf_mlp.mlp_forward(P1, ts, layers, **kw)
        assert rel_err(raw, c['raw']) < 1e-5, name
        lw = [(w.clone().requires_grad_(), b.clone().requires_grad_()) for w, b in layers]
        p = P1.clone().requires_grad_()
        sf = sf_mlp.sf_multi_step(p, ts, g['dt'], g['steps'], lw, sf_mag_div=100.0, **kw)
        assert rel_err(sf, c['sf']) < 1e-5, name
        (sf * c['cot'].double()).sum().backward()
        assert frac_within(p.grad, c['g_p'], 2e-3) > 0.999, name
        assert frac_within(lw[0][0].grad, c['g_w0'].reshape(lw[0][0].shape), 2e-3) > 0.999, name
        assert frac_within(lw[0][1].grad, c['g_b0'], 2e-3) > 0.999, name


def test_state_dict_matches_reference_constructor(cfg_golden):
    from dvd_b200.networks.sceneflow_field import SceneFlowFieldNet
    for name, c in zip(_ids(cfg_golden), cfg_golden['configs']):
        net = SceneFlowFieldNet(net_width=256, n_layers=4, time_dependent=c['time_dependent'], N_freq_xyz=c['n_freq_xyz'],
                                N_freq_t=c['n_freq_t'])
        sd = net.state_dict()
        assert list(sd) == c['keys'], name
        assert {k: tuple(v.shape) for k, v in sd.items()} == c['shapes'], name


def test_make_mlp_cfg_carries_the_reference_frequencies(cfg_golden):
    from dvd_b200 import ops
    for c in cfg_golden['configs']:
        fx, ft, td = c['n_freq_xyz'], c['n_freq_t'], c['time_dependent']
        cfg = ops.make_mlp_cfg(fx, ft, td)
        assert ops.mlp_n_in(fx, ft, td) == c['nin']
        assert list(cfg.freq_xyz)[:fx] == torch.linspace(1, fx + 1, steps=fx).tolist()
        assert all(f == 0.0 for f in list(cfg.freq_xyz)[fx:])
        n_t = ft if td else 0
        assert list(cfg.freq_t)[:n_t] == torch.linspace(1, n_t + 1, steps=n_t).tolist()
        assert all(f == 0.0 for f in list(cfg.freq_t)[n_t:])


@pytest.mark.parametrize('fx,ft,td', [(37, 16, True), (43, 16, False), (0, 127, True), (-1, 16, True)])
def test_over_bound_configurations_are_rejected(fx, ft, td, cfg_golden):
    from dvd_b200 import ops
    from dvd_b200.networks.sceneflow_field import SceneFlowFieldNet
    with pytest.raises(ValueError):
        ops.make_mlp_cfg(fx, ft, td)
    with pytest.raises(ValueError):
        SceneFlowFieldNet(net_width=256, n_layers=4, time_dependent=td, N_freq_xyz=fx, N_freq_t=ft)
    if fx >= 0:
        assert ops.mlp_n_in(fx, ft, td) > 256
    assert [tuple(x) for x in cfg_golden['over_bound']] == [(37, 16, True), (43, 16, False)]


def test_model_rejects_an_over_bound_encoding_at_construction():
    from dvd_b200 import synthetic
    from dvd_b200.models import get_model
    opt = synthetic.default_opt(n_freq_xyz=37, n_freq_t=16, midas=False)
    with pytest.raises(ValueError, match='256'):
        get_model('scene_flow_motion_field')(opt, None)
