"""TEST INFRASTRUCTURE — generates tests/golden/mlp_cfg_golden.pt: the reference's SceneFlowFieldNet and
Model.forward_sf_net_multi_step (imported unmodified through oracle/ref_harness.py) for positional encodings other
than the default 16 / 16, on a small ragged pixel set (1 x 17 x 23).

Run in the authoring container only:   python -m oracle.gen_golden_mlp_cfg
Every configuration shares the hidden and output layers (stored once); per configuration the fixture keeps the
first layer, the state-dict keys and shapes of the reference constructor, the raw single-eval output, the 3-step
chain, and the gradients w.r.t. the points and the first layer for a cotangent zeroed on the LeakyReLU kink band.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_harness, sf_mlp  # noqa: E402
from oracle.gen_golden import GOLD, mlp_inputs  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402

# (n_freq_xyz, n_freq_t, time_dependent); n_freq_t of a time-independent field is unused (the Model passes its flag anyway)
CONFIGS = [(8, 4, True), (0, 0, True), (0, 16, True), (16, 0, True), (10, 16, False), (1, 1, True), (5, 3, True),
           (36, 16, True), (42, 16, False), (0, 126, True)]
OVER_BOUND = [(37, 16, True), (43, 16, False)]
STEPS = 3
# Half-width of the LeakyReLU kink band whose pixels get a zero cotangent. Wider than kink_band's default 3e-5: with only 4 input
# features (0, 0, time-dependent) the first-layer pre-activations are large and an fp32 implementation's absolute error
# there reaches a few 1e-5, enough to take the other slope at a pre-activation of 3.4e-5.
KINK_WIDTH = 1e-4


def _reference_net(ns, fx, ft, td, seed):
    torch.manual_seed(seed)
    net = ns.sff.SceneFlowFieldNet(net_width=256, n_layers=4, time_dependent=td, N_freq_xyz=fx, N_freq_t=ft)
    ns.smf.Model.init_weight(None, net, 'kaiming', 0.01, a=0.2)     # reference init (smf.py:123)
    with torch.no_grad():
        for p in net.parameters():
            if p.dim() == 1:
                p.normal_(0, 0.05)                                      # exercise the bias path
    return net


def main():
    ns = ref_harness.import_reference()
    P1, ts, dt = mlp_inputs(B=1, H=17, W=23, seed=7)
    shared = _reference_net(ns, 16, 16, True, 100).state_dict()
    hidden = {k: v.clone() for k, v in shared.items() if not k.startswith('convs.0.')}
    out = {'P1': P1, 'ts': ts, 'dt': dt, 'steps': STEPS, 'hidden': hidden, 'over_bound': OVER_BOUND, 'configs': []}
    for i, (fx, ft, td) in enumerate(CONFIGS):
        net = _reference_net(ns, fx, ft, td, 200 + i)
        with torch.no_grad():
            for k, v in hidden.items():
                net.state_dict()[k].copy_(v)
        sd = net.state_dict()
        model = ns.smf.Model.__new__(ns.smf.Model)
        model.opt = ref_harness.default_opt(time_dependent=td, n_freq_xyz=fx, n_freq_t=ft)
        model.net_sceneflow = net
        with torch.no_grad():
            raw = net(P1.clone(), ts) if td else net(P1.clone())
        kw = dict(n_freq_xyz=fx, n_freq_t=ft, time_dependent=td)
        band = sf_mlp.kink_band(P1, ts, dt, STEPS, sf_mlp.layers_from_state_dict(sd), width=KINK_WIDTH, **kw)
        cot = torch.randn(P1.shape, generator=torch.Generator().manual_seed(30 + i)) * (~band).unsqueeze(1).float()
        net.zero_grad()
        p = P1.clone().requires_grad_()
        sf = model.forward_sf_net_multi_step(p, ts, time_step=dt, steps=STEPS)
        (sf * cot).sum().backward()
        out['configs'].append({
            'n_freq_xyz': fx, 'n_freq_t': ft, 'time_dependent': td, 'nin': sd['convs.0.conv.weight'].shape[1],
            'keys': list(sd), 'shapes': {k: tuple(v.shape) for k, v in sd.items()},
            'w0': sd['convs.0.conv.weight'].clone(), 'b0': sd['convs.0.conv.bias'].clone(),
            'raw': raw.detach(), 'cot': cot, 'kink_band_pixels': int(band.sum()),
            'sf': sf.detach(), 'g_p': p.grad.clone(),
            'g_w0': net.convs[0].conv.weight.grad.clone(), 'g_b0': net.convs[0].conv.bias.grad.clone()})
        print('(%d, %d, %s) nin=%d |raw|max=%.3g band=%d' % (fx, ft, td, out['configs'][-1]['nin'], raw.abs().max(),
                                                            int(band.sum())))
    save_golden(out, GOLD, 'mlp_cfg_golden')
    print('wrote mlp_cfg_golden')


if __name__ == '__main__':
    main()
