"""The flat Adam checker (oracle/adam_fp32.py) on the CPU: torch.optim.Adam in fp32, handed the fp32 betas the kernel
receives, passes it at steps 1-6, and each planted defect of the update fails it. So the bound the GPU step tests hold
`dvd_adam_flat_dev` to is neither vacuous nor tighter than correctly rounded fp32 arithmetic."""
import numpy as np
import pytest
import torch

from oracle.adam_fp32 import adam_fp32_numpy, check_adam, f32

LR, BETAS, EPS, GSCALE = 1e-3, (f32(0.5), f32(0.9)), 1e-8, 0.5
# tensor sizes of a flat buffer, each start 4-aligned (16 bytes) as FlatParams lays them out, and the weight scale of each:
# conv-like, BatchNorm-like (~1) and a large head bias whose ulp is close to one update
LAYOUT = [(1, 2000.0), (3, 1.0), (64, 1.0), (1000, 0.02), (4096, 0.02), (9, 0.3), (20000, 0.05)]


def _layout():
    segs, o = [], 0
    for n, _ in LAYOUT:
        segs.append((o, n))
        o += (n + 3) // 4 * 4
    return segs, (o + 3) // 4 * 4


def _flat(parts, numel):
    out = torch.zeros(numel, dtype=torch.float32)
    for (o, n), x in zip(_layout()[0], parts):
        out[o:o + n] = x.reshape(-1)
    return out


def _grads(steps, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(steps):
        gs = []
        for n, _ in LAYOUT:
            x = torch.randn(n, generator=g) * 10 ** float(torch.empty(1).uniform_(-4, -2, generator=g))
            x[torch.rand(n, generator=g) < 0.05] = 0.0           # parameters without a gradient this step
            x[torch.rand(n, generator=g) < 0.02] *= 1e-17          # g^2 subnormal in fp32
            gs.append(x)
        out.append(gs)
    return out


def _params(seed=1):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, generator=g) * s + (s if s >= 1 else 0.0)) for n, s in LAYOUT]


def _torch_run(steps=6):
    segs, numel = _layout()
    ps = [torch.nn.Parameter(x.clone()) for x in _params()]
    opt = torch.optim.Adam(ps, lr=LR, betas=BETAS, eps=EPS)
    reps = []
    for t, gs in enumerate(_grads(steps), 1):
        p0 = _flat([p.detach() for p in ps], numel)
        st = [opt.state.get(p, {}) for p in ps]
        m0 = _flat([s['exp_avg'] if s else torch.zeros(p.numel()) for s, p in zip(st, ps)], numel)
        v0 = _flat([s['exp_avg_sq'] if s else torch.zeros(p.numel()) for s, p in zip(st, ps)], numel)
        for p, gr in zip(ps, gs):
            p.grad = (gr * GSCALE).float()      # what the kernel forms as gk = g * gscale
        opt.step()
        m1 = _flat([opt.state[p]['exp_avg'] for p in ps], numel)
        v1 = _flat([opt.state[p]['exp_avg_sq'] for p in ps], numel)
        reps.append(check_adam(p0, m0, v0, _flat(gs, numel), _flat([p.detach() for p in ps], numel), m1, v1, t=t, lr=LR,
                               betas=BETAS, eps=EPS, gscale=GSCALE, segments=segs))
    return reps


def _numpy_run(steps=6, **defect):
    segs, numel = _layout()
    p = _flat(_params(), numel).numpy()
    m, v = np.zeros_like(p), np.zeros_like(p)
    reps = []
    for t, gs in enumerate(_grads(steps), 1):
        g = _flat(gs, numel).numpy()
        kw = dict(defect)
        if kw.pop('bc_lags', False):          # bias correction one step behind (from step 2: 1 - b^0 = 0 would be inf)
            kw['bc_step'] = max(t - 1, 1)
        p1, m1, v1 = adam_fp32_numpy(p, g, m, v, t, LR, BETAS, EPS, GSCALE, **kw)
        T = torch.from_numpy
        reps.append(check_adam(T(p), T(m), T(v), T(g), T(p1), T(m1), T(v1), t=t, lr=LR, betas=BETAS, eps=EPS, gscale=GSCALE,
                               segments=segs))
        p, m, v = p1, m1, v1
    return reps


def test_torch_adam_fp32_passes_at_steps_1_to_6():
    reps = _torch_run()
    for t, r in enumerate(reps, 1):
        print('step %d: m %.2f units, v %.2f units, p %.3f of bound, slope %.3f of tolerance'
              % (t, r['m_units'], r['v_units'], r['p_ratio'], r['slope_ratio']))
        assert not r['fail'], (t, r['fail'])


def test_kernel_restatement_passes():
    for t, r in enumerate(_numpy_run(), 1):
        assert not r['fail'], (t, r['fail'])


@pytest.mark.parametrize('defect,expect', [
    ({'bc_lags': True}, "p'"),
    ({'lr_scale': 1.01}, "p'"),
    ({'use_gscale': False}, "m'"),
    ({'fp64_betas': (0.5, 0.9)}, "v'"),
])
def test_planted_defects_fail(defect, expect):
    reps = _numpy_run(**defect)
    fails = [f for r in reps for f in r['fail']]
    assert fails, defect
    assert any(f.startswith(expect) for f in fails), (defect, fails[:3])


def test_lagging_bias_correction_is_seen_at_every_step():
    """From step 2 on, a bias correction one step behind changes each update by a few per cent at most (β = 0.5, 0.9); the
    checker sees it at every one of those steps on its own."""
    reps = _numpy_run(bc_lags=True)
    assert not reps[0]['fail']
    for t in range(2, 7):
        assert any(f.startswith("p'") for f in reps[t - 1]['fail']), (t, reps[t - 1]['fail'])
