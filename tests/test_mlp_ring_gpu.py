"""GPU: the scene-flow MLP chain kernels give every pixel the same bits whether its pair runs in a batch or alone.

A pixel's forward and data gradient depend only on its own inputs, so any difference between the two runs comes from the
weight ring's bookkeeping (stage index, barrier phase) going wrong at some ring position. The batch sizes are chosen so that
the ring positions differ: CTAs own one or two tiles, pixel counts are ragged, and the number of ring stages a CTA consumes
is not a multiple of the ring depth. Compared: acc, s_steps, p_steps and every evaluation's a_out (not g_bias5, whose
atomicAdd order is not fixed)."""
import pytest
import torch

from tools.mlp_kernel_dump import CONFIGS, make_inputs, make_weights, run_chain

pytestmark = pytest.mark.gpu

# (B, H, W, n_eval): 3072 px = 24 tiles per pair; 1665 px per pair leaves a partial tile. On 132 SMs, 144 tiles give some
# CTAs two tiles and the others one.
CASES = [(6, 48, 64, 9), (3, 48, 64, 5), (11, 37, 45, 1), (10, 37, 45, 2), (2, 37, 45, 7)]


@pytest.fixture(scope='module', params=sorted(CONFIGS))
def packed(request):
    from dvd_b200 import _lib, ops
    fx, ft, td = CONFIGS[request.param]
    ws, bs = make_weights(ops.mlp_n_in(fx, ft, td), seed=21)
    return _lib, ops, ops.PackedMlp(ops.make_mlp_cfg(n_freq_xyz=fx, n_freq_t=ft, time_dependent=td), 'cuda').refresh(ws, bs)


@pytest.mark.parametrize('B,H,W,n_eval', CASES)
def test_batch_equals_pairs_bitwise(packed, B, H, W, n_eval):
    _lib, ops, pk = packed
    p0, t0, g_acc, g_steps = make_inputs(B, H, W, n_eval, seed=22)
    n_acc = n_eval - n_eval // 3
    full = run_chain(_lib, ops, pk, p0, t0, g_acc, g_steps, n_eval, n_acc)
    keys = ['acc', 's_steps', 'p_steps'] + ['a_out_e%d' % e for e in range(n_eval)]
    for b in range(B):
        one = run_chain(_lib, ops, pk, p0[b:b + 1].contiguous(), t0[b:b + 1].contiguous(), g_acc[b:b + 1].contiguous(),
                        [g[b:b + 1].contiguous() for g in g_steps], n_eval, n_acc)
        for k in keys:
            mine = full[k][:, b:b + 1] if k in ('s_steps', 'p_steps') else full[k][b:b + 1]
            assert torch.equal(mine.view(torch.int32), one[k].view(torch.int32)), (k, b)
