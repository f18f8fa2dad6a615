"""Ordered reductions under torch.use_deterministic_algorithms(True) (DESIGN.md 2.11 and 3).

With the mode on, every backward launch that adds partial sums with fp32 atomics takes its ordered variant. Checked here:
  * per kernel: two launches on the same inputs are bitwise equal, and each ordered variant meets the fp64 bounds the
    existing tests hold the atomic path to (the weight gradient of every depth-net layer class at 8 and 1 images, with
    ragged tiles; the scene-flow MLP kernels against their bf16 emulation, including empty weight-gradient splits; g_depth_2
    per element within k * 2^-24 * sum|contributions| of the emulated contributions; the CUDA-core stem, head, column sums
    and the hourglass BatchNorm against the default launches);
  * whole steps: a step restored from a snapshot into the same buffers and run again is bitwise equal in every parameter,
    gradient and Adam moment (MiDaS and hourglass, gaps 1 and 8, warm and joint phase, 2 pairs at 64x96 and 8 at 224x384);
    a captured and replayed step graph is bitwise equal to the eager step from the same state; a graph captured in one
    mode is never replayed in the other;
  * two `python -m dvd_b200.train --deterministic` processes write bitwise equal checkpoints and print equal epoch logs;
  * one ordered step still meets the reference fixture's bounds of test_step_gpu.py.
"""
import contextlib
import os
import subprocess
import sys

import pytest
import torch

from conftest import GOLDEN, rel_err
from test_reproject_fp32_emulation_gpu import emu  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def deterministic(flag=True):
    """torch.use_deterministic_algorithms(flag) for the block; torch raises on a cuBLAS call in that mode unless
    CUBLAS_WORKSPACE_CONFIG is set, which it reads at the call"""
    prev, prev_env = torch.are_deterministic_algorithms_enabled(), os.environ.get('CUBLAS_WORKSPACE_CONFIG')
    torch.use_deterministic_algorithms(flag)
    os.environ['CUBLAS_WORKSPACE_CONFIG'] = prev_env or ':4096:8'
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)
        if prev_env is None:
            os.environ.pop('CUBLAS_WORKSPACE_CONFIG', None)


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------------
# per kernel

def _conv_cases():
    from test_conv_wgrad_bench_shapes_gpu import CASES
    cases = [(8,) + c[1:] for c in CASES]
    cases += [(1, 14, 24, 1024, 1024, 1, 1, 1, 'bn', 1),      # one image: split-K over few pixel tiles
              (1, 56, 96, 256, 256, 3, 1, 32, 'bn', 5),
              (1, 17, 23, 256, 128, 3, 1, 1, 'bias', 1),      # ragged tiles in both directions
              (1, 9, 13, 512, 512, 3, 2, 32, 'bn', 1)]        # stride 2, ragged, more splits than pixel tiles
    return cases


@pytest.mark.parametrize('case', _conv_cases(), ids=lambda c: 'n%d_%dx%d_%d_%d_k%d_s%d_g%d_%s' % c[:9])
def test_conv_weight_gradient_ordered(case):
    from dvd_b200 import conv_ops as co
    from test_conv_wgrad_bench_shapes_gpu import TOL, tf32
    N, H, W, ci, co_, k, stride, groups, extra, slack = case
    g = torch.Generator(device='cuda').manual_seed(ci + 3 * co_ + 7 * H + 11 * k + stride + groups + N)
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
    c = co.Conv(conv, bn)
    grads = (lambda: [conv.weight.grad, bn.weight.grad, bn.bias.grad]) if bn is not None else (lambda: [conv.weight.grad, conv.bias.grad])
    runs = []
    for ordered in (True, True, False):
        conv.weight.grad = torch.zeros_like(conv.weight)
        if bn is not None:
            bn.weight.grad, bn.bias.grad = torch.zeros_like(bn.weight), torch.zeros_like(bn.bias)
        else:
            conv.bias.grad = torch.zeros_like(conv.bias)
        with deterministic(ordered):
            for rep in (1, 2):                # the second launch accumulates
                c.wgrad(x, gm, sums=True)
                torch.cuda.synchronize()
                if ordered:
                    assert rel_err(conv.weight.grad, rep * ref) < TOL * slack
                    if bn is not None:
                        assert rel_err(bn.weight.grad, rep * ref_dgamma) < 5e-5 * slack
                        assert rel_err(bn.bias.grad, rep * ref_sum) < 2e-5
                    else:
                        assert rel_err(conv.bias.grad, rep * ref_sum) < 2e-5
        runs.append([t.clone() for t in grads()])
    assert all(same_bits(a, b) for a, b in zip(runs[0], runs[1])), 'two ordered launches differ'
    # the atomic path sums the same partials in another order
    for a, b in zip(runs[0], runs[2]):
        assert rel_err(a, b) < 2 * TOL * slack


@pytest.mark.parametrize('name,shape', [('16-16-T', (1, 17, 23)), ('16-16-T', (1, 27, 33)), ('16-0-F', (1, 128, 192)),
                                        ('36-16-T', (1, 27, 33)), ('8-4-T', (1, 128, 192))])
def test_mlp_kernels_ordered_against_emulation(name, shape, monkeypatch):
    """test_mlp_bf16_emulation_gpu's whole check with the mode on: the autograd path (ordered data and weight gradients,
    one- and two-stream) against the per-eval raw results the emulation bounds; (1, 27, 33) leaves weight-gradient splits
    empty."""
    from test_mlp_bf16_emulation_gpu import _check_case
    with deterministic():
        _check_case(name, *shape, monkeypatch)


@pytest.mark.parametrize('B', [1, 8])
def test_mlp_chain_backward_ordered_is_bitwise_repeatable(B):
    from dvd_b200 import ops
    from test_mlp_bf16_emulation_gpu import DT, N_ACC, N_EVAL, make_case
    H, W = 64, 96
    layers, p0, t0, g_acc, g_steps = make_case('16-16-T', B, H, W)
    ws = [w.cuda().contiguous() for w, _ in layers]
    bs = [b.cuda().contiguous() for _, b in layers]
    p0, t0, g_acc, g_steps = p0.cuda(), t0.cuda(), g_acc.cuda(), g_steps.cuda()
    pk = ops.PackedMlp(ops.make_mlp_cfg(), 'cuda').refresh(ws, bs)
    out = []
    for ordered in (True, True, False):
        with deterministic(ordered):
            p = p0.clone().requires_grad_()
            wr = [w.clone().requires_grad_() for w in ws]
            br = [b.clone().requires_grad_() for b in bs]
            acc, s = ops.scene_flow_chain(p, t0, pk, DT, N_EVAL, N_ACC, wr, br)
            ((acc * g_acc).sum() + (s * g_steps).sum()).backward()
            torch.cuda.synchronize()
        out.append([p.grad] + [w.grad for w in wr] + [b.grad for b in br])
    assert all(same_bits(a, b) for a, b in zip(out[0], out[1]))
    for a, b in zip(out[0], out[2]):
        assert rel_err(a, b) < 3.5e-6        # test_mlp_bf16_emulation_gpu.ATOMIC_REL: atomic-order spread


@pytest.mark.parametrize('shape', [(1, 17, 23), (3, 30, 50), (8, 64, 96), (4, 224, 384)], ids=lambda s: 'x'.join(map(str, s)))
def test_reproject_backward_ordered_against_emulation(emu, shape):  # noqa: F811
    """g_sf bit for bit and g_depth_2 within k * 2^-24 * sum|c| of the emulated contributions (test_reproject_fp32_emulation_gpu's
    _check_loss), on the path the ordered variant takes for every shape; two launches bitwise equal."""
    from oracle import reproject_fp32 as R
    from test_reproject_fp32_emulation_gpu import SUBSET, Case, _check_loss, _loss_cfg, _staged
    from dvd_b200 import ops
    B, H, W = shape
    case = Case(emu, B, H, W, seed=B + H, sigma=14.0)
    cfgs = R.all_cfgs(flow_mul=1.0, disp_mul=0.7) if B * H * W < 5000 else SUBSET
    with deterministic():
        for cfg in cfgs:
            _check_loss(case, cfg, case.g, _staged(B, H, W))
        lc = _loss_cfg(cfgs[0])
        outs = [ops.reproject_loss_bwd(*case.g, lc, ops.reproject_loss_fwd(*case.g, lc)) for _ in range(2)]
    torch.cuda.synchronize()
    assert same_bits(outs[0][0], outs[1][0]) and same_bits(outs[0][1], outs[1][1])


def test_cuda_core_reductions_ordered():
    """stem, head, column sums and the hourglass BatchNorm backward: two ordered launches bitwise equal, and within fp32
    reordering noise of the atomic launches"""
    from dvd_b200 import conv_ops as co, ops
    dev = torch.device('cuda')
    N, H, W = 8, 224, 384
    res = {}
    for ordered in (True, True, False):
        g = torch.Generator(device='cuda').manual_seed(5)
        torch.manual_seed(0)
        conv = torch.nn.Conv2d(3, 64, 7, 2, 3, bias=False).cuda()
        bn = torch.nn.BatchNorm2d(64).eval().cuda()
        for p in (conv.weight, bn.weight, bn.bias):
            p.grad = torch.zeros_like(p)
        x = torch.rand(N, 3, H, W, generator=g, device=dev)
        a0 = co.stem_fwd(x, conv, bn)
        ga = torch.randn(a0.shape, generator=g, device=dev).contiguous(memory_format=torch.channels_last)
        hx = torch.relu(torch.randn(N, 32, H, W, generator=g, device=dev)).contiguous(memory_format=torch.channels_last)
        hw, hb = torch.randn(32, generator=g, device=dev) * 0.1, torch.full((1,), 0.5, device=dev)
        gd = torch.randn(N, 1, H, W, generator=g, device=dev)
        gw, gb = torch.zeros(32, device=dev), torch.zeros(1, device=dev)
        gc = torch.randn(N, 256, 56, 96, generator=g, device=dev).contiguous(memory_format=torch.channels_last)
        mean, var = torch.randn(256, generator=g, device=dev) * 0.1, torch.rand(256, generator=g, device=dev) + 0.5
        cs, dg = torch.zeros(256, device=dev), torch.zeros(256, device=dev)
        bnx = torch.randn(N, 128, 56, 96, generator=g, device=dev).contiguous(memory_format=torch.channels_last)
        bnh = torch.nn.BatchNorm2d(128).eval().cuda()
        with torch.no_grad():
            bnh.running_mean.normal_(0, 0.1, generator=g), bnh.running_var.uniform_(0.5, 1.5, generator=g)
        with deterministic(ordered):
            co.stem_wgrad(x, ga, a0, conv, bn, (0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
            co.head_bwd(hx, hw, hb, gd, gw, gb)
            co.relu_bwd_colsum(gc, colsum=cs, bn=(mean, var, 1e-5), dgamma=dg, round_out=False)
            xb = bnx.clone().requires_grad_()
            y = ops.bn_act(xb, bnh, None, True)
            gy = torch.randn(y.shape, generator=g, device=dev).contiguous(memory_format=torch.channels_last)
            y.backward(gy)
            torch.cuda.synchronize()
        res.setdefault(ordered, []).append([conv.weight.grad.clone(), bn.weight.grad.clone(), bn.bias.grad.clone(), gw, gb, cs, dg,
                                            bnh.weight.grad.clone(), bnh.bias.grad.clone()])
    a, b = res[True]
    assert all(same_bits(u, v) for u, v in zip(a, b))
    for u, v in zip(a, res[False][0]):
        assert rel_err(u, v) < 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# whole steps

def _harness():
    from test_step_graph_replay_gpu import Harness

    class OrderedHarness(Harness):
        def _sig(self, batch):
            s = super()._sig(batch)
            return s + ('ordered',) if torch.are_deterministic_algorithms_enabled() else s
    return OrderedHarness


def _build_model(opt):
    from dvd_b200 import synthetic
    from dvd_b200.models import get_model
    model = get_model('scene_flow_motion_field')(opt, None)
    synthetic.seed_net_(model.net_depth, 0, 2000.0 if opt.midas else None)
    synthetic.seed_net_(model.net_sceneflow, 1)
    model.to(torch.device('cuda:0'))
    return model


def _bitwise(e, g, what):
    bad = []
    for i, (a, b) in enumerate(zip(e['fwd'], g['fwd'])):
        if not same_bits(a, b):
            bad.append('%s: forward %s' % (what, ('logs', 'd1', 'd2', 'sf')[i]))
    if e['log'] != g['log']:
        bad.append('%s: batch logs' % what)
    for n in ('depth', 'scene'):
        for k in ('data', 'grad', 'm', 'v', 'state'):
            a, b = e['post'][n][k], g['post'][n][k]
            if not same_bits(a, b):
                nd = int((a.view(torch.int32) != b.view(torch.int32)).sum())
                bad.append('%s: %s %s differs in %d elements (max |diff| %.3g)' % (what, n, k, nd, float((a - b).abs().max())))
    return bad


STEP_SCENARIOS = {
    'midas_64x96_gap1_warm': dict(midas=True, H=64, W=96, pairs=[(3, 4), (20, 21)], epoch='warm'),
    'midas_64x96_gap8_joint': dict(midas=True, H=64, W=96, pairs=[(3, 11), (20, 28)], epoch='joint'),
    'hourglass_64x96_gap1_joint': dict(midas=False, H=64, W=96, pairs=[(3, 4), (20, 21)], epoch='joint'),
    'hourglass_64x96_gap8_warm': dict(midas=False, H=64, W=96, pairs=[(3, 11), (20, 28)], epoch='warm'),
    'midas_224x384_gap8_joint': dict(midas=True, H=224, W=384, pairs=[(j * 7, j * 7 + 8) for j in range(8)], epoch='joint'),
    'midas_224x384_gap1_joint': dict(midas=True, H=224, W=384, pairs=[(j * 7, j * 7 + 1) for j in range(8)], epoch='joint'),
}


@pytest.mark.timeout(1200)
@pytest.mark.parametrize('name', sorted(STEP_SCENARIOS))
def test_step_is_bitwise_reproducible(name):
    """eager vs eager from one snapshot, then the graph path (two eager warm-ups, the capture, a replay) against the eager
    step from the same snapshot, all bitwise. In the first scenario the mode is then switched off: the graph path must start
    a signature of its own (eager warm-ups), not replay the ordered graph."""
    from dvd_b200 import synthetic
    from test_step_graph_replay_gpu import make_batch
    sc = STEP_SCENARIOS[name]
    dev = torch.device('cuda:0')
    opt = synthetic.default_opt(lr=1e-4, scene_lr_mul=10.0, midas=sc['midas'])
    h = _harness()(_build_model(opt), name)
    epoch = 1 if sc['epoch'] == 'warm' else opt.warm_sf + 1
    bad = []
    with deterministic():
        for i in range(4):
            batch = make_batch(sc['pairs'], sc['H'], sc['W'], seed=10 + i, resident=bool(i % 2), dev=dev)
            pre = h.snapshot()
            e = h.run(epoch, batch, False, 'eager %d' % i)
            if i == 0:
                h.restore(pre)
                bad += _bitwise(e, h.run(epoch, batch, False, 'eager again'), 'eager vs eager')
            h.restore(pre)
            gr = h.run(epoch, batch, True, 'graph %d' % i) if sc['midas'] else h.run(epoch, batch, False, 'eager %d' % i)
            bad += _bitwise(e, gr, 'step %d %s vs eager' % (i, gr['kind']))
            if sc['midas']:
                want = ('eager', 'eager', 'capture', 'replay')[i]
                if gr['kind'] != want:
                    bad.append('step %d: %s, expected %s' % (i, gr['kind'], want))
    assert not bad, '\n'.join(bad[:30])
    if name == 'midas_64x96_gap8_joint':
        m = h.m
        n_graphs = sum(1 for v in m._graphs.values() if v.get('graph') is not None)
        with deterministic(False):
            kinds = [h.run(epoch, make_batch(sc['pairs'], sc['H'], sc['W'], seed=50 + i, resident=False, dev=dev), True,
                           'default %d' % i)['kind'] for i in range(3)]
        assert kinds == ['eager', 'eager', 'capture'], kinds
        assert sum(1 for v in m._graphs.values() if v.get('graph') is not None) == n_graphs + 1
        with deterministic():
            assert h.run(epoch, make_batch(sc['pairs'], sc['H'], sc['W'], seed=60, resident=False, dev=dev), True,
                         'ordered again')['kind'] == 'replay'


def test_ordered_step_meets_reference_fixture(step_golden):
    """test_step_gpu's reference-fixture bounds for one joint-phase step with the mode on"""
    from test_step_gpu import test_train_step_matches_reference_fixture
    with deterministic():
        test_train_step_matches_reference_fixture(step_golden, 'joint')


@pytest.fixture(scope='module')
def step_golden():
    from oracle.golden_io import load_golden
    return load_golden(GOLDEN, 'step_golden')


# ---------------------------------------------------------------------------------------------------------------------
# process to process

TRAIN = ('--net scene_flow_motion_field --dataset synthetic_sequence --gaps 1 --n_frames 8 --height 64 --width 96 --epoch_batches 5 '
         '--lr 1e-6 --batch_size 1 --optim adam --gpu 0 --workers 0 --save_net 1 --save_net_opt --one_way --loss_type l1 --l1_mul 0 '
         '--acc_mul 1 --disp_mul 1 --warm_sf 1 --scene_lr_mul 1000 --repeat 1 --flow_mul 1 --sf_mag_div 100 --time_dependent --midas '
         '--use_disp --vis_batches_train 0 --manual_seed 0 --deterministic --epoch 3 --validate --vali_batches 2').split()


def _train(logdir):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    env.pop('CUBLAS_WORKSPACE_CONFIG', None)
    r = subprocess.run([sys.executable, '-m', 'dvd_b200.train'] + TRAIN + ['--logdir', logdir], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    logs = []
    for line in r.stdout.splitlines():
        if line.startswith('epoch '):
            log = eval(line.split(':', 1)[1])          # the driver prints a plain dict of floats
            logs.append({k: v for k, v in log.items() if not k.endswith('_time')})      # wall-clock fields differ
    return logs


def _tensors(obj, prefix=''):
    if torch.is_tensor(obj):
        yield prefix, obj
    elif isinstance(obj, dict):
        for k in sorted(obj, key=str):
            yield from _tensors(obj[k], '%s/%s' % (prefix, k))
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            yield from _tensors(v, '%s/%d' % (prefix, i))


@pytest.mark.timeout(1800)
def test_two_training_processes_write_identical_checkpoints(tmp_path):
    """5 steps per epoch at one gap: two eager steps, the capture and replays in the warm epoch, a new signature in each joint
    epoch; --validate every epoch. checkpoint.pt (both nets, both optimizers with their Adam moments) bit for bit, and the
    printed epoch logs, loss_eval included, equal."""
    logs, ckpts = [], []
    for run in ('a', 'b'):
        logdir = str(tmp_path / run)
        logs.append(_train(logdir))
        f = os.path.join(logdir, 'scene_flow_motion_field_synthetic_sequence', '0', 'checkpoint.pt')
        ckpts.append(torch.load(f, map_location='cpu', weights_only=False))
    assert len(logs[0]) == 3 and all('loss_eval' in l for l in logs[0]) and logs[0] == logs[1], logs
    ta, tb = list(_tensors(ckpts[0])), list(_tensors(ckpts[1]))
    assert [k for k, _ in ta] == [k for k, _ in tb] and len(ta) > 100
    assert any('exp_avg_sq' in k for k, _ in ta)
    raw = lambda t: t.contiguous().reshape(-1).view(torch.uint8)  # noqa: E731
    bad = [k for (k, a), (_, b) in zip(ta, tb) if not (a.shape == b.shape and a.dtype == b.dtype and torch.equal(raw(a), raw(b)))]
    assert not bad, bad[:20]
