"""GPU: the scene-flow MLP kernels for positional encodings other than the default 16 / 16 (the generic kernels: counts read
at run time, first layer padded to a multiple of 64 input channels). Against the reference-generated fixture
tests/golden/mlp_cfg_golden.pt and the fp64 CPU oracle, the raw C ABI's refusal of encodings wider than 256 features, whole
optimisation steps against oracle/step.py, and the training command line."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from conftest import GOLDEN, rel_err
from test_oracle_step import frac_within

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TIGHT = 1e-4
WTOL_SMALL = 1e-2


@pytest.fixture(scope='module')
def cfg_golden():
    from oracle.golden_io import load_golden
    return load_golden(GOLDEN, 'mlp_cfg_golden')


def _name(c):
    return '%d-%d-%s' % (c['n_freq_xyz'], c['n_freq_t'], 'T' if c['time_dependent'] else 'F')


def _kw(c):
    return dict(n_freq_xyz=c['n_freq_xyz'], n_freq_t=c['n_freq_t'], time_dependent=c['time_dependent'])


def _params(g, c):
    sd = dict(g['hidden'])
    sd['convs.0.conv.weight'], sd['convs.0.conv.bias'] = c['w0'], c['b0']
    ws = [sd['convs.%d.conv.weight' % l].reshape(sd['convs.%d.conv.weight' % l].shape[0], -1).cuda().contiguous()
          for l in range(6)]
    bs = [sd['convs.%d.conv.bias' % l].cuda().contiguous() for l in range(6)]
    return ws, bs


def _packed(ws, bs, **kw):
    from dvd_b200 import ops
    return ops.PackedMlp(ops.make_mlp_cfg(**kw), 'cuda').refresh(ws, bs)


def test_forward_chain_and_gradients_match_reference_fixture(cfg_golden):
    """Every configuration of the fixture (ragged 1 x 17 x 23 pixels): the raw single eval, the 3-step chain, dL/dp and the
    first layer's weight and bias gradients."""
    from dvd_b200 import ops
    g = cfg_golden
    P1, ts = g['P1'].cuda(), g['ts'].cuda()
    for c in g['configs']:
        name, td = _name(c), c['time_dependent']
        ws, bs = _params(g, c)
        pk = _packed(ws, bs, **_kw(c))
        out = ops.mlp_chain_fwd(pk, P1, ts if td else None, g['dt'], 1, 1)
        assert rel_err(out['acc'] * 100.0, c['raw']) < TIGHT, name
        ws = [w.requires_grad_() for w in ws]
        bs = [b.requires_grad_() for b in bs]
        pk = _packed(ws, bs, **_kw(c))
        p = P1.clone().requires_grad_()
        acc, _ = ops.scene_flow_chain(p, ts if td else None, pk, g['dt'], g['steps'], g['steps'], ws, bs)
        assert rel_err(acc, c['sf']) < TIGHT, name
        (acc * c['cot'].cuda()).sum().backward()
        assert rel_err(p.grad, c['g_p']) < 5e-4, (name, rel_err(p.grad, c['g_p']))
        assert rel_err(ws[0].grad, c['g_w0'].reshape(ws[0].shape)) < WTOL_SMALL, name
        assert rel_err(bs[0].grad, c['g_b0']) < WTOL_SMALL, name


def test_every_layer_gradient_vs_fp64_oracle(cfg_golden):
    """All six layers' weight and bias gradients at 128 x 192 pixels with a coherent cotangent (see test_mlp_gpu.py:
    test_weight_gradient_single_plane_noise for why the weight gradient is compared at this size)."""
    from dvd_b200 import ops
    from oracle import sf_mlp
    H, W = 128, 192
    gen = torch.Generator().manual_seed(H)
    p = torch.randn(1, 3, H, W, generator=gen) * 3.0
    t = torch.full((1, 1, H, W), 0.3)
    cot = 1.0 + 0.3 * torch.nn.functional.interpolate(torch.randn(1, 3, 5, 7, generator=gen), size=(H, W), mode='bilinear')
    for i, c in enumerate(cfg_golden['configs']):
        name, kw, td = _name(c), _kw(c), c['time_dependent']
        layers = sf_mlp.init_layers(n_in=c['nin'], seed=20 + i)
        layers = [(w, torch.randn(b.shape, generator=torch.Generator().manual_seed(i)) * 0.05) for w, b in layers]
        lw = [(w.double().requires_grad_(), b.double().requires_grad_()) for w, b in layers]
        ref = sf_mlp.sf_multi_step(p.double(), t.double(), 1.0 / 80, 2, lw, **kw)
        (ref * cot.double()).sum().backward()
        ws = [w.cuda().contiguous().requires_grad_() for w, _ in layers]
        bs = [b.cuda().contiguous().requires_grad_() for _, b in layers]
        pk = _packed(ws, bs, **kw)
        acc, _ = ops.scene_flow_chain(p.cuda(), t.cuda() if td else None, pk, 1.0 / 80, 2, 2, ws, bs)
        assert rel_err(acc, ref) < TIGHT, name
        (acc * cot.cuda()).sum().backward()
        for l in range(6):
            assert rel_err(ws[l].grad, lw[l][0].grad.reshape(ws[l].shape)) < WTOL_SMALL, (name, 'dW%d' % l)
            assert rel_err(bs[l].grad, lw[l][1].grad) < WTOL_SMALL, (name, 'db%d' % l)


def test_over_bound_configurations_fail_in_the_c_abi(cfg_golden):
    """rc -2 from every MLP entry point, before anything is launched (null buffers: nothing may be touched)."""
    from dvd_b200 import _lib
    lib = _lib.load()
    for fx, ft, td in cfg_golden['over_bound']:
        cfg = _lib.MlpCfg()
        cfg.n_freq_xyz, cfg.n_freq_t, cfg.time_dependent, cfg.sf_mag_div = fx, ft, int(td), 100.0
        ref = ctypes.byref(cfg)
        ptrs = (ctypes.c_void_p * 6)()
        calls = {
            'dvd_mlp_pack_weights': lambda: lib.dvd_mlp_pack_weights(ref, ptrs, None, None, None),
            'dvd_mlp_chain_fwd': lambda: lib.dvd_mlp_chain_fwd(ref, None, None, None, None, 0.0, 1, 1, None, None, None, None,
                                                               128, 128, None),
            'dvd_mlp_dgrad': lambda: lib.dvd_mlp_dgrad(ref, None, None, None, 0.0, 0, 0, None, None, None, None, None, None,
                                                       None, 128, 128, None),
            'dvd_mlp_wgrad': lambda: lib.dvd_mlp_wgrad(ref, None, None, ptrs, ptrs, 128, None),
        }
        for what, call in calls.items():
            rc = call()
            assert rc == -2, (what, fx, ft, td, rc)
            with pytest.raises(RuntimeError, match='at most 256'):
                _lib.check(rc, what)
    torch.cuda.synchronize()


# ---- whole optimisation steps ---------------------------------------------------------------------------------------------
H, W = 64, 96
STEP_CONFIGS = {'8-4-T': dict(n_freq_xyz=8, n_freq_t=4), '0-0-T': dict(n_freq_xyz=0, n_freq_t=0),
                '36-16-T': dict(n_freq_xyz=36, n_freq_t=16)}


def _build(over):
    from dvd_b200 import synthetic
    from dvd_b200.models import get_model
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    opt = synthetic.default_opt(lr=1e-4, **over)
    model = get_model('scene_flow_motion_field')(opt, None)
    synthetic.seed_net_(model.net_depth, 0, 2000.0)
    synthetic.seed_net_(model.net_sceneflow, 1)
    sd_d = {k: v.clone() for k, v in model.net_depth.state_dict().items()}
    sd_m = {k: v.clone() for k, v in model.net_sceneflow.state_dict().items()}
    model.to(torch.device('cuda:0'))
    return model, opt, sd_d, sd_m


@pytest.mark.parametrize('name', sorted(STEP_CONFIGS))
@pytest.mark.parametrize('epoch', [1, 6])
def test_train_step_matches_oracle(name, epoch):
    """Model._train_on_batch (2 pairs, MiDaS) against oracle.step.train_step in the warm-up (1) and the joint (6) epoch, then
    enough further steps for the CUDA-graph path to capture and replay."""
    from dvd_b200 import synthetic
    from oracle import step
    model, opt, sd_d, sd_m = _build(STEP_CONFIGS[name])
    batch = synthetic.make_batch([(10, 12), (30, 32)], H=H, W=W, seed=11, smooth_flow=True, flow_sigma=2.0)
    ob = {k: (v.squeeze(0) if torch.is_tensor(v) and v.dim() > 0 else v) for k, v in batch.items()}
    log_o, _, _, ex = step.train_step(sd_d, sd_m, ob, opt, epoch)
    log = model._train_on_batch(epoch, 0, batch)
    for k in ('loss', 'flow_loss_1_2', 'disp_loss_1_2', 'sf_loss', 'acc_reg'):
        assert abs(log[k] - log_o[k]) <= 1e-3 * abs(log_o[k]) + 1e-9, (name, epoch, k, log[k], log_o[k])
    grads = dict(model.net_sceneflow.named_parameters())
    for k, ref in ex['grads_mlp'].items():
        assert grads[k].grad.shape == ref.shape, (name, k)
        assert frac_within(grads[k].grad, ref, 5e-3) > 0.99, (name, k)
    for i in range(1, 6):
        log = model._train_on_batch(epoch, i, batch)
        assert all(v == v and abs(v) < float('inf') for k, v in log.items() if isinstance(v, float)), (name, log)
    torch.cuda.synchronize()
    assert model.graph_stats['replayed'] > 0, (name, model.graph_stats)


BASE = ('--net scene_flow_motion_field --dataset synthetic_sequence --gaps 1,2 --n_frames 8 --height 64 --width 96 --epoch_batches 4 '
        '--lr 1e-6 --batch_size 1 --optim adam --gpu 0 --workers 0 --save_net 1 --save_net_opt --one_way --loss_type l1 --l1_mul 0 '
        '--acc_mul 1 --disp_mul 1 --warm_sf 1 --scene_lr_mul 1000 --repeat 1 --flow_mul 1 --sf_mag_div 100 --time_dependent --midas '
        '--use_disp --vis_batches_train 0 --manual_seed 1 --epoch 2 --n_freq_xyz 8 --n_freq_t 4').split()


@pytest.mark.timeout(900)
def test_train_cli_with_a_non_default_encoding(tmp_path):
    logdir = str(tmp_path / 'ckpt')
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', 'dvd_b200.train'] + BASE + ['--logdir', logdir], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    losses = [eval(l.split(':', 1)[1])['loss'] for l in r.stdout.splitlines() if l.startswith('epoch ')]
    assert len(losses) == 2 and all(v == v and v > 0 for v in losses), r.stdout[-1500:]
    full = os.path.join(logdir, 'scene_flow_motion_field_synthetic_sequence', '0')
    sd = torch.load(os.path.join(full, 'checkpoint.pt'), map_location='cpu', weights_only=False)
    mlp = sd['nets'][1]
    assert mlp['convs.0.conv.weight'].shape == (256, 60, 1, 1)
    from dvd_b200.networks.sceneflow_field import SceneFlowFieldNet
    net = SceneFlowFieldNet(net_width=256, n_layers=4, time_dependent=True, N_freq_xyz=8, N_freq_t=4)
    net.load_state_dict(mlp)
    assert all(torch.isfinite(v).all() for v in mlp.values())
