"""GPU: validation and export — `dvd_disp_vali` (csrc/eval_ops.cu) against its fp32 restatement (oracle/disp_vali.py),
`Model.validate_sequence` against the reference's `_vali_on_batch`, validation between replayed step graphs, the `--validate`
training driver (opt.pt, best.pt) and the `dvd_b200.test` export driver against the CPU oracle and the reference's npz layout."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_err

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32)


def _check_kernel(d, g):
    """terms bitwise, sums within γ_n·Σ|t| of the fp64 sum, a second launch bitwise equal"""
    from dvd_b200 import _lib, ops
    from oracle import disp_vali
    N, _, H, W = d.shape
    sse, terms = ops.disp_vali(d, g, want_terms=True)
    sse2 = ops.disp_vali(d, g)
    torch.cuda.synchronize()
    ref = torch.from_numpy(disp_vali.terms_fp32(d.cpu(), g.cpu()))
    bad = (_bits(terms) != _bits(ref)) & ~(torch.isnan(terms.cpu()) & torch.isnan(ref))
    assert not bad.any(), (int(bad.sum()), bad.nonzero()[:5].tolist())
    assert torch.equal(_bits(sse), _bits(sse2))
    exact, asum = disp_vali.frame_sse_fp64(ref.numpy())
    P = _lib.load().dvd_disp_vali_partials_size(N, H, W) // N
    got = sse.cpu().double().numpy()
    finite = np.isfinite(exact)
    assert (np.abs(got - exact)[finite] <= disp_vali.sum_bound(asum, H, W, P)[finite]).all(), (got, exact)
    return sse


@pytest.mark.parametrize('N,H,W', [(1, 37, 53), (3, 64, 96), (16, 33, 65), (3, 224, 384)])
def test_disp_vali_terms_and_sums(N, H, W):
    from dvd_b200 import synthetic
    d = synthetic.make_depths(N, H, W, seed=11, lo=-0.05, hi=9.0).cuda()
    g = synthetic.make_depths(N, H, W, seed=12, lo=-0.5, hi=8.0).clamp_min(0).cuda()
    # plant exact thresholds, zeros and their neighbours
    t = np.float32(1e-2)
    for i, v in enumerate([t, np.nextafter(t, np.float32(1)), np.nextafter(t, np.float32(0)), 0.0, -0.0, 1e-8]):
        d.view(-1)[i * 7::97] = float(v)
        g.view(-1)[i * 11::89] = float(v)
    _check_kernel(d.contiguous(), g.contiguous())


def test_disp_vali_degenerate_inputs_and_scalar_path():
    from dvd_b200 import ops, synthetic
    N, H, W = 3, 64, 96
    d = synthetic.make_depths(N, H, W, seed=13).cuda()
    g = synthetic.make_depths(N, H, W, seed=14).cuda()
    assert (_check_kernel(d, torch.zeros_like(g)).cpu() == 0).all()          # gt = 0 everywhere: nothing is valid
    s = _check_kernel(torch.zeros_like(d), g)                                  # depth = 0: the term is disp(gt)²
    ref = ((1 / g.double()) ** 2).reshape(N, -1).sum(1).cpu()
    assert rel_err(s, ref) < 1e-5
    # storage offset of one element: neither pointer is 16-byte aligned, the scalar path runs
    buf_d = torch.empty(N * H * W + 1, device='cuda')
    buf_g = torch.empty(N * H * W + 1, device='cuda')
    dd, gg = buf_d[1:].view(N, 1, H, W), buf_g[1:].view(N, 1, H, W)
    dd.copy_(d), gg.copy_(g)
    assert rel_err(_check_kernel(dd, gg), ops.disp_vali(d, g)) < 1e-5       # same terms, another summation order
    # caller-owned output slice
    out = torch.full((N + 2,), -1.0, device='cuda')
    ops.disp_vali(d, g, out=out[1:N + 1])
    assert out[0].item() == -1 and out[-1].item() == -1 and torch.equal(_bits(out[1:N + 1]), _bits(ops.disp_vali(d, g)))


def test_disp_vali_argument_checks():
    from dvd_b200 import _lib, ops
    lib = _lib.load()
    x = torch.ones(2, 1, 8, 8, device='cuda')
    p = ctypes.c_void_p
    assert lib.dvd_disp_vali(p(x.data_ptr()), None, p(x.data_ptr()), None, p(x.data_ptr()), 2, 8, 8, None) == -2
    assert b'null pointer' in lib.dvd_last_error()
    assert lib.dvd_disp_vali(p(x.data_ptr()), p(x.data_ptr()), p(x.data_ptr()), None, p(x.data_ptr()), 0, 8, 8, None) == -2
    assert lib.dvd_disp_vali_partials_size(0, 8, 8) == -1
    with pytest.raises(ValueError):
        ops.disp_vali(x, torch.ones(2, 1, 8, 9, device='cuda'))
    with pytest.raises(ValueError):
        ops.disp_vali(x.cpu(), x.cpu())


def _seeded_model(**over):
    from dvd_b200 import synthetic
    from dvd_b200.models import get_model
    model = get_model('scene_flow_motion_field')(synthetic.default_opt(**over), None)
    synthetic.seed_net_(model.net_depth, 0, 2000.0)
    synthetic.seed_net_(model.net_sceneflow, 1)
    model.to(torch.device('cuda:0'))
    return model


def _frames(n, H, W, n_frames=None):
    from dvd_b200 import synthetic
    from dvd_b200.train import stack_frames
    return stack_frames([synthetic.make_frame(i, H=H, W=W, n_frames=n_frames or n) for i in range(n)], n, torch.device('cuda:0'))


def test_validate_sequence_equals_the_mean_of_vali_on_batch():
    from oracle import disp_vali
    model = _seeded_model()
    H, W, n = 64, 96, 5
    fr = _frames(n, H, W)
    per = []
    for i in range(n):
        batch = {k: (v[i:i + 1] if torch.is_tensor(v) else v[i:i + 1]) for k, v in fr.items()}
        per.append(model._vali_on_batch(1, i, batch)['loss'])
    ref = sum(per) / n
    bound = 2 * disp_vali.gamma(H * W) * ref            # both sides are fp32 sums of the same non-negative terms
    model.train()
    v1 = model.validate_sequence(fr, chunk=1)
    assert abs(v1 - ref) <= bound, (v1, ref, bound)
    assert all(net.training for net in model._nets)     # the nets' modes are restored
    v4 = model.validate_sequence(fr, chunk=4)           # other forward batch sizes: the same depth up to convolution order
    assert abs(v4 - ref) <= 1e-4 * ref, (v4, ref)
    assert model.validate_sequence(fr, chunk=1) == v1   # reproducible
    # batches of 2 with drop_last: the mean over the first 4 frames
    v2 = model.validate_sequence(fr, batch_size=2, chunk=1)
    assert abs(v2 - sum(per[:4]) / 4) <= bound
    with pytest.raises(ValueError):
        model.validate_sequence({k: v.cpu() if torch.is_tensor(v) else v for k, v in fr.items()})


def test_validation_between_replayed_steps_leaves_the_next_step_unchanged():
    """snapshot method of test_step_graph_replay_gpu.py: the same replayed step from the same state, once without and once
    after a validation pass, must compute a bitwise-equal forward"""
    from dvd_b200 import synthetic
    model = _seeded_model(full_logdir=None)
    batch = synthetic.make_batch([(3, 5)], H=64, W=96, seed=2)
    fr = _frames(4, 64, 96)
    for i in range(4):                  # eager, eager, capture, replay
        model._train_on_batch(6, i, batch)
    assert model.graph_stats['replayed'] >= 1 and model.graph_stats['captured'] == 1

    def snapshot():
        s = {}
        for n, o in (('depth', model.optimizer_depth), ('scene', model.optimizer_scene)):
            a = o.adam
            s[n] = dict(data=o.flat.data.clone(), grad=o.flat.grad.clone(), m=a.exp_avg.clone(), v=a.exp_avg_sq.clone(),
                        state=a.step_state.clone(), count=a.step_count)
        s['bufs'] = [b.clone() for net in model._nets for b in net.buffers()]
        return s

    def restore(s):
        for n, o in (('depth', model.optimizer_depth), ('scene', model.optimizer_scene)):
            a, x = o.adam, s[n]
            o.flat.data.copy_(x['data']), o.flat.grad.copy_(x['grad'])
            a.exp_avg.copy_(x['m']), a.exp_avg_sq.copy_(x['v']), a.step_state.copy_(x['state'])
            a.step_count = x['count']
        for b, x in zip([b for net in model._nets for b in net.buffers()], s['bufs']):
            b.copy_(x)
        torch.cuda.synchronize()

    def step():
        before = model.graph_stats['replayed']
        log = model._train_on_batch(6, 9, batch)
        torch.cuda.synchronize()
        assert model.graph_stats['replayed'] == before + 1
        ent = next(e for e in model._graphs.values() if e.get('graph') is not None)
        return log, [t.clone() for t in ent['vis'][:3]]

    snap = snapshot()
    log_a, fwd_a = step()
    restore(snap)
    v = model.validate_sequence(fr, chunk=2)
    assert v == v and v > 0
    log_b, fwd_b = step()
    assert log_a == log_b
    for x, y in zip(fwd_a, fwd_b):
        assert torch.equal(_bits(x), _bits(y))
    # the eval forward after the steps runs the MLP with the current weights and still matches the oracle path
    assert model.graph_stats['eager'] == 2 and model.graph_stats['captured'] == 1


BASE = ('--net scene_flow_motion_field --dataset synthetic_sequence --gaps 1,2 --n_frames 8 --height 64 --width 96 --epoch_batches 4 '
        '--lr 1e-6 --batch_size 1 --optim adam --gpu 0 --workers 0 --save_net 1 --save_net_opt --one_way --loss_type l1 --l1_mul 0 '
        '--acc_mul 1 --disp_mul 1 --warm_sf 1 --scene_lr_mul 1000 --repeat 1 --flow_mul 1 --sf_mag_div 100 --time_dependent --midas '
        '--use_disp --vis_batches_train 0 --manual_seed 1').split()


def _run(module, args):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', module] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    return r.stdout


def _epochs(out):
    res = {}
    for line in out.splitlines():
        if line.startswith('epoch '):
            res[int(line.split()[1].rstrip(':'))] = eval(line.split(':', 1)[1])
    return res


@pytest.mark.timeout(2400)
def test_train_validate_best_checkpoint_and_test_export(tmp_path):
    from oracle.gen_golden_eval import oracle_forward
    from oracle.golden_io import load_golden
    # --validate: loss_eval in every epoch log (epoch 0 from --vali_at_start), best.pt at the lowest one
    logdir = str(tmp_path / 'val')
    ep = _epochs(_run('dvd_b200.train', BASE + ['--logdir', logdir, '--epoch', '2', '--validate', '--vali_at_start',
                                                '--vali_batches', '6']))
    assert sorted(ep) == [0, 1, 2] and all(v['loss_eval'] > 0 for v in ep.values()), ep
    full = os.path.join(logdir, 'scene_flow_motion_field_synthetic_sequence', '0')
    opt = torch.load(os.path.join(full, 'opt.pt'))
    assert opt['validate'] and opt['n_frames'] == 8 and os.path.exists(os.path.join(full, 'opt.txt'))
    best = torch.load(os.path.join(full, 'best.pt'), map_location='cpu', weights_only=False)
    assert set(best) == {'nets', 'optimizers', 'epoch', 'loss_eval'}
    e_best = min(ep, key=lambda e: ep[e]['loss_eval'])
    assert best['epoch'] == e_best and best['loss_eval'] == ep[e_best]['loss_eval'], (best['epoch'], best['loss_eval'], ep)

    # the same run without --validate: no best.pt, and the same training logs
    plain = str(tmp_path / 'plain')
    ep_plain = _epochs(_run('dvd_b200.train', BASE + ['--logdir', plain, '--epoch', '2']))
    full_plain = os.path.join(plain, 'scene_flow_motion_field_synthetic_sequence', '0')
    assert not os.path.exists(os.path.join(full_plain, 'best.pt')) and os.path.exists(os.path.join(full_plain, 'opt.pt'))
    assert sorted(ep_plain) == [1, 2]
    # epoch 1 (warm-up, depth net frozen) agrees to the printed precision. Epoch 2 trains the depth net, whose weight gradients
    # are summed with fp32 atomics, so two runs of the same command differ there (1.0e-4 relative in disp_loss_1_2 seen on an
    # H100); a validation that moved weights, consumed the sampler's RNG or changed a phase would show at epoch 1 already.
    for e, tol in ((1, 5e-5), (2, 1e-3)):
        a, b = ep_plain[e], {k: v for k, v in ep[e].items() if k != 'loss_eval'}
        assert set(a) == set(b)
        for k in ('loss', 'flow_loss_1_2', 'disp_loss_1_2', 'sf_loss', 'acc_reg'):
            assert abs(a[k] - b[k]) <= 2e-6 + tol * abs(a[k]), (e, k, a[k], b[k])

    # test / export driver on best.pt
    out_root = str(tmp_path / 'test') + '/'
    _run('dvd_b200.test', ['--net', 'scene_flow_motion_field', '--dataset', 'synthetic_sequence', '--checkpoint_path', full,
                           '--epoch', '-1', '--batch_size', '1', '--output_dir', out_root, '--gpu', '0', '--workers', '0',
                           '--html_logger', '--manual_seed', '3'])
    outdir = os.path.join(out_root + 'scene_flow_motion_field_synthetic_sequence_epoch_-1', 'epochbest_test')
    files = sorted(os.listdir(outdir))
    assert files == ['batch%04d.npz' % i for i in range(8)], files
    gold = load_golden(GOLDEN, 'eval_export_golden')
    model = _seeded_model()
    model.load_state_dict(os.path.join(full, 'best.pt'))
    sd_d = {k: v.cpu() for k, v in model.net_depth.state_dict().items()}
    sd_m = {k: v.cpu() for k, v in model.net_sceneflow.state_dict().items()}
    fr = _frames(8, 64, 96)
    for i, f in enumerate(files):
        z = np.load(os.path.join(outdir, f))
        assert {k: (tuple(z[k].shape), z[k].dtype.str) for k in z.files} == gold['layout']
        batch = {k: (v[i:i + 1] if torch.is_tensor(v) else v[i:i + 1]) for k, v in fr.items()}
        d, sf = oracle_forward(sd_d, sd_m, batch)
        assert rel_err(torch.from_numpy(z['depth']), d) < 1e-3
        assert rel_err(torch.from_numpy(z['sf_1_2']), sf) < 1e-2
        assert np.array_equal(z['depth_gt'], batch['depth_mvs'].cpu().numpy()) and str(z['pair_path'][0]) == batch['pair_path'][0]


def test_test_on_batch_export_matches_the_reference_files(tmp_path):
    """the reference's own exported depth / scene flow (tests/golden/eval_export_golden.pt) on the same seeded weights"""
    from oracle.golden_io import load_golden
    gold = load_golden(GOLDEN, 'eval_export_golden')
    m = gold['meta']
    model = _seeded_model(output_dir=str(tmp_path), epoch=-1)
    fr = _frames(m['n_frames'], m['H'], m['W'])
    for i in range(m['n_frames']):
        ret = model.test_on_batch(i, {k: v[i:i + 1] for k, v in fr.items()})
        z = np.load(os.path.join(str(tmp_path), 'epochbest_test', 'batch%04d.npz' % i))
        assert {k: (tuple(z[k].shape), z[k].dtype.str) for k in z.files} == gold['layout']
        assert np.array_equal(z['depth'], ret['depth']) and np.array_equal(z['sf_1_2'], ret['sf_1_2'])
        assert rel_err(torch.from_numpy(z['depth']), gold['depth'][i:i + 1]) < 1e-3
        assert rel_err(torch.from_numpy(z['sf_1_2']), gold['sf_1_2'][i:i + 1]) < 1e-2
    # the reference's batch-223 row copy (video_base.py:148-150) goes to the file only
    model.opt.epoch = 7
    ret = model.test_on_batch(223, {k: v[:1] for k, v in fr.items()})
    z = np.load(os.path.join(str(tmp_path), 'epoch0007_test', 'batch0223.npz'))
    assert np.array_equal(z['depth'][0, 0, 0], ret['depth'][0, 0, 2]) and np.array_equal(z['depth'][0, 0, 1], ret['depth'][0, 0, 2])
    assert np.array_equal(z['depth'][0, 0, 2:], ret['depth'][0, 0, 2:]) and not np.array_equal(ret['depth'][0, 0, 0], ret['depth'][0, 0, 2])
