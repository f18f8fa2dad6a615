"""Replayed step graphs against eager steps from the same state, and every flat Adam update against its fp32 contract.

bench.py times replays of `Model._graph_step`: static input buffers, one memory pool shared by several graphs, side-stream
weight gradients captured as fork/join, the staged re-projection's pose slots and the device-side Adam counter. Each step
below is teacher-forced: the full training state (flat parameters and gradients, Adam moments, device counter, host counter,
BatchNorm buffers) is snapshot, the step runs eagerly, the snapshot is copied back into the same buffers (the graphs captured
their addresses) and the same batch runs on the graph path - an eager warm-up, the capture or a replay. Training continues
from the graph path's state, so the same model interleaves eager steps and replays, as bench.py's roofline probe does.

Checked at every step:
  * forward, bit for bit: d1, d2, sf and the 9 log floats (every forward kernel is deterministic);
  * gradients of both nets per parameter tensor (slope, relative L2, max-norm), within fp32-atomic-order noise: the two
    eager warm-up steps of each signature measure that noise directly and it is printed;
  * the Adam identity of oracle/adam_fp32.py on both paths, over the whole flat buffer including its zero padding, the
    device counter bit for bit and the host counter; in the warm phase the depth net must not move at all;
  * the graph path was really taken: no capture error, and exact captured / replayed / eager counts.
At the end of each scenario the checkpoint reports the steps taken and loads into torch.optim.Adam, a fresh model loaded from
it takes the next step eagerly with a forward bitwise equal to the original model's replay, and `test_on_batch` runs the MLP
with the current weights.
"""
import pytest
import torch

from oracle.adam_fp32 import check_adam, state_matches

pytestmark = pytest.mark.gpu

# Gradient agreement of a step against the eager step from the same state, per parameter tensor: |slope - 1|, relative L2
# and max-norm error relative to the tensor's maximum. fp32 atomics (convolution and MLP weight gradients, column sums,
# g_depth_2) make two eager runs differ in the last bits. In the depth net those differences flip the TF32 rounding of some
# data-gradient operands and grow through ~100 layers to ~1e-3 relative L2. The bounds are about 4x the largest spread
# between two eager runs measured on an H100 SXM (80 GB HBM3, 700 W power limit), over both scenarios and two runs: depth
# net |slope - 1| 2.3e-4, L2 1.18e-3, max-norm 1.85e-3 (all at 64x96); scene-flow MLP 1.7e-6, 1.7e-6, 1.7e-6 (224x384).
GRAD_BOUND = {'depth': {'slope': 1e-3, 'l2': 5e-3, 'max': 8e-3},
              'scene': {'slope': 7e-6, 'l2': 7e-6, 'max': 7e-6}}


def _squeeze(batch):
    lead = batch['img_1'].dim() == 5
    return {k: (v.squeeze(0) if (lead and torch.is_tensor(v) and v.dim() > 0) else v) for k, v in batch.items()}


def make_batch(pairs, H, W, seed, resident, dev):
    """bench.py's two kinds of batch: host-pinned, or device-resident with `steps_hint` and a host `time_step`."""
    from dvd_b200 import synthetic
    hb = {k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in synthetic.make_batch(pairs, H=H, W=W, seed=seed).items()}
    if not resident:
        return hb
    rb = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in hb.items()}
    rb['time_step'] = hb['time_step']
    rb['steps_hint'] = int(round(float(hb['frame_id_2'].reshape(-1)[0] - hb['frame_id_1'].reshape(-1)[0])))
    return rb


def build_model(opt):
    from dvd_b200 import synthetic
    from dvd_b200.models import get_model
    model = get_model('scene_flow_motion_field')(opt, None)
    synthetic.seed_net_(model.net_depth, 0, 2000.0)
    synthetic.seed_net_(model.net_sceneflow, 1)
    model.to(torch.device('cuda:0'))
    return model


def _segments(flat):
    return [(o, p.numel()) for p, o in zip(flat.params, flat.offsets)]


class Harness:
    """Runs teacher-forced steps of one model and collects every deviation in `problems`."""

    def __init__(self, model, name):
        self.m, self.name = model, name
        self.betas = model.optim_params['betas']
        self.t = {'depth': 0, 'scene': 0}
        self.sig_seen = {}
        self.expect = {'captured': 0, 'replayed': 0, 'eager': 0}
        self.problems = []
        self.spread = {(c, n): {'slope': 0.0, 'l2': 0.0, 'max': 0.0} for c in ('eager', 'graph') for n in ('depth', 'scene')}
        self.adam_worst = {'m_units': 0.0, 'v_units': 0.0, 'p_ratio': 0.0, 'slope_ratio': 0.0}

    def _opts(self):
        return [('depth', self.m.optimizer_depth), ('scene', self.m.optimizer_scene)]

    def snapshot(self):
        s = {}
        for n, o in self._opts():
            a = o.adam
            s[n] = dict(data=o.flat.data.clone(), grad=o.flat.grad.clone(), m=a.exp_avg.clone(), v=a.exp_avg_sq.clone(),
                        state=a.step_state.clone(), count=a.step_count)
        s['bufs'] = [b.clone() for net in self.m._nets for b in net.buffers()]
        return s

    def restore(self, s):
        for n, o in self._opts():
            a, x = o.adam, s[n]
            o.flat.data.copy_(x['data']), o.flat.grad.copy_(x['grad'])
            a.exp_avg.copy_(x['m']), a.exp_avg_sq.copy_(x['v']), a.step_state.copy_(x['state'])
            a.step_count = x['count']
        for b, x in zip([b for net in self.m._nets for b in net.buffers()], s['bufs']):
            b.copy_(x)

    def _sig(self, batch):
        b = _squeeze(batch)
        steps, dt = self.m._host_steps(b)
        return (b['img_1'].shape[0], tuple(b['img_1'].shape[-2:]), steps, bool(self.m.warm), round(float(dt), 9))

    def run(self, epoch, batch, graph, tag):
        """One step on the eager (graph=False) or the graph path. Returns the record of what it computed and left behind."""
        from dvd_b200.models.scene_flow_motion_field import Model
        m = self.m
        m.opt.cuda_graph = graph
        rec = {}

        def body(inp, steps, dt):
            out = Model._step_body(m, inp, steps, dt)
            rec['out'] = out
            return out
        m._step_body = body
        before = dict(getattr(m, 'graph_stats', {'captured': 0, 'replayed': 0, 'eager': 0}))
        try:
            log = m._train_on_batch(epoch, 0, batch)
        finally:
            del m._step_body
        torch.cuda.synchronize()
        kind = 'eager'
        if graph:
            if getattr(m, 'graph_error', None) is not None or getattr(m, '_graph_broken', False):
                self.problems.append('%s: graph path broken: %s' % (tag, getattr(m, 'graph_error', None)))
                raise AssertionError('\n'.join(self.problems))
            st = m.graph_stats
            kind = 'eager' if st['eager'] > before['eager'] else ('capture' if st['captured'] > before['captured'] else 'replay')
        if kind == 'eager':
            logs, d1, d2, sf, _ = rec['out']
            fwd = (logs.cpu(), d1.clone(), d2.clone(), sf.clone())
        else:
            ent = m._graphs.get(self._sig(batch))
            if ent is None or ent.get('graph') is None:
                self.problems.append('%s: no step graph under this batch\'s signature %s (have %s)' % (tag, self._sig(batch), list(m._graphs)))
                raise AssertionError('\n'.join(self.problems))
            fwd = (ent['pinned'].clone(),) + tuple(x.clone() for x in ent['vis'][:3])
        post = {}
        for n, o in self._opts():
            a = o.adam
            post[n] = dict(data=o.flat.data.clone(), grad=o.flat.grad.clone(), m=a.exp_avg.clone(), v=a.exp_avg_sq.clone(),
                           state=a.step_state.clone(), count=a.step_count)
        return {'kind': kind, 'log': log, 'fwd': fwd, 'post': post}

    def check_adam(self, pre, rec, tag):
        m = self.m
        for n, o in self._opts():
            a, x, y = o.adam, pre[n], rec['post'][n]
            t = self.t[n]
            stepped = n == 'scene' or not m.warm
            if not stepped:
                same = all(torch.equal(x[k], y[k]) for k in ('data', 'm', 'v', 'state')) and x['count'] == y['count']
                if not same:
                    self.problems.append('%s: depth net changed in the warm phase' % tag)
                continue
            if y['count'] != t:
                self.problems.append('%s %s: host step_count %d, expected %d' % (tag, n, y['count'], t))
            if not state_matches(y['state'], t, self.betas):
                self.problems.append('%s %s: device counter %s, expected step %d' % (tag, n, y['state'].cpu().tolist(), t))
            r = check_adam(x['data'], x['m'], x['v'], y['grad'], y['data'], y['m'], y['v'], t=t, lr=a.lr, betas=a.betas,
                           eps=a.eps, segments=_segments(o.flat))
            for k in self.adam_worst:
                self.adam_worst[k] = max(self.adam_worst[k], r.get(k, float('inf')))
            for f in r['fail'][:4]:
                self.problems.append('%s %s Adam: %s' % (tag, n, f))

    def compare(self, e, g, tag):
        """g (graph path, or a second eager run) against e (eager) from the same state."""
        for i, (a, b) in enumerate(zip(e['fwd'], g['fwd'])):
            if a.shape != b.shape or not torch.equal(a.view(torch.int32), b.view(torch.int32)):
                what = ('logs', 'd1', 'd2', 'sf')[i]
                diff = float((a.double() - b.double()).abs().max()) if a.shape == b.shape else None
                self.problems.append('%s: %s forward %s differs from eager (max |diff| %s)' % (tag, g['kind'], what, diff))
        if e['log'] != g['log']:
            self.problems.append('%s: batch logs differ: %s vs %s' % (tag, e['log'], g['log']))
        cat = 'eager' if g['kind'] == 'eager' else 'graph'
        for n, o in self._opts():
            ge, gg = e['post'][n]['grad'], g['post'][n]['grad']
            for j, (off, num) in enumerate(_segments(o.flat)):
                a, b = gg[off:off + num].double(), ge[off:off + num].double()
                den = float((b * b).sum())
                if den == 0.0:
                    if bool((a != 0).any()):
                        self.problems.append('%s %s tensor %d: gradient where the eager step has none' % (tag, n, j))
                    continue
                dev = {'slope': abs(float((a * b).sum()) / den - 1.0), 'l2': float(((a - b) ** 2).sum().sqrt()) / den ** 0.5,
                       'max': float((a - b).abs().max() / b.abs().max())}
                for k, v in dev.items():
                    self.spread[cat, n][k] = max(self.spread[cat, n][k], v)
                    if v > GRAD_BOUND[n][k]:
                        self.problems.append('%s %s tensor %d: gradient %s %.3g > %.3g' % (tag, n, j, k, v, GRAD_BOUND[n][k]))

    def step(self, epoch, batch, tag):
        """Teacher-forced pair: eager from the snapshot, then the graph path from the same snapshot; continue from the latter."""
        m = self.m
        m.warm = epoch <= m.opt.warm_sf
        self.t['scene'] += 1
        if not m.warm:
            self.t['depth'] += 1
        pre = self.snapshot()
        e = self.run(epoch, batch, False, tag + ' eager')
        self.check_adam(pre, e, tag + ' eager')
        self.restore(pre)
        sig = self._sig(batch)
        n = self.sig_seen.get(sig, 0)
        self.sig_seen[sig] = n + 1
        want = 'eager' if n < 2 else ('capture' if n == 2 else 'replay')
        self.expect['eager' if want == 'eager' else 'replayed'] += 1
        self.expect['captured'] += want == 'capture'
        g = self.run(epoch, batch, True, tag + ' graph')
        if g['kind'] != want:
            self.problems.append('%s: graph path ran a %s step, expected a %s' % (tag, g['kind'], want))
        if dict(m.graph_stats) != self.expect:
            self.problems.append('%s: graph_stats %s, expected %s' % (tag, m.graph_stats, self.expect))
        self.check_adam(pre, g, tag + ' ' + g['kind'])
        self.compare(e, g, tag)
        del pre, e
        return g


def end_of_scenario(h, epoch, batch, tmp_path):
    """Checkpoint round trip, a fresh model's eager step against the original model's replay, and the eval forward."""
    import copy
    from dvd_b200 import ops
    m = h.m
    f = str(tmp_path / ('%s.pt' % h.name))
    m.save_state_dict(f, save_optimizer=True, additional_values={'epoch': epoch})
    sd = torch.load(f, map_location='cpu', weights_only=False)
    for (n, o), osd, net in zip(h._opts(), sd['optimizers'], m._nets):
        steps = {int(float(s['step'])) for s in osd['state'].values()}
        if steps != ({h.t[n]} if h.t[n] else set()):
            h.problems.append('checkpoint %s reports steps %s, %d taken' % (n, steps, h.t[n]))
        if osd['state']:
            torch.optim.Adam(net.parameters(), lr=o.lr, betas=o.betas).load_state_dict(osd)

    fresh = type(m)(copy.copy(m.opt), None)
    fresh.load_state_dict(f)
    fresh.to(torch.device('cuda:0'))
    hf = Harness(fresh, h.name + ' fresh')
    hf.t = dict(h.t)
    for k in ('depth', 'scene'):
        if k == 'scene' or epoch > m.opt.warm_sf:
            hf.t[k] += 1
    fresh.warm = epoch <= m.opt.warm_sf
    pre_f = hf.snapshot()
    rf = hf.run(epoch, batch, False, 'fresh model')
    hf.check_adam(pre_f, rf, 'fresh model eager')
    del pre_f
    g = h.step(epoch, batch, 'after checkpoint')
    if g['kind'] != 'replay':
        h.problems.append('after checkpoint: the original model ran a %s step, expected a replay' % g['kind'])
    for i, (a, b) in enumerate(zip(g['fwd'], rf['fwd'])):
        if not torch.equal(a.view(torch.int32), b.view(torch.int32)):
            h.problems.append('fresh model: forward %s differs from the original model\'s replay' % ('logs', 'd1', 'd2', 'sf')[i])
    h.problems += hf.problems
    del fresh, hf, rf

    # eval forward after training: the MLP must run with the weights the last Adam step wrote
    b = _squeeze(batch)
    ev = {'img': b['img_1'], 'R_1': b['R_1'], 't_1': b['t_1'], 'K_inv': b['K_inv'], 'time_stamp_1': b['time_stamp_1'],
          'time_step': b['time_step']}
    out = m.test_on_batch(0, ev)
    dev = torch.device('cuda:0')
    with torch.no_grad():
        depth = torch.from_numpy(out['depth']).to(dev).contiguous()
        B = depth.shape[0]
        K_inv, R_1, t_1 = (ev[k].to(dev) for k in ('K_inv', 'R_1', 't_1'))
        Rt = R_1.reshape(B, 3, 3).transpose(1, 2)
        poses = ops.pack_poses(K_inv.reshape(B, 3, 3).transpose(1, 2), K_inv, Rt, Rt, t_1, t_1)
        P = ops.unproject_fwd(depth, poses, 1)
        ts = ev['time_stamp_1'].to(dev).contiguous() if m.opt.time_dependent else None
        dt = float(ev['time_step'].reshape(-1)[0])
        want = ops.mlp_chain_fwd(m.net_sceneflow.packed(m.opt.sf_mag_div, force=True), P, ts, dt, 1, 1, want_steps=False)['acc']
    got = torch.from_numpy(out['sf_1_2']).to(dev)
    if not torch.equal(got.view(torch.int32), want.view(torch.int32)):
        h.problems.append('test_on_batch: sf_1_2 is not the MLP with the current weights (max |diff| %.3g)'
                          % float((got - want).abs().max()))


def report(h):
    for (c, n), s in h.spread.items():
        print('\n[%s] %s gradient spread, %s vs eager: %s' % (h.name, n, c, {k: '%.3g' % v for k, v in s.items()}))
    print('[%s] Adam worst: %s' % (h.name, {k: '%.3g' % v for k, v in h.adam_worst.items()}))
    print('[%s] graph_stats %s' % (h.name, getattr(h.m, 'graph_stats', None)))
    assert not h.problems, '\n'.join(h.problems[:40])


@pytest.mark.timeout(900)
def test_small_replays_match_eager_steps(tmp_path):
    """64x96 (the re-projection's generic path): warm phase then joint phase, three signatures interleaved after capture,
    host-pinned and device-resident batches alternating; lr 1e-4 with scene_lr_mul 10 so one Adam update is well above one
    ulp of a typical weight."""
    from dvd_b200 import synthetic
    dev = torch.device('cuda:0')
    opt = synthetic.default_opt(lr=1e-4, scene_lr_mul=10.0)
    h = Harness(build_model(opt), 'small')
    H, W = 64, 96
    sigs = {'A': [(3, 4)], 'B': [(10, 12), (30, 32)], 'C': [(5, 8), (40, 43)]}
    warm, joint = 1, opt.warm_sf + 1
    sched = [(warm, 'A')] * 4 + [(joint, s) for s in 'AABBCC' + 'ABC' + 'BACACB']
    for i, (epoch, s) in enumerate(sched):
        pairs = [(f + i % 3, f + i % 3 + (g - f)) for f, g in sigs[s]]
        batch = make_batch(pairs, H, W, seed=100 + i, resident=bool(i % 2), dev=dev)
        h.step(epoch, batch, 'step %d (%s, epoch %d)' % (i, s, epoch))
    end_of_scenario(h, joint, make_batch(sigs['B'], H, W, seed=999, resident=True, dev=dev), tmp_path)
    report(h)


@pytest.mark.timeout(1800)
def test_bench_configuration_replays_match_eager_steps(tmp_path):
    """bench.py's configuration: 224x384, 8 pairs, synthetic.default_opt(), joint phase; gaps 8 and 1, largest first. For each
    gap 2 eager steps and the capture, then 3 replays alternating between the gaps. Only at this size does the re-projection
    take its staged path with pose slots."""
    from dvd_b200 import synthetic
    dev = torch.device('cuda:0')
    opt = synthetic.default_opt()
    h = Harness(build_model(opt), 'bench')
    H, W, n_frames = 224, 384, 80
    joint = opt.warm_sf + 1
    gaps = [8, 1] * 6
    for i, gap in enumerate(gaps):
        pairs = [((i * 7 + j) % (n_frames - 1 - gap), (i * 7 + j) % (n_frames - 1 - gap) + gap) for j in range(8)]
        batch = make_batch(pairs, H, W, seed=i, resident=bool(i % 2 == 0), dev=dev)
        h.step(joint, batch, 'step %d (gap %d)' % (i, gap))
    last = [((j * 5) % 70, (j * 5) % 70 + 8) for j in range(8)]
    end_of_scenario(h, joint, make_batch(last, H, W, seed=77, resident=True, dev=dev), tmp_path)
    report(h)
