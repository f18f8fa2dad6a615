"""Model plug-in `scene_flow_motion_field` — H100-native mirror of the reference's
models/scene_flow_motion_field.py:32-367 (`Model(VideoBaseModel(NetInterface))`).

Same alias (`--net scene_flow_motion_field`), same flags (dead ones accepted as no-ops), same
`_nets` / `_optimizers` order, same 7-key `batch_log`, same checkpoint layout. What differs is HOW one
step runs:

  reference (≈2000 ATen launches, 7 host syncs)            here
  ------------------------------------------------------   ---------------------------------------------
  net_depth(img_1); net_depth(img_2)     (smf.py:232-238)   ONE forward over the 2B images (BN is in eval mode)
  flow_by_depth → global_p1              (:240-245)         dvd_unproject_fwd
  `steps` MLP evals, each 6 convs+64 trig (:252,:360-367)   dvd_mlp_chain_fwd  (one persistent wgmma kernel)
  scene_flow_projection_slack + _calc_loss (:256-324)       dvd_reproject_loss_fwd (fused, partial sums only)
  loss.backward(retain_graph) + _opt_reg's own backward     ONE backward: the acceleration regulariser reuses
    and 2 extra MLP evals (:192-195,:326-344)                 the chain's s_0, s_1 (identical values) and its
                                                              gradient is merged before the depth-net backward
  13 x pred.cpu().numpy() every step     (:201-202)         only on visualised batches
  5 x .item()                            (:321-323)         one 8-float D2H per step
  2 x torch.optim.Adam over ~430 tensors (:212-213)         dvd_adam_flat on flat buffers (+ NCCL all-reduce)
"""
from os import makedirs
from os.path import join

import numpy as np
import torch

from .netinterface import NetInterface
from .. import ops
from ..flat import FlatAdam, FlatParams
from ..networks.sceneflow_field import SceneFlowFieldNet
from ..third_party.MiDaS import MidasNet
from ..third_party.hourglass import HourglassModel_Embed

try:   # the reference keeps checkpoint locations in configs/__init__.py:15-16
    from configs import depth_pretrain_path, midas_pretrain_path   # noqa: F401
except Exception:   # stand-alone use
    depth_pretrain_path, midas_pretrain_path = None, None


class _AccReg(torch.autograd.Function):
    """Model._opt_reg (smf.py:326-344) on the chain's own (s_0, s_1)."""

    @staticmethod
    def forward(ctx, s0, s1, acc_mul):
        val, g0, g1 = ops.acc_reg(s0.contiguous(), s1.contiguous(), acc_mul)
        ctx.save_for_backward(g0, g1)
        return val.reshape(())

    @staticmethod
    def backward(ctx, g):
        g0, g1 = ctx.saved_tensors
        return g0 * g, g1 * g, None


class _DeferredAdam:
    """Adam whose flat buffers are created when the model reaches its device (`Model.to`)."""

    def __init__(self, net, lr, betas, channels_last=False):
        self.net, self.lr, self.betas, self.channels_last = net, lr, betas, channels_last
        self.flat, self.adam, self._pending = None, None, None

    def materialize(self):
        if self.adam is None:
            self.flat = FlatParams(self.net, channels_last=self.channels_last)
            self.adam = FlatAdam(self.flat, self.lr, self.betas)
            if self._pending is not None:
                self.adam.load_state_dict(self._pending)
                self._pending = None
        return self

    def state_dict(self):
        return self.adam.state_dict() if self.adam is not None else (self._pending or {'state': {}, 'param_groups': []})

    def load_state_dict(self, sd):
        if self.adam is not None:
            self.adam.load_state_dict(sd)
        else:
            self._pending = sd

    def step(self, gscale=1.0):
        self.adam.step(gscale)

    def zero_grad(self):
        self.flat.zero_grad()


class Model(NetInterface):
    @classmethod
    def add_arguments(cls, parser):
        a = parser.add_argument
        # live flags (models/scene_flow_motion_field.py:33-67)
        a('--disp_mul', type=float, default=10, help='disparity multiplier')
        a('--scene_lr_mul', type=float, default=1, help='lr multiplier for scene flow network')
        a('--n_down', type=int, default=3, help='sf net size (FCN variant only)')
        a('--weight_steps', action='store_true', help='weight steps by baselines')
        a('--flow_mul', type=float, default=10, help='multiplier for flow losses')
        a('--acc_mul', type=float, default=100, help='multiplier for acceleration regularization losses')
        a('--interp_steps', type=int, default=5, help='steps for interpolation')
        a('--use_disp', action='store_true', help='flag for using disp losses')
        a('--use_disp_ratio', action='store_true', help='use disp ratio losses')
        a('--time_dependent', action='store_true', help='flag for time dependent scene flow model')
        a('--use_cnn', action='store_true', help='CNN scene-flow model (not implemented here: SURVEY.md §8(f))')
        a('--use_embedding', action='store_true', help='optimizable embedding for each frame')
        a('--use_motion_seg', action='store_true', help='flag for using motion seg')
        a('--warm_reg', action='store_true', help='use reg for warm up as well')
        a('--warm_sf', type=int, default=0, help='warm up flow network for k epochs')
        a('--n_freq_xyz', type=int, default=16, help='xyz_embeddings')
        a('--n_freq_t', type=int, default=16, help='time embeddings')
        a('--sf_mag_div', type=float, default=100, help='divident for sceneflow network output')
        a('--midas', action='store_true', help='use midas for depth prediction')
        # flags the reference parses but never reads — accepted, no effect
        a('--l1_mul', type=float, default=1e-4)
        a('--one_way', action='store_true')
        a('--loss_type', type=str, default='l2')
        a('--sf_min_mul', type=float, default=0)
        a('--sf_quantile', type=float, default=0.5)
        a('--static', action='store_true')
        a('--static_mul', type=float, default=1)
        a('--si_mul', type=float, default=0)
        a('--cos_mul', type=float, default=0)
        a('--motion_seg_hard', action='store_true')
        a('--warm_mul', type=float, default=1)
        a('--warm_static', action='store_true')
        return parser, set()

    def __init__(self, opt, loggers):
        super().__init__(opt, loggers)
        self.input_names = ['img', 'img_1', 'img_2', 'pose', 'intrinsic', 'mask_1', 'mask_2', 'R_1', 'R_1_T', 'R_2',
                            'R_2_T', 't_1', 't_2', 'flow_1_2', 'flow_2_1', 'K', 'K_inv', 'motion_seg_1',
                            'time_stamp_1', 'time_stamp_2', 'frame_id_1', 'frame_id_2', 'time_step']
        self.gt_names = []
        self.requires = list(set().union(self.input_names, self.gt_names))
        if opt.use_cnn:
            raise NotImplementedError('--use_cnn (FCNUnet scene-flow model) is outside the native hot path (SURVEY.md §8(f))')
        if opt.midas:
            resize = [224, 384] if any(k in (opt.dataset or '') for k in ('real_video', 'korean', 'mctest', 'cube')) else None
            self.net_depth = MidasNet(path=midas_pretrain_path, non_negative=True, normalize_input=True, resize=resize)
        else:
            self.net_depth = HourglassModel_Embed(noexp=False, use_embedding=opt.use_embedding)
            if depth_pretrain_path:
                self.net_depth.net_depth.load_state_dict(torch.load(depth_pretrain_path, map_location='cpu'))
        self.net_sceneflow = SceneFlowFieldNet(net_width=256, n_layers=4, time_dependent=opt.time_dependent,
                                               N_freq_xyz=opt.n_freq_xyz, N_freq_t=opt.n_freq_t)
        self.global_rank = getattr(opt, 'global_rank', 0)
        self._nets = [self.net_depth, self.net_sceneflow]
        self.optimizer_depth = _DeferredAdam(self.net_depth, opt.lr, self.optim_params['betas'], channels_last=bool(opt.midas))
        self.optimizer_scene = _DeferredAdam(self.net_sceneflow, opt.lr * opt.scene_lr_mul, self.optim_params['betas'])
        self._optimizers = [self.optimizer_depth, self.optimizer_scene]
        self._metrics = ['flow_loss_1_2', 'loss', 'disp_loss_1_2', 'data_time', 'acc_reg', 'sf_loss']
        self.init_vars(add_path=False)
        self.init_weight(self.net_sceneflow, 'kaiming', 0.01, a=0.2)
        self.visualizer = None
        self.warm = False
        self.steps = 1
        self._world = 1

    # ---- device -------------------------------------------------------------------------------------------
    def to(self, device):
        super().to(device)
        if self.device.type == 'cuda':
            for o in self._optimizers:
                o.materialize()

    def _after_load(self):
        self.net_sceneflow._packed_version = None

    def sync_parameters(self, src=0):
        """train.py:290-292 of the reference broadcasts every tensor; here: one flat broadcast per net."""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            self._world = dist.get_world_size()
            for o in self._optimizers:
                o.materialize().flat.broadcast(src)
            # BatchNorm running statistics are buffers, not parameters: the reference relies on every rank having
            # loaded the same checkpoint (train.py:290-292 broadcasts parameters only); broadcast them as well.
            for net in self._nets:
                for buf in net.buffers():
                    if buf.dtype.is_floating_point:
                        dist.broadcast(buf, src)
            self.net_sceneflow._packed_version = None

    # ---- helpers ------------------------------------------------------------------------------------------
    def _loss_cfg(self):
        o = self.opt
        return ops.make_loss_cfg(midas=o.midas, warm=self.warm, use_disp=o.use_disp, use_disp_ratio=o.use_disp_ratio,
                                 flow_mul=o.flow_mul, disp_mul=o.disp_mul)

    def _set_depth_trainable(self, flag):
        self.net_depth.eval()   # BN is in eval mode in both phases (smf.py:157,168; hourglass.py:200-208)
        for p in self.net_depth.parameters():
            p.requires_grad = flag

    @staticmethod
    def _host_steps(batch):
        """steps = round(mean(ts_2 - ts_1) / time_step) (smf.py:247-250), taken from the batch BEFORE it
        is moved to the device so that no host sync is needed."""
        ts1, ts2, dt = batch['time_stamp_1'], batch['time_stamp_2'], batch['time_step']
        dt = float(dt.reshape(-1)[0]) if torch.is_tensor(dt) else float(dt)
        if 'steps_hint' in batch:   # GPU-resident batches carry the gap so that no device read-back is needed
            return int(batch['steps_hint']), dt
        gap = float((ts2.reshape(ts2.shape[0], -1)[:, 0] - ts1.reshape(ts1.shape[0], -1)[:, 0]).float().mean())
        return int(round(gap / dt)), dt

    def _depths(self, img_1, img_2):
        B = img_1.shape[0]
        if self.opt.midas:
            d = self.net_depth(torch.cat([img_1, img_2], 0))
        else:
            d = self.net_depth(torch.cat([img_1, img_2], 0), None)
        return d[:B].contiguous(), d[B:].contiguous()

    # ---- one optimisation step (smf.py:152-227) --------------------------------------------------------------
    def _step_body(self, inp, steps, dt):
        """Everything of one step that runs on the device, with NO host synchronisation (so it can be captured in a CUDA
        graph): forward, losses, ONE backward, gradient exchange, both Adam updates. `inp` = namespace of device tensors.
        Returns (logs [9] on the device: flow, disp, sf, loss, mask-sum, cf, cd, -, acc_reg; d1, d2, sf, poses for visualisation).
        Under torch.use_deterministic_algorithms(True), read once here, every backward launch of the step takes its ordered
        variant (DESIGN.md 2.11)."""
        with ops.ordered_reductions(torch.are_deterministic_algorithms_enabled()):
            return self._step_launches(inp, steps, dt)

    def _step_launches(self, inp, steps, dt):
        o = self.opt
        for opt_ in self._optimizers:
            opt_.materialize().zero_grad()
        B, _, H, W = inp.img_1.shape
        use_reg = o.interp_steps > 0 and (not self.warm or o.warm_reg) and o.acc_mul > 0
        n_eval = max(steps, 2) if use_reg else steps
        if self.warm:
            with torch.no_grad():
                d1, d2 = self._depths(inp.img_1, inp.img_2)
        else:
            d1, d2 = self._depths(inp.img_1, inp.img_2)
        poses = ops.pack_poses(inp.K, inp.K_inv, inp.R_1_T, inp.R_2_T, inp.t_1, inp.t_2)
        P1 = ops.unproject(d1, poses, 1)
        ts1 = inp.time_stamp_1.contiguous() if o.time_dependent else None
        self.net_sceneflow._packed_version = None   # weights changed behind autograd's back last step: re-pack
        acc, s_steps = self.net_sceneflow.chain(P1, ts1, dt, n_eval, steps, o.sf_mag_div)
        sf = acc
        if o.use_motion_seg:
            sf = sf * inp.motion_seg_1.reshape(B, 1, H, W)
        mask = inp.mask_2.reshape(B, H, W).contiguous()
        loss, scal = ops.reproject_loss(d1, d2, sf, inp.flow_1_2.contiguous(), mask, poses, self._loss_cfg(),
                                        gscale=float(steps) if o.weight_steps else 1.0)
        total = loss
        reg = None
        if use_reg:
            reg = _AccReg.apply(s_steps[0], s_steps[1], float(o.acc_mul))
            total = total + reg
        # gradient exchange (the reference's DDP wrappers are discarded, train.py:284-287; this is what they intended): sum
        # all-reduce of the flat gradient buffers. The depth net's 422 MB go in three buckets, each launched the moment the
        # explicit backward (depth_engine.py) has finished that block - decoder + layer4 (190 MB), layer3 (220 MB), the rest -
        # on NCCL's stream, overlapping the remaining backward; the MLP's 1.2 MB follow the scene-flow chain's backward.
        works = []
        overlap = self._world > 1 and o.midas and not self.warm
        if overlap:
            flat = self.optimizer_depth.flat
            if getattr(self, '_buckets', None) is None:
                r = flat.bucket_ranges(self.net_depth, ['pretrained.layer3.', 'pretrained.layer4.'])
                self._buckets = {'rest': r[0], 'layer3': r[1], 'decoder+layer4': r[2]}
            first = [True]

            def hook(stage):
                if first[0]:      # the scene-flow MLP's gradients were final before the depth net's backward began
                    works.append(self.optimizer_scene.flat.allreduce_grad(async_op=True))
                    first[0] = False
                a, b_ = self._buckets[stage]
                works.append(flat.allreduce_range(a, b_))
            self.net_depth.engine().grad_hook = hook
        total.backward()
        gscale = 1.0
        if self._world > 1:
            if overlap:
                self.net_depth.engine().grad_hook = None
                for w in works:
                    w.wait()
            else:
                for opt_ in self._optimizers:
                    if opt_ is self.optimizer_depth and self.warm:
                        continue
                    opt_.flat.allreduce_grad()
            gscale = 1.0 / self._world
        if not self.warm:
            self.optimizer_depth.step(gscale)
        self.optimizer_scene.step(gscale)
        logs = torch.cat([scal, (reg.detach().reshape(1) if reg is not None else scal.new_zeros(1))])
        return logs, d1.detach(), d2.detach(), sf.detach(), poses

    def _train_on_batch(self, epoch, batch_ind, batch):
        o = self.opt
        self.warm = epoch <= o.warm_sf
        self._set_depth_trainable(not self.warm)
        # the DataLoader's batch dim of 1 is dropped without touching the caller's dict (smf.py:177-179)
        lead = batch['img_1'].dim() == 5
        b = {k: (v.squeeze(0) if (lead and torch.is_tensor(v) and v.dim() > 0) else v) for k, v in batch.items()}
        steps, dt = self._host_steps(b)
        self.steps = steps
        if self._graph_ok():
            logs, vis = self._graph_step(b, steps, dt)
        else:
            self.load_batch(b)
            dev_logs, d1, d2, sf, poses = self._step_body(self._input, steps, dt)
            logs = dev_logs.cpu()    # ONE device->host read per step
            vis = (d1, d2, sf, poses)
        # the Adam step wrote the MLP weights through a raw pointer (no version bump, same address): the cached wgmma pack of
        # the eval forward (`_predict_on_batch`) is stale on both branches - captured graphs re-pack inside `_step_body`
        self.net_sceneflow._packed_version = None
        # `**loss_data` overrides the step-weighted 'loss' in the reference's dict literal (smf.py:226,321)
        has_reg = o.interp_steps > 0 and (not self.warm or o.warm_reg) and o.acc_mul > 0
        batch_log = {'size': o.batch_size, 'loss': float(logs[3]), 'total_loss': float(logs[3]),
                     'flow_loss_1_2': float(logs[0]), 'disp_loss_1_2': float(logs[1]), 'sf_loss': float(logs[2]),
                     'acc_reg': float(logs[8]) if has_reg else 0}

        # smf.py:215-225. Without --vis_at_start the reference counts back from opt.epoch_batches (a TypeError when that is
        # None, so there is no behaviour to keep): no dump then, and only indices 0 <= indx <= vis_batches_train dump.
        vis_every = getattr(o, 'vis_every_train', 0)
        if vis_every and np.mod(epoch, vis_every) == 0 and self.full_logdir:
            if getattr(o, 'vis_at_start', False):
                indx = batch_ind
            else:
                indx = (o.epoch_batches - batch_ind) if getattr(o, 'epoch_batches', None) else -1
            if 0 <= indx <= getattr(o, 'vis_batches_train', 0):
                self.load_batch(b)
                d1, d2, sf, poses = vis
                self._dump_visual(epoch, batch_ind, indx, b, d1, d2, sf, poses)
        return batch_log

    # ---- CUDA-graph replay of the step ------------------------
    # One graph per step signature (pairs, resolution, Euler steps, phase): the ~1200 kernel launches of a step (104 convolutions
    # x {pack, forward, data gradient, weight gradient, column sums} + MLP chain + re-projection + Adam) are captured once and
    # replayed with one cudaGraphLaunch; inputs are copied into static buffers, the 9 log floats come back through a pinned
    # buffer. The first `graph_warmup` steps of a signature run eagerly (they are real optimisation steps), then the next one is
    # captured and replayed. Graphs share one memory pool (they never run concurrently). Single-GPU only: with the NCCL gradient
    # exchange the eager path (which overlaps the all-reduce with the backward) is used.
    _GRAPH_KEYS = ('img_1', 'img_2', 'mask_2', 'R_1_T', 'R_2_T', 't_1', 't_2', 'flow_1_2', 'K', 'K_inv', 'motion_seg_1', 'time_stamp_1')

    def _graph_ok(self):
        # with several ranks the captured step contains the bucketed NCCL all-reduces (side stream forked from and joined to the
        # capture stream): every rank captures at the same step because the step signature (pairs, gap, phase) is rank-uniform
        return (getattr(self.opt, 'cuda_graph', True) and (self._world == 1 or getattr(self.opt, 'cuda_graph_dist', True))
                and self.device.type == 'cuda' and self.opt.midas and not getattr(self, '_graph_broken', False))

    def _graph_sig(self, b, steps, dt):
        sig = (b['img_1'].shape[0], tuple(b['img_1'].shape[-2:]), steps, bool(self.warm), round(float(dt), 9))
        if torch.are_deterministic_algorithms_enabled():
            sig += ('ordered',)    # a graph captured with ordered reductions never replays without them, and vice versa
        return sig

    def _graph_step(self, b, steps, dt):
        sig = self._graph_sig(b, steps, dt)
        if not hasattr(self, '_graphs'):
            self._graphs, self._graph_pool, self.graph_stats = {}, None, {'captured': 0, 'replayed': 0, 'eager': 0}
        ent = self._graphs.setdefault(sig, {'seen': 0, 'graph': None})
        if ent['graph'] is None and ent['seen'] < getattr(self.opt, 'graph_warmup', 2):
            ent['seen'] += 1
            self.graph_stats['eager'] += 1
            self.load_batch(b)
            dev_logs, d1, d2, sf, poses = self._step_body(self._input, steps, dt)
            return dev_logs.cpu(), (d1, d2, sf, poses)
        if ent['graph'] is None:
            static = lambda: None   # noqa: E731
            for k in self._GRAPH_KEYS:
                setattr(static, k, torch.empty(b[k].shape, dtype=torch.float32, device=self.device))
            ent['static'] = static
            ent['pinned'] = torch.empty(9, dtype=torch.float32).pin_memory()
            for k in self._GRAPH_KEYS:
                getattr(static, k).copy_(b[k], non_blocking=True)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            n0 = ops.LAUNCHES['n']
            try:
                # thread_local: NCCL's watchdog thread queries events while this thread captures
                with torch.cuda.graph(g, pool=self._graph_pool, capture_error_mode='thread_local'):
                    dev_logs, d1, d2, sf, poses = self._step_body(static, steps, dt)
                    ent['pinned'].copy_(dev_logs, non_blocking=True)
            except Exception as e:   # noqa: BLE001  capture is an optimisation: report and keep stepping eagerly
                self._graph_broken = True
                self.graph_error = repr(e)[:500]
                torch.cuda.synchronize()
                for o_ in self._optimizers:      # the host-side counters advanced during the aborted capture
                    if o_.adam is not None:
                        o_.adam.step_count -= 0 if (o_ is self.optimizer_depth and self.warm) else 1
                self.load_batch(b)
                dev_logs, d1, d2, sf, poses = self._step_body(self._input, steps, dt)
                return dev_logs.cpu(), (d1, d2, sf, poses)
            if self._graph_pool is None:
                self._graph_pool = g.pool()
            ent.update(graph=g, vis=(d1, d2, sf, poses), launches=ops.LAUNCHES['n'] - n0, captured_now=True)
            self.graph_stats['captured'] += 1
        else:
            for k in self._GRAPH_KEYS:
                getattr(ent['static'], k).copy_(b[k], non_blocking=True)
            ops.LAUNCHES['n'] += ent['launches']
        if ent.pop('captured_now', False):
            pass          # capture recorded the step (and advanced the host-side Adam counters) without executing it
        else:
            if not self.warm:
                self.optimizer_depth.adam.note_replayed()
            self.optimizer_scene.adam.note_replayed()
        ent['graph'].replay()
        self.graph_stats['replayed'] += 1
        torch.cuda.current_stream().synchronize()      # the log of THIS step (NaN guard of the loggers), no run-ahead needed
        return ent['pinned'].clone(), ent['vis']

    def release_graphs(self):
        """Drop every captured step graph (and its static buffers). Required before torch.distributed.destroy_process_group():
        NCCL does not tear a communicator down while CUDA graphs that captured its collectives are alive."""
        if getattr(self, '_graphs', None):
            torch.cuda.synchronize()
            self._graphs.clear()
            self._graph_pool = None
            torch.cuda.synchronize()

    def _dump_visual(self, epoch, batch_ind, indx, batch, d1, d2, sf, poses):
        """The 13 `pred` arrays of the reference (smf.py:201-202, video_base.py:105-126), materialised only
        on visualised batches."""
        inp = self._input
        o = ops.reproject_materialize(d1.contiguous(), d2.contiguous(), inp.flow_1_2.contiguous(), sf.contiguous(), poses)
        pred = {'dflow_1_2': o['dflow_1_2'].permute(0, 2, 3, 1), 'depth_image_1_2': o['depth_image_1_2'],
                'depth_warp_1_2': o['depth_warp_1_2'], 'depth_1': d1, 'depth_2': d2,
                'scenef_1_2': sf.permute(0, 2, 3, 1).unsqueeze(3), 'global_p1': o['global_p1'],
                'staticflow_1_2': o['staticflow_1_2'].permute(0, 2, 3, 1),
                'p1_camera_2': o['p1_camera_2'].permute(0, 2, 3, 1).unsqueeze(3),
                'warped_p2_camera_2': o['warped_p2_camera_2'].permute(0, 2, 3, 1).unsqueeze(3), 'sf_1_2': sf,
                'sf_by_dep_1_2': o['sf_by_depth'].permute(0, 2, 3, 1).unsqueeze(3),
                'sf_loss_pp': (o['sf_by_depth'] - sf).abs().sum(1)}
        out = {k: v.cpu().numpy() for k, v in pred.items()}
        out.update(batch_size=len(batch.get('pair_path', [])), img_1=batch['img_1'].cpu().numpy(),
                   img_2=batch['img_2'].cpu().numpy(), flow_1_2=inp.flow_1_2.cpu().numpy(),
                   flow_2_1=inp.flow_2_1.cpu().numpy(), pair_path=batch.get('pair_path', []))
        if 'depth_pred_1' in batch:
            out['depth_nn_1'] = batch['depth_pred_1'].cpu().numpy()
        outdir = join(self.full_logdir, 'visualize', 'epoch%04d_train' % epoch)
        makedirs(outdir, exist_ok=True)
        if self.global_rank == 0 and self.visualizer is not None:
            # the page images are rendered from the device tensors the npz arrays above were copied from
            dev = dict(pred, img_1=inp.img_1, img_2=inp.img_2, flow_1_2=inp.flow_1_2, flow_2_1=inp.flow_2_1)
            if 'depth_pred_1' in batch:
                dev['depth_nn_1'] = batch['depth_pred_1'].to(self.device)
            self.visualizer.visualize(dev, indx + (1000 * epoch), outdir)
        np.savez(join(outdir, 'rank%04d_batch%04d' % (self.global_rank, batch_ind)), **out)

    # ---- eval / test forward (smf.py:265-276; video_base.py:66-103,128-155) ---------------------------------
    def _predict_on_batch(self, is_train=True):
        if is_train:
            raise RuntimeError('the training forward is fused inside _train_on_batch')
        inp = self._input
        with torch.no_grad():
            depth = self.net_depth(inp.img) if self.opt.midas else self.net_depth(inp.img, None)
            B = depth.shape[0]
            poses = ops.pack_poses(inp.K_inv.reshape(B, 3, 3).transpose(1, 2), inp.K_inv,
                                   inp.R_1.reshape(B, 3, 3).transpose(1, 2), inp.R_1.reshape(B, 3, 3).transpose(1, 2),
                                   inp.t_1, inp.t_1)
            P = ops.unproject_fwd(depth.contiguous(), poses, 1)
            dt = inp.time_step
            dt = float(dt.reshape(-1)[0]) if torch.is_tensor(dt) else float(dt)
            ts = inp.time_stamp_1.contiguous() if self.opt.time_dependent else None
            out = ops.mlp_chain_fwd(self.net_sceneflow.packed(self.opt.sf_mag_div), P, ts, dt, 1, 1, want_steps=False)
        return {'depth': depth, 'sf_1_2': out['acc']}

    @staticmethod
    def depth2disp(depth):
        valid = (depth > 1e-2).float()
        return (1 / (depth + (1 - valid) * 1e-8)) * valid

    def disp_vali(self, d1, d2):
        vali = d2 > 1e-2
        return torch.nn.functional.mse_loss(self.depth2disp(d1) * vali, self.depth2disp(d2) * vali)

    def _vali_on_batch(self, epoch, batch_idx, batch):
        self.eval()
        self.load_batch(batch)
        pred = self._predict_on_batch(is_train=False)
        gt = batch['depth_mvs'].to(pred['depth'].device)
        return {'size': batch['img'].shape[0], 'loss': self.disp_vali(pred['depth'], gt).item()}

    def validate_sequence(self, frames, batch_size=1, chunk=8, epoch=None):
        """The reference's validation pass (train.py:234,319-346 with `_vali_on_batch`) over a device-resident sequence.

        `frames` holds the `vali` items of the dataset stacked along dim 0 (at least 'img' [F,3,H,W] and 'depth_mvs'
        [F,1,H,W], on the model's device). Batches of `batch_size` frames are formed as the reference's loader does
        (drop_last=True). Depth runs `chunk` frames at a time through the inference forward of the depth net (no saved
        activations), and `dvd_disp_vali` writes each frame's squared-error sum into one device buffer that is read back once.

        Returns the reference's `loss_eval`: the size-weighted mean of the per-batch `disp_vali` losses, i.e. the mean per-frame
        MSE over the frames of the complete batches. The step graphs, the MLP's wgmma pack and the nets' train / eval modes are
        left as they were.

        With `epoch` given and a visualizer set, the first `vis_batches_vali` batches of an epoch with epoch % vis_every_vali
        == 0 are also handled as the reference's `_vali_on_batch` visualises them (`_vali_visual`), after the loss."""
        img, gt = frames['img'], frames['depth_mvs']
        n = (img.shape[0] // batch_size) * batch_size
        if n < 1:
            raise ValueError('validate_sequence needs at least one batch of %d frames, got %d' % (batch_size, img.shape[0]))
        if img.device != self.device or gt.device != self.device:
            raise ValueError('validate_sequence expects the frames on %s (move the sequence to the device once)' % self.device)
        H, W = gt.shape[-2:]
        modes = [net.training for net in self._nets]
        for net in self._nets:
            net.eval()
        sse = torch.empty(n, dtype=torch.float32, device=self.device)
        try:
            with torch.no_grad():
                for s in range(0, n, chunk):
                    e = min(s + chunk, n)
                    x = img[s:e]
                    depth = self.net_depth(x) if self.opt.midas else self.net_depth(x, None)
                    ops.disp_vali(depth.contiguous(), gt[s:e].float().contiguous(), out=sse[s:e])
            vis_every = getattr(self.opt, 'vis_every_vali', 0)
            if epoch is not None and self.visualizer is not None and vis_every and epoch % vis_every == 0 and self.full_logdir:
                for bi in range(min(getattr(self.opt, 'vis_batches_vali', 0), n // batch_size)):
                    s, e = bi * batch_size, (bi + 1) * batch_size
                    self._vali_visual(epoch, bi, {k: v[s:e] for k, v in frames.items() if torch.is_tensor(v) or isinstance(v, list)})
                self.visualizer.flush()
        finally:
            for net, m in zip(self._nets, modes):
                net.train(m)
        per_frame = sse.cpu().double() / float(H * W)      # the one read-back of the pass
        batch_losses = per_frame.reshape(-1, batch_size).mean(1)
        return float(batch_losses.mean())

    def _vali_visual(self, epoch, batch_idx, batch):
        """video_base.py:89-99: the page images and `rank%04d_batch%04d.npz` of one validation batch (device tensors)."""
        self.load_batch(batch)
        pred = self._predict_on_batch(is_train=False)
        outdir = join(self.full_logdir, 'visualize', 'epoch%04d_vali' % epoch)
        makedirs(outdir, exist_ok=True)
        dev = dict(pred, img_1=batch['img'], img_2=batch['img'], depth_nn=batch['depth_pred'], depth_gt=batch['depth_mvs'].float())
        self.visualizer.visualize(dev, batch_idx + (1000 * epoch), outdir)
        out = self.pack_output({k: v.cpu().numpy() for k, v in pred.items()}, batch)
        np.savez(join(outdir, 'rank%04d_batch%04d' % (self.global_rank, batch_idx)), **out)

    def pack_output(self, pred_all, batch):
        """video_base.py:105-126 for the per-frame (`img`) batches of the test pass."""
        out = {'batch_size': len(batch['pair_path']), 'img_1': batch['img'].cpu().numpy(), 'img_2': batch['img'].cpu().numpy()}
        out.update(pred_all)
        out['depth_nn'] = batch['depth_pred'].cpu().numpy()
        out['depth_gt'] = batch['depth_mvs'].cpu().numpy()
        out['cam_c2w'] = batch['cam_c2w'].cpu().numpy()
        out['K'] = batch['K'].cpu().numpy()
        out['pair_path'] = batch['pair_path']
        return out

    def test_on_batch(self, batch_idx, batch):
        """Refined depth and scene flow of one per-frame batch. With `opt.output_dir` set (the test driver sets it), also writes
        <output_dir>/epoch{best|%04d}_test/batch%04d.npz with the reference's `pack_output` keys (video_base.py:128-155)."""
        self.eval()
        self.load_batch(batch)
        pred = self._predict_on_batch(is_train=False)
        pred = {k: v.cpu().numpy() for k, v in pred.items()}
        out_root = getattr(self.opt, 'output_dir', None)
        if out_root:
            epoch_string = 'best' if self.opt.epoch < 0 else '%04d' % self.opt.epoch
            outdir = join(out_root, 'epoch%s_test' % epoch_string)
            makedirs(outdir, exist_ok=True)
            output = self.pack_output({k: v.copy() for k, v in pred.items()}, batch)
            if batch_idx == 223:
                # kept on purpose: the reference overwrites the first two depth rows of batch 223 with the third
                # (video_base.py:148-150), so exported files stay interchangeable with its own
                output['depth'][0, 0, 0, :] = output['depth'][0, 0, 2, :]
                output['depth'][0, 0, 1, :] = output['depth'][0, 0, 2, :]
            np.savez(join(outdir, 'batch%04d' % batch_idx), **output)
        return pred
