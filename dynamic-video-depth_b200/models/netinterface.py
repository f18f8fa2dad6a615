"""NetInterface-compatible training runtime (surface of models/netinterface.py:35-562 of the reference).

Only the surface the driver and the Model plug-in rely on is provided — epoch/batch loop with the
Keras-style logger callbacks, batch loading, device moves, checkpoint save/load in the reference's
`{'nets': [...], 'optimizers': [...], 'epoch': n}` layout. The loggers / visualisers themselves are out
of scope: any object implementing the callback protocol works, including the
reference's own `loggers.ComposeLogger`.
"""
import time

import torch
from torch.nn import init


class NullLogger:
    """Accepts every callback of the reference's logger protocol (loggers/loggers.py:445-515)."""

    def __init__(self):
        self.batch_logs = []
        self.epoch_logs = []

    def add_logger(self, l):
        pass

    def get_html_logger(self):
        return None

    def set_params(self, p):
        self.params = p

    def set_model(self, m):
        pass

    def train(self):
        pass

    def eval(self):
        pass

    def on_train_begin(self, logs=None):
        pass

    def on_train_end(self, logs=None):
        pass

    def on_epoch_begin(self, epoch, logs=None):
        pass

    def on_epoch_end(self, epoch, logs=None):
        self.epoch_logs.append((epoch, logs))

    def on_batch_begin(self, batch, logs=None):
        pass

    def on_batch_end(self, batch, logs=None):
        self.batch_logs.append(logs)


class _EpochMeans:
    """Size-weighted running means of the batch logs (what loggers._LogCumulator provides, :88-110)."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.sums, self.n = {}, 0

    def update(self, log):
        size = log.get('size', 1)
        self.n += size
        for k, v in log.items():
            if k in ('size', 'batch', 'epoch') or not isinstance(v, (int, float)):
                continue
            self.sums[k] = self.sums.get(k, 0.0) + v * size

    def get_epoch_log(self):
        out = {k: v / max(self.n, 1) for k, v in self.sums.items()}
        self.reset()
        return out


class NetInterface(object):
    """Derived classes set `_nets`, `_optimizers`, `_metrics`, `input_names` and implement
    `_train_on_batch` / `_vali_on_batch` / `test_on_batch` (reference contract, netinterface.py:35-50).
    batch_log values are sample-wise means; it must contain 'loss' and 'size'."""

    @staticmethod
    def preprocess(sample_loaded):
        return sample_loaded

    @classmethod
    def add_arguments(cls, parser):
        return parser, set()

    def __init__(self, opt, logger):
        if opt.optim != 'adam':
            raise NotImplementedError('dvd_b200 implements the Adam path of the reference (optimizer %s requested)' % opt.optim)
        self._internal_logger = _EpochMeans()
        if logger is not None and hasattr(logger, 'add_logger'):
            logger.add_logger(self._internal_logger)
        self._logger = logger if logger is not None else NullLogger()
        self.opt = opt
        self.full_logdir = getattr(opt, 'full_logdir', None)
        self._nets, self._optimizers, self._moveable_vars, self._metrics = [], [], [], []
        self.input_names, self.gt_names, self.aux_names = [], [], []
        self._input, self._gt, self._aux = (lambda: None), (lambda: None), (lambda: None)
        self.optim_params = {'betas': (opt.adam_beta1, opt.adam_beta2)}
        self.device = torch.device('cpu')

    # ---- weight init (models/netinterface.py:55-84) -------------------------------------------------
    def init_weight(self, net=None, init_type='kaiming', init_param=0.02, a=0, turnoff_tracking=False):
        def fn(m):
            name = m.__class__.__name__
            if hasattr(m, 'weight') and m.weight is not None and ('Conv' in name or 'Linear' in name):
                if init_type == 'normal':
                    init.normal_(m.weight.data, 0.0, init_param)
                elif init_type == 'xavier':
                    init.xavier_normal_(m.weight.data, gain=init_param)
                elif init_type == 'kaiming':
                    init.kaiming_normal_(m.weight.data, a=a, mode='fan_in')
                elif init_type == 'orth':
                    init.orthogonal_(m.weight.data, gain=init_param)
                else:
                    raise NotImplementedError('initialization method [%s] is not implemented' % init_type)
                if getattr(m, 'bias', None) is not None:
                    init.constant_(m.bias.data, 0.0)
            elif 'BatchNorm' in name and getattr(m, 'affine', False):
                init.normal_(m.weight.data, 1.0, init_param)
                init.constant_(m.bias.data, 0.0)
        (net if net is not None else self.net).apply(fn)

    # ---- batch plumbing (netinterface.py:140-177,442-459) ---------------------------------------------
    def init_vars(self, add_path=True):
        for name in self.input_names:
            setattr(self._input, name, torch.empty(0))
            self._moveable_vars.append('_input.' + name)
        for name in self.gt_names:
            setattr(self._gt, name, torch.empty(0))
            self._moveable_vars.append('_gt.' + name)

    def load_batch(self, batch, include_gt=True):
        """References to the caller's tensors are stored and moved with non_blocking copies; the
        caller's dict is never mutated."""
        for name in self.input_names:
            if name in batch:
                v = batch[name]
                if torch.is_tensor(v):
                    v = v.to(self.device, non_blocking=True)
                setattr(self._input, name, v)
        if include_gt:
            for name in self.gt_names:
                if name in batch:
                    setattr(self._gt, name, batch[name].to(self.device, non_blocking=True))

    def _train_on_batch(self, epoch, batch_ind, batch):
        raise NotImplementedError

    def _vali_on_batch(self, epoch, batch_ind, batch):
        raise NotImplementedError

    def test_on_batch(self, batch_ind, batch):
        raise NotImplementedError

    def _register_tensorboard(self, tblogger):
        self.tensorboard_logger = tblogger

    # ---- epoch loop (netinterface.py:193-360) ---------------------------------------------------------
    def train_epoch(self, dataloader, *, dataloader_vali=None, max_batches_per_train=None, max_batches_per_vali=None,
                    epochs=1, initial_epoch=1, verbose=1, reset_dataset=None, vali_at_start=False, global_rank=0,
                    train_epoch_callback=None):
        logger = self._logger
        steps = len(dataloader) if max_batches_per_train is None else min(max_batches_per_train, len(dataloader))
        steps_eval = 0
        if dataloader_vali is not None:
            steps_eval = len(dataloader_vali) if max_batches_per_vali is None else min(max_batches_per_vali, len(dataloader_vali))
        logger.set_params({'epochs': epochs + initial_epoch - 1, 'steps': steps, 'steps_eval': steps_eval,
                           'samples': steps * getattr(self.opt, 'batch_size', 1),
                           'samples_eval': steps_eval * getattr(self.opt, 'batch_size', 1),
                           'verbose': verbose, 'metrics': self._metrics})
        logger.set_model(self)
        logger.on_train_begin()

        def run(loader, n, epoch, fn, is_train):
            (self.train if is_train else self.eval)()
            (logger.train if is_train else logger.eval)()
            logger.on_epoch_begin(epoch)
            end = time.time()
            for i, data in enumerate(loader):
                if i >= n:
                    break
                t0 = time.time()
                logger.on_batch_begin(i)
                log = fn(epoch, i, data)
                if log is None:
                    raise ValueError('Batch log is not returned by the batch method. Aborting.')
                log.update(batch=i, epoch=epoch, data_time=t0 - end, batch_time=time.time() - t0)
                self._internal_logger.update(log)
                logger.on_batch_end(i, log)
                end = time.time()
            epoch_log = self._internal_logger.get_epoch_log()
            if getattr(self.opt, 'multiprocess_distributed', False):
                epoch_log = self._reduce_epoch_log(epoch_log)
            logger.on_epoch_end(epoch, epoch_log)

        if vali_at_start:
            if dataloader_vali is None:
                raise ValueError('eval_at_beginning is set to True but no eval data is given.')
            run(dataloader_vali, steps_eval, initial_epoch - 1, self._vali_on_batch, False)
        for epoch in range(initial_epoch, initial_epoch + epochs):
            if reset_dataset is not None:
                reset_dataset.reset()
            run(dataloader, steps, epoch, self._train_on_batch, True)
            if getattr(self, 'visualizer', None) is not None:
                self.visualizer.flush()    # the epoch's page images are on disk before the epoch counts as done
            if train_epoch_callback is not None:
                train_epoch_callback(epoch)
            if dataloader_vali is not None:
                run(dataloader_vali, steps_eval, epoch, self._vali_on_batch, False)
        logger.on_train_end()

    def _reduce_epoch_log(self, epoch_log):
        """Mean of the scalar epoch metrics over ranks in ONE small all-reduce (the reference issues one
        dist.reduce per key and then divides by world_size*ngpus, netinterface.py:306-313)."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            return epoch_log
        keys = sorted(epoch_log)
        dev = self.device if self.device.type == 'cuda' else torch.device('cpu')
        v = torch.tensor([float(epoch_log[k]) for k in keys], dtype=torch.float64, device=dev)
        dist.all_reduce(v)
        v = (v / dist.get_world_size()).cpu().tolist()
        return dict(zip(keys, v))

    # ---- mode / device ----------------------------------------------------------------------------------
    def train(self):
        for m in self._nets:
            m.train()

    def eval(self):
        for m in self._nets:
            m.eval()

    def num_parameters(self, return_list=False):
        counts = [sum(p.numel() for p in net.parameters()) for net in self._nets]
        return counts if return_list else sum(counts)

    def to(self, device):
        for net in self._nets:
            net.to(device)
        self.device = torch.device(device)

    def cuda(self):
        self.to(torch.device('cuda', torch.cuda.current_device()))

    def cpu(self):
        self.to(torch.device('cpu'))

    # ---- checkpoints (netinterface.py:528-574) --------------------------------------------------------
    def save_state_dict(self, filepath, *, save_optimizer=False, additional_values={}):
        sd = {'nets': [net.state_dict() for net in self._nets]}
        if save_optimizer:
            sd['optimizers'] = [o.state_dict() for o in self._optimizers]
        sd.update(additional_values)
        torch.save(sd, filepath)

    def load_state_dict(self, filepath, *, load_optimizer='auto'):
        sd = torch.load(filepath, map_location='cpu', weights_only=False)
        if load_optimizer == 'auto':
            load_optimizer = 'optimizers' in sd
        assert len(self._nets) == len(sd['nets'])
        for net, s in zip(self._nets, sd['nets']):
            net.load_state_dict(s)
        if load_optimizer:
            assert len(self._optimizers) == len(sd['optimizers'])
            for o, s in zip(self._optimizers, sd['optimizers']):
                o.load_state_dict(s)   # hyper-parameters (lr) of the current run are kept
        self._after_load()
        return {k: v for k, v in sd.items() if k not in ('optimizers', 'nets')}

    def _after_load(self):
        pass
