"""Driver with the reference's CLI (train.py:30-364): `python -m dvd_b200.train --net scene_flow_motion_field
--dataset <alias> <flags of experiments/*/train_sequence.sh>`.

One process per GPU. Multi-GPU runs are launched with torchrun (RANK / WORLD_SIZE / LOCAL_RANK) or with the
reference's `--multiprocess_distributed` (mp.spawn). Unlike the reference — whose DistributedDataParallel
wrappers are discarded (train.py:284-287) — gradients really are mean-all-reduced every step (flat buffers,
NCCL over NVLink), after ONE flat parameter broadcast from rank 0.
"""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from .models import get_model
from .datasets import get_dataset
from .models.netinterface import NullLogger
from .options import options_train


def stack_frames(dataset, n, device):
    """The first `n` items of a per-frame (`vali`) dataset as one batch dict (what a DataLoader with batch_size=n yields), its
    tensors moved to `device` once."""
    batch = torch.utils.data.default_collate([dataset[i] for i in range(n)])
    return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in batch.items()}


class _Validator:
    """--validate: the reference's per-epoch validation (train.py:234,319-346) and its best-model rule (ModelSaveLogger with
    save_best, loggers/loggers.py:259-306; train.py:150-166): best.pt is written, with the optimizers, whenever loss_eval is
    strictly lower than the best so far, which on resume is read from the existing best.pt."""

    def __init__(self, opt, model, Dataset, device):
        self.opt, self.model = opt, model
        ds = Dataset(opt, mode='vali', model=model)
        bs = max(1, opt.batch_size)
        n = len(ds) if opt.vali_batches is None else min(len(ds), opt.vali_batches * bs)
        n = (n // bs) * bs                       # the reference's vali loader drops the last incomplete batch
        if n < 1:
            raise SystemExit('--validate: the vali set has %d frames, fewer than one batch of --batch_size %d' % (len(ds), bs))
        self.batch_size = bs
        self.frames = stack_frames(ds, n, device)
        self.best_path = os.path.join(opt.full_logdir, 'best.pt') if opt.full_logdir else None
        self.best = None
        if opt.resume != 0 and self.best_path and os.path.isfile(self.best_path):
            self.best = torch.load(self.best_path, map_location='cpu', weights_only=False).get('loss_eval')
        self.loss_eval = {}

    def __call__(self, epoch):
        v = self.model.validate_sequence(self.frames, batch_size=self.batch_size, epoch=epoch)
        self.loss_eval[epoch] = v
        if self.best_path and (self.best is None or v < self.best):
            self.best = v
            self.model.save_state_dict(self.best_path, save_optimizer=True, additional_values={'epoch': epoch, 'loss_eval': v})


def save_opt(opt):
    """opt.pt (the options as a dict, what the reference's test.py loads) and opt.txt in the log directory (train.py:88-96)."""
    logdir = opt.full_logdir
    if os.path.exists(os.path.join(logdir, 'opt.pt')) and opt.pt_no_overwrite:
        return
    os.makedirs(logdir, exist_ok=True)
    torch.save(vars(opt), os.path.join(logdir, 'opt.pt'))
    with open(os.path.join(logdir, 'opt.txt'), 'w') as fout:
        for k, v in vars(opt).items():
            fout.write('%20s\t%-20s\n' % (k, v))


def main_worker(local_rank, ngpus, opt):
    if opt.deterministic:
        # before CUDA initialises: cuBLAS reads its workspace setting once, and torch raises on a cuBLAS call without it
        os.environ.setdefault('CUBLAS_WORKSPACE_CONFIG', ':4096:8')
        torch.use_deterministic_algorithms(True)
    env_world = int(os.environ.get('WORLD_SIZE', '1'))
    distributed = opt.multiprocess_distributed or env_world > 1
    if opt.gpu == '-1':
        raise SystemExit('dvd_b200 has no CPU path (--gpu -1 is the reference CPU mode; use the reference for that)')
    if distributed:
        if env_world > 1:
            rank, world, local_rank = int(os.environ['RANK']), env_world, int(os.environ.get('LOCAL_RANK', 0))
            dist.init_process_group(opt.dist_backend)
        else:
            world = opt.world_size * ngpus
            rank = opt.node_rank * ngpus + local_rank
            dist.init_process_group(opt.dist_backend, init_method=opt.init_url, world_size=world, rank=rank)
    else:
        rank, world = 0, 1
        local_rank = int(opt.gpu) if opt.gpu not in ('none', '') else 0
    torch.cuda.set_device(local_rank)
    device = torch.device('cuda', local_rank)
    opt.global_rank = rank
    if opt.manual_seed is not None:
        torch.manual_seed(opt.manual_seed + rank)
    logger = NullLogger()
    model = get_model(opt.net)(opt, logger)
    if opt.dataset == 'synthetic_sequence' and opt.resume == 0 and getattr(opt, 'midas', False):
        # no pretrained MiDaS checkpoint ships with the synthetic sequence: with default-initialised weights 10000 / out leaves the
        # valid depth range and every loss is identically zero (SURVEY.md 8(d)) - use the seeded synthetic weights of the benchmark
        from . import synthetic
        synthetic.seed_net_(model.net_depth, opt.manual_seed or 0, 2000.0)
    Dataset = get_dataset(opt.dataset)
    ds = Dataset(opt, mode='train', model=model)
    initial_epoch = 1
    ckpt_dir = os.path.join(opt.full_logdir, 'nets') if opt.full_logdir else None
    if opt.resume != 0 and ckpt_dir:
        name = 'checkpoint.pt' if opt.resume == -1 else ('best.pt' if opt.resume == -2 else '%04d.pt' % opt.resume)
        extra = model.load_state_dict(os.path.join(opt.full_logdir, name if opt.resume < 0 else os.path.join('nets', name)))
        initial_epoch = int(extra.get('epoch', 0)) + 1
    model.to(device)
    sampler = None
    if distributed:
        dist.barrier()
        model.sync_parameters(0)
    if getattr(opt, 'resident', False):
        # SURVEY.md 8(f2) / 8(e): the sequence lives on the GPU, batches are gap-uniform and disjoint across ranks
        from .datasets.resident import GapBucketSampler, ResidentLoader, ResidentSequence
        seq = ResidentSequence(ds, device)
        sampler = GapBucketSampler(seq.gaps, opt.pairs_per_step, world, rank, seed=opt.manual_seed or 0)
        loader = ResidentLoader(seq, sampler)
    else:
        if distributed:
            sampler = torch.utils.data.distributed.DistributedSampler(ds)
        loader = torch.utils.data.DataLoader(ds, batch_size=1, shuffle=sampler is None, sampler=sampler,
                                             num_workers=opt.workers, pin_memory=True, drop_last=True)

    validator = _Validator(opt, model, Dataset, device) if (opt.validate and rank == 0) else None
    if opt.html_logger and rank == 0 and opt.full_logdir:
        from .train_vis import PageWriter
        model.visualizer = PageWriter(opt.full_logdir)

    def on_epoch(epoch):
        if sampler is not None:
            sampler.set_epoch(epoch)
        if rank == 0 and ckpt_dir and opt.save_net > 0 and epoch % opt.save_net == 0:
            os.makedirs(ckpt_dir, exist_ok=True)
            model.save_state_dict(os.path.join(ckpt_dir, '%04d.pt' % epoch), save_optimizer=opt.save_net_opt,
                                  additional_values={'epoch': epoch})
            model.save_state_dict(os.path.join(opt.full_logdir, 'checkpoint.pt'), save_optimizer=True,
                                  additional_values={'epoch': epoch})
        if validator is not None:
            validator(epoch)
    try:
        if validator is not None and opt.vali_at_start:
            validator(initial_epoch - 1)
        model.train_epoch(loader, epochs=opt.epoch, initial_epoch=initial_epoch, max_batches_per_train=opt.epoch_batches,
                          global_rank=rank, train_epoch_callback=on_epoch)
    finally:
        if model.visualizer is not None:
            model.visualizer.close()     # every page image is written (or its failure raised) before the run ends
    if rank == 0 and validator is None:
        for e, log in logger.epoch_logs:
            print('epoch %d:' % e, {k: round(v, 6) for k, v in log.items()})
    elif rank == 0:
        # the validation of epoch e joins that epoch's training log; --vali_at_start adds epoch initial_epoch - 1
        logs = dict(logger.epoch_logs)
        for e in sorted(set(logs) | set(validator.loss_eval)):
            log = {k: round(v, 6) for k, v in logs.get(e, {}).items()}
            if e in validator.loss_eval:
                log['loss_eval'] = validator.loss_eval[e]     # unrounded: it is the value best.pt records
            print('epoch %d:' % e, log)
    if distributed:
        model.release_graphs()
        dist.destroy_process_group()


def main(argv=None):
    opt, _ = options_train.parse(argv)
    if opt.full_logdir is None and opt.logdir:
        opt.full_logdir = os.path.join(opt.logdir, '%s_%s' % (opt.net, opt.dataset), str(opt.expr_id))
    if opt.full_logdir and int(os.environ.get('RANK', '0')) == 0:
        save_opt(opt)
    ngpus = max(1, len([g for g in str(opt.gpu).split(',') if g not in ('none', '')]))
    if opt.multiprocess_distributed and int(os.environ.get('WORLD_SIZE', '1')) == 1:
        mp.spawn(main_worker, nprocs=ngpus, args=(ngpus, opt))
    else:
        main_worker(0, 1, opt)


if __name__ == '__main__':
    mp.set_start_method('spawn', force=True)
    main()
