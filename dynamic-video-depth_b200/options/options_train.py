"""Flag surface of the reference's options/options_train.py:23-189, kept name for name: general flags,
then the dataset's and the model's own flags through their `add_arguments` (two-pass parse, :165-189).
`--html_logger` writes the training and validation pages (dvd_b200/train_vis.py). The other flags that only drive
out-of-scope subsystems (CSV / TensorBoard loggers, `--vis_workers`, `--vis_param_f`) are accepted and ignored."""
import argparse
import sys


def add_general_arguments(parser):
    unique_params = {'gpu', 'resume', 'epoch', 'workers', 'batch_size', 'save_net', 'epoch_batches', 'logdir',
                     'pt_no_overwrite', 'full_logdir', 'vis_batches_vali', 'vali_batches', 'vali_at_start', 'vis_every_vali'}
    a = parser.add_argument
    a('--gpu', default='none', type=str, help="gpu to use ('-1' is rejected: dvd_b200 has no CPU path)")
    a('--manual_seed', type=int, default=None)
    a('--deterministic', action='store_true',
      help='bitwise reproducible training on one GPU: torch.use_deterministic_algorithms(True), ordered gradient reductions')
    a('--resume', type=int, default=0, help='0 scratch, -1 last checkpoint, -2 best, N epoch')
    a('--suffix', default='', type=str)
    a('--epoch', type=int, default=0, help='number of epochs to train')
    a('--force_overwrite', action='store_true')
    a('--dataset', type=str, default=None)
    a('--workers', type=int, default=4)
    a('--batch_size', type=int, default=16)
    a('--no_batching', action='store_true')
    a('--epoch_batches', default=None, type=int)
    a('--vali_batches', default=None, type=int)
    a('--vali_at_start', action='store_true')
    a('--log_time', action='store_true')
    a('--print_net', action='store_true')
    a('--multiprocess_distributed', action='store_true')
    a('--world_size', type=int, default=1)
    a('--node_rank', type=int, default=0)
    a('--dist_backend', type=str, default='nccl', choices=['nccl', 'gloo', 'mpi'])
    a('--init_url', type=str, default='tcp://127.0.0.1:60504')
    a('--net', type=str, required=True)
    a('--optim', type=str, default='adam')
    a('--lr', type=float, default=1e-4)
    a('--adam_beta1', type=float, default=0.5)
    a('--adam_beta2', type=float, default=0.9)
    a('--sgd_momentum', type=float, default=0.9)
    a('--sgd_dampening', type=float, default=0)
    a('--wdecay', type=float, default=0.0)
    a('--init_type', type=str, default='normal')
    a('--mixed_precision_training', action='store_true', help='parsed, never read (as in the reference)')
    a('--loss_scaling', type=float, default=255)
    a('--logdir', type=str, default=None)
    a('--full_logdir', type=str, default=None)
    a('--exprdir_no_prefix', action='store_true')
    a('--pt_no_overwrite', action='store_true')
    a('--log_batch', action='store_true')
    a('--progbar_interval', type=float, default=0.05)
    a('--no_accum', action='store_true')
    a('--expr_id', type=int, default=0)
    a('--save_net', type=int, default=1)
    a('--save_net_opt', action='store_true')
    a('--vis_every_vali', default=1, type=int)
    a('--vis_every_train', default=1, type=int)
    a('--vis_batches_vali', type=int, default=10)
    a('--vis_batches_train', type=int, default=10)
    a('--tensorboard', action='store_true')
    a('--tensorboard_keyword', type=str, default='checkpoints')
    a('--html_logger', action='store_true')
    a('--vis_workers', default=2, type=int)
    a('--vis_param_f', default=None, type=str)
    a('--vis_at_start', action='store_true')
    a('--test_template', type=str, default=None)
    # dvd_b200 extensions (the reference ignores unknown flags, options_train.py:184-186)
    a('--resident', action='store_true', help='keep the whole sequence on the GPU and draw gap-bucketed, rank-disjoint batches '
                                              '(datasets/resident.py) instead of one pair file per step through a DataLoader')
    a('--pairs_per_step', type=int, default=1, help='frame pairs per step and GPU with --resident (the reference ships 1 per file)')
    a('--validate', action='store_true', help='validate after every epoch (and before the first with --vali_at_start) on the '
                                              "dataset's vali frames, at most --vali_batches batches, log loss_eval and keep "
                                              'best.pt at the lowest loss_eval (train.py:150-166,319-346 of the reference)')
    return parser, unique_params


def parse(argv=None, get_dataset=None, get_model=None):
    from ..models import get_model as _gm
    from ..datasets import get_dataset as _gd
    get_model, get_dataset = get_model or _gm, get_dataset or _gd
    argv = sys.argv[1:] if argv is None else argv
    parser = argparse.ArgumentParser()
    parser, unique = add_general_arguments(parser)
    first, _ = parser.parse_known_args(argv)
    parser, u_d = get_dataset(first.dataset).add_arguments(parser)
    parser, u_m = get_model(first.net).add_arguments(parser)
    opt, unknown = parser.parse_known_args(argv)
    if unknown:
        print('[warning] ignoring unknown argument', unknown)
    return opt, unique.union(u_d).union(u_m)
