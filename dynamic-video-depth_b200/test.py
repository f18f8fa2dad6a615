"""Test / export driver with the reference's CLI (test.py, options/options_test.py): `python -m dvd_b200.test --net
scene_flow_motion_field --dataset <alias> --checkpoint_path <training log dir> --epoch -1 --output_dir <dir> --batch_size 1
--gpu 0 [dataset flags]`.

Loads the training options from <checkpoint_path>/opt.pt and the weights from best.pt (--epoch < 0) or nets/<epoch>.pt, reads
the dataset's `vali` frames once and keeps them on the GPU, and writes one
<output_dir><net>_<dataset>[_<suffix>]/epoch{best|%04d}_test/batch%04d.npz per batch with the refined depth, the scene flow and
the reference's `pack_output` keys (Model.test_on_batch). The reference's `on_test_end` videos and HTML page are not produced.
"""
import os
from argparse import Namespace
from os.path import join
from shutil import rmtree

import torch

from .datasets import get_dataset
from .models import get_model
from .models.netinterface import NullLogger
from .options import options_test


def output_dir_for(opt):
    """test.py:50-62 of the reference, including its overwrite rule (which looks at epoch_%04d, not at the epoch*_test
    directory the files go to)."""
    out = opt.output_dir
    out += (opt.net + '_' + opt.dataset + '_' + opt.suffix.format(**vars(opt))) if opt.suffix != '' else (opt.net + '_' + opt.dataset)
    if os.path.isdir(join(out, 'epoch_%04d' % opt.epoch)):
        if opt.overwrite:
            rmtree(join(out, 'epoch_%04d' % opt.epoch))
        else:
            raise ValueError('%s already exists, but no overwrite flag' % out)
    os.makedirs(out, exist_ok=True)
    return out


def main(argv=None):
    opt = options_test.parse(argv)
    if opt.gpu == '-1':
        raise SystemExit('dvd_b200 has no CPU path (--gpu -1 is the reference CPU mode; use the reference for that)')
    gpus = [g for g in str(opt.gpu).split(',') if g not in ('none', '')]
    device = torch.device('cuda', int(gpus[0]) if gpus else 0)
    torch.cuda.set_device(device)
    if opt.manual_seed is not None:
        torch.manual_seed(opt.manual_seed)
    output_dir = output_dir_for(opt)

    opt_train = Namespace(**torch.load(join(opt.checkpoint_path, 'opt.pt'), weights_only=False))
    opt_train.global_rank = 0
    opt_train.output_dir = output_dir
    model = get_model(opt.net)(opt_train, NullLogger())
    net_file = join(opt.checkpoint_path, 'best.pt') if opt.epoch < 0 else join(opt.checkpoint_path, 'nets', '%04d.pt' % opt.epoch)
    dataset = get_dataset(opt_train.dataset)(opt_train, mode='vali', model=model)
    loader = torch.utils.data.DataLoader(dataset, batch_size=opt.batch_size, num_workers=opt.workers, pin_memory=True,
                                         drop_last=False, shuffle=False)
    # the whole sequence goes to the GPU once, before the first forward
    batches = [{k: (v.to(device, non_blocking=True) if torch.is_tensor(v) else v) for k, v in b.items()} for b in loader]
    model.load_state_dict(net_file)
    model.to(device)
    model.eval()
    model.opt.epoch = opt.epoch
    for i, batch in enumerate(batches):
        model.test_on_batch(i, batch)
    print('wrote %d batches to %s' % (len(batches), join(output_dir, 'epoch%s_test' % ('best' if opt.epoch < 0 else '%04d' % opt.epoch))))


if __name__ == '__main__':
    main()
