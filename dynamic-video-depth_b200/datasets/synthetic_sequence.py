"""Synthetic stand-in for datasets/davis_sequence.py: yields batch dicts of the reference's pair-file
format (keys / shapes of datasets/davis_sequence.py:86-113) for an `n_frames`-frame sequence.

mode='vali' yields one frame per item with the keys of davis_sequence's `vali` items (davis_sequence.py:117-152), a seeded
synthetic `depth_mvs` included (about 10 % of its pixels are 0, i.e. invalid)."""
import torch

from .. import synthetic


class Dataset(torch.utils.data.Dataset):
    @classmethod
    def add_arguments(cls, parser):
        parser.add_argument('--gaps', type=str, default='1,2,3,4', help='gaps for sequences')
        parser.add_argument('--repeat', type=int, default=1)
        parser.add_argument('--n_frames', type=int, default=80)
        parser.add_argument('--height', type=int, default=224)
        parser.add_argument('--width', type=int, default=384)
        parser.add_argument('--track_id', default='train', type=str)
        return parser, set()

    def __init__(self, opt, mode='train', model=None):
        assert mode in ('train', 'vali')
        self.opt, self.mode = opt, mode
        gaps = [int(g) for g in str(opt.gaps).split(',')]
        self.pairs = synthetic.pair_list(opt.n_frames, gaps)
        self.n_frames = float(opt.n_frames)

    def __len__(self):
        if self.mode == 'vali':
            return int(self.n_frames)
        return len(self.pairs) * max(1, getattr(self.opt, 'repeat', 1))

    def __getitem__(self, idx):
        if self.mode == 'vali':
            return synthetic.make_frame(idx, H=self.opt.height, W=self.opt.width, n_frames=int(self.n_frames))
        pair = self.pairs[idx % len(self.pairs)]
        b = synthetic.make_batch([pair], H=self.opt.height, W=self.opt.width, n_frames=int(self.n_frames), seed=idx,
                                 leading_dim=False)
        b['time_step'] = float(b['time_step'])
        return b
