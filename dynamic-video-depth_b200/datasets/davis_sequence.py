"""The reference's DAVIS dataset (datasets/davis_sequence.py): the same flags and the same `train` / `vali` items, read from
the reference's files. `--data_root` replaces its hard-wired './datafiles/davis_processed' (still the default).

  train  one sequence .pt file per item, <data_root>/sequences_select_pairs_midas/<track>/{001|subsample}/
         shuffle_False_gap_XX_*.pt for every gap of --gaps, repeated --repeat times
  vali   one frame per item, <data_root>/frames_midas/<track>/*.npz
"""
import glob
import os

import numpy as np
import torch

from ..flow_pairs import to_dataset_item


class Dataset(torch.utils.data.Dataset):
    DEFAULT_ROOT = './datafiles/davis_processed'

    @classmethod
    def add_arguments(cls, parser):
        parser.add_argument('--cache', action='store_true', help='cache the data into ram')
        parser.add_argument('--subsample', action='store_true', help='subsample the video in time')
        cls.add_track_argument(parser)
        parser.add_argument('--overfit', action='store_true', help='overfit and see if things works')
        parser.add_argument('--gaps', type=str, default='1,2,3,4', help='gaps for sequences')
        parser.add_argument('--repeat', type=int, default=1, help='number of repeatition')
        parser.add_argument('--select', action='store_true', help='pred')
        parser.add_argument('--data_root', type=str, default=cls.DEFAULT_ROOT,
                            help='directory holding frames_midas/, flow_pairs/ and sequences_select_pairs_midas/')
        return parser, set()

    @classmethod
    def add_track_argument(cls, parser):
        parser.add_argument('--track_id', default='train', type=str, help='the track id to load')

    def track_name(self, data_root):
        return self.opt.track_id

    def __init__(self, opt, mode='train', model=None):
        super().__init__()
        self.opt, self.mode = opt, mode
        assert mode in ('train', 'vali')
        data_root = getattr(opt, 'data_root', None) or self.DEFAULT_ROOT
        track_name = self.track_name(data_root)
        if model is None:
            self.required, self.preproc = ['img', 'flow'], None
        elif mode == 'train':
            self.required, self.preproc = getattr(model, 'requires', None), getattr(model, 'preprocess', None)
        else:
            self.required, self.preproc = ['img'], getattr(model, 'preprocess', None)
        self.frame_dir = os.path.join(data_root, 'frames_midas', track_name)
        if mode == 'train':
            self.init_train(data_root, track_name)
        else:
            self.file_list = sorted(glob.glob(os.path.join(self.frame_dir, '*.npz')))
            self.n_frames = len(self.file_list) + 0.0

    def init_train(self, data_root, track_name):
        sub = 'subsample' if self.opt.subsample else '%03d' % 1
        data_path = os.path.join(data_root, 'sequences_select_pairs_midas', track_name, sub)
        self.file_list = []
        for g in [int(x) for x in self.opt.gaps.split(',')]:
            self.file_list += sorted(glob.glob(os.path.join(data_path, 'shuffle_False_gap_%02d_*.pt' % g)))
        self.n_frames = len(sorted(glob.glob(os.path.join(self.frame_dir, '*.npz')))) + 0.0

    def __len__(self):
        return len(self.file_list) if self.mode != 'train' else len(self.file_list) * self.opt.repeat

    @property
    def unit(self):
        return 2.0 if self.opt.subsample else 1.0

    def train_item(self, idx):
        sample = to_dataset_item(torch.load(self.file_list[idx]), self.n_frames, self.unit)
        sample['pair_path'] = self.file_list[idx]
        return sample

    def __getitem__(self, idx):
        idx = idx % self.opt.capat if self.opt.overfit else idx % len(self.file_list)
        if self.mode == 'train':
            return self.train_item(idx)
        d = np.load(self.file_list[idx])
        H, W, _ = d['img'].shape
        s = {'time_stamp_1': np.ones([1, H, W]) * idx / self.n_frames, 'img': np.transpose(d['img'], [2, 0, 1]),
             'frame_id_1': idx, 'time_step': self.unit / self.n_frames, 'depth_pred': d['depth_pred'][None, ...],
             'cam_c2w': d['pose_c2w'], 'depth_mvs': d['depth_mvs'][None, ...]}
        R_1, t_1, K = d['pose_c2w'][:3, :3], d['pose_c2w'][:3, 3], d['intrinsics']
        s['R_1'] = np.broadcast_to(R_1.T, (1, 1, 3, 3)).astype(np.float64)
        s['R_1_T'] = np.broadcast_to(R_1, (1, 1, 3, 3)).astype(np.float64)
        s['t_1'] = np.broadcast_to(t_1, (1, 1, 1, 3)).astype(np.float64)
        s['K'] = np.broadcast_to(K.T, (1, 1, 3, 3)).astype(np.float64)
        s['K_inv'] = np.broadcast_to(np.linalg.inv(K).T, (1, 1, 3, 3)).astype(np.float64)
        s['pair_path'] = self.file_list[idx]
        for k, v in s.items():
            if isinstance(v, np.ndarray):
                s[k] = torch.from_numpy(v).float()
        return s
