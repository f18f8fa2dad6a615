"""A video read straight from its frames and optical flows: davis_sequence's flags and `vali` items, but the `train` pairs are
built at construction by flow_pairs.PairBuilder from <data_root>/frames_midas/<track> and <data_root>/flow_pairs/<track>
(finished flowpair_*.npz as generate_flows.py writes them, or raw flows of any resolution, resized and masked on the GPU).
No sequence .pt files are read or written; item i equals what davis_sequence returns for the file the reference would write."""
import os

from ..flow_pairs import PairBuilder
from . import davis_sequence


class Dataset(davis_sequence.Dataset):
    def init_train(self, data_root, track_name):
        gaps = [int(x) for x in self.opt.gaps.split(',')]
        self.builder = PairBuilder(self.frame_dir, os.path.join(data_root, 'flow_pairs', track_name), gaps, unit=self.unit,
                                   name=track_name)
        self.file_list = list(range(len(self.builder)))
        self.n_frames = self.builder.n_frames

    def train_item(self, idx):
        return self.builder[idx]
