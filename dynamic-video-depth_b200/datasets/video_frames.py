"""A video read straight from its frames and optical flows: davis_sequence's flags and `vali` items, but the `train` pairs are
built at construction by flow_pairs.PairBuilder from <data_root>/frames_midas/<track> and <data_root>/flow_pairs/<track>
(finished flowpair_*.npz as generate_flows.py writes them, or raw flows of any resolution, resized and masked on the GPU).
No sequence .pt files are read or written; item i equals what davis_sequence returns for the file the reference would write.
A track without a flow_pairs/ directory is prepared from its frames alone when --raft_ckpt names a RAFT checkpoint: the flows
are estimated by dvd_b200.raft on the GPU."""
import os

from ..flow_pairs import PairBuilder
from . import davis_sequence


class Dataset(davis_sequence.Dataset):
    @classmethod
    def add_arguments(cls, parser):
        parser, unique = super().add_arguments(parser)
        parser.add_argument('--raft_ckpt', type=str, default=None,
                            help='RAFT checkpoint; used only when the track has no flow_pairs/ directory')
        parser.add_argument('--raft_iters', type=int, default=20, help='RAFT update iterations')
        return parser, unique

    def init_train(self, data_root, track_name):
        gaps = [int(x) for x in self.opt.gaps.split(',')]
        flows_dir, raft = os.path.join(data_root, 'flow_pairs', track_name), None
        if not os.path.isdir(flows_dir):
            ckpt = getattr(self.opt, 'raft_ckpt', None)
            if not ckpt:
                raise FileNotFoundError('%s does not exist: prepare the flows, or give --raft_ckpt to estimate them' % flows_dir)
            from ..raft import load_raft
            flows_dir, raft = None, load_raft(ckpt)
        self.builder = PairBuilder(self.frame_dir, flows_dir, gaps, unit=self.unit, name=track_name, raft=raft,
                                   raft_iters=getattr(self.opt, 'raft_iters', 20))
        self.file_list = list(range(len(self.builder)))
        self.n_frames = self.builder.n_frames

    def train_item(self, idx):
        return self.builder[idx]
