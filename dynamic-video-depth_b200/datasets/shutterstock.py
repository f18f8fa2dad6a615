"""The reference's Shutterstock dataset (datasets/shutterstock.py): davis_sequence with an integer --track_id that indexes
the sorted track directories under <data_root>/frames_midas, and './datafiles/shutterstock' as the default --data_root."""
import glob
import os

from . import davis_sequence


class Dataset(davis_sequence.Dataset):
    DEFAULT_ROOT = './datafiles/shutterstock'

    @classmethod
    def add_track_argument(cls, parser):
        parser.add_argument('--track_id', default=0, type=int, help='the track id to load')

    def track_name(self, data_root):
        tracks = sorted(glob.glob(os.path.join(data_root, 'frames_midas', '*')))
        return [x.split('/')[-1] for x in tracks][self.opt.track_id]
