"""Write a video's training pairs in the reference's file formats.

    python -m dvd_b200.prepare_pairs --frames <root>/frames_midas/<track> --flows <root>/flow_pairs/<track> \
        --out <root>/sequences_select_pairs_midas/<track>/001 [--flows_out DIR] --gaps 1,2,3,4,5,6,7,8

Reads frame_%05d.npz and flowpair_%05d_%05d.npz (raw flows at any resolution are resized and masked on the GPU, see
flow_pairs.py; with --raft_ckpt instead of --flows the flows are estimated here by dvd_b200.raft from the frames' images) and writes shuffle_False_gap_XX_sequence_XXXXX.pt under --out, plus the finished flowpair_*.npz under
--flows_out when given, so that the reference's own train.py and datasets read what this builds.
"""
import argparse
import time

from .flow_pairs import PairBuilder


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument('--frames', required=True, help='directory of frame_%%05d.npz')
    p.add_argument('--flows', default=None, help='directory of flowpair_%%05d_%%05d.npz (finished or raw flows)')
    p.add_argument('--raft_ckpt', default=None, help='RAFT checkpoint (raft-sintel.pth): estimate the flows instead of reading --flows')
    p.add_argument('--raft_iters', type=int, default=20, help='RAFT update iterations (generate_flows.py:130)')
    p.add_argument('--out', required=True, help='directory for the sequence .pt files')
    p.add_argument('--flows_out', default=None, help='directory for the finished flowpair_*.npz (not written if omitted)')
    p.add_argument('--gaps', default='1,2,3,4,5,6,7,8', help='frame gaps (generate_sequence_midas.py:178)')
    a = p.parse_args(argv)
    if (a.flows is None) == (a.raft_ckpt is None):
        p.error('give exactly one of --flows and --raft_ckpt')
    t0 = time.time()
    raft = None
    if a.raft_ckpt is not None:
        from .raft import load_raft
        raft = load_raft(a.raft_ckpt)
    b = PairBuilder(a.frames, a.flows, [int(g) for g in a.gaps.split(',')], raft=raft, raft_iters=a.raft_iters)
    n = b.write(a.out, a.flows_out)
    print('%d pairs (%d from raw flows) of %d frames written to %s in %.1f s' % (n, b.raw_pairs, int(b.n_frames), a.out,
                                                                                 time.time() - t0))


if __name__ == '__main__':
    main()
