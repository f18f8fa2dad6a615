"""TEST INFRASTRUCTURE — writes tests/golden/shutterstock_frames_golden.pt by running the UNMODIFIED reference script
scripts/preprocess/shutterstock/generate_frame_midas.py (runpy, CPU) on a synthetic ShutterStock layout.

    python -m oracle.gen_golden_shutterstock

The temporary directory holds datafiles/shutterstock/triangulation/<track>/<track>_<timestamp>.h5 for the five tracks of
oracle.shutterstock_frames.TRACKS: empty files, which only the script's glob sees. Their contents are the seeded arrays of
oracle.shutterstock_frames.synthetic_frame, so the fixture stores checksums of the inputs, not the inputs. The seeded MiDaS
checkpoint (dvd_b200.synthetic.seed_net_, head bias shifted) is written where configs.midas_pretrain_path points; its
weights are not stored, only a checksum.

Shims: `h5py` is a stub module whose File(path) returns a handle of the synthetic arrays (datasets that are truthy and
convert with np.asarray, as h5py's do); the torch.hub ResNeXt of oracle.ref_harness; `.cuda()` as a no-op;
skimage.transform.resize as oracle.frames.sk_resize, the one shim that touches arithmetic (skimage is not installed); and
`tqdm` as a pass-through that, when the save loop of a track starts, copies the script's per-track globals (depths,
scales, s), which the next track overwrites.

Stored per prepared track: the frame order and the script's scales and s; the full-resolution MiDaS depth of the frames
listed in FULL; the written arrays of those frames (img only for the first of them); for every frame, the meta (keys,
shapes, dtypes), intrinsics, pose_c2w and checksums of img, depth_pred and depth_mvs.
"""
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

from . import golden_io
from . import shutterstock_frames as ssf
from .gen_golden_frames import install_shims as install_davis_shims
from .gen_golden_frames import seeded_midas_state, GOLDEN_DIR, WEIGHT_SEED, HEAD_BIAS
from .ref_harness import REF_ROOT

SCRIPT = os.path.join(REF_ROOT, 'scripts', 'preprocess', 'shutterstock', 'generate_frame_midas.py')
# frames (positions in the prepared list) whose full arrays are stored; the others are kept as checksums
FULL = {0: (0, 1, 2), 1: (0, 1, 2), 3: (0, 133), 4: (0, 1, 2)}


class FakeDataset:
    def __init__(self, a):
        self.a = a

    def __bool__(self):
        return True

    def __array__(self, dtype=None, copy=None):
        return self.a if dtype is None else self.a.astype(dtype)


class FakeFile:
    def __init__(self, path, mode='r'):
        track = os.path.basename(os.path.dirname(path))
        t = [x[0] for x in ssf.TRACKS].index(track)
        f = dict(ssf.track_files(t))[os.path.basename(path)]
        self.items = {k: FakeDataset(v) for k, v in ssf.synthetic_frame(t, f).items()}
        self.attrs = {}

    def __getitem__(self, key):
        return self.items[key]


SNAPSHOTS = {}


def tqdm_stub(it, *a, **k):
    if isinstance(it, enumerate):                                      # the save loop: this track's scale is final
        g = sys._getframe(1).f_globals
        SNAPSHOTS[int(g['track_id'])] = dict(depths=[np.array(d) for d in g['depths']], scales=list(g['scales']), s=g['s'])
    return it


def install_shims():
    install_davis_shims()
    sys.modules['h5py'] = types.SimpleNamespace(File=FakeFile)
    sys.modules['tqdm'] = types.SimpleNamespace(tqdm=tqdm_stub)


def checksum(a):
    return float(np.asarray(a).astype(np.float64).sum())


def main():
    install_shims()
    sd = seeded_midas_state()
    out = dict(weight_seed=WEIGHT_SEED, head_bias=HEAD_BIAS,
               weight_checksum=float(sum(v.double().abs().sum() for v in sd.values())), tracks={})
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        for name, *_ in ssf.TRACKS:
            t = [x[0] for x in ssf.TRACKS].index(name)
            d = os.path.join(tmp, 'datafiles', 'shutterstock', 'triangulation', name)
            os.makedirs(d)
            for fn, _ in ssf.track_files(t):
                open(os.path.join(d, fn), 'wb').close()
        os.makedirs(os.path.join(tmp, 'pretrained_depth_ckpt'))
        torch.save(sd, os.path.join(tmp, 'pretrained_depth_ckpt', 'midas_cpkt.pt'))
        os.chdir(tmp)
        try:
            g = runpy.run_path(SCRIPT, run_name='__main__')
        finally:
            os.chdir(cwd)
        names = list(g['track_names'])
        assert names == [x[0] for x in ssf.TRACKS]
        for t, name in enumerate(names):
            order = [dict(ssf.track_files(t))[os.path.basename(p)] for p in g['valid_track_lut'][t]]
            frames_dir = os.path.join(tmp, 'datafiles', 'shutterstock', 'frames_midas', name)
            if not os.path.isdir(frames_dir):
                assert t not in SNAPSHOTS
                out['tracks'][name] = dict(skipped=True, order=order)
                continue
            assert order == ssf.kept_frames(t)
            snap = SNAPSHOTS[t]
            rec = dict(skipped=False, order=order, scales=torch.from_numpy(np.asarray(snap['scales'])),
                       s=torch.from_numpy(np.asarray(snap['s'])), depths={}, frames=[])
            for i in range(len(order)):
                with np.load(os.path.join(frames_dir, 'frame_%05d.npz' % i), allow_pickle=True) as z:
                    a = {k: z[k] for k in z.keys()}
                assert a['motion_seg'].dtype == object and a['motion_seg'].item() is None
                inp = ssf.synthetic_frame(t, order[i])
                assert np.array_equal(a['img_orig'], inp['prediction/img'])
                fr = dict(meta={k: (tuple(v.shape), str(v.dtype)) for k, v in a.items()},
                          intrinsics=torch.from_numpy(a['intrinsics']), pose_c2w=torch.from_numpy(a['pose_c2w']),
                          checksums={k: checksum(a[k]) for k in ('img', 'depth_pred', 'depth_mvs', 'img_orig')})
                if i in FULL[t]:
                    rec['depths'][i] = torch.from_numpy(snap['depths'][i])
                    for k in ('depth_pred', 'depth_mvs') + (('img',) if i == FULL[t][0] else ()):
                        fr[k] = torch.from_numpy(a[k])
                rec['frames'].append(fr)
            out['tracks'][name] = rec
            print('%s: %d frames, s = %r (%s)' % (name, len(order), snap['s'], np.asarray(snap['s']).dtype))
    golden_io.save_golden(out, GOLDEN_DIR, 'shutterstock_frames_golden')


if __name__ == '__main__':
    main()
