"""TEST INFRASTRUCTURE — writes tests/golden/frames_golden.pt by running the UNMODIFIED reference script
scripts/preprocess/davis/generate_frame_midas.py (runpy, CPU) on a synthetic DAVIS layout.

    python -m oracle.gen_golden_frames

The temporary directory holds datafiles/DAVIS/{JPEGImages,Annotations}/1080p/<track> and triangulation/<track>.* for the two
track names the script hard-codes, `train` and `dog`: 3 frames each at 160x400 (W > 384: working size 128x384), JPEG frames,
RGB PNG masks with an object region (so that the mask test rejects points), and a vertex set with points behind the camera
and outside the image. The seeded MiDaS checkpoint (dvd_b200.synthetic.seed_net_, head bias shifted) is written where
configs.midas_pretrain_path points; its weights are not stored, only a checksum.

Shims: the torch.hub ResNeXt of oracle.ref_harness; `.cuda()` as a no-op; `trimesh.load` as a reader of the `v` lines; and
skimage.transform.resize as oracle.frames.sk_resize, the scipy calls of skimage >= 0.19 — the only shim that touches
arithmetic (skimage is not installed).

Stored: every input file's bytes, the written arrays of both tracks (img_orig as a checksum; the full working-size img of
`dog`, a checksum of `train`'s), and from the run's globals after the last track: full_pred_depths, pts_list, mvs_depths,
pred_depths, scales, s, intrinsics, extrinsics (scaled in place by the script's save loop) and h_pt.
"""
import io
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch
from PIL import Image

from . import golden_io
from . import frames as oracle_frames
from .ref_harness import REF_ROOT, import_reference

TRACKS = ('train', 'dog')
H, W, N_FRAMES, N_POINTS = 160, 400, 3, 3000
WEIGHT_SEED, HEAD_BIAS = 0, 2000.0
SCRIPT = os.path.join(REF_ROOT, 'scripts', 'preprocess', 'davis', 'generate_frame_midas.py')
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')


def seeded_midas_state():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from dvd_b200 import synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    return synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True), WEIGHT_SEED, HEAD_BIAS).state_dict()


def synthetic_track(t):
    """-> {relative path: bytes} of one track."""
    g = np.random.default_rng(10 + t)
    name = TRACKS[t]
    files = {}
    yy, xx = np.mgrid[0:H, 0:W]
    for f in range(N_FRAMES):
        base = np.stack([np.sin(xx / (17.0 + 3 * c) + f * 0.3 + t) * np.cos(yy / (11.0 + 2 * c)) for c in range(3)], -1)
        img = np.clip(127.5 + 90 * base + g.normal(0, 12, base.shape), 0, 255).astype(np.uint8)
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format='JPEG', quality=92)
        files['JPEGImages/1080p/%s/%05d.jpg' % (name, f)] = buf.getvalue()
        mask = np.zeros((H, W, 3), np.uint8)
        mask[40 + 5 * f:110 + 5 * f, 150 + 10 * f:260 + 10 * f, 0] = 255
        mask[60:70, 20:40, :] = 128                                     # a grey region: partial mask values
        buf = io.BytesIO()
        Image.fromarray(mask).save(buf, format='PNG')
        files['Annotations/1080p/%s/%05d.png' % (name, f)] = buf.getvalue()
    files['triangulation/%s.intrinsics.txt' % name] = ''.join('%d %.6f %.6f %.6f %.6f\n' % (f, 310.0 + t, 305.5, 199.25, 81.5)
                                                              for f in range(N_FRAMES)).encode()
    rows = []
    for f in range(N_FRAMES):
        a = 0.02 * f + 0.01 * t
        c2w = np.eye(4)
        c2w[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
        c2w[:3, 3] = [0.1 * f, 0.02 * f, 0.05 * t]
        rows.append('%d ' % f + ' '.join('%.12g' % v for v in c2w.reshape(-1)))
    files['triangulation/%s.matrices.txt' % name] = ('\n'.join(rows) + '\n').encode()
    pts = np.stack([g.uniform(-5, 5, N_POINTS), g.uniform(-2.5, 2.5, N_POINTS), g.uniform(-9, -1.5, N_POINTS)], 1)
    pts[:200, 2] = g.uniform(0.5, 3, 200)                                # behind the camera
    files['triangulation/%s.obj' % name] = ''.join('v %.9g %.9g %.9g\n' % tuple(p) for p in pts).encode() + b'f 1 2 3\n'
    assert len(np.unique(pts, axis=0)) == N_POINTS                       # trimesh could merge repeated vertices
    return files


def _obj_vertices(path):
    return np.asarray([[float(x) for x in ln.split()[1:4]] for ln in open(path) if ln.startswith('v ')], dtype=np.float64)


def install_shims():
    import_reference()                                                    # reference modules + the hub ResNeXt shim
    torch.nn.Module.cuda = lambda self, *a, **k: self
    torch.Tensor.cuda = lambda self, *a, **k: self
    sys.modules['trimesh'] = types.SimpleNamespace(load=lambda p: types.SimpleNamespace(vertices=_obj_vertices(p)))
    sk = types.ModuleType('skimage')
    sk.transform = types.ModuleType('skimage.transform')
    sk.transform.resize = lambda image, output_shape, preserve_range=True: oracle_frames.sk_resize(image, output_shape)
    sys.modules.update({'skimage': sk, 'skimage.transform': sk.transform})


def as_u8(b):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).clone()


def main():
    install_shims()
    sd = seeded_midas_state()
    out = dict(H=H, W=W, weight_seed=WEIGHT_SEED, head_bias=HEAD_BIAS,
               weight_checksum=float(sum(v.double().abs().sum() for v in sd.values())), inputs={}, outputs={})
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        for t in range(len(TRACKS)):
            for rel, data in synthetic_track(t).items():
                path = os.path.join(tmp, 'datafiles', 'DAVIS', rel)
                os.makedirs(os.path.dirname(path), exist_ok=True)
                with open(path, 'wb') as f:
                    f.write(data)
                out['inputs'][rel] = as_u8(data)
        os.makedirs(os.path.join(tmp, 'pretrained_depth_ckpt'))
        torch.save(sd, os.path.join(tmp, 'pretrained_depth_ckpt', 'midas_cpkt.pt'))
        os.chdir(tmp)
        try:
            g = runpy.run_path(SCRIPT, run_name='__main__')
        finally:
            os.chdir(cwd)
        for name in TRACKS:
            frames = []
            for f in range(N_FRAMES):
                with np.load(os.path.join(tmp, 'datafiles', 'davis_processed', 'frames_midas', name, 'frame_%05d.npz' % f)) as d:
                    a = {k: d[k] for k in d.keys()}
                assert np.array_equal(a['depth_mvs'], a['depth_pred'])
                rec = {k: torch.from_numpy(a[k]) for k in ('pose_c2w', 'intrinsics', 'depth_pred')}
                rec['motion_seg'] = torch.from_numpy(a['motion_seg'].astype(np.uint8))
                rec['meta'] = {k: (tuple(v.shape), str(v.dtype)) for k, v in a.items()}
                rec['img_orig_checksum'] = float(a['img_orig'].astype(np.float64).sum())
                rec['img_checksum'] = float(a['img'].astype(np.float64).sum())
                if name == TRACKS[-1]:
                    rec['img'] = torch.from_numpy(a['img'])
                frames.append(rec)
            out['outputs'][name] = frames
    out['globals'] = dict(full_pred_depths=[torch.from_numpy(d) for d in g['full_pred_depths']],
                          pts_list=[torch.from_numpy(p) for p in g['pts_list']],
                          mvs_depths=[torch.from_numpy(d) for d in g['mvs_depths']],
                          pred_depths=[torch.from_numpy(d) for d in g['pred_depths']],
                          scales=[float(s) for s in g['scales']], s=float(g['s']),
                          intrinsics=torch.from_numpy(g['intrinsics']), extrinsics=torch.from_numpy(g['extrinsics']),
                          h_pt=torch.from_numpy(g['h_pt']))
    golden_io.save_golden(out, GOLDEN_DIR, 'frames_golden')
    print('s = %r, points per frame %s' % (out['globals']['s'], [p.shape[1] for p in g['pts_list']]))


if __name__ == '__main__':
    main()
