"""TEST INFRASTRUCTURE — generates tests/golden/flow_pairs_golden*.pt from the reference's own preprocessing code.

1. Writes a tiny video in the reference's formats to a temporary directory: 6 frames at 40x56 (frame_%05d.npz) and, for every
   pair of gaps 1-4, raw flows at 24x32: smooth random fields, a shift that sends pixels out of the image and a patch of
   deliberately inconsistent backward flow.
2. Runs the reference on it:
   - `resize_flow`, `backward_flow_warp`, `get_oob_mask` and the mask lines of scripts/preprocess/davis/generate_flows.py
     (:139-148). That module is never imported (at import it builds RAFT on the GPU and may pip-install cv2): it is parsed with
     `ast` and only those function definitions and statements are executed;
   - generate_sequence_midas.collate_sequence_fix_gap, with its module-level paths pointed at the temporary directory, saved
     as the reference's __main__ block saves it;
   - datasets/davis_sequence.Dataset and datasets/shutterstock.Dataset on the written files (train and vali).
3. Stores the inputs, the reference's flows and masks, a band flag per pixel (round-trip error within 1e-4 of the threshold
   or target within 1e-4 px of the border) and SHA-256 digests of every tensor the reference's datasets return.

Run from the repository root: python -m oracle.gen_golden_flow_pairs
"""
import ast
import glob
import importlib.util
import os
import shutil
import sys
import tempfile

import numpy as np
import torch
import torch.nn.functional as F

from oracle.flow_pairs import digest, digest_item
from oracle.golden_io import save_golden
from oracle.ref_harness import REF_ROOT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_FRAMES, H, W, RAW_H, RAW_W, GAPS = 6, 40, 56, 24, 32, (1, 2, 3, 4)
TRACK = 'clip'
BAND = 1e-4


def band_flags(err, flow):
    h, w = flow.shape[:2]
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing='ij')
    qx, qy = xs + flow[..., 0], ys + flow[..., 1]
    near = np.minimum.reduce([np.abs(qx), np.abs(qx - (w - 1)), np.abs(qy), np.abs(qy - (h - 1))]) <= BAND
    return torch.from_numpy(np.packbits(near | (np.abs(err.astype(np.float64) - 1.0) <= BAND)))   # bits, row-major


def reference_flow_code():
    """the three functions and the mask statements of generate_flows.py, executed from its syntax tree"""
    path = os.path.join(REF_ROOT, 'scripts', 'preprocess', 'davis', 'generate_flows.py')
    tree = ast.parse(open(path).read(), path)
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ('resize_flow', 'get_oob_mask', 'backward_flow_warp')]
    assert len(fns) == 3
    import cv2
    ns = {'np': np, 'torch': torch, 'F': F, 'cv2': cv2}
    exec(compile(ast.Module(body=fns, type_ignores=[]), path, 'exec'), ns)
    gen = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == 'generate_pair_data')
    first = next(i for i, s in enumerate(gen.body) if isinstance(s, ast.Assign) and getattr(s.targets[0], 'id', None) == 'warp_flow_1_2')
    last = next(i for i, s in enumerate(gen.body) if isinstance(s, ast.Assign) and getattr(s.targets[0], 'id', None) == 'save_dict')
    mask_code = compile(ast.Module(body=gen.body[first:last], type_ignores=[]), path, 'exec')

    def masks(flow_1_2, flow_2_1):
        env = dict(ns, flow_1_2=flow_1_2, flow_2_1=flow_2_1)
        exec(mask_code, env)
        return env['mask_1'], env['mask_2'], env['err_1'], env['err_2']
    return ns['resize_flow'], masks


def smooth(rng, h, w, scale):
    lo = torch.from_numpy(rng.standard_normal((1, 2, 4, 5)).astype(np.float32))
    return (F.interpolate(lo, size=(h, w), mode='bicubic', align_corners=False)[0].permute(1, 2, 0).numpy() * scale).astype(np.float32)


def make_raw_flows(rng, gap):
    f12 = smooth(rng, RAW_H, RAW_W, 0.3 * gap)
    f12[..., 0] += 1.2 * gap                         # a shift: the right border's pixels leave the image
    f21 = -f12 + smooth(rng, RAW_H, RAW_W, 0.15) + rng.standard_normal((RAW_H, RAW_W, 2)).astype(np.float32) * 0.08
    y0, x0 = rng.integers(2, RAW_H - 8), rng.integers(2, RAW_W - 10)
    f21[y0:y0 + 5, x0:x0 + 7] += rng.standard_normal((5, 7, 2)).astype(np.float32) * 3.0   # inconsistent patch
    return f12.astype(np.float32), f21.astype(np.float32)


def make_frames(rng):
    frames = []
    for f in range(N_FRAMES):
        ang = 0.05 * f
        R = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]])
        pose = np.eye(4)
        pose[:3, :3], pose[:3, 3] = R, rng.standard_normal(3) * 0.1
        K = np.array([[50.0, 0, 27.5], [0, 48.0, 19.5], [0, 0, 1]], dtype=np.float32) + rng.random((3, 3)).astype(np.float32) * np.float32(0.01)
        K[2] = (0, 0, 1)
        d = {'img': rng.random((H, W, 3)).astype(np.float32), 'pose_c2w': pose, 'intrinsics': K,
             'depth_mvs': (1 + rng.random((H, W)) * 3).astype(np.float32), 'depth_pred': (1 + rng.random((H, W)) * 3).astype(np.float32)}
        if f < 2:
            d['motion_seg'] = (rng.random((H, W)) > 0.7).astype(np.uint8)
        frames.append(d)
    return frames


def odd_width_case(rng, resize_flow, masks):
    """five pairs at 15x21 (odd width) straight at working resolution"""
    hh, ww = 15, 21
    out = {'flow_1_2': [], 'flow_2_1': [], 'mask_1': [], 'mask_2': [], 'band_1': [], 'band_2': []}
    for g in range(1, 6):
        f12 = smooth(rng, hh, ww, 0.8 * g)
        f12[..., 1] -= 1.2 * g
        f21 = -f12 + smooth(rng, hh, ww, 0.2) + rng.standard_normal((hh, ww, 2)).astype(np.float32) * 0.1
        f21[4:8, 6:12] += 2.5
        m1, m2, e1, e2 = masks(f12, f21)
        for k, v in (('flow_1_2', f12), ('flow_2_1', f21), ('mask_1', m1.astype(np.uint8)), ('mask_2', m2.astype(np.uint8)),
                     ('band_1', band_flags(e1, f21)), ('band_2', band_flags(e2, f12))):
            out[k].append(v if torch.is_tensor(v) else torch.from_numpy(np.ascontiguousarray(v)))
    return {k: torch.stack(v) for k, v in out.items()}


def main():
    rng = np.random.default_rng(20260501)
    resize_flow, masks = reference_flow_code()
    tmp = tempfile.mkdtemp(prefix='dvd_flow_pairs_')
    cwd = os.getcwd()
    try:
        root = os.path.join(tmp, 'datafiles', 'davis_processed')
        fdir, pdir = os.path.join(root, 'frames_midas', TRACK), os.path.join(root, 'flow_pairs', TRACK)
        sdir = os.path.join(root, 'sequences_select_pairs_midas', TRACK, '001')
        for d in (fdir, pdir, sdir):
            os.makedirs(d)
        frames = make_frames(rng)
        for f, d in enumerate(frames):
            np.savez(os.path.join(fdir, 'frame_%05d.npz' % f), **d)
        pairs = [(f, f + g) for g in GAPS for f in range(N_FRAMES - 1 - g)]
        flows = []
        for a, b in pairs:
            r12, r21 = make_raw_flows(rng, b - a)
            f12, f21 = resize_flow(r12.copy(), [W, H]), resize_flow(r21.copy(), [W, H])
            m1, m2, e1, e2 = masks(f12, f21)
            np.savez(os.path.join(pdir, 'flowpair_%05d_%05d.npz' % (a, b)), flow_1_2=f12.astype(np.float32),
                     flow_2_1=f21.astype(np.float32), mask_1=m1.astype(np.uint8), mask_2=m2.astype(np.uint8), frame_id_1=a,
                     frame_id_2=b)
            flows.append({'raw_1_2': torch.from_numpy(r12), 'raw_2_1': torch.from_numpy(r21),
                          'flow_1_2': torch.from_numpy(f12.astype(np.float32)), 'flow_2_1': torch.from_numpy(f21.astype(np.float32)),
                          'mask_1': torch.from_numpy(m1.astype(np.uint8)), 'mask_2': torch.from_numpy(m2.astype(np.uint8)),
                          'band_1': band_flags(e1, f21), 'band_2': band_flags(e2, f12),
                          'pair': (a, b)})
        # generate_sequence_midas: its own collate, saved as its __main__ block does
        spec = importlib.util.spec_from_file_location(
            'ref_generate_sequence_midas', os.path.join(REF_ROOT, 'scripts', 'preprocess', 'davis', 'generate_sequence_midas.py'))
        gsm = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(gsm)
        gsm.data_list_root, gsm.flow_path = os.path.join(root, 'frames_midas'), os.path.join(root, 'flow_pairs')
        pair_files = []
        for gap in GAPS:
            for cnt, f in enumerate(np.arange(N_FRAMES - 1 - gap)):
                seq = gsm.collate_sequence_fix_gap(TRACK, np.arange(f, f + 1), gap=gap)
                name = 'shuffle_False_gap_%02d_sequence_%05d.pt' % (gap, cnt)
                torch.save(seq, os.path.join(sdir, name))
                pair_files.append({'name': name, 'keys': list(seq), 'digests': {k: digest(v) for k, v in seq.items()}})
        # the shutterstock layout: same files under datafiles/shutterstock
        shutil.copytree(root, os.path.join(tmp, 'datafiles', 'shutterstock'))
        os.chdir(tmp)
        if REF_ROOT not in sys.path:
            sys.path.insert(0, REF_ROOT)
        for m in [m for m in sys.modules if m == 'datasets' or m.startswith('datasets.')]:
            del sys.modules[m]
        from datasets import davis_sequence, shutterstock

        class Opt:
            subsample = False
            overfit = False
            repeat = 2
            gaps = ','.join(str(g) for g in GAPS)
        items = {}
        for alias, mod, track in (('davis_sequence', davis_sequence, TRACK), ('shutterstock', shutterstock, 0)):
            opt = Opt()
            opt.track_id = track
            for mode in ('train', 'vali'):
                ds = mod.Dataset(opt, mode=mode)
                items['%s/%s' % (alias, mode)] = [digest_item(ds[i]) for i in range(len(ds))]
        os.chdir(cwd)
        rng_odd = np.random.default_rng(7)
        golden = {'meta': {'n_frames': N_FRAMES, 'H': H, 'W': W, 'raw_h': RAW_H, 'raw_w': RAW_W, 'gaps': list(GAPS),
                           'track': TRACK, 'repeat': Opt.repeat, 'band': BAND},
                  'frames': [{k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in d.items()} for d in frames],
                  'flows': flows, 'pair_files': pair_files, 'items': items,
                  'odd': odd_width_case(rng_odd, resize_flow, masks)}
        save_golden(golden, os.path.join(ROOT, 'tests', 'golden'), 'flow_pairs_golden')
        total = sum(os.path.getsize(p) for p in glob.glob(os.path.join(ROOT, 'tests', 'golden', 'flow_pairs_golden*.pt')))
        print('wrote flow_pairs_golden (%d pairs, %.0f kB)' % (len(pairs), total / 1e3))
    finally:
        os.chdir(cwd)
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    main()
