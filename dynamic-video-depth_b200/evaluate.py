"""Scores of a test export: `python -m dvd_b200.evaluate --test_dir OUT/<net>_<dataset>_epoch_-1/epochbest_test --frames DIR
(--flows DIR | --raft_ckpt FILE [--raft_iters 20]) [--gaps 1,2,4,8] [--out DIR] [--chunk 16] [--gpu 0]`.

The method claims that the refined depth is more consistent across frames than its per-frame initialisation and no less
accurate. This measures both, for the refined `depth` and for the initial `depth_nn` of the export's `batch%04d.npz` files,
and writes OUT/metrics.json, OUT/frames.csv (one row per frame) and OUT/pairs.csv (one row per pair); OUT defaults to
--test_dir. It prints a refined-versus-initial table.

Frames. The export's frames are read in file order (export_io.Frames: depth, depth_nn, depth_gt, K and cam_c2w, the
poses with points.camera_block's conventions, and pair_path). A frame's number is the N of its pair_path basename
`frame_N.npz`, else its position in the export.

Accuracy against depth_gt, per frame and over the sequence. A pixel counts when depth_gt g and the evaluated depth d are valid
(finite and > 1e-2). Three scales s: `none` (1: the refined depth is in the poses' scale), `frame` (med(g) / med(d) over the
frame's valid pixels) and `sequence` (the same over all valid pixels of all frames), med the lower median (rank (n - 1) // 2).
On d' = s d: abs_rel = mean |d' - g| / g, sq_rel = mean (d' - g)^2 / g, rmse, rmse_log (natural log), d1, d2, d3 = the
fractions with max(d'/g, g/d') < 1.25^k. Sequence values pool the pixels: sums over all frames over the total count, square
roots last. `depth_gt_is_depth_nn` records whether depth_gt and depth_nn are bitwise equal (DAVIS and COLMAP frame files
calibrate MiDaS itself into depth_mvs), in which case accuracy is not an independent measure.

Consistency along the flow, per pair a -> b = a + g of flow_pairs.pair_list(n frame files, --gaps) whose frames are both in the
export. Flows and masks come from flow_pairs.PairBuilder (finished or raw flowpair files under --flows, or RAFT with
--raft_ckpt). Pixel x of frame a counts when the flowpair mask_2 is 0 there, D_a(x) is valid and so are the four bilinear taps
of D_b at q = x + flow_1_2(x) (align_corners, border-clamped). With P = c2w_a (D_a(x) K_a^-1 (x, 1)), c = w2c_b P, z = c.z and
p = (K_b c).xy / z: e_r = |p - q| pixels, e_d = |z - D_b~(q)| / D_b~(q). z <= 1e-3 counts as `behind` and is left out of the
means. Per region (`all`; `static` where the frame files' motion_seg of frame a is 0, when they carry one): count, behind,
mean e_r, mean e_d and the fractions of e_r < 1 and < 3 pixels, per pair, per gap and over all pairs (pooled over pixels). No
scale alignment: the units are the poses'.

Numerics: per-pixel arithmetic in fp64, fp64 sums in a fixed order (csrc/depth_metrics.cu); the host pools frames and pairs in
index order. The files are bitwise identical from run to run and for every --chunk. An empty set (a frame without a valid
pixel) has count 0 and NaN metrics (null in metrics.json, nan in the CSV files) and adds nothing to the pooled values.
Device memory: the three depth maps of every frame stay resident (12 bytes per pixel per frame, sent `--chunk` frames per
copy); the flows of `--chunk` pairs at a time follow, one copy per chunk.
"""
import argparse
import csv
import json
import os
import re
import time

import numpy as np
import torch

from . import ops
from .export_io import Frames, chunk_size, cuda_device, list_files
from .flow_pairs import PairBuilder, pair_list, read_npz
from .points import camera_block

F32 = np.float32
KEYS = ('depth', 'depth_nn', 'depth_gt', 'img_1', 'K', 'cam_c2w')
SOURCES = ('refined', 'initial')                 # depth, depth_nn
ALIGNMENTS = ('none', 'frame', 'sequence')
ACC_METRICS = ('abs_rel', 'sq_rel', 'rmse', 'rmse_log', 'd1', 'd2', 'd3')
REGIONS = ('all', 'static')
PAIR_METRICS = ('count', 'behind', 'e_r', 'e_d', 'e_r_lt1', 'e_r_lt3')
DEFAULT_GAPS = (1, 2, 4, 8)


# ---- inputs ---------------------------------------------------------------------------------------------------------------------
def frame_number(pair_path, position):
    """the N of a pair_path basename `frame_N.npz` (the frame files' names), else the frame's position in the export"""
    m = re.fullmatch(r'frame_(\d+)\.npz', os.path.basename(str(pair_path)))
    return int(m.group(1)) if m else int(position)


class Export:
    """The frames of a test export in file order (export_io.Frames, each file opened once): depth, depth_nn, depth_gt
    [N,H,W] fp32, cam [N,30] fp32 (camera_block) and the frame numbers."""

    def __init__(self, test_dir):
        ex = Frames(list_files(test_dir), keys=KEYS, optional=('pair_path',))
        self.N, self.H, self.W = ex.N, ex.H, ex.W
        self.depth, self.depth_nn, self.depth_gt = ex.depth, ex.depth_nn, ex.depth_gt
        self.cam = camera_block(ex.K, ex.c2w)
        self.numbers = np.asarray([frame_number(p, i) if p is not None else i for i, p in enumerate(ex.pair_path)],
                                  dtype=np.int64)
        if len(set(self.numbers.tolist())) != self.N:
            raise ValueError('the frames of %s do not have distinct numbers' % test_dir)

    def gt_is_nn(self):
        return bool(np.array_equal(self.depth_gt.view(np.uint32), self.depth_nn.view(np.uint32)))


def select_pairs(n_frames, gaps, numbers):
    """{gap: [(a, b) frame numbers]}: flow_pairs.pair_list(n_frames, gaps) restricted to pairs whose two frames are in
    `numbers`, in pair_list's order; ValueError for a gap without a pair"""
    have = set(int(v) for v in numbers)
    out = {}
    for g in gaps:
        out[g] = [p for p in pair_list(n_frames, [g]) if p[0] in have and p[1] in have]
        if not out[g]:
            raise ValueError('gap %d gives no pair of two exported frames (%d frame files, %d exported frames)'
                             % (g, n_frames, len(have)))
    return out


def check_gaps(gaps):
    gaps = [int(g) for g in gaps]
    if not gaps or any(g < 1 for g in gaps) or len(set(gaps)) != len(gaps):
        raise ValueError('gaps must be distinct integers >= 1, got %r' % (gaps,))
    return gaps


# ---- accuracy -----------------------------------------------------------------------------------------------------------------
def _div(a, n):
    with np.errstate(all='ignore'):
        return np.where(n > 0, a / np.where(n > 0, n, 1), np.nan)


def accuracy_from_sums(s):
    """sums [..., 22] of one source (dvd_depth_metrics' layout) -> {alignment: {metric: [...]}, 'count': [...]}"""
    s = np.asarray(s, dtype=np.float64)
    n = s[..., 0]
    out = {'count': n}
    for a, name in enumerate(ALIGNMENTS):
        b = 1 + 7 * a
        out[name] = {'abs_rel': _div(s[..., b], n), 'sq_rel': _div(s[..., b + 1], n), 'rmse': np.sqrt(_div(s[..., b + 2], n)),
                     'rmse_log': np.sqrt(_div(s[..., b + 3], n)), 'd1': _div(s[..., b + 4], n), 'd2': _div(s[..., b + 5], n),
                     'd3': _div(s[..., b + 6], n)}
    return out


def _scale(mg, md):
    mg, md = np.asarray(mg, np.float64), np.asarray(md, np.float64)
    with np.errstate(all='ignore'):
        return mg / md


def depth_accuracy(depth, depth_nn, depth_gt, chunk=None):
    """Device maps depth, depth_nn, depth_gt [N,H,W] fp32 -> dict with, per source: 'sums' [N,22] (frames), 'median_gt',
    'median' [N+1] (frames, then the pool), 'scale' [N+1] (frame scales, then the sequence scale) as host arrays. The sums are
    computed `chunk` frames per launch (all at once by default); they do not depend on it."""
    N = depth.shape[0]
    res, scales = {}, np.ones((N, 2, 3))
    for j, (name, d) in enumerate(zip(SOURCES, (depth, depth_nn))):
        mg, cg = ops.masked_select_median(depth_gt, d)
        md, _ = ops.masked_select_median(d, depth_gt)
        mg, md = mg.cpu().numpy(), md.cpu().numpy()
        sc = _scale(mg, md)
        res[name] = {'median_gt': mg, 'median': md, 'count': cg.cpu().numpy(), 'scale': sc}
        scales[:, j, 1], scales[:, j, 2] = sc[:N], sc[N]
    sd = torch.from_numpy(scales).to(depth.device)
    step = N if not chunk else int(chunk)
    sums = torch.cat([ops.depth_metrics(depth[s:s + step], depth_nn[s:s + step], depth_gt[s:s + step], sd[s:s + step])
                      for s in range(0, N, step)]).cpu().numpy()
    for j, name in enumerate(SOURCES):
        res[name]['sums'] = sums[:, j]
    return res


# ---- consistency --------------------------------------------------------------------------------------------------------------
def consistency_from_sums(s):
    """sums [..., 6] of one source and region -> {metric: [...]} (PAIR_METRICS)"""
    s = np.asarray(s, dtype=np.float64)
    n = s[..., 0]
    return {'count': n, 'behind': s[..., 1], 'e_r': _div(s[..., 2], n), 'e_d': _div(s[..., 3], n), 'e_r_lt1': _div(s[..., 4], n),
            'e_r_lt3': _div(s[..., 5], n)}


def pair_consistency(depth, depth_nn, cam, ia, ib, flows, masks, motion_seg=None, chunk=16):
    """Device resident frames depth, depth_nn [F,H,W], cam [F,30] and optional motion_seg [F,H,W] uint8; pairs ia, ib (frame
    indices) with host flows [P,H,W,2] fp32 and masks [P,H,W] uint8 (sequences of arrays or tensors). The flows go to the device
    `chunk` pairs per copy. Returns host sums [P,2,2,6] (dvd_pair_consistency's layout)."""
    F, H, W = depth.shape
    HW, P = H * W, len(ia)
    out = []
    for s in range(0, P, int(chunk)):
        e = min(s + int(chunk), P)
        n = e - s
        buf = np.empty(n * HW * 9 + 8 * n, dtype=np.uint8)     # flows, then ia, ib, then masks: the chunk's one copy
        buf[:n * HW * 8].view(F32).reshape(n, H, W, 2)[:] = np.stack([np.asarray(flows[i], F32) for i in range(s, e)])
        buf[n * HW * 8:n * HW * 8 + 8 * n].view(np.int32)[:] = np.concatenate([np.asarray(ia[s:e]), np.asarray(ib[s:e])])
        buf[n * HW * 8 + 8 * n:].reshape(n, H, W)[:] = np.stack([np.asarray(masks[i], np.uint8) for i in range(s, e)])
        g = torch.from_numpy(buf).to(depth.device)
        fl = g[:n * HW * 8].view(torch.float32).view(n, H, W, 2)
        idx = g[n * HW * 8:n * HW * 8 + 8 * n].view(torch.int32)
        mk = g[n * HW * 8 + 8 * n:].view(n, H, W)
        out.append(ops.pair_consistency(depth, depth_nn, cam, idx[:n], idx[n:], fl, mk, motion_seg))
    return torch.cat(out).cpu().numpy()


# ---- the whole export ---------------------------------------------------------------------------------------------------------
def _json_num(v):
    v = float(v)
    return v if np.isfinite(v) else None


def _csv_num(v):
    return repr(float(v))


def _frame_files(frames_dir):
    files = sorted(f for f in os.listdir(frames_dir) if re.fullmatch(r'frame_\d+\.npz', f)) if os.path.isdir(frames_dir) else []
    if not files:
        raise FileNotFoundError('no frame_*.npz under %s' % frames_dir)
    return files


def evaluate_export(test_dir, frames_dir, flows_dir=None, raft=None, gaps=DEFAULT_GAPS, out=None, chunk=16, device=None,
                    raft_iters=20):
    """Scores the export in `test_dir` (see the module docstring) and writes metrics.json, frames.csv and pairs.csv to `out`
    (default test_dir). raft: a dvd_b200.raft.RaftNet (instead of flows_dir) or a checkpoint path, run for raft_iters
    update iterations. Returns a dict with the
    record written to metrics.json, the per-frame and per-pair rows, the paths and host timings."""
    t0 = time.perf_counter()
    gaps = check_gaps(gaps)
    chunk = chunk_size(chunk)
    if (flows_dir is None) == (raft is None):
        raise ValueError('give exactly one of flows_dir and raft')
    out = test_dir if out is None else out
    ex = Export(test_dir)
    files = _frame_files(frames_dir)
    fh, fw = read_npz(os.path.join(frames_dir, files[0]))['img'].shape[:2]
    if (fh, fw) != (ex.H, ex.W):
        raise ValueError('the frame files are %dx%d, the export %dx%d' % (fh, fw, ex.H, ex.W))
    by_gap = select_pairs(len(files), gaps, ex.numbers)
    t_read = time.perf_counter() - t0
    dev = cuda_device(device)
    if isinstance(raft, str):
        from .raft import load_raft
        raft = load_raft(raft, dev)
    t1 = time.perf_counter()
    pb = PairBuilder(frames_dir, flows_dir, gaps, raft=raft, raft_iters=raft_iters, device=dev)
    if (pb.H, pb.W) != (ex.H, ex.W):
        raise ValueError('the frame files are %dx%d, the export %dx%d' % (pb.H, pb.W, ex.H, ex.W))
    t_flows = time.perf_counter() - t1

    t2 = time.perf_counter()
    N, H, W = ex.N, ex.H, ex.W
    maps = torch.empty(3, N, H, W, dtype=torch.float32, device=dev)
    for s in range(0, N, chunk):
        e = min(s + chunk, N)
        maps[:, s:e].copy_(torch.from_numpy(np.stack([ex.depth[s:e], ex.depth_nn[s:e], ex.depth_gt[s:e]])))
    acc = depth_accuracy(maps[0], maps[1], maps[2], chunk)
    slot = {int(v): i for i, v in enumerate(ex.numbers)}
    index = {p: i for i, p in enumerate(pb.pairs)}
    pairs = [p for g in gaps for p in by_gap[g]]
    firsts = sorted({a for a, _ in pairs})
    has_seg = ['motion_seg' in pb.frames[a] for a in firsts]
    if any(has_seg) and not all(has_seg):
        raise ValueError('motion_seg is in %d of the %d frame files that begin a pair; it must be in all or none'
                         % (sum(has_seg), len(has_seg)))
    seg = None
    if all(has_seg):
        hs = np.ones((N, H, W), dtype=np.uint8)
        for a in firsts:
            hs[slot[a]] = (pb.frames[a]['motion_seg'].reshape(H, W).numpy() != 0)
        seg = torch.from_numpy(hs).to(dev)
    cam = torch.from_numpy(ex.cam).to(dev)
    psums = pair_consistency(maps[0], maps[1], cam, [slot[a] for a, _ in pairs], [slot[b] for _, b in pairs],
                             [pb.flows[index[p]][0] for p in pairs], [pb.flows[index[p]][3] for p in pairs], seg, chunk)
    torch.cuda.synchronize(dev)
    t_device = time.perf_counter() - t2

    rec = record(test_dir, frames_dir, flows_dir, raft is not None, gaps, ex, acc, pairs, psums, seg is not None)
    frame_rows, pair_rows = frame_table(ex, acc), pair_table(pairs, psums, seg is not None)
    paths = write_outputs(out, rec, frame_rows, pair_rows)
    return {'record': rec, 'frames': frame_rows, 'pairs': pair_rows, 'paths': paths,
            'timing': {'read_s': t_read, 'flows_s': t_flows, 'device_s': t_device, 'total_s': time.perf_counter() - t0}}


def write_outputs(out, rec, frame_rows, pair_rows):
    """metrics.json, frames.csv and pairs.csv under `out`; returns their paths"""
    os.makedirs(out, exist_ok=True)
    paths = {k: os.path.join(out, k) for k in ('metrics.json', 'frames.csv', 'pairs.csv')}
    with open(paths['metrics.json'], 'w') as f:
        json.dump(rec, f, indent=1)
    for key, rows in (('frames.csv', frame_rows), ('pairs.csv', pair_rows)):
        with open(paths[key], 'w', newline='') as f:
            w = csv.writer(f, lineterminator='\n')
            w.writerow(list(rows[0].keys()))
            for r in rows:
                w.writerow(list(r.values()))
    return paths


def _acc_block(m, i=None):
    pick = (lambda v: v) if i is None else (lambda v: v[i])
    return dict({'count': int(pick(m['count']))}, **{a: {k: _json_num(pick(m[a][k])) for k in ACC_METRICS} for a in ALIGNMENTS})


def _cons_block(m):
    return {k: (int(m[k]) if k in ('count', 'behind') else _json_num(m[k])) for k in PAIR_METRICS}


def record(test_dir, frames_dir, flows_dir, used_raft, gaps, ex, acc, pairs, psums, static):
    """The contents of metrics.json"""
    rec = {'test_dir': os.path.abspath(test_dir), 'frames_dir': os.path.abspath(frames_dir),
           'flows': 'raft' if used_raft else os.path.abspath(flows_dir), 'gaps': list(gaps), 'height': ex.H, 'width': ex.W,
           'n_frames': ex.N, 'frames': [int(v) for v in ex.numbers], 'n_pairs': len(pairs),
           'depth_gt_is_depth_nn': ex.gt_is_nn(), 'static_region': bool(static), 'accuracy': {}, 'consistency': {}}
    gap_of = np.asarray([b - a for a, b in pairs])
    for j, name in enumerate(SOURCES):
        a = acc[name]
        seq = accuracy_from_sums(a['sums'].sum(0))
        rec['accuracy'][name] = dict(_acc_block(seq), median_gt=_json_num(a['median_gt'][-1]), median=_json_num(a['median'][-1]),
                                     scale_sequence=_json_num(a['scale'][-1]))
        c = {}
        for r, region in enumerate(REGIONS):
            if r == 1 and not static:
                c[region] = None
                continue
            c[region] = dict(_cons_block(consistency_from_sums(psums[:, j, r].sum(0))),
                             per_gap={str(g): _cons_block(consistency_from_sums(psums[gap_of == g, j, r].sum(0))) for g in gaps})
        rec['consistency'][name] = c
    return rec


def frame_table(ex, acc):
    rows = []
    for i in range(ex.N):
        r = {'frame': int(ex.numbers[i])}
        for name in SOURCES:
            m = accuracy_from_sums(acc[name]['sums'][i])
            r['%s_count' % name] = int(m['count'])
            r['%s_scale_frame' % name] = _csv_num(acc[name]['scale'][i])
            for al in ALIGNMENTS:
                for k in ACC_METRICS:
                    r['%s_%s_%s' % (name, al, k)] = _csv_num(m[al][k])
        rows.append(r)
    return rows


def pair_table(pairs, psums, static):
    rows = []
    for p, (a, b) in enumerate(pairs):
        r = {'frame_a': a, 'frame_b': b, 'gap': b - a}
        for j, name in enumerate(SOURCES):
            for reg, region in enumerate(REGIONS[:2 if static else 1]):
                m = consistency_from_sums(psums[p, j, reg])
                for k in PAIR_METRICS:
                    r['%s_%s_%s' % (name, region, k)] = int(m[k]) if k in ('count', 'behind') else _csv_num(m[k])
        rows.append(r)
    return rows


def summary(rec):
    """the refined-versus-initial table the command prints"""
    acc, con = rec['accuracy'], rec['consistency']
    fmt = lambda v: '%10s' % ('-' if v is None else '%.4g' % v)
    lines = ['%-34s %10s %10s' % ('', 'refined', 'initial')]
    for al in ALIGNMENTS:
        for k in ('abs_rel', 'rmse', 'd1'):
            lines.append('%-34s %s %s' % ('accuracy %s %s' % (al, k), fmt(acc['refined'][al][k]), fmt(acc['initial'][al][k])))
    for region in REGIONS:
        if con['refined'][region] is None:
            continue
        for k, label in (('e_r', 'mean reprojection error (px)'), ('e_d', 'mean depth error'), ('e_r_lt1', 'e_r < 1 px')):
            lines.append('%-34s %s %s' % ('%s %s' % (region, label), fmt(con['refined'][region][k]), fmt(con['initial'][region][k])))
    lines.append('depth_gt is depth_nn: %s (accuracy is %san independent measure)'
                 % (rec['depth_gt_is_depth_nn'], 'not ' if rec['depth_gt_is_depth_nn'] else ''))
    return '\n'.join(lines)


def parse_gaps(s):
    try:
        return check_gaps(s.split(','))
    except ValueError:
        raise argparse.ArgumentTypeError('gaps must be distinct integers >= 1 separated by commas, got %r' % s) from None


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog='python -m dvd_b200.evaluate', description=__doc__.split('\n\n')[0])
    p.add_argument('--test_dir', required=True, help='directory of the batch%%04d.npz files the test driver wrote')
    p.add_argument('--frames', required=True, help='directory of the video\'s frame_%%05d.npz files')
    g = p.add_mutually_exclusive_group(required=True)
    g.add_argument('--flows', default=None, help='directory of flowpair_%%05d_%%05d.npz (finished or raw flows)')
    g.add_argument('--raft_ckpt', default=None, help='RAFT checkpoint: estimate the flows from the frame files instead')
    p.add_argument('--raft_iters', type=int, default=20, help='RAFT update iterations (as prepare_pairs)')
    p.add_argument('--gaps', type=parse_gaps, default=list(DEFAULT_GAPS), help='frame gaps of the pairs (default 1,2,4,8)')
    p.add_argument('--out', default=None, help='output directory (default: --test_dir)')
    p.add_argument('--chunk', type=chunk_size, default=16, help='frames (pairs) per device copy')
    p.add_argument('--gpu', type=int, default=0)
    return p.parse_args(argv)


def main(argv=None):
    a = parse_args(argv)
    res = evaluate_export(a.test_dir, a.frames, a.flows, a.raft_ckpt, a.gaps, a.out, a.chunk, device=a.gpu, raft_iters=a.raft_iters)
    print(summary(res['record']))
    t = res['timing']
    print('%d frames, %d pairs: metrics.json, frames.csv, pairs.csv in %s (%.2f s: reading %.2f s, flows %.2f s, device %.2f s)'
          % (res['record']['n_frames'], res['record']['n_pairs'], os.path.dirname(res['paths']['metrics.json']), t['total_s'],
             t['read_s'], t['flows_s'], t['device_s']))
    return res


if __name__ == '__main__':
    main()
