"""The learned scene flow over a test export: `python -m dvd_b200.tracks --test_dir OUT/<net>_<dataset>_epoch_-1/epochbest_test
--checkpoint_path LOGDIR [--epoch -1] --frames DIR (--flows DIR | --raft_ckpt FILE [--raft_iters 20]) [--gaps 1,2,4,8]
[--query_every 10] [--stride 16] [--length 30] [--tail 10] [--moving_only] [--out DIR] [--chunk 16] [--gpu 0]`.

The method makes depth consistent for moving objects by fitting a scene-flow field with the depth. This reads the field back
and writes, under OUT (default --test_dir/tracks):
  tracks.json, pairs.csv   flow consistency of the refined depth per pair, per gap and over all pairs, for the regions all,
                           static and moving, without the scene flow (the static assumption: evaluate's refined figures) and
                           with it. The headline is the moving region's mean e_r with against without.
  tracks.npz, tracks_%05d.png, tracks.mp4
                           3D tracks integrated through the field from a grid of query pixels and drawn over the frames.

The field. opt.pt and best.pt (--epoch < 0) or nets/%04d.pt under --checkpoint_path, as the test driver reads them; only the
SceneFlowFieldNet (nets[1]) is built, with the training's time_dependent, n_freq_xyz, n_freq_t and sf_mag_div. Frame number N
(evaluate.frame_number) has the time stamp t = N / n_frames in fp64 rounded to fp32, n_frames the frame files under --frames,
as the test pass's items; one Euler step advances t by dt = 1 / n_frames. A pair a -> b takes steps = round(mean(ts_2 - ts_1)
/ dt), as the training step does: b - a. A checkpoint trained with --subsample (unit 2: a one-frame advance would be half a
step) is refused with ValueError.

Scene flow of a pair a -> b: P = the unprojection of D_a (points.world_points, the training's fp32 global_p1), the chain
ops.mlp_chain_fwd from t_a with n_eval = n_acc = steps, times frame a's motion_seg when the training used --use_motion_seg
(the pair's valid mask when the frame files have none, as the pair files carry it): the sf_1_2 the training loss saw for this
pair. The pairs of one gap go `--chunk` per launch.

Consistency (csrc/tracks.cu: dvd_pair_consistency_sf): evaluate's rule for the refined depth with the scene flow added to the
world point before the change to camera b, P' = P + sf. Regions: all; static and moving where frame a's motion_seg is 0 and
not 0, when the frame files carry it. fp64 per pixel and fixed-order fp64 sums: the files are bitwise identical from run to run
and for every --chunk.

Tracks. Query frames are every --query_every-th exported frame; query pixels a --stride grid at offset stride // 2 with a valid
refined depth (finite, > 1e-2), and with --moving_only also motion_seg != 0. Seeds are gathered from the frame's full
unprojection. One chain per query frame runs min(--length, last exported frame number - N) steps; X[0] = P and X[j+1] = X[j] +
s_j in fp32, position j belonging to frame number N + j. Output frame f draws every track alive at f with its last --tail
segments and a head mark, in frame f's camera, hidden behind the refined depth, with the exact rule of include/dvd_b200.h
(dvd_draw_tracks). A track's colour is the flow wheel at its query pixel (hue the angle about the image centre, saturation
the distance over the half-diagonal). tracks.npz: query_frame [M], query_pixel [M,2] (x, y), positions [M,L+1,3] (NaN past
the alive length), alive [M], colour [M,3] RGB, and per step the head's projection proj [M,L+1,3] (u, v, z) in that step's own
frame and visible [M,L+1] (NaN and 0 where that frame is not exported).

Backward-in-time tracks (they need the field's inverse), --subsample checkpoints and compensating depth_nn are not offered.
"""
import argparse
import csv
import json
import os
import time
import zipfile
from argparse import Namespace

import numpy as np
import torch

from . import ops
from .evaluate import (_csv_num, _frame_files, _json_num, check_gaps, consistency_from_sums, frame_number, parse_gaps,
                       select_pairs, upload_pairs, DEFAULT_GAPS, PAIR_METRICS)
from .export_io import Frames, Writer, chunk_size, cuda_device, list_files, to_device
from .flow_pairs import FRAME_FMT, PairBuilder, read_npz
from .points import camera_block, world_points
from .render_views import view_cams

F32 = np.float32
REGIONS = ('all', 'static', 'moving')
MODES = ('static_assumption', 'scene_flow')
MAX_STEPS = 64             # Euler steps per chain launch (dvd_mlp_chain_fwd)


# ---- the field ------------------------------------------------------------------------------------------------------------------
def training_options(checkpoint_path):
    """the training options in <checkpoint_path>/opt.pt as a Namespace; ValueError for a --subsample checkpoint"""
    o = torch.load(os.path.join(checkpoint_path, 'opt.pt'), weights_only=False)
    o = Namespace(**(vars(o) if isinstance(o, Namespace) else o))
    if getattr(o, 'subsample', False):
        raise ValueError('%s was trained with --subsample: time steps of two frames, so a one-frame advance would be half an '
                         'Euler step; tracks and scene-flow consistency need a checkpoint trained on every frame' % checkpoint_path)
    return o


def checkpoint_file(checkpoint_path, epoch):
    return os.path.join(checkpoint_path, 'best.pt') if epoch < 0 else os.path.join(checkpoint_path, 'nets', '%04d.pt' % epoch)


class Field:
    """The trained scene-flow MLP (nets[1] of the checkpoint) on the device, with the training options it ran under."""

    def __init__(self, checkpoint_path, epoch=-1, device=None):
        from .networks.sceneflow_field import SceneFlowFieldNet
        o = training_options(checkpoint_path)
        self.time_dependent, self.sf_mag_div = bool(o.time_dependent), float(o.sf_mag_div)
        self.use_motion_seg = bool(getattr(o, 'use_motion_seg', False))
        self.n_freq_xyz, self.n_freq_t = int(o.n_freq_xyz), int(o.n_freq_t)
        net = SceneFlowFieldNet(net_width=256, n_layers=4, time_dependent=self.time_dependent, N_freq_xyz=self.n_freq_xyz,
                                N_freq_t=self.n_freq_t)
        sd = torch.load(checkpoint_file(checkpoint_path, epoch), map_location='cpu', weights_only=False)
        net.load_state_dict(sd['nets'][1])
        self.net = net.to(device).eval()
        self.packed = self.net.packed(self.sf_mag_div)

    def chain(self, p0, t, dt, steps, want_steps=False):
        """ops.mlp_chain_fwd from p0 [B,3,H,W] at the time stamps t [B] (fp32 device tensor), n_eval = n_acc = steps"""
        B, _, H, W = p0.shape
        t0 = t.reshape(B, 1, 1, 1).expand(B, 1, H, W).contiguous() if self.time_dependent else None
        return ops.mlp_chain_fwd(self.packed, p0, t0, dt, steps, steps, want_steps=want_steps)


def time_stamps(numbers, n_frames):
    """t = N / n_frames in fp64 rounded to fp32 (the test pass's time_stamp_1, datasets/davis_sequence.py)"""
    return (np.asarray(numbers, np.float64) / float(n_frames)).astype(F32)


def time_step(n_frames, unit=1.0):
    """dt = unit / n_frames (datasets' time_step)"""
    return float(unit) / float(n_frames)


def euler_steps(a, b, n_frames, unit=1.0):
    """steps = round(mean(ts_2 - ts_1) / time_step) of the training step for the pair a -> b, with the training items' fp32
    time stamps fid / n_frames (a gap g takes g / unit steps: with unit 2, --subsample, a one-frame gap would take half a step,
    which is why training_options refuses such checkpoints)"""
    ts1 = torch.tensor([float(a)]) / float(n_frames)
    ts2 = torch.tensor([float(b)]) / float(n_frames)
    return int(round(float((ts2 - ts1).float().mean()) / time_step(n_frames, unit)))


# ---- consistency ------------------------------------------------------------------------------------------------------------------
def pair_scene_flow(field, depth, cam, ts, ia, dt, steps, mul=None):
    """sf [n,3,H,W] of pairs starting at resident frames ia [n] (int64 device indices): the chain from the unprojection of
    their refined depth, times `mul` [n,H,W] when given"""
    n, H, W = ia.shape[0], depth.shape[1], depth.shape[2]
    P = world_points(depth[ia].contiguous(), cam[ia].contiguous())
    sf = field.chain(P, ts[ia], dt, steps)['acc']
    return sf * mul.reshape(n, 1, H, W) if mul is not None else sf


def consistency(field, depth, cam, ts, dt, steps_of, ia, ib, flows, masks, motion_seg=None, seg_mul=None, chunk=16):
    """Device resident depth [F,H,W], cam [F,30], ts [F] fp32; pairs ia, ib (frame indices) with host flows and masks and
    their Euler steps steps_of [P] (pairs of one step count must be contiguous for them to share launches); motion_seg [F,H,W]
    uint8 (regions) and seg_mul [F,H,W] fp32 (the training's multiplier; None: the pair's valid mask) when the training used
    --use_motion_seg. Returns host sums [P,2,3,6]: without the scene flow, then with it."""
    P, (H, W) = len(ia), depth.shape[1:]
    zeros = None
    out = []
    s = 0
    while s < P:
        e = s
        while e < P and e - s < chunk and steps_of[e] == steps_of[s]:
            e += 1
        fl, ia_d, ib_d, mk = upload_pairs(depth.device, (H, W), ia, ib, flows, masks, s, e)
        mul = None
        if field.use_motion_seg:
            mul = seg_mul[ia_d.long()] if seg_mul is not None else 1.0 - mk.float()
        sf = pair_scene_flow(field, depth, cam, ts, ia_d.long(), dt, int(steps_of[s]), mul)
        if zeros is None or zeros.shape[0] < e - s:
            zeros = torch.zeros(chunk, 3, H, W, dtype=torch.float32, device=depth.device)
        without = ops.pair_consistency_sf(depth, cam, ia_d, ib_d, fl, mk, zeros[:e - s], motion_seg)
        out.append(torch.stack([without, ops.pair_consistency_sf(depth, cam, ia_d, ib_d, fl, mk, sf.contiguous(), motion_seg)], 1))
        s = e
    return torch.cat(out).cpu().numpy()


# ---- tracks ---------------------------------------------------------------------------------------------------------------------
def query_pixels(depth, H, W, stride, seg=None):
    """flat pixel indices of the stride grid at offset stride // 2 with a valid depth (and seg != 0 when seg is given)"""
    ys, xs = np.meshgrid(np.arange(stride // 2, H, stride), np.arange(stride // 2, W, stride), indexing='ij')
    idx = (ys * W + xs).reshape(-1)
    d = np.asarray(depth, F32).reshape(-1)[idx]
    keep = np.isfinite(d) & (d > F32(1e-2))
    if seg is not None:
        keep &= np.asarray(seg).reshape(-1)[idx] != 0
    return idx[keep]


def track_colours(qx, qy, H, W):
    """the flow wheel at the query pixels: hue the angle about the image centre, saturation the distance over the
    half-diagonal, value 1; fp64, rounded half up to uint8 RGB [M,3]"""
    dx, dy = np.asarray(qx, np.float64) - (W - 1) / 2.0, np.asarray(qy, np.float64) - (H - 1) / 2.0
    h = (np.arctan2(dy, dx) / (2 * np.pi)) % 1.0 * 6.0
    s = np.minimum(np.hypot(dx, dy) / max(np.hypot(W - 1, H - 1) / 2.0, 1e-12), 1.0)
    i = np.floor(h).astype(np.int64) % 6
    f = h - np.floor(h)
    p, q, t = 1 - s, 1 - s * f, 1 - s * (1 - f)
    one = np.ones_like(s)
    r = np.choose(i, [one, q, p, p, t, one])
    g = np.choose(i, [t, one, one, q, p, p])
    b = np.choose(i, [p, p, t, one, one, q])
    return np.clip(np.floor(np.stack([r, g, b], 1) * 255 + 0.5), 0, 255).astype(np.uint8)


def integrate(field, depth_dev, cam_dev, ts, dt, host_depth, numbers, query_every, stride, length, seg=None, last=None):
    """Tracks from every query_every-th frame, clipped at frame number `last` (default the last of `numbers`): dict of host
    arrays first [M] (frame number), slot [M] (export position), pixel [M] (flat index), X [M,length+1,3] fp32 (NaN past the
    alive length), alive [M]"""
    F, H, W = host_depth.shape
    last = int(np.max(numbers)) if last is None else int(last)
    parts = []
    for s in range(0, F, query_every):
        idx = query_pixels(host_depth[s], H, W, stride, None if seg is None else seg[s])
        M = idx.shape[0]
        if M == 0:
            continue
        a = int(numbers[s])
        L = min(length, last - a)
        P = world_points(depth_dev[s:s + 1].contiguous(), cam_dev[s:s + 1].contiguous())
        p0 = P[0].reshape(3, -1)[:, torch.from_numpy(idx).to(P.device)].reshape(1, 3, 1, M).contiguous()
        X = torch.full((length + 1, 3, M), float('nan'), dtype=torch.float32, device=P.device)
        X[0] = p0.reshape(3, M)
        if L > 0:
            steps = field.chain(p0, ts[s:s + 1], dt, L, want_steps=True)['s_steps']
            x = p0
            for j in range(L):
                x = x + steps[j]
                X[j + 1] = x.reshape(3, M)
        parts.append({'first': np.full(M, a, np.int32), 'slot': np.full(M, s, np.int64), 'pixel': idx,
                      'X': X.permute(2, 0, 1).contiguous().cpu().numpy(), 'alive': np.full(M, L + 1, np.int32)})
    if not parts:
        raise ValueError('no query pixel with a valid depth%s' % (' and motion_seg != 0' if seg is not None else ''))
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def draw_frames(tr, colours, host_depth, K, c2w, numbers, images, tail, chunk, device, on_chunk):
    """draws the tracks over every frame, `chunk` frames per launch; on_chunk(s, frames [n,H,W,3] BGR) receives each chunk.
    Returns the head projections proj [M,L1,3] and visibility [M,L1] (host)."""
    F, H, W = host_depth.shape
    M, L1 = tr['X'].shape[:2]
    X, first, alive, rgb = (torch.from_numpy(np.ascontiguousarray(a)).to(device)
                            for a in (tr['X'], tr['first'], tr['alive'], colours))
    proj = torch.full((M, L1, 3), float('nan'), dtype=torch.float32, device=device)
    vis = torch.zeros(M, L1, dtype=torch.uint8, device=device)
    cams = view_cams(K, c2w)
    for s in range(0, F, chunk):
        e = min(s + chunk, F)
        d, img, cm = to_device(device, host_depth[s:e], images(s, e), cams[s:e])
        num = torch.from_numpy(np.asarray(numbers[s:e], np.int32)).to(device)
        on_chunk(s, ops.draw_tracks(X, first, alive, rgb, cm.contiguous(), d, img, num, tail, proj=proj, vis=vis).cpu().numpy())
    return proj.cpu().numpy(), vis.cpu().numpy()


# ---- the whole export -------------------------------------------------------------------------------------------------------------
def _block(s):
    m = consistency_from_sums(s)
    return {k: (int(m[k]) if k in ('count', 'behind') else _json_num(m[k])) for k in PAIR_METRICS}


def record(args, ex_n, numbers, H, W, n_files, field, pairs, steps_of, sums, moving, tr):
    gap_of = np.asarray([b - a for a, b in pairs])
    rec = {'test_dir': os.path.abspath(args['test_dir']), 'checkpoint': os.path.abspath(args['checkpoint']),
           'frames_dir': os.path.abspath(args['frames_dir']), 'flows': args['flows'], 'gaps': list(args['gaps']),
           'height': H, 'width': W, 'n_frame_files': n_files, 'n_frames': ex_n, 'frames': [int(v) for v in numbers],
           'time_dependent': field.time_dependent, 'sf_mag_div': field.sf_mag_div, 'use_motion_seg': field.use_motion_seg,
           'steps_per_gap': {str(g): int(steps_of[list(gap_of).index(g)]) for g in args['gaps']},
           'n_pairs': len(pairs), 'moving_region': bool(moving), 'consistency': {}}
    for m, mode in enumerate(MODES):
        c = {}
        for r, region in enumerate(REGIONS):
            if r > 0 and not moving:
                c[region] = None
                continue
            c[region] = dict(_block(sums[:, m, r].sum(0)),
                             per_gap={str(g): _block(sums[gap_of == g, m, r].sum(0)) for g in args['gaps']})
        rec['consistency'][mode] = c
    rec['headline'] = {'moving_e_r_static_assumption': rec['consistency'][MODES[0]]['moving']['e_r'] if moving else None,
                       'moving_e_r_scene_flow': rec['consistency'][MODES[1]]['moving']['e_r'] if moving else None}
    rec['tracks'] = {'n_tracks': int(tr['X'].shape[0]), 'query_every': args['query_every'], 'stride': args['stride'],
                     'length': args['length'], 'tail': args['tail'], 'moving_only': args['moving_only'],
                     'query_frames': sorted({int(v) for v in tr['first']})}
    return rec


def pair_table(pairs, steps_of, sums, moving):
    rows = []
    for p, (a, b) in enumerate(pairs):
        r = {'frame_a': a, 'frame_b': b, 'gap': b - a, 'steps': int(steps_of[p])}
        for m, mode in enumerate(MODES):
            for reg, region in enumerate(REGIONS[:3 if moving else 1]):
                mm = consistency_from_sums(sums[p, m, reg])
                for k in PAIR_METRICS:
                    r['%s_%s_%s' % (mode, region, k)] = int(mm[k]) if k in ('count', 'behind') else _csv_num(mm[k])
        rows.append(r)
    return rows


def _seg_of(frames_dir, numbers):
    """motion_seg of the frame files of `numbers` ([n,H,W] fp32), or None when none has one; ValueError when only some do"""
    segs = [read_npz(os.path.join(frames_dir, FRAME_FMT % n)).get('motion_seg') for n in numbers]
    have = [s is not None for s in segs]
    if not any(have):
        return None
    if not all(have):
        raise ValueError('motion_seg is in %d of %d frame files; it must be in all or none' % (sum(have), len(have)))
    return np.stack([np.asarray(s, F32) for s in segs])


def check_options(query_every, stride, length, tail):
    for name, v, lo, hi in (('query_every', query_every, 1, None), ('stride', stride, 1, None), ('length', length, 1, MAX_STEPS),
                            ('tail', tail, 0, ops._lib.DVD_TRACK_MAX_TAIL)):
        if int(v) != v or v < lo or (hi is not None and v > hi):
            raise ValueError('%s must be an integer in [%d, %s], got %r' % (name, lo, hi if hi is not None else 'inf', v))


def trace_export(test_dir, checkpoint_path, frames_dir, flows_dir=None, raft=None, epoch=-1, gaps=DEFAULT_GAPS, query_every=10,
                 stride=16, length=30, tail=10, moving_only=False, out=None, chunk=16, device=None, raft_iters=20):
    """Writes tracks.json, pairs.csv, tracks.npz, tracks_%05d.png and tracks.mp4 under `out` (default test_dir/tracks); see the
    module docstring. raft: a dvd_b200.raft.RaftNet (instead of flows_dir) or a checkpoint path. Returns a dict with the record,
    the pair rows, the paths and host timings."""
    t0 = time.perf_counter()
    gaps = check_gaps(gaps)
    chunk = chunk_size(chunk)
    check_options(query_every, stride, length, tail)
    if (flows_dir is None) == (raft is None):
        raise ValueError('give exactly one of flows_dir and raft')
    if max(gaps) > MAX_STEPS:
        raise ValueError('gaps above %d take more Euler steps than one chain runs' % MAX_STEPS)
    out = os.path.join(test_dir, 'tracks') if out is None else out
    training_options(checkpoint_path)                         # refuses --subsample before anything is read
    ex = Frames(list_files(test_dir), keys=('depth', 'img_1', 'K', 'cam_c2w'), optional=('pair_path',))
    N, H, W = ex.N, ex.H, ex.W
    numbers = np.asarray([frame_number(p, i) if p is not None else i for i, p in enumerate(ex.pair_path)], dtype=np.int64)
    if len(set(numbers.tolist())) != N:
        raise ValueError('the frames of %s do not have distinct numbers' % test_dir)
    files = _frame_files(frames_dir)
    n_files = len(files)
    fh, fw = read_npz(os.path.join(frames_dir, files[0]))['img'].shape[:2]
    if (fh, fw) != (H, W):
        raise ValueError('the frame files are %dx%d, the export %dx%d' % (fh, fw, H, W))
    by_gap = select_pairs(n_files, gaps, numbers)
    seg = _seg_of(frames_dir, numbers)
    if moving_only and seg is None:
        raise ValueError('--moving_only needs motion_seg in the frame files')
    t_read = time.perf_counter() - t0

    dev = cuda_device(device)
    field = Field(checkpoint_path, epoch, dev)
    if isinstance(raft, str):
        from .raft import load_raft
        raft = load_raft(raft, dev)
    t1 = time.perf_counter()
    pb = PairBuilder(frames_dir, flows_dir, gaps, raft=raft, raft_iters=raft_iters, device=dev)
    if (pb.H, pb.W) != (H, W):
        raise ValueError('the frame files are %dx%d, the export %dx%d' % (pb.H, pb.W, H, W))
    t_flows = time.perf_counter() - t1

    t2 = time.perf_counter()
    depth, cam = to_device(dev, ex.depth, camera_block(ex.K, ex.c2w))
    cam = cam.contiguous()
    ts = torch.from_numpy(time_stamps(numbers, n_files)).to(dev)
    dt = time_step(n_files)
    seg_u8 = torch.from_numpy((seg != 0).astype(np.uint8)).to(dev) if seg is not None else None
    seg_mul = torch.from_numpy(seg).to(dev) if seg is not None else None
    slot = {int(v): i for i, v in enumerate(numbers)}
    index = {p: i for i, p in enumerate(pb.pairs)}
    pairs = [p for g in gaps for p in by_gap[g]]
    steps_of = [euler_steps(a, b, n_files) for a, b in pairs]
    sums = consistency(field, depth, cam, ts, dt, steps_of, [slot[a] for a, _ in pairs], [slot[b] for _, b in pairs],
                       [pb.flows[index[p]][0] for p in pairs], [pb.flows[index[p]][3] for p in pairs], seg_u8, seg_mul, chunk)
    torch.cuda.synchronize(dev)
    t_cons = time.perf_counter() - t2

    t3 = time.perf_counter()
    tr = integrate(field, depth, cam, ts, dt, ex.depth, numbers, query_every, stride, length, seg if moving_only else None)
    colours = track_colours(tr['pixel'] % W, tr['pixel'] // W, H, W)
    torch.cuda.synchronize(dev)
    t_int = time.perf_counter() - t3

    t4 = time.perf_counter()
    os.makedirs(out, exist_ok=True)
    paths = {k: os.path.join(out, k) for k in ('tracks.json', 'pairs.csv', 'tracks.npz', 'tracks.mp4')}
    with Writer() as wr:
        video = wr.video(paths['tracks.mp4'], 24, (H, W))

        def on_chunk(s, frames):
            for j, fr in enumerate(frames):
                wr.png(os.path.join(out, 'tracks_%05d.png' % int(numbers[s + j])), fr)
                video.write(fr)
        proj, vis = draw_frames(tr, colours, ex.depth, ex.K, ex.c2w, numbers, ex.images, tail, chunk, dev, on_chunk)
    t_draw = time.perf_counter() - t4

    args = {'test_dir': test_dir, 'checkpoint': checkpoint_file(checkpoint_path, epoch), 'frames_dir': frames_dir,
            'flows': 'raft' if raft is not None else os.path.abspath(flows_dir), 'gaps': gaps, 'query_every': query_every,
            'stride': stride, 'length': length, 'tail': tail, 'moving_only': bool(moving_only)}
    rec = record(args, N, numbers, H, W, n_files, field, pairs, steps_of, sums, seg is not None, tr)
    rows = pair_table(pairs, steps_of, sums, seg is not None)
    with open(paths['tracks.json'], 'w') as f:
        json.dump(rec, f, indent=1)
    with open(paths['pairs.csv'], 'w', newline='') as f:
        w = csv.writer(f, lineterminator='\n')
        w.writerow(list(rows[0].keys()))
        for r in rows:
            w.writerow(list(r.values()))
    X = tr['X']
    write_npz(paths['tracks.npz'], query_frame=tr['first'].astype(np.int64), query_pixel=np.stack([tr['pixel'] % W, tr['pixel'] // W], 1),
              positions=X, alive=tr['alive'].astype(np.int64), colour=colours, proj=proj, visible=vis.astype(bool))
    t_files = time.perf_counter() - t4
    return {'record': rec, 'pairs': rows, 'paths': paths, 'tracks': tr, 'proj': proj, 'visible': vis,
            'timing': {'read_s': t_read, 'flows_s': t_flows, 'consistency_s': t_cons, 'integrate_s': t_int,
                       'draw_s': t_draw, 'files_s': t_files, 'total_s': time.perf_counter() - t0}}


def write_npz(path, **arrays):
    """np.savez with a fixed member time stamp, so that equal arrays give equal bytes (np.savez stamps the current time)"""
    with zipfile.ZipFile(path, 'w', compression=zipfile.ZIP_STORED) as z:
        for k, a in arrays.items():
            info = zipfile.ZipInfo(k + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            with z.open(info, 'w', force_zip64=True) as f:
                np.lib.format.write_array(f, np.asanyarray(a), allow_pickle=False)


def summary(rec):
    con = rec['consistency']
    fmt = lambda v: '%12s' % ('-' if v is None else '%.4g' % v)
    lines = ['%-34s %12s %12s' % ('', 'static asm.', 'scene flow')]
    for region in REGIONS:
        if con[MODES[0]][region] is None:
            continue
        for k, label in (('e_r', 'mean reprojection error (px)'), ('e_d', 'mean depth error'), ('e_r_lt1', 'e_r < 1 px')):
            lines.append('%-34s %s %s' % ('%s %s' % (region, label), fmt(con[MODES[0]][region][k]), fmt(con[MODES[1]][region][k])))
    lines.append('%d tracks from %d query frames' % (rec['tracks']['n_tracks'], len(rec['tracks']['query_frames'])))
    return '\n'.join(lines)


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog='python -m dvd_b200.tracks', description=__doc__.split('\n\n')[0])
    p.add_argument('--test_dir', required=True, help='directory of the batch%%04d.npz files the test driver wrote')
    p.add_argument('--checkpoint_path', required=True, help='training log directory (opt.pt, best.pt, nets/)')
    p.add_argument('--epoch', type=int, default=-1, help='checkpoint epoch (< 0: best.pt)')
    p.add_argument('--frames', required=True, help='directory of the video\'s frame_%%05d.npz files')
    g = p.add_mutually_exclusive_group(required=True)
    g.add_argument('--flows', default=None, help='directory of flowpair_%%05d_%%05d.npz (finished or raw flows)')
    g.add_argument('--raft_ckpt', default=None, help='RAFT checkpoint: estimate the flows from the frame files instead')
    p.add_argument('--raft_iters', type=int, default=20, help='RAFT update iterations (as prepare_pairs)')
    p.add_argument('--gaps', type=parse_gaps, default=list(DEFAULT_GAPS), help='frame gaps of the pairs (default 1,2,4,8)')
    p.add_argument('--query_every', type=int, default=10, help='seed tracks on every k-th exported frame')
    p.add_argument('--stride', type=int, default=16, help='query pixel grid spacing')
    p.add_argument('--length', type=int, default=30, help='Euler steps (frames) per track, at most %d' % MAX_STEPS)
    p.add_argument('--tail', type=int, default=10, help='segments drawn behind a track\'s head')
    p.add_argument('--moving_only', action='store_true', help='seed only where motion_seg != 0')
    p.add_argument('--out', default=None, help='output directory (default: --test_dir/tracks)')
    p.add_argument('--chunk', type=chunk_size, default=16, help='pairs (frames) per launch')
    p.add_argument('--gpu', type=int, default=0)
    a = p.parse_args(argv)
    try:
        check_options(a.query_every, a.stride, a.length, a.tail)
    except ValueError as e:
        p.error(str(e))
    return a


def main(argv=None):
    a = parse_args(argv)
    res = trace_export(a.test_dir, a.checkpoint_path, a.frames, a.flows, a.raft_ckpt, a.epoch, a.gaps, a.query_every, a.stride,
                       a.length, a.tail, a.moving_only, a.out, a.chunk, device=a.gpu, raft_iters=a.raft_iters)
    print(summary(res['record']))
    t = res['timing']
    print('%d frames, %d pairs: tracks.json, pairs.csv, tracks.npz, tracks_*.png, tracks.mp4 in %s (%.2f s: consistency %.2f s, '
          'tracks %.2f s, drawing and files %.2f s)' % (res['record']['n_frames'], res['record']['n_pairs'],
                                                        os.path.dirname(res['paths']['tracks.json']), t['total_s'],
                                                        t['consistency_s'], t['integrate_s'], t['files_s']))
    return res


if __name__ == '__main__':
    main()
