"""The learned scene flow over a test export (dvd_b200.tracks, csrc/tracks.cu): per-stage times of one whole run.

    python tools/bench_tracks.py [--configs 80x224x384,200x288x512] [--gaps 1,2,4,8] [--out FILE.json]

Per configuration (frames x H x W) a seeded video is written to a temporary directory: frame files with motion_seg, finished
flowpair files for every pair of the gaps, a test export and a checkpoint with a seeded scene-flow field. Then, after a
warm-up run of the whole command on the same data:

  chain        the scene flow of every pair (tracks.pair_scene_flow: unprojection + dvd_mlp_chain_fwd, pairs of one gap 16 per
               launch), CUDA events, best of 3
  consistency  dvd_pair_consistency_sf over every pair, without and with the scene flow, 16 pairs per launch, best of 3
  integrate    the tracks (one chain per query frame, --query_every 10, --stride 16, --length 30), host clock after a sync
  drawing      dvd_draw_tracks over every frame (16 per launch) including the device-to-host copy of the frames, best of 3
  command      tracks.trace_export as a whole, with its own split: reading, flows, consistency (chain + kernels + copies),
               integration, drawing and file writes (PNG files, tracks.mp4, JSON, CSV, NPZ)
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
F32 = np.float32


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'nvidia-smi unavailable'


def best_of(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    best = float('inf')
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b) / 1e3)
    return best


def write_video(root, n, H, W, gaps, seed=0):
    """a plane at depth 4 seen by a camera moving along x, a square at depth 2 moving across it; flows from the static scene"""
    from dvd_b200.networks.sceneflow_field import SceneFlowFieldNet
    from dvd_b200.flow_pairs import pair_list
    rng = np.random.default_rng(seed)
    f = 0.8 * W
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]])
    dirs = {k: os.path.join(root, k) for k in ('frames', 'flows', 'export', 'ckpt')}
    for d in dirs.values():
        os.makedirs(d)
    y, x = np.mgrid[0:H, 0:W]
    depth, seg = np.full((n, H, W), 4.0, F32), np.zeros((n, H, W), F32)
    for i in range(n):
        x0 = int(W * 0.1 + (W * 0.6) * i / n)
        on = (x >= x0) & (x < x0 + W // 4) & (y >= H // 3) & (y < H // 3 + H // 4)
        depth[i][on], seg[i][on] = 2.0, 1.0
    poses = np.tile(np.eye(4), (n, 1, 1))
    poses[:, 0, 3] = 0.01 * np.arange(n)
    for i in range(n):
        img = rng.random((H, W, 3)).astype(F32)
        np.savez(os.path.join(dirs['frames'], 'frame_%05d.npz' % i), img=img, img_orig=img, pose_c2w=poses[i], intrinsics=K,
                 depth_mvs=depth[i], depth_pred=depth[i], motion_seg=seg[i])
        np.savez(os.path.join(dirs['export'], 'batch%04d.npz' % i), depth=depth[i][None, None], depth_nn=depth[i][None, None],
                 depth_gt=depth[i][None, None], img_1=img.transpose(2, 0, 1)[None], K=K.T[None].astype(F32),
                 cam_c2w=poses[i][None].astype(F32), pair_path=np.asarray([os.path.join(dirs['frames'], 'frame_%05d.npz' % i)]))
    for a, b in pair_list(n, gaps):
        f12 = np.stack([-f * 0.01 * (b - a) / depth[a], np.zeros((H, W))], -1).astype(F32)
        m2 = np.zeros((H, W), np.uint8)
        np.savez(os.path.join(dirs['flows'], 'flowpair_%05d_%05d.npz' % (a, b)), flow_1_2=f12, flow_2_1=-f12, mask_1=m2, mask_2=m2)
    torch.manual_seed(seed)
    net = SceneFlowFieldNet(net_width=256, n_layers=4, time_dependent=True, N_freq_xyz=16, N_freq_t=16)
    for p in net.parameters():
        torch.nn.init.normal_(p, std=0.05)
    torch.save({'time_dependent': True, 'n_freq_xyz': 16, 'n_freq_t': 16, 'sf_mag_div': 100.0, 'use_motion_seg': False},
               os.path.join(dirs['ckpt'], 'opt.pt'))
    torch.save({'nets': [{}, net.state_dict()]}, os.path.join(dirs['ckpt'], 'best.pt'))
    return dirs, seg


def run(n, H, W, gaps):
    from dvd_b200 import ops, tracks
    from dvd_b200.evaluate import select_pairs, upload_pairs
    from dvd_b200.export_io import Frames, list_files, to_device
    from dvd_b200.flow_pairs import PairBuilder
    from dvd_b200.points import camera_block
    res = {'frames': n, 'height': H, 'width': W}
    with tempfile.TemporaryDirectory() as tmp:
        d, seg = write_video(tmp, n, H, W, gaps)
        kw = dict(gaps=gaps, out=os.path.join(tmp, 'out'), chunk=16)
        tracks.trace_export(d['export'], d['ckpt'], d['frames'], d['flows'], **kw)          # warm-up
        t0 = time.perf_counter()
        cmd = tracks.trace_export(d['export'], d['ckpt'], d['frames'], d['flows'], **kw)
        res['command_s'] = time.perf_counter() - t0
        res['command_split_s'] = cmd['timing']
        res['n_pairs'] = cmd['record']['n_pairs']
        res['n_tracks'] = cmd['record']['tracks']['n_tracks']
        res['moving_e_r'] = cmd['record']['headline']

        dev = torch.device('cuda')
        field = tracks.Field(d['ckpt'], device=dev)
        ex = Frames(list_files(d['export']), keys=('depth', 'img_1', 'K', 'cam_c2w'))
        depth, cam = to_device(dev, ex.depth, camera_block(ex.K, ex.c2w))
        ts = torch.from_numpy(tracks.time_stamps(np.arange(n), n)).to(dev)
        dt = tracks.time_step(n)
        pb = PairBuilder(d['frames'], d['flows'], gaps, device=dev)
        by_gap = select_pairs(n, gaps, np.arange(n))
        seg = torch.from_numpy((seg != 0).astype(np.uint8)).to(dev)
        chunks = []
        for g in gaps:
            ps = by_gap[g]
            ia, ib = [a for a, _ in ps], [b for _, b in ps]
            index = {p: i for i, p in enumerate(pb.pairs)}
            for s in range(0, len(ps), 16):
                e = min(s + 16, len(ps))
                fl, ia_d, ib_d, mk = upload_pairs(dev, (H, W), ia, ib, [pb.flows[index[p]][0] for p in ps],
                                                  [pb.flows[index[p]][3] for p in ps], s, e)
                chunks.append((g, fl, ia_d, ib_d, mk))
        sfs = []

        def chain():
            sfs.clear()
            for g, fl, ia_d, ib_d, mk in chunks:
                sfs.append(tracks.pair_scene_flow(field, depth, cam, ts, ia_d.long(), dt, g).contiguous())
        res['chain_s'] = best_of(chain)
        zeros = torch.zeros(16, 3, H, W, device=dev)

        def cons():
            for (g, fl, ia_d, ib_d, mk), sf in zip(chunks, sfs):
                ops.pair_consistency_sf(depth, cam, ia_d, ib_d, fl, mk, zeros[:ia_d.shape[0]], seg)
                ops.pair_consistency_sf(depth, cam, ia_d, ib_d, fl, mk, sf, seg)
        res['consistency_kernels_s'] = best_of(cons)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tr = tracks.integrate(field, depth, cam, ts, dt, ex.depth, np.arange(n), 10, 16, 30)
        torch.cuda.synchronize()
        res['integrate_s'] = time.perf_counter() - t0
        colours = tracks.track_colours(tr['pixel'] % W, tr['pixel'] // W, H, W)

        def draw():
            tracks.draw_frames(tr, colours, ex.depth, ex.K, ex.c2w, np.arange(n), ex.images, 10, 16, dev, lambda s, f: None)
        t = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            draw()
            torch.cuda.synchronize()
            t.append(time.perf_counter() - t0)
        res['drawing_with_uploads_s'] = min(t)
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--configs', default='80x224x384,200x288x512')
    p.add_argument('--gaps', default='1,2,4,8')
    p.add_argument('--out', default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_tracks measures the GPU; no CUDA device is available')
    gaps = [int(g) for g in a.gaps.split(',')]
    out = {'gpu': gpu_info(), 'runs': []}
    for c in a.configs.split(','):
        n, H, W = (int(v) for v in c.split('x'))
        r = run(n, H, W, gaps)
        out['runs'].append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps({'gpu': out['gpu']}))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
