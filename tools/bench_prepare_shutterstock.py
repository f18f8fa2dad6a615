"""Frame preparation of one ShutterStock track (dvd_b200.frames.ShutterstockFrameBuilder): time per stage and for the whole
track, against the reference's path on the same GPU (eager PyTorch MiDaS at the stored size, then numpy / scipy on the CPU for
the dense calibration and the three resizes), a few frames timed and scaled to the track.

    python tools/bench_prepare_shutterstock.py [--frames 100] [--size 416,736] [--ref_frames 3] [--out results/bench_ss.json]

Synthetic frames (seeded image, MVS map with holes, cameras) are held in memory as h5-like handles; MiDaS has seeded weights.
Device stages are timed with CUDA events on one pass over the track, after a warm-up pass.
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


def make_track(n, H, W, seed=0):
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    out = []
    for f in range(n):
        img = np.stack([0.5 + 0.4 * np.sin(xx / (40.0 + 7 * c) + 0.05 * f) * np.cos(yy / (30.0 + 5 * c)) for c in range(3)], -1)
        mvs = (2.0 + np.sin(xx / 50.0 + 0.03 * f) * np.cos(yy / 35.0)).astype(np.float32)
        mvs[g.random((H, W)) < 0.15] = 0                                         # MVS holes
        T = np.eye(4)
        T[:3, 3] = [0.02 * f, 0.01, 0.5]
        out.append({'prediction/img': img.astype(np.float32), 'prediction/mvs_depth': mvs, 'prediction/T_1_G': T,
                    'prediction/K': np.array([[1.1 * W, 0, W / 2], [0, 1.1 * W, H / 2], [0, 0, 1]])})
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--frames', type=int, default=100)
    p.add_argument('--size', default='416,736')
    p.add_argument('--chunk', type=int, default=8)
    p.add_argument('--ref_frames', type=int, default=3)
    p.add_argument('--out', default=None)
    a = p.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    from dvd_b200 import frames as fr, ops, synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    from oracle import depth_nets, shutterstock_frames as ssf
    H, W = (int(x) for x in a.size.split(','))
    res = dict(gpu=torch.cuda.get_device_name(0), frames=a.frames, size=[H, W])
    try:
        res['nvidia_smi'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        res['nvidia_smi'] = repr(e)
    net = synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True, resize=None), 0, 2000.0).cuda().eval()
    hs = make_track(a.frames, H, W)
    fr.ShutterstockFrameBuilder(hs, net, chunk=a.chunk)                         # warm-up: engine plan, allocator
    torch.cuda.synchronize()
    # per stage, on the same work ShutterstockFrameBuilder does
    dev = torch.device('cuda')
    th, tw = (int(x) for x in fr.get_im_size(H, W))
    res['target'] = [th, tw]
    wts = [torch.from_numpy(ops.gaussian_weights(i, o)[1]).to(dev) for i, o in ((H, th), (W, tw))]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    t_up = t_midas = t_cal = t_aa = 0.0
    meds = []
    for c in range(0, a.frames, a.chunk):
        ev[0].record()
        img = torch.from_numpy(np.stack([h['prediction/img'] for h in hs[c:c + a.chunk]])).to(dev)
        mvs = torch.from_numpy(np.stack([h['prediction/mvs_depth'] for h in hs[c:c + a.chunk]])).to(dev)
        n = img.shape[0]
        ev[1].record()
        with torch.no_grad():
            nn = net.engine().forward(img.permute(0, 3, 1, 2).contiguous(), train=False).reshape(n, H, W)
        ev[2].record()
        meds.append(ops.row_medians(ops.dense_ratios(nn, mvs))[0])
        ev[3].record()
        ops.aa_resize(img, th, tw, wts)
        ops.aa_resize(nn.reshape(n, H, W, 1), th, tw, wts)
        ops.aa_resize((mvs * 2.5).float().unsqueeze(-1).contiguous(), th, tw, wts)
        ev[4].record()
        torch.cuda.synchronize()
        t_up += ev[0].elapsed_time(ev[1]) / 1e3
        t_midas += ev[1].elapsed_time(ev[2]) / 1e3
        t_cal += ev[2].elapsed_time(ev[3]) / 1e3
        t_aa += ev[3].elapsed_time(ev[4]) / 1e3
    np.mean(torch.cat(meds).cpu().numpy())
    res.update(upload_s=t_up, midas_s=t_midas, calibration_s=t_cal, aa_resize_s=t_aa)
    # whole track: construction (device passes, medians, s) and write
    t0 = time.perf_counter()
    b = fr.ShutterstockFrameBuilder(hs, net, chunk=a.chunk)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    with tempfile.TemporaryDirectory() as tmp:
        b.write(tmp)
    t2 = time.perf_counter()
    res.update(build_s=t1 - t0, write_s=t2 - t1, track_s=t2 - t0, scale=float(b.scale))
    # the reference's path: eager MiDaS on the GPU at the stored size, numpy / scipy on the CPU, per frame
    sd = {k: v.to(dev) for k, v in net.state_dict().items()}
    k = a.ref_frames
    x0 = torch.from_numpy(hs[0]['prediction/img']).permute(2, 0, 1)[None].to(dev)
    with torch.no_grad():
        depth_nets.midas_forward(sd, x0, True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    deps = []
    with torch.no_grad():
        for f in range(k):
            d = depth_nets.midas_forward(sd, torch.from_numpy(hs[f]['prediction/img']).permute(2, 0, 1)[None].to(dev), True)
            deps.append(d[0, 0].cpu().numpy())
    t1 = time.perf_counter()
    _, s = ssf.calibrate(deps, [h['prediction/mvs_depth'] for h in hs[:k]])
    t2 = time.perf_counter()
    for f in range(k):
        h = hs[f]
        ssf.frame_outputs(h['prediction/img'], deps[f], h['prediction/mvs_depth'], h['prediction/K'], h['prediction/T_1_G'], s)
    t3 = time.perf_counter()
    sc = a.frames / k
    res.update(ref_midas_s=(t1 - t0) * sc, ref_calibration_s=(t2 - t1) * sc, ref_resize_s=(t3 - t2) * sc,
               ref_track_s=(t3 - t0) * sc + res['write_s'])
    res['speedup_calibration'] = res['ref_calibration_s'] / res['calibration_s']
    res['speedup_resize'] = res['ref_resize_s'] / res['aa_resize_s']
    res['speedup_track'] = res['ref_track_s'] / res['track_s']
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
