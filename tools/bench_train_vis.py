"""Training-page images (dvd_b200.train_vis, csrc/train_vis.cu): device time of one visualised training pack, its copy back,
its PNG writes, and the numpy oracle on the CPU for the same pack.

    python tools/bench_train_vis.py [--configs 1x224x384,8x224x384,1x288x512,8x288x512] [--out results/train_vis.json]

A pack is what `--html_logger` renders for one training batch of B pairs: five depth maps [B,1,H,W], four flows (two read
through permuted [B,2,H,W] views, two [B,H,W,2]) and two images [B,3,H,W]. CUDA events time dvd_vis_ranges and dvd_vis_tiles
(best of 3 after a warm-up, 20 launches each). GB/s is the compulsory traffic over kernel time next to the 3.35 TB/s data-sheet
HBM3 peak of an H100 SXM: the ranges kernel reads every source element once (4 B per depth pixel, 8 B per flow pixel, 12 B
per image pixel); the tile kernel reads the same and writes 3 B per pixel. Host clocks time the device-to-host copy of the
tiles, the PNG writes on the writer's thread pool, and oracle/train_vis.py on the same pack (checked equal to the tiles).
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK_GBS = 3350.0
DEPTHS = ('depth_1', 'depth_2', 'depth_image_1_2', 'depth_warp_1_2', 'depth_nn_1')


def make_pack(B, H, W, dev):
    g = torch.Generator(device='cpu').manual_seed(0)
    pack = {k: (torch.rand(B, 1, H, W, generator=g) * 8 + 1) for k in DEPTHS}
    pack['dflow_1_2'] = torch.randn(B, 2, H, W, generator=g).permute(0, 2, 3, 1)
    pack['staticflow_1_2'] = torch.randn(B, 2, H, W, generator=g).permute(0, 2, 3, 1)
    pack['flow_1_2'] = torch.randn(B, H, W, 2, generator=g) * 4
    pack['flow_2_1'] = torch.randn(B, H, W, 2, generator=g) * 4
    pack['img_1'] = torch.rand(B, 3, H, W, generator=g)
    pack['img_2'] = torch.rand(B, 3, H, W, generator=g)
    return {k: v.to(dev) for k, v in pack.items()}


def bench(B, H, W, dev, reps=20):
    from dvd_b200 import _lib, ops, train_vis
    from oracle import train_vis as ov
    pack = make_pack(B, H, W, dev)
    keys = sorted(pack)
    maps = [(train_vis.image_kind(k), pack[k].permute(0, 3, 1, 2) if train_vis.image_kind(k) == 'flow' else pack[k]) for k in keys]
    turbo = torch.from_numpy(train_vis.turbo_table()).to(dev)
    wheel = torch.from_numpy(np.ascontiguousarray(train_vis.color_wheel() / 255)).to(dev)
    arr, H_, W_, n = ops.vis_map_array(maps, turbo, wheel)
    ranges = torch.empty(2 * n, dtype=torch.float32, device=dev)
    tiles = torch.empty(n, H, W, 3, dtype=torch.uint8, device=dev)
    lib = _lib.load()
    st = ops._stream()

    def ranges_call():
        _lib.check(lib.dvd_vis_ranges(arr, len(maps), H, W, ops._ptr(ranges), st), 'dvd_vis_ranges')

    def tiles_call():
        _lib.check(lib.dvd_vis_tiles(arr, len(maps), H, W, ops._ptr(ranges), ops._ptr(turbo), ops._ptr(wheel), ops._ptr(tiles), st),
                   'dvd_vis_tiles')

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        best = float('inf')
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1) / reps)
        return best

    ms_ranges = timed(ranges_call)
    ms_tiles = timed(tiles_call)
    px = B * H * W
    read = px * (4 * len(DEPTHS) + 8 * 4 + 12 * 2)
    written = px * 3 * len(keys)
    t0 = time.perf_counter()
    host = tiles.cpu().numpy()
    ms_d2h = (time.perf_counter() - t0) * 1e3
    with tempfile.TemporaryDirectory() as d:
        w = train_vis.PageWriter(d)
        out = os.path.join(d, 'visualize', 'epoch0001_train')
        t0 = time.perf_counter()
        w.visualize(pack, 1000, out)
        w.flush()
        ms_page = (time.perf_counter() - t0) * 1e3
        w.close()
    t0 = time.perf_counter()
    want = ov.pack_images({k: v.cpu().numpy() for k, v in pack.items()}, train_vis.turbo_table(), train_vis.color_wheel(),
                          train_vis.image_kind)
    ms_cpu = (time.perf_counter() - t0) * 1e3
    equal = all(np.array_equal(host[q * B:(q + 1) * B], want[k]) for q, k in enumerate(keys))
    return {'B': B, 'H': H, 'W': W, 'images': n, 'ms_ranges': ms_ranges, 'ms_tiles': ms_tiles,
            'gbs_ranges': read / ms_ranges / 1e6, 'gbs_tiles': (read + written) / ms_tiles / 1e6,
            'share_of_peak_tiles': (read + written) / ms_tiles / 1e6 / PEAK_GBS, 'ms_d2h': ms_d2h,
            'ms_visualize_and_pngs': ms_page, 'ms_cpu_oracle': ms_cpu, 'oracle_equal': equal}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--configs', default='1x224x384,8x224x384,1x288x512,8x288x512')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_train_vis needs a GPU')
    dev = torch.device('cuda')
    res = {'device': torch.cuda.get_device_name(dev), 'results': []}
    for c in a.configs.split(','):
        B, H, W = (int(x) for x in c.split('x'))
        r = bench(B, H, W, dev)
        print(json.dumps(r))
        res['results'].append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
