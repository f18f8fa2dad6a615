"""Throughput of the validation pass and of the export pass, in frames/s, timed with CUDA events.

  validation  Model.validate_sequence over a device-resident sequence (MiDaS inference forward in chunks of 8 frames +
              dvd_disp_vali, one read-back), 384x224 / 80 frames and 512x288 / 200 frames, seeded synthetic weights.
  metric      on the depths of that pass: dvd_disp_vali over all frames (one launch pair) against the ATen formula of
              `_vali_on_batch` (depth2disp twice, masks, mse_loss) run frame by frame as the reference's loop does, without its
              per-frame .item() (which would add one host sync per frame).
  export      Model.test_on_batch for every frame at batch size 1 (forward, scene flow, npz file into a temporary directory),
              the `dvd_b200.test` loop.

Prints one JSON object (and writes it to --json PATH when given). Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:       # noqa: BLE001 - informational only
        return 'unknown (%s)' % e


def timed(fn, reps=3):
    """(best, worst) seconds of fn() over `reps` runs, CUDA events around each"""
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1) * 1e-3)
    return min(out), max(out)


def one_size(H, W, n, export_frames):
    from dvd_b200 import ops, synthetic
    from dvd_b200.models import get_model
    from dvd_b200.train import stack_frames
    from oracle.disp_vali import reference_mse
    dev = torch.device('cuda:0')
    with tempfile.TemporaryDirectory() as tmp:
        model = get_model('scene_flow_motion_field')(synthetic.default_opt(output_dir=tmp, epoch=-1), None)
        synthetic.seed_net_(model.net_depth, 0, 2000.0)
        synthetic.seed_net_(model.net_sceneflow, 1)
        model.to(dev)
        frames = stack_frames([synthetic.make_frame(i, H=H, W=W, n_frames=n) for i in range(n)], n, dev)
        model.validate_sequence(frames)                       # warm-up: packs, allocator
        torch.cuda.synchronize()
        vb, vw = timed(lambda: model.validate_sequence(frames))
        loss = model.validate_sequence(frames)

        with torch.no_grad():
            model.net_depth.eval()
            depth = torch.cat([model.net_depth(frames['img'][s:s + 8]) for s in range(0, n, 8)])
        gt = frames['depth_mvs']
        kb, kw = timed(lambda: ops.disp_vali(depth, gt), reps=20)
        aten = lambda: torch.stack([reference_mse(depth[i:i + 1], gt[i:i + 1]) for i in range(n)])  # noqa: E731
        aten()
        ab, aw = timed(aten, reps=5)
        kernel_loss = float((ops.disp_vali(depth, gt).double() / (H * W)).mean())
        aten_loss = float(aten().double().mean())

        def export():
            for i in range(export_frames):
                model.test_on_batch(i, {k: v[i:i + 1] for k, v in frames.items()})
        export()
        eb, ew = timed(export, reps=2)
        model.train()
    return {'H': H, 'W': W, 'frames': n,
            'vali_fps': n / vb, 'vali_ms': vb * 1e3, 'vali_ms_worst': vw * 1e3, 'loss_eval': loss,
            'metric_kernel_ms': kb * 1e3, 'metric_kernel_ms_worst': kw * 1e3, 'metric_aten_ms': ab * 1e3,
            'metric_aten_ms_worst': aw * 1e3, 'metric_speedup': ab / kb,
            'metric_loss_kernel': kernel_loss, 'metric_loss_aten': aten_loss,
            'export_frames': export_frames, 'export_fps': export_frames / eb, 'export_fps_worst': export_frames / ew}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    t0 = time.time()
    res = {'gpu': gpu_info(), 'sizes': [one_size(224, 384, 80, 80), one_size(288, 512, 200, 200)]}
    res['wall_s'] = time.time() - t0
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
