"""Generate tests/golden/train_vis_golden.pt from the UNMODIFIED reference on the CPU (authoring container only):

    python oracle/gen_golden_train_vis.py

Runs `HTMLVisualizer._visualize` (util/util_visualize.py's Converter, util/util_flow.py's flow2img) and
`HTMLVisualizer.prepare_HTML_string` with n_workers=0 over planted packs. `PIL.Image.fromarray` is intercepted to record each
uint8 image and its file name; `heatmap_to_pseudo_color` is wrapped to record every depth heat-map input. The reference's
float turbo table and its colour wheel are recorded as data. Packs: constant and ramped depths, depths with zeros, flows with
zero images, components above 1e7, NaN components and exact wheel-sector angles, images in {0, 1}, in 0..255 and in [-1, 1],
B = 1 and 3, and keys that produce no image."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden', 'train_vis_golden.pt')
BATCH_IDX = (1003, 2001)
H, W = 20, 36


def _ramp(h, w, lo, hi):
    return np.linspace(lo, hi, h * w, dtype=np.float32).reshape(1, h, w)


def planted_packs():
    rng = np.random.default_rng(7)
    B = 3
    rnd = lambda *s: rng.standard_normal(s).astype(np.float32)  # noqa: E731
    depth_1 = np.stack([_ramp(H, W, 0.5, 9.0), _ramp(H, W, 3.0, 3.5), rng.uniform(1, 8, (1, H, W)).astype(np.float32)])
    depth_2 = np.full((B, 1, H, W), 5.0, np.float32)                       # constant: h = 0 everywhere
    depth_image = rng.uniform(1, 8, (B, 1, H, W)).astype(np.float32)
    depth_image[rng.random((B, 1, H, W)) < 0.2] = 0.0                      # zeros: t = 1e6
    sector = np.zeros((H, W, 2), np.float32)                               # exact wheel-sector angles, radius 2
    j = np.arange(H * W) % 55
    theta = np.pi * (2 * j / 54.0 - 1)
    sector[..., 0] = (-2 * np.cos(theta)).astype(np.float32).reshape(H, W)
    sector[..., 1] = (-2 * np.sin(theta)).astype(np.float32).reshape(H, W)
    sector[0, :4] = [[1, 0], [0, 1], [-1, 0], [0, -1]]                     # axis directions
    big = rnd(H, W, 2) * 3
    big[2, 5, 0] = 2e7
    big[4, 7, 1] = -3e7
    static = np.stack([np.zeros((H, W, 2), np.float32), big, sector])
    flow = rnd(B, H, W, 2) * 4
    flow[1, 3, 3, 0] = np.nan                                              # NaN: maxrad = -1 for that image
    flow[2] = 0.0                                                          # all-zero image: NaN everywhere, black
    img01 = (rng.random((B, 3, H, W)) < 0.5).astype(np.float32)
    img255 = np.round(rng.uniform(0, 255, (B, 3, H, W))).astype(np.float32)
    img255[0, :, 0, 0] = [0, 255, 255]
    train = {'batch_size': B, 'depth_1': depth_1, 'depth_2': depth_2, 'depth_image_1_2': depth_image,
             'depth_warp_1_2': rng.uniform(2, 6, (B, 1, H, W)).astype(np.float32), 'depth_nn_1': depth_1[::-1].copy(),
             'dflow_1_2': rnd(B, H, W, 2), 'staticflow_1_2': static, 'flow_1_2': flow, 'flow_2_1': rnd(B, H, W, 2) * 0.01,
             'img_1': img01, 'img_2': img255, 'scenef_1_2': rnd(B, H, W, 1, 3), 'sf_1_2': rnd(B, 3, H, W),
             'global_p1': rnd(B, 3, H, W), 'pair_path': ['a', 'b', 'c']}
    gt = rng.uniform(2, 8, (1, 1, H, W)).astype(np.float32)
    gt[rng.random((1, 1, H, W)) < 0.1] = 0.0
    img = rng.uniform(-1, 1, (1, 3, H, W)).astype(np.float32)
    vali = {'batch_size': 1, 'depth': _ramp(H, W, 9.0, 1.0)[None], 'sf_1_2': rnd(1, 3, H, W), 'img_1': img, 'img_2': img,
            'depth_nn': rng.uniform(1.5, 9, (1, 1, H, W)).astype(np.float32), 'depth_gt': gt,
            'cam_c2w': np.eye(4, dtype=np.float32)[None], 'K': np.eye(3, dtype=np.float32)[None], 'pair_path': ['f0']}
    return [('epoch0001_train', train), ('epoch0002_vali', vali)]


def main():
    ns = ref_harness.import_reference()  # noqa: F841  (installs the shims and the reference's module roots)
    import third_party.util_colormap as ucm
    import util.util_flow as uflow
    import util.util_visualize as uvis
    import visualize.html_visualizer as hv

    recorded, heats = {}, []

    class _Img:
        def __init__(self, arr):
            self.arr = np.array(arr)

        def save(self, path, fmt):
            assert fmt == 'PNG'
            recorded[os.path.basename(path)] = self.arr

    class _PIL:
        fromarray = _Img

    hv.Image = _PIL
    real_heat = uvis.heatmap_to_pseudo_color

    def heat(x):
        heats.append(np.array(x))
        return real_heat(x)
    uvis.heatmap_to_pseudo_color = heat

    class _Logger:
        epoch_content = None

    out = {'turbo_ref': torch.from_numpy(np.asarray(ucm.turbo_colormap_data_np, dtype=np.float64)),
           'wheel_ref': torch.from_numpy(uflow.make_color_wheel()), 'packs': []}
    for (folder, pack), bidx in zip(planted_packs(), BATCH_IDX):
        logger = _Logger()
        vis = hv.HTMLVisualizer(logger, n_workers=0)
        vis.prepare_HTML_string(pack, bidx, folder)
        recorded.clear()
        heats.clear()
        ref_pack = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pack.items()}   # flow2img zeroes in place
        vis._visualize(ref_pack, bidx, '/nonexistent/' + folder)
        out['packs'].append({
            'folder': folder, 'batch_idx': bidx,
            'inputs': {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in pack.items()},
            'images': {k: torch.from_numpy(v) for k, v in recorded.items()},
            'heat': torch.from_numpy(np.stack(heats)), 'heat_keys': [k for k in pack if 'depth' in k],   # 'depth' is the first keyword
            'header': logger.epoch_content['header'], 'rows': logger.epoch_content['content']})
    torch.save(out, OUT)
    print('wrote %s (%d bytes)' % (OUT, os.path.getsize(OUT)))


if __name__ == '__main__':
    main()
