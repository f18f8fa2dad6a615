"""TEST INFRASTRUCTURE — export fixture: runs the UNMODIFIED reference `test_on_batch` / `pack_output`
(models/video_base.py:105-155) through oracle/ref_harness.py on a seeded 6-frame 64x96 synthetic video (the `vali` items of
dvd_b200's synthetic_sequence, batch size 1) with name-seeded weights (dvd_b200.synthetic.seed_net_), and stores the keys, shapes
and dtypes of every batch%04d.npz it writes plus its `depth` and `sf_1_2`. Authoring container only."""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_harness  # noqa: E402
from oracle.golden_io import save_golden  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
H, W, N_FRAMES = 64, 96, 6
DEPTH_SEED, MLP_SEED, HEAD_BIAS = 0, 1, 2000.0


def frames():
    from dvd_b200 import synthetic
    return [synthetic.make_frame(i, H=H, W=W, n_frames=N_FRAMES) for i in range(N_FRAMES)]


def oracle_forward(sd_depth, sd_mlp, batch):
    """CPU oracle of `_predict_on_batch(is_train=False)` (smf.py:265-276) on a per-frame batch: MiDaS depth, un-projection with
    the frame's own pose, one Euler step of the scene-flow MLP."""
    from oracle import depth_nets, geometry, sf_mlp
    B = batch['img'].shape[0]
    with torch.no_grad():
        d = depth_nets.midas_forward(sd_depth, batch['img'].cpu())
        R = batch['R_1_T'].cpu().reshape(B, 3, 3)
        t = batch['t_1'].cpu().reshape(B, 3)
        Kinv = batch['K_inv'].cpu().reshape(B, 3, 3).transpose(1, 2)
        P = geometry.unproject(d, R, t, Kinv)
        dt = batch['time_step']
        dt = float(dt.reshape(-1)[0]) if torch.is_tensor(dt) else float(dt)
        sf = sf_mlp.sf_multi_step(P, batch['time_stamp_1'].cpu(), dt, 1, sf_mlp.layers_from_state_dict(sd_mlp))
    return d, sf


def run():
    from dvd_b200 import synthetic
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    model, _ = ref_harness.build_reference_model(ref_harness.default_opt(), seed=0)
    synthetic.seed_net_(model.net_depth, DEPTH_SEED, HEAD_BIAS)
    synthetic.seed_net_(model.net_sceneflow, MLP_SEED)
    loader = torch.utils.data.DataLoader(frames(), batch_size=1, shuffle=False, drop_last=False)
    with tempfile.TemporaryDirectory() as tmp:
        model.opt.output_dir = tmp
        model.opt.epoch = -1
        for i, batch in enumerate(loader):
            model.test_on_batch(i, batch)
        files = sorted(os.listdir(os.path.join(tmp, 'epochbest_test')))
        assert files == ['batch%04d.npz' % i for i in range(N_FRAMES)], files
        layout, depth, sf = None, [], []
        for f in files:
            d = np.load(os.path.join(tmp, 'epochbest_test', f))
            lay = {k: (tuple(d[k].shape), d[k].dtype.str) for k in d.files}
            assert layout is None or {k: v[0] for k, v in lay.items()} == {k: v[0] for k, v in layout.items()}
            layout = lay
            depth.append(torch.from_numpy(d['depth'].copy()))
            sf.append(torch.from_numpy(d['sf_1_2'].copy()))
    return {'layout': layout, 'depth': torch.cat(depth), 'sf_1_2': torch.cat(sf),
            'meta': {'H': H, 'W': W, 'n_frames': N_FRAMES, 'depth_seed': DEPTH_SEED, 'mlp_seed': MLP_SEED, 'head_bias': HEAD_BIAS}}


def main():
    os.makedirs(GOLD, exist_ok=True)
    out = run()
    save_golden(out, GOLD, 'eval_export_golden')
    print('wrote eval_export_golden', out['layout'])


if __name__ == '__main__':
    main()
