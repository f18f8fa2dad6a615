"""CPU: the validation / export surface — `options_test` flags, the test driver's output naming, `opt.pt`, the synthetic `vali`
items, the fp32 restatement of `dvd_disp_vali` (oracle/disp_vali.py) against torch's own terms of the reference formula, the
exported npz layout of the reference (tests/golden/eval_export_golden.pt) and the CPU oracle against the reference's exported
depth and scene flow."""
import argparse
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_err

VALI_KEYS = {'img', 'R_1', 'R_1_T', 't_1', 'K', 'K_inv', 'time_stamp_1', 'time_step', 'frame_id_1', 'depth_pred', 'cam_c2w',
             'pair_path', 'depth_mvs'}
NPZ_KEYS = {'batch_size', 'img_1', 'img_2', 'depth', 'sf_1_2', 'depth_nn', 'depth_gt', 'cam_c2w', 'K', 'pair_path'}


def test_options_test_accepts_the_reference_test_command():
    from dvd_b200.options import options_test
    from dvd_b200.test import output_dir_for
    # experiments/davis/test_cmd.txt, formatted as train.py:355 formats it
    argv = ('--net scene_flow_motion_field --dataset davis_sequence --workers 4 --output_dir ./test_results/davis_sequence/ '
            '--epoch -1 --html_logger --batch_size 1 --gpu 0 --track_id dog --suffix epoch_-1 '
            '--checkpoint_path ./checkpoints/davis/sequence/scene_flow_motion_field_davis_sequence/0').split()
    opt = options_test.parse(argv)
    assert opt.epoch == -1 and opt.batch_size == 1 and opt.html_logger and opt.workers == 4 and opt.track_id == 'dog'
    assert opt.checkpoint_path.endswith('/0') and opt.suffix == 'epoch_-1' and not opt.overwrite and opt.manual_seed is None
    assert options_test.parse(['--net', 'scene_flow_motion_field', '--dataset', 'synthetic_sequence', '--gpu', '0',
                               '--checkpoint_path', 'x', '--output_dir', 'y']).suffix == 'epoch_{epoch}'


def test_test_driver_output_directory_and_overwrite_rule(tmp_path):
    from dvd_b200.test import output_dir_for
    o = argparse.Namespace(output_dir=str(tmp_path) + '/', net='scene_flow_motion_field', dataset='synthetic_sequence',
                           suffix='epoch_{epoch}', epoch=3, overwrite=False)
    out = output_dir_for(o)      # test.py:52-53: plain concatenation, the suffix formatted with the options
    assert out == str(tmp_path) + '/scene_flow_motion_field_synthetic_sequence_epoch_3' and os.path.isdir(out)
    os.makedirs(os.path.join(out, 'epoch_0003'))
    with pytest.raises(ValueError):
        output_dir_for(o)
    o.overwrite = True
    assert output_dir_for(o) == out and not os.path.exists(os.path.join(out, 'epoch_0003'))
    o.suffix = ''
    assert output_dir_for(o) == str(tmp_path) + '/scene_flow_motion_field_synthetic_sequence'


def test_train_driver_writes_a_loadable_opt_pt(tmp_path):
    from dvd_b200.options import options_train
    from dvd_b200.train import save_opt
    opt, _ = options_train.parse(['--net', 'scene_flow_motion_field', '--dataset', 'synthetic_sequence', '--midas', '--validate',
                                  '--full_logdir', str(tmp_path / 'log')])
    assert opt.validate and not options_train.parse(['--net', 'scene_flow_motion_field'])[0].validate
    save_opt(opt)
    d = torch.load(str(tmp_path / 'log' / 'opt.pt'))        # the reference's test.py loads it with torch.load's defaults
    assert d == vars(opt) and argparse.Namespace(**d).midas
    assert 'midas' in open(str(tmp_path / 'log' / 'opt.txt')).read()


def test_synthetic_vali_items_have_the_davis_vali_keys():
    from dvd_b200.datasets import get_dataset
    from dvd_b200.options import options_train
    opt, _ = options_train.parse(['--net', 'scene_flow_motion_field', '--dataset', 'synthetic_sequence', '--n_frames', '6',
                                  '--height', '32', '--width', '48'])
    ds = get_dataset('synthetic_sequence')(opt, mode='vali')
    assert len(ds) == 6
    s = ds[4]
    assert set(s) == VALI_KEYS
    shapes = {'img': (3, 32, 48), 'R_1': (1, 1, 3, 3), 'R_1_T': (1, 1, 3, 3), 't_1': (1, 1, 1, 3), 'K': (1, 1, 3, 3),
              'K_inv': (1, 1, 3, 3), 'time_stamp_1': (1, 32, 48), 'depth_pred': (1, 32, 48), 'cam_c2w': (4, 4),
              'depth_mvs': (1, 32, 48)}
    for k, sh in shapes.items():
        assert tuple(s[k].shape) == sh and s[k].dtype == torch.float32, k
    assert s['frame_id_1'] == 4 and s['time_step'] == 1 / 6 and float(s['time_stamp_1'][0, 0, 0]) == np.float32(4 / 6)
    # R_1 holds R_c2w^T, R_1_T holds R_c2w (davis_sequence.py:141-145), consistent with cam_c2w
    assert torch.equal(s['R_1_T'].reshape(3, 3), s['cam_c2w'][:3, :3]) and torch.equal(s['R_1'].reshape(3, 3), s['cam_c2w'][:3, :3].t())
    gt = s['depth_mvs']
    assert 0.03 < float((gt == 0).float().mean()) < 0.2 and float(gt.max()) <= 8.0
    assert torch.equal(ds[4]['depth_mvs'], gt)                    # seeded
    # train mode is untouched
    tr = get_dataset('synthetic_sequence')(opt)
    assert len(tr) == 10 and tr[5]['img_1'].shape == (1, 3, 32, 48)


def _edge_depths():
    """every branch of the formula: exactly 1e-2f, its neighbours, 0, -0, tiny, huge, negative, and a random bulk"""
    f = np.float32
    t = f(1e-2)
    edges = np.array([t, np.nextafter(t, f(1)), np.nextafter(t, f(0)), 0.0, -0.0, 1e-8, f(1e-8) * 2, 1e-30, 3.0, 1e6, 1e30,
                      -1.0, -2e-8, 0.5, 7.25], dtype=np.float32)
    g = torch.Generator().manual_seed(5)
    d = torch.from_numpy(np.concatenate([edges.repeat(len(edges)), (torch.rand(3000, generator=g) * 10).numpy()]))
    gt = torch.from_numpy(np.concatenate([np.tile(edges, len(edges)), (torch.rand(3000, generator=g) * 10).numpy()]))
    gt[len(edges) ** 2::7] = 0.0
    return d.reshape(1, 1, 1, -1).contiguous(), gt.reshape(1, 1, 1, -1).contiguous()


def test_fp32_restatement_reproduces_torch_terms_bitwise():
    from oracle import disp_vali
    d, g = _edge_depths()
    ref = disp_vali.reference_terms(d, g).numpy()
    mine = disp_vali.terms_fp32(d, g)
    assert mine.dtype == np.float32 and mine.shape == ref.shape
    same = (mine.view(np.uint32) == ref.view(np.uint32)) | (np.isnan(mine) & np.isnan(ref))
    assert same.all(), np.argwhere(~same)[:10]
    # the threshold is strict and taken in fp32: depth == 1e-2f is invalid, its upper neighbour valid
    t = np.float32(1e-2)
    dd = torch.tensor([t, np.nextafter(t, np.float32(1))]).reshape(1, 1, 1, 2)
    gg = torch.full((1, 1, 1, 2), 1.0)
    assert disp_vali.terms_fp32(dd, gg)[0, 0, 0, 0] == 1.0 and disp_vali.terms_fp32(dd, gg)[0, 0, 0, 1] > 1e3
    assert (disp_vali.terms_fp32(dd, torch.zeros_like(dd)) == 0).all()        # gt == 0: no contribution


def test_fp64_frame_sums_equal_the_reference_mse():
    from dvd_b200 import synthetic
    from oracle import disp_vali
    N, H, W = 3, 37, 53
    d = synthetic.make_depths(N, H, W, seed=3, lo=0.005, hi=9.0)
    g = synthetic.make_depths(N, H, W, seed=4, lo=-0.5, hi=8.0).clamp_min(0)
    sse, asum = disp_vali.frame_sse_fp64(disp_vali.terms_fp32(d, g))
    assert (asum == sse).all() and (sse > 0).all()
    for n in range(N):
        ref = disp_vali.reference_terms(d[n:n + 1], g[n:n + 1]).double().mean().item()
        assert abs(sse[n] / (H * W) - ref) <= 1e-12 * abs(ref)
        # the reference's fp32 `mse_loss` (its own summation order) agrees to fp32 accuracy
        assert abs(sse[n] / (H * W) - disp_vali.reference_mse(d[n:n + 1], g[n:n + 1]).item()) <= 1e-5 * abs(ref)
    # a batch's mse_loss is the mean of its frames' MSEs (equal frame sizes)
    assert abs(sse.mean() / (H * W) - disp_vali.reference_mse(d, g).item()) <= 1e-5 * sse.mean() / (H * W)
    assert disp_vali.sum_depth(224, 384, 42) == 8 + 3 + 20


def test_library_exports_the_validation_entry_points():
    """the C ABI rows of include/dvd_b200.h for csrc/eval_ops.cu are declared, bound and exported"""
    import ctypes
    import test_capi_symbols
    from dvd_b200 import _lib
    names = {'dvd_disp_vali', 'dvd_disp_vali_partials_size'}
    assert names <= set(test_capi_symbols._declared()) and names <= set(_lib.SIGNATURES)
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert all(hasattr(lib, n) for n in names)
    lib = _lib.load()
    assert lib.dvd_version() >= 103
    assert lib.dvd_disp_vali_partials_size(80, 224, 384) == 80 * 42 and lib.dvd_disp_vali_partials_size(2, 1, 1) == 2
    assert lib.dvd_disp_vali_partials_size(1, 4096, 4096) == 128 and lib.dvd_disp_vali_partials_size(0, 8, 8) == -1


@pytest.fixture(scope='module')
def export_golden():
    from oracle.golden_io import load_golden
    return load_golden(GOLDEN, 'eval_export_golden')


def test_export_fixture_layout(export_golden):
    lay = export_golden['layout']
    assert set(lay) == NPZ_KEYS
    m = export_golden['meta']
    H, W = m['H'], m['W']
    assert lay['depth'] == ((1, 1, H, W), '<f4') and lay['sf_1_2'] == ((1, 3, H, W), '<f4')
    assert lay['img_1'] == ((1, 3, H, W), '<f4') and lay['K'] == ((1, 1, 1, 3, 3), '<f4') and lay['cam_c2w'] == ((1, 4, 4), '<f4')
    assert lay['batch_size'] == ((), '<i8') and lay['pair_path'][0] == (1,) and lay['pair_path'][1].startswith('<U')
    assert export_golden['depth'].shape == (m['n_frames'], 1, H, W)


def test_cpu_oracle_matches_the_reference_export(export_golden):
    """the oracle the GPU export test compares against equals what the reference's test_on_batch wrote"""
    from dvd_b200 import synthetic
    from dvd_b200.models import get_model
    from oracle.gen_golden_eval import oracle_forward
    m = export_golden['meta']
    model = get_model('scene_flow_motion_field')(synthetic.default_opt(), None)
    synthetic.seed_net_(model.net_depth, m['depth_seed'], m['head_bias'])
    synthetic.seed_net_(model.net_sceneflow, m['mlp_seed'])
    frames = [synthetic.make_frame(i, H=m['H'], W=m['W'], n_frames=m['n_frames']) for i in range(m['n_frames'])]
    batch = torch.utils.data.default_collate(frames)
    d, sf = oracle_forward(model.net_depth.state_dict(), model.net_sceneflow.state_dict(), batch)
    assert rel_err(d, export_golden['depth']) < 1e-5
    assert rel_err(sf, export_golden['sf_1_2']) < 1e-4
