"""GPU: the flow-pair kernels (csrc/flow_pairs.cu) against the reference's preprocessing stored in the fixture
(tests/golden/flow_pairs_golden*), the pair builder on raw flows, one optimisation step on a built pair against the same pair read
from written files, the training driver on a video read from frames and flows, and the raw C ABI's argument checks."""
import ctypes
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_err
from oracle import flow_pairs as ofp
from oracle.golden_io import load_golden
from test_flow_pairs_cpu import write_video

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def golden():
    return load_golden(GOLDEN, 'flow_pairs_golden')


def _band(ref, k, shape):
    bits = ref['band_' + k]
    if bits.dim() == 2:
        return np.stack([ofp.unpack_band(b.numpy(), shape[1:]) for b in bits])
    return ofp.unpack_band(bits.numpy(), shape)


def _assert_masks(m, ref_u8, band, convention):
    m = m.cpu().numpy()
    if convention == 'pair_file':
        assert m.shape == ref_u8.shape + (1, 1) and m.dtype == np.float32
        m = (1 - m[..., 0, 0]).astype(np.uint8)
    else:
        assert m.shape == ref_u8.shape and m.dtype == np.uint8
    keep = ~band
    assert keep.mean() > 0.99
    assert np.array_equal(m[keep], ref_u8[keep])


def test_resize_kernel_matches_cv2(golden):
    from dvd_b200 import ops
    H, W = golden['meta']['H'], golden['meta']['W']
    for raw, ref in (('raw_1_2', 'flow_1_2'), ('raw_2_1', 'flow_2_1')):
        src = torch.stack([fl[raw] for fl in golden['flows']]).cuda()
        out = ops.flow_resize_cubic(src, H, W)
        for j, fl in enumerate(golden['flows']):
            assert rel_err(out[j], fl[ref]) <= 1e-5, (fl['pair'], raw, rel_err(out[j], fl[ref]))
        # and the CPU restatement's operation order
        assert rel_err(out.cpu(), torch.from_numpy(ofp.resize_flow_cubic(src.cpu().numpy(), H, W))) <= 1e-6
    # down-sampling, non-integer ratios, odd sizes
    g = torch.Generator().manual_seed(0)
    for (h, w, Ho, Wo) in ((288, 512, 224, 384), (17, 23, 40, 31), (40, 56, 13, 9)):
        src = torch.randn(3, h, w, 2, generator=g) * 4
        out = ops.flow_resize_cubic(src.cuda(), Ho, Wo).cpu()
        assert rel_err(out, torch.from_numpy(ofp.resize_flow_cubic(src.numpy(), Ho, Wo))) <= 1e-6, (h, w, Ho, Wo)


@pytest.mark.parametrize('convention', ['flowpair', 'pair_file'])
def test_mask_kernel_matches_reference(golden, convention):
    from dvd_b200 import ops
    fl = golden['flows']
    f12 = torch.stack([f['flow_1_2'] for f in fl]).cuda()
    f21 = torch.stack([f['flow_2_1'] for f in fl]).cuda()
    m1, m2 = ops.flow_pair_masks(f12, f21, convention=convention)
    for j, f in enumerate(fl):
        for k, m in (('1', m1), ('2', m2)):
            ref = f['mask_' + k].numpy()
            _assert_masks(m[j], ref, _band(f, k, ref.shape), convention)
    # odd width, B = 5 and B = 1
    odd = golden['odd']
    for sl in (slice(0, 5), slice(2, 3)):
        m1, m2 = ops.flow_pair_masks(odd['flow_1_2'][sl].contiguous().cuda(), odd['flow_2_1'][sl].contiguous().cuda(),
                                     convention=convention)
        for k, m in (('1', m1), ('2', m2)):
            ref = odd['mask_' + k][sl].numpy()
            band = _band({'band_' + k: odd['band_' + k][sl]}, k, ref.shape)
            _assert_masks(m, ref, band, convention)
    # the kernel and the CPU restatement agree bitwise (same operation order), band included
    a, b = odd['flow_1_2'].numpy(), odd['flow_2_1'].numpy()
    m1, m2 = ops.flow_pair_masks(odd['flow_1_2'].cuda(), odd['flow_2_1'].cuda(), convention=convention)
    o1, o2 = ofp.pair_masks(a, b, convention)
    assert np.array_equal(m1.cpu().numpy(), o1) and np.array_equal(m2.cpu().numpy(), o2)


@pytest.mark.parametrize('flows', ['raw', 'raw_full'])
def test_builder_on_raw_flows_equals_the_reference(golden, tmp_path, flows):
    from dvd_b200.flow_pairs import PairBuilder
    fdir, pdir = write_video(golden, str(tmp_path), flows=flows)
    b = PairBuilder(fdir, pdir, golden['meta']['gaps'])
    assert b.raw_pairs == len(b) == len(golden['flows'])
    ref_items = golden['items']['davis_sequence/train']
    masked = ('mask_1', 'mask_2', 'motion_seg_1')
    for i, fl in enumerate(golden['flows']):
        it = b[i]
        d = ofp.digest_item(it)
        for k, v in ref_items[i].items():
            if k in masked or (flows == 'raw' and k in ('flow_1_2', 'flow_2_1')):
                continue
            assert d[k] == v, (i, k)
        for k in ('flow_1_2', 'flow_2_1'):
            assert rel_err(it[k][0], fl[k]) <= 1e-5, (i, k)
        a, bb = fl['pair']
        for k in ('1', '2'):
            ref = fl['mask_' + k].numpy()
            _assert_masks(it['mask_' + k][0], ref, _band(fl, k, ref.shape), 'pair_file')
        if 'motion_seg' not in golden['frames'][a]:
            assert torch.equal(it['motion_seg_1'], it['mask_2'])
        else:
            assert d['motion_seg_1'] == ref_items[i]['motion_seg_1']


def make_video(root, track='clip', n=6, H=64, W=96, raw=(36, 48), seed=0):
    """a small video in the reference's layout: frames at HxW and raw flows at `raw` resolution (no masks)"""
    rng = np.random.default_rng(seed)
    fdir, pdir = os.path.join(root, 'frames_midas', track), os.path.join(root, 'flow_pairs', track)
    os.makedirs(fdir)
    os.makedirs(pdir)
    for f in range(n):
        pose = np.eye(4)
        pose[:3, 3] = rng.standard_normal(3) * 0.05
        K = np.array([[60.0, 0, W / 2 - 0.5], [0, 60.0, H / 2 - 0.5], [0, 0, 1]])
        np.savez(os.path.join(fdir, 'frame_%05d.npz' % f), img=rng.random((H, W, 3)).astype(np.float32), pose_c2w=pose,
                 intrinsics=K, depth_mvs=(2 + rng.random((H, W))).astype(np.float32),
                 depth_pred=(2 + rng.random((H, W))).astype(np.float32))
    for g in range(1, n):
        for f in range(n - g):
            f12 = (rng.standard_normal((raw[0], raw[1], 2)) * 0.3 + 0.5 * g).astype(np.float32)
            f21 = (-f12 + rng.standard_normal(f12.shape) * 0.1).astype(np.float32)
            np.savez(os.path.join(pdir, 'flowpair_%05d_%05d.npz' % (f, f + g)), flow_1_2=f12, flow_2_1=f21)
    return fdir, pdir


def _step(over, batch):
    from dvd_b200 import synthetic
    from dvd_b200.models import get_model
    opt = synthetic.default_opt(**over)
    model = get_model('scene_flow_motion_field')(opt, None)
    synthetic.seed_net_(model.net_depth, 0, 2000.0 if opt.midas else None)
    synthetic.seed_net_(model.net_sceneflow, 1)
    model.to(torch.device('cuda:0'))
    log = model._train_on_batch(6, 0, batch)
    torch.cuda.synchronize()
    params = [p.detach().cpu().clone() for net in (model.net_depth, model.net_sceneflow) for p in net.parameters()]
    return {k: float(v) for k, v in log.items() if isinstance(v, (float, int)) or (torch.is_tensor(v) and v.numel() == 1)}, params


@pytest.mark.parametrize('midas', [False, True], ids=['hourglass', 'midas'])
def test_step_on_built_pair_equals_step_on_written_pair(tmp_path, midas):
    from dvd_b200.datasets import get_dataset
    from dvd_b200.flow_pairs import PairBuilder
    root = str(tmp_path / 'data')
    fdir, pdir = make_video(root)
    b = PairBuilder(fdir, pdir, [2])
    b.write(os.path.join(root, 'sequences_select_pairs_midas', 'clip', '001'))
    opt = types.SimpleNamespace(subsample=False, overfit=False, repeat=1, gaps='2', data_root=root, track_id='clip')
    ds = get_dataset('davis_sequence')(opt, mode='train')
    i = 1
    collate = torch.utils.data.default_collate
    bb, bd = collate([b[i]]), collate([ds[i]])
    assert set(bb) == set(bd)
    for k in bb:
        if torch.is_tensor(bb[k]):
            assert bb[k].dtype == bd[k].dtype and torch.equal(bb[k], bd[k]), k
    over = dict(midas=midas, lr=1e-4)
    log_b, p_b = _step(over, bb)
    log_d, p_d = _step(over, bd)
    assert log_b == log_d, (log_b, log_d)
    assert all(np.isfinite(v) for v in log_b.values())
    # the weight gradients are summed with fp32 atomics, so two steps on one batch can differ in the last bits of a gradient,
    # and Adam's first step (lr * g / (|g| + eps)) turns a last-bit change of a near-zero gradient into up to lr: the batches
    # are bitwise equal (above); the updated weights agree element for element except where that reordering reaches them
    same = sum(int((x == y).sum()) for x, y in zip(p_b, p_d))
    total = sum(x.numel() for x in p_b)
    for x, y in zip(p_b, p_d):
        assert (x - y).abs().max() <= 2 * over['lr'], rel_err(x, y)
    assert same >= 0.9 * total, (same, total)
    print('bitwise-equal weights after the step: %d of %d' % (same, total))


@pytest.mark.timeout(1200)
def test_train_driver_on_video_frames(tmp_path):
    root = str(tmp_path / 'data')
    make_video(root, n=8)
    args = ('--net scene_flow_motion_field --dataset video_frames --track_id clip --gaps 1,2 --epoch 1 --epoch_batches 2 '
            '--resident --lr 1e-6 --batch_size 1 --optim adam --gpu 0 --workers 0 --one_way --loss_type l1 --l1_mul 0 '
            '--acc_mul 1 --disp_mul 1 --warm_sf 1 --scene_lr_mul 1000 --flow_mul 1 --sf_mag_div 100 --time_dependent --use_disp '
            '--vis_batches_train 0 --manual_seed 1').split() + ['--data_root', root, '--logdir', str(tmp_path / 'log')]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', 'dvd_b200.train'] + args, cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=1100)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    lines = [l for l in r.stdout.splitlines() if l.startswith('epoch 1:')]
    assert lines, r.stdout[-2000:]
    log = eval(lines[0].split(':', 1)[1])
    assert all(np.isfinite(v) for v in log.values()), log


def test_raw_abi_rejects_bad_arguments_before_launch():
    from dvd_b200 import _lib
    lib = _lib.load()
    P = ctypes.c_void_p
    src = torch.zeros(2, 8, 10, 2, device='cuda')
    dst = torch.full((2, 16, 20, 2), 7.0, device='cuda')
    m = torch.full((2, 16, 20), 5, dtype=torch.uint8, device='cuda')
    m2 = m.clone()
    mf = torch.full((2, 16, 20), 5.0, device='cuda')
    s = P(torch.cuda.current_stream().cuda_stream)
    nb_s, nb_d = src.numel() * 4, dst.numel() * 4
    bad_resize = [
        (P(src.data_ptr()), nb_s - 8, P(dst.data_ptr()), nb_d, 2, 8, 10, 16, 20),        # size mismatch
        (P(src.data_ptr()), nb_s, P(dst.data_ptr()), nb_d + 4, 2, 8, 10, 16, 20),
        (P(src.data_ptr() + 4), nb_s, P(dst.data_ptr()), nb_d, 2, 8, 10, 16, 20),        # misaligned
        (P(src.data_ptr()), nb_s, P(dst.data_ptr() + 4), nb_d, 2, 8, 10, 16, 20),
        (P(0), nb_s, P(dst.data_ptr()), nb_d, 2, 8, 10, 16, 20),                         # null
        (P(src.data_ptr()), nb_s, P(dst.data_ptr()), nb_d, 0, 8, 10, 16, 20),            # shape
    ]
    for a in bad_resize:
        assert lib.dvd_flow_resize_cubic(*a, s) == -2, a
        assert lib.dvd_last_error()
    f = dst  # [2,16,20,2]
    nb_f = f.numel() * 4
    bad_masks = [
        (P(f.data_ptr()), P(f.data_ptr()), nb_f - 8, P(m.data_ptr()), P(m2.data_ptr()), m.numel(), 2, 16, 20, 0),
        (P(f.data_ptr()), P(f.data_ptr()), nb_f, P(m.data_ptr()), P(m2.data_ptr()), m.numel() * 4, 2, 16, 20, 0),
        (P(f.data_ptr() + 4), P(f.data_ptr()), nb_f, P(m.data_ptr()), P(m2.data_ptr()), m.numel(), 2, 16, 20, 0),
        (P(f.data_ptr()), P(f.data_ptr()), nb_f, P(mf.data_ptr() + 2), P(mf.data_ptr()), mf.numel() * 4, 2, 16, 20, 1),
        (P(f.data_ptr()), P(f.data_ptr()), nb_f, P(m.data_ptr()), P(m2.data_ptr()), m.numel(), 2, 16, 20, 7),
        (P(f.data_ptr()), P(f.data_ptr()), nb_f, P(m.data_ptr()), P(0), m.numel(), 2, 16, 20, 0),
        (P(f.data_ptr()), P(f.data_ptr()), 2 * 16 * 1 * 8, P(m.data_ptr()), P(m2.data_ptr()), 2 * 16, 2, 16, 1, 0),
    ]
    for a in bad_masks:
        assert lib.dvd_flow_pair_masks(*a, s) == -2, a
    torch.cuda.synchronize()
    assert (dst == 7).all() and (m == 5).all() and (m2 == 5).all() and (mf == 5).all()   # nothing was launched
    with pytest.raises(ValueError):
        from dvd_b200 import ops
        ops.flow_pair_masks(f, f[:, :8].contiguous())
