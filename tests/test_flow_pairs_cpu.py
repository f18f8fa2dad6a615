"""CPU: the flow-pair oracle against the reference's preprocessing (tests/golden/flow_pairs_golden*, written by
oracle/gen_golden_flow_pairs.py), and the pair builder, its writer and the davis_sequence / shutterstock / video_frames datasets
against the reference's datasets on the fixture video (flows with masks, so no kernel runs)."""
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import flow_pairs as ofp
from oracle.golden_io import load_golden


@pytest.fixture(scope='module')
def golden():
    return load_golden(GOLDEN, 'flow_pairs_golden')


def write_video(g, root, flows='finished'):
    """the fixture video in the reference's layout under root/{frames_midas,flow_pairs}/<track>; flows: 'finished' (the
    reference's flowpair files), 'raw' (24x32 flows, no masks) or 'raw_full' (working-resolution flows, no masks)"""
    track = g['meta']['track']
    fdir, pdir = os.path.join(root, 'frames_midas', track), os.path.join(root, 'flow_pairs', track)
    os.makedirs(fdir, exist_ok=True)
    os.makedirs(pdir, exist_ok=True)
    for f, d in enumerate(g['frames']):
        np.savez(os.path.join(fdir, 'frame_%05d.npz' % f), **{k: v.numpy() for k, v in d.items()})
    for fl in g['flows']:
        a, b = fl['pair']
        if flows == 'finished':
            d = dict(flow_1_2=fl['flow_1_2'].numpy(), flow_2_1=fl['flow_2_1'].numpy(), mask_1=fl['mask_1'].numpy(),
                     mask_2=fl['mask_2'].numpy(), frame_id_1=a, frame_id_2=b)
        elif flows == 'raw':
            d = dict(flow_1_2=fl['raw_1_2'].numpy(), flow_2_1=fl['raw_2_1'].numpy())
        else:
            d = dict(flow_1_2=fl['flow_1_2'].numpy(), flow_2_1=fl['flow_2_1'].numpy())
        np.savez(os.path.join(pdir, 'flowpair_%05d_%05d.npz' % (a, b)), **d)
    return fdir, pdir


def opt_for(g, root, track=None):
    return types.SimpleNamespace(subsample=False, overfit=False, repeat=g['meta']['repeat'], cache=False, select=False,
                                 gaps=','.join(str(x) for x in g['meta']['gaps']), data_root=root,
                                 track_id=g['meta']['track'] if track is None else track)


def test_oracle_resize_matches_cv2(golden):
    H, W = golden['meta']['H'], golden['meta']['W']
    for fl in golden['flows']:
        for raw, ref in (('raw_1_2', 'flow_1_2'), ('raw_2_1', 'flow_2_1')):
            mine = ofp.resize_flow_cubic(fl[raw].numpy(), H, W)
            b = fl[ref].numpy()
            assert mine.shape == b.shape and mine.dtype == np.float32
            assert np.abs(mine - b).max() <= 1e-6 * np.abs(b).max(), (fl['pair'], raw)


def _check_masks(mine_1, mine_2, ref, batch=False):
    n_bad = 0
    for k, mine in (('1', mine_1), ('2', mine_2)):
        r = ref['mask_' + k].numpy()
        band = ofp.unpack_band(ref['band_' + k].numpy(), r.shape) if not batch else np.stack(
            [ofp.unpack_band(bits, r.shape[1:]) for bits in ref['band_' + k].numpy()])
        keep = ~band
        assert keep.mean() > 0.99
        assert np.array_equal(np.asarray(mine)[keep], r[keep]), k
        n_bad += int(r.sum())
    assert n_bad > 0


def test_oracle_masks_match_reference(golden):
    for fl in golden['flows']:
        m1, m2 = ofp.pair_masks(fl['flow_1_2'].numpy(), fl['flow_2_1'].numpy(), 'flowpair')
        _check_masks(m1, m2, fl)
        v1, v2 = ofp.pair_masks(fl['flow_1_2'].numpy(), fl['flow_2_1'].numpy(), 'pair_file')
        assert v1.shape == m1.shape + (1, 1) and v1.dtype == np.float32
        assert np.array_equal(v1[..., 0, 0], 1 - m1) and np.array_equal(v2[..., 0, 0], 1 - m2)
    # every pixel class is exercised: out of bounds, inconsistent inside the image, valid
    m = np.stack([fl['mask_1'].numpy() for fl in golden['flows']])
    assert 0.02 < m.mean() < 0.6
    odd = golden['odd']
    m1, m2 = ofp.pair_masks(odd['flow_1_2'].numpy(), odd['flow_2_1'].numpy(), 'flowpair')
    _check_masks(m1, m2, odd, batch=True)


def test_pair_list_follows_the_reference_rule():
    from dvd_b200.flow_pairs import pair_list
    assert pair_list(6, [1, 4]) == [(0, 1), (1, 2), (2, 3), (3, 4), (0, 4)]
    assert pair_list(3, [2]) == []


def test_builder_writer_and_mirrors_equal_the_reference(golden, tmp_path):
    from dvd_b200.datasets import get_dataset
    from dvd_b200.flow_pairs import PairBuilder
    root = str(tmp_path / 'davis_processed')
    fdir, pdir = write_video(golden, root)
    track = golden['meta']['track']
    b = PairBuilder(fdir, pdir, golden['meta']['gaps'], device='cpu')
    assert b.raw_pairs == 0 and len(b) == len(golden['pair_files'])
    # the writer emits the reference's pair files, bitwise
    out = os.path.join(root, 'sequences_select_pairs_midas', track, '001')
    assert b.write(out, flows_out=str(tmp_path / 'flows_out')) == len(b)
    for pf in golden['pair_files']:
        d = torch.load(os.path.join(out, pf['name']))
        assert list(d) == pf['keys']
        assert {k: ofp.digest(v) for k, v in d.items()} == pf['digests'], pf['name']
    for fl in golden['flows']:
        z = np.load(str(tmp_path / 'flows_out' / ('flowpair_%05d_%05d.npz' % fl['pair'])))
        assert all(np.array_equal(z[k], fl[k].numpy()) for k in ('flow_1_2', 'flow_2_1', 'mask_1', 'mask_2'))
        assert (int(z['frame_id_1']), int(z['frame_id_2'])) == fl['pair']
    # the davis_sequence mirror reads them back as the reference's Dataset does, train and vali
    ref_train = golden['items']['davis_sequence/train']
    for mode in ('train', 'vali'):
        ds = get_dataset('davis_sequence')(opt_for(golden, root), mode=mode)
        ref = golden['items']['davis_sequence/' + mode]
        assert len(ds) == len(ref)
        for i in range(len(ds)):
            assert ofp.digest_item(ds[i]) == ref[i], (mode, i)
    # the builder's own items are those dicts
    n = len(b)
    for i in range(n):
        assert ofp.digest_item(b[i]) == ref_train[i], i
    # shutterstock: an integer track id into the sorted track directories
    sroot = str(tmp_path / 'shutterstock')
    os.symlink(root, sroot)
    for mode in ('train', 'vali'):
        ds = get_dataset('shutterstock')(opt_for(golden, sroot, track=0), mode=mode)
        ref = golden['items']['shutterstock/' + mode]
        assert [ofp.digest_item(ds[i]) for i in range(len(ds))] == ref, mode
    # video_frames: pairs built at construction from the frames and the flow files, no sequence files read
    os.rename(out, out + '.moved')
    vf = get_dataset('video_frames')(opt_for(golden, root), mode='train')
    assert len(vf) == len(ref_train)
    for i in range(len(vf)):
        it = ofp.digest_item(vf[i])
        assert it == ref_train[i], i
    vv = get_dataset('video_frames')(opt_for(golden, root), mode='vali')
    assert [ofp.digest_item(vv[i]) for i in range(len(vv))] == golden['items']['davis_sequence/vali']


def test_dataset_flags_mirror_the_reference():
    from dvd_b200.options import options_train
    base = ['--net', 'scene_flow_motion_field']
    for alias, track in (('davis_sequence', 'dog'), ('shutterstock', 3), ('video_frames', 'dog')):
        opt, _ = options_train.parse(base + ['--dataset', alias, '--track_id', str(track), '--gaps', '1,3', '--repeat', '2',
                                             '--subsample', '--cache', '--overfit', '--select', '--data_root', '/data'])
        assert (opt.track_id, opt.gaps, opt.repeat, opt.subsample, opt.cache, opt.overfit, opt.select, opt.data_root) == \
            (track, '1,3', 2, True, True, True, True, '/data')
    opt, _ = options_train.parse(base + ['--dataset', 'davis_sequence'])
    assert opt.data_root == './datafiles/davis_processed' and opt.track_id == 'train'
    opt, _ = options_train.parse(base + ['--dataset', 'shutterstock'])
    assert opt.data_root == './datafiles/shutterstock' and opt.track_id == 0


def test_builder_without_a_gpu_refuses_raw_flows(golden, tmp_path):
    from dvd_b200.flow_pairs import PairBuilder
    fdir, pdir = write_video(golden, str(tmp_path), flows='raw')
    with pytest.raises(RuntimeError):
        PairBuilder(fdir, pdir, [1], device='cpu')


def test_flow_ops_reject_cpu_and_bad_tensors():
    from dvd_b200 import ops
    with pytest.raises(ValueError):
        ops.flow_resize_cubic(torch.zeros(1, 8, 8, 2), 16, 16)
    with pytest.raises(ValueError):
        ops.flow_pair_masks(torch.zeros(1, 8, 8, 2), torch.zeros(1, 8, 8, 2))
    with pytest.raises(ValueError):
        ops.flow_pair_masks(torch.zeros(1, 8, 8, 2), torch.zeros(1, 8, 8, 2), convention='bad')
