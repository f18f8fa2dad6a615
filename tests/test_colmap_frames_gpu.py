"""GPU: dvd_b200.frames.ColmapFrameBuilder against FrameBuilder on a twin scene, written once as a DAVIS track and once as a
COLMAP model over the same image files (test_colmap_frames_cpu.write_twin). FrameBuilder is pinned to the unmodified reference
script by tests/golden/frames_golden.pt, so equal frame files chain the COLMAP path to it. Then a COLMAP scene through the
prepare_frames, prepare_pairs and train command lines."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_colmap_frames_cpu as cm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def seeded(resize=(256, 512)):
    from dvd_b200 import synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    return synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True, resize=list(resize)), 0, 2000.0)


@pytest.fixture(scope='module')
def net():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    return seeded().cuda().eval()


def written(b, out_dir):
    assert b.write(out_dir) == b.n_frames
    files = []
    for i in range(b.n_frames):
        with np.load(os.path.join(out_dir, 'frame_%05d.npz' % i)) as z:
            files.append({k: z[k] for k in z.keys()})
    return files


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize('case', ['masks_bin', 'zero_masks_txt'])
def test_colmap_frames_equal_the_davis_twin_bitwise(net, tmp_path, case):
    from dvd_b200 import frames as fr
    zero = case.startswith('zero')
    sc = cm.scene(n=6, V=3000, seed=11)
    images_dir, masks_dir = cm.write_twin(str(tmp_path), sc, zero_masks=zero)
    davis = fr.FrameBuilder(str(tmp_path), 'clip', net, chunk=4)
    model = str(tmp_path / ('sparse_txt' if zero else 'sparse_bin'))
    colmap = fr.ColmapFrameBuilder(images_dir, model, net, masks_dir=None if zero else masks_dir, chunk=4)
    assert colmap.names == ['%05d.jpg' % f for f in range(6)]
    assert same_bits(colmap.scale, davis.scale) and same_bits(colmap.medians, davis.medians)
    assert np.array_equal(colmap.counts, davis.counts) and 0 < colmap.counts.min()
    assert zero or colmap.counts.max() < 3000                                    # the masks reject points in every frame
    ref, got = written(davis, str(tmp_path / 'davis_out')), written(colmap, str(tmp_path / 'colmap_out'))
    for i, (r, g) in enumerate(zip(ref, got)):
        assert sorted(g) == sorted(r)
        for k in r:
            assert same_bits(g[k], r[k]), (i, k)
        seg = g['motion_seg']
        assert (seg == 0).all() if zero else 0 < seg.sum() < seg.size
    print('%s: s = %r, points per frame %s' % (case, float(colmap.scale), colmap.counts.tolist()))


def test_general_rotations_agree_within_ulps(net, tmp_path):
    from dvd_b200 import frames as fr
    sc = cm.scene(n=6, V=3000, exact=False, seed=5)
    images_dir, masks_dir = cm.write_twin(str(tmp_path), sc)
    davis = fr.FrameBuilder(str(tmp_path), 'clip', net, chunk=4)
    colmap = fr.ColmapFrameBuilder(images_dir, str(tmp_path / 'sparse_bin'), net, masks_dir=masks_dir, chunk=4)
    # the DAVIS matrices are inverted twice in fp64; the selection is the same, the ratios move by a few ulps
    assert np.array_equal(colmap.counts, davis.counts)
    ulps = lambda a, b: float(np.max(np.abs(np.subtract(a, b)) / np.spacing(np.abs(b))))      # noqa: E731
    print('medians %.1f ulp, s %.1f ulp' % (ulps(colmap.medians, davis.medians), ulps(colmap.scale, davis.scale)))
    assert ulps(colmap.medians, davis.medians) <= 16 and ulps(colmap.scale, davis.scale) <= 16
    for i in range(6):
        g, r = colmap.frame(i), davis.frame(i)
        for k in ('img', 'img_orig', 'depth_pred', 'depth_mvs', 'intrinsics', 'motion_seg'):
            assert same_bits(g[k], r[k]), (i, k)
        # pose_c2w before the fp32 cast, then as stored
        p64 = [np.linalg.inv(np.block([[E[i][:3, :3], E[i][:3, 3:] * s], [E[i][3:]]]))
               for E, s in ((colmap.extrinsics, colmap.scale), (davis.extrinsics, davis.scale))]
        assert np.abs(p64[0] - p64[1]).max() <= 16 * np.spacing(np.abs(p64[1]).max())
        assert np.abs(g['pose_c2w'] - r['pose_c2w']).max() <= np.spacing(np.abs(r['pose_c2w']).max())


@pytest.mark.timeout(1200)
def test_prepare_frames_pairs_and_train_clis_on_a_colmap_model(net, tmp_path):
    from dvd_b200 import frames as fr, prepare_frames, prepare_pairs
    from oracle import raft as oracle_raft
    n, gaps = 6, [1, 2]
    sc = cm.scene(n=n, V=3000, seed=2)
    cm.write_txt(str(tmp_path / 'sparse'), sc['cameras'], sc['images'], sc['points'])
    images_dir, masks_dir = str(tmp_path / 'images'), str(tmp_path / 'masks')
    cm.write_images(images_dir, n, masks_dir)
    ckpt = str(tmp_path / 'midas_cpkt.pt')
    torch.save(seeded().state_dict(), ckpt)
    data = tmp_path / 'data'
    frames_dir = str(data / 'frames_midas' / 'clip')
    prepare_frames.main(['--colmap_model', str(tmp_path / 'sparse'), '--images', images_dir, '--masks', masks_dir,
                         '--midas_ckpt', ckpt, '--out', frames_dir, '--chunk', '4'])
    assert sorted(os.listdir(frames_dir)) == ['frame_%05d.npz' % i for i in range(n)]
    b = fr.ColmapFrameBuilder(images_dir, str(tmp_path / 'sparse'), net, masks_dir=masks_dir, chunk=4)
    for i, got in enumerate(written(b, str(tmp_path / 'direct'))):
        with np.load(os.path.join(frames_dir, 'frame_%05d.npz' % i)) as z:
            assert all(same_bits(z[k], got[k]) for k in got), i                   # the checkpoint's weights, the same files
    raft_ckpt = str(tmp_path / 'raft.pth')
    torch.save({'module.' + k: v for k, v in oracle_raft.seeded_state_dict(0, 0.7).items()}, raft_ckpt)
    seq = str(data / 'sequences_select_pairs_midas' / 'clip' / '001')
    prepare_pairs.main(['--frames', frames_dir, '--raft_ckpt', raft_ckpt, '--raft_iters', '2', '--out', seq,
                        '--flows_out', str(data / 'flow_pairs' / 'clip'), '--gaps', ','.join(map(str, gaps))])
    assert len(os.listdir(seq)) == sum(n - 1 - g for g in gaps)
    args = ('--net scene_flow_motion_field --dataset video_frames --track_id clip --gaps 1,2 --epoch 1 --epoch_batches 2 '
            '--resident --lr 1e-6 --batch_size 1 --optim adam --gpu 0 --workers 0 --one_way --loss_type l1 --l1_mul 0 '
            '--acc_mul 1 --disp_mul 1 --warm_sf 1 --scene_lr_mul 1000 --flow_mul 1 --sf_mag_div 100 --time_dependent '
            '--use_disp --vis_batches_train 0 --manual_seed 1').split()
    args += ['--data_root', str(data), '--logdir', str(tmp_path / 'log')]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', 'dvd_b200.train'] + args, cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=1100)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith('epoch 1:')]
    assert lines, r.stdout[-2000:]
    log = eval(lines[0].split(':', 1)[1])                                          # the driver prints a plain dict of floats
    assert all(v == v and abs(v) != float('inf') for v in log.values()), log
