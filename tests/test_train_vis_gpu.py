"""GPU: the training-page tiles (csrc/train_vis.cu through ops.vis_tiles) equal the numpy oracle (oracle/train_vis.py) bit for
bit, and a `train --html_logger` run writes every PNG, npz and page, each PNG the oracle of the npz beside it, without changing
what the run computes."""
import glob
import os
import re
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from dvd_b200 import ops, train_vis
from oracle import train_vis as ov

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tables(dev):
    return (torch.from_numpy(train_vis.turbo_table()).to(dev),
            torch.from_numpy(np.ascontiguousarray(train_vis.color_wheel() / 255)).to(dev))


def _planted(N, H, W, seed):
    g = np.random.default_rng(seed)
    depth = g.uniform(0.5, 9, (N, 1, H, W)).astype(np.float32)
    depth[0, 0, 0, :3] = [0.0, -2.0, 1e-3]
    if N > 1:
        depth[1, 0, 1, 1] = np.nan                       # the whole image is black
        depth[1, 0, 2, 2] = np.inf
    if N > 2:
        depth[2, 0, 0, 0] = -1e-6                        # t = inf: that pixel is NaN, the rest 0
        depth[2, 0, 3, 3] = -np.inf
    flow = (g.standard_normal((N, H, W, 2)) * 5).astype(np.float32)
    flow[0, 0, 0] = [2e7, 1.0]
    flow[0, 1, 1] = [0.0, 0.0]
    if N > 1:
        flow[1, 2, 2, 1] = np.nan
    if N > 2:
        flow[2] = 0.0
    img = g.uniform(0, 1, (N, 3, H, W)).astype(np.float32)
    img[0, 0, 0, 0] = np.nan
    img255 = np.round(g.uniform(-5, 260, (N, 3, H, W))).astype(np.float32)
    imgpm = g.uniform(-1.2, 1.1, (N, 3, H, W)).astype(np.float32)
    return {'depth_a': depth, 'flow_a': flow, 'img_a': img, 'img_b': img255, 'img_c': imgpm}


@pytest.mark.parametrize('N', [1, 3, 17])
@pytest.mark.parametrize('HW', [(64, 96), (224, 384), (37, 101)])
def test_tiles_equal_the_oracle(N, HW):
    H, W = HW
    pack = _planted(N, H, W, seed=N * 1000 + W)
    dev = torch.device('cuda')
    turbo, wheel = _tables(dev)
    t = {k: torch.from_numpy(v).to(dev) for k, v in pack.items()}
    flow_planar = t['flow_a'].permute(0, 3, 1, 2).contiguous()             # [N,2,H,W], read back through a permuted view
    depth_strided = torch.empty(N, 1, H, W + 3, device=dev)[..., 1:W + 1]  # non-contiguous rows
    depth_strided.copy_(t['depth_a'])
    maps = [('depth', t['depth_a']), ('depth', depth_strided), ('flow', t['flow_a'].permute(0, 3, 1, 2)),
            ('flow', flow_planar), ('img', t['img_a']), ('img', t['img_b']), ('img', t['img_c'])]
    tiles = ops.vis_tiles(maps, turbo, wheel)
    again = ops.vis_tiles(maps, turbo, wheel)
    torch.cuda.synchronize()
    assert torch.equal(tiles, again)
    got = tiles.cpu().numpy()
    turbo_h, wheel_h = train_vis.turbo_table(), train_vis.color_wheel()
    dep = np.stack([ov.depth_image(d[0], turbo_h) for d in pack['depth_a']])
    flo = np.stack([ov.flow_image(f, wheel_h) for f in pack['flow_a']])
    want = [dep, dep, flo, flo, ov.img_images(pack['img_a']), ov.img_images(pack['img_b']), ov.img_images(pack['img_c'])]
    for q, w in enumerate(want):
        np.testing.assert_array_equal(got[q * N:(q + 1) * N], w, err_msg='map %d (%s)' % (q, maps[q][0]))
    if N > 1:
        assert got[1].max() == 0                          # NaN depth: black, and the rest of the pack is written


BASE = ('--net scene_flow_motion_field --dataset synthetic_sequence --gaps 1 --n_frames 8 --height 64 --width 96 --epoch_batches 4 '
        '--lr 1e-6 --batch_size 1 --optim adam --gpu 0 --workers 0 --one_way --loss_type l1 --l1_mul 0 --acc_mul 1 --disp_mul 1 '
        '--warm_sf 1 --scene_lr_mul 1000 --repeat 1 --flow_mul 1 --sf_mag_div 100 --time_dependent --midas --use_disp '
        '--manual_seed 1 --epoch 2 --vis_every_train 1 --vis_batches_train 2 --vis_at_start --validate --vali_at_start '
        '--vis_batches_vali 2').split()


def _run(args, logdir):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    r = subprocess.run([sys.executable, '-m', 'dvd_b200.train'] + BASE + ['--logdir', logdir] + args, cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    logs = {}
    for line in r.stdout.splitlines():
        if line.startswith('epoch '):
            log = eval(line.split(':', 1)[1])      # the driver prints a plain dict of floats
            logs[int(line.split()[1].rstrip(':'))] = {k: v for k, v in log.items() if k not in ('data_time', 'batch_time')}
    return logs


def _files(root):
    return sorted(os.path.relpath(p, root) for p in glob.glob(os.path.join(root, '**', '*'), recursive=True) if os.path.isfile(p))


@pytest.mark.timeout(1800)
def test_train_html_logger_end_to_end(tmp_path):
    with_pages = _run(['--html_logger'], str(tmp_path / 'a'))
    without = _run([], str(tmp_path / 'b'))
    # the pages read the step's outputs and change nothing the run computes. The training step is not bitwise reproducible
    # from process to process: two plain runs of this configuration differ by up to 1e-4 relative in the printed losses and
    # 1e-5 in loss_eval (measured on an H100), so the logs are compared to 1e-3 relative, above that noise and far below
    # what a change of the computation would move
    assert sorted(with_pages) == sorted(without) == [0, 1, 2]
    for e in without:
        assert with_pages[e].keys() == without[e].keys()
        for k, v in without[e].items():
            assert with_pages[e][k] == pytest.approx(v, rel=1e-3, abs=1e-6), (e, k)
    a = glob.glob(str(tmp_path / 'a' / '*' / '*'))[0]
    b = glob.glob(str(tmp_path / 'b' / '*' / '*'))[0]
    files_a, files_b = _files(a), _files(b)
    assert not [f for f in files_b if f.endswith(('.png', '.html', '.json')) or '_vali' in f]
    assert set(files_b) - {'opt.pt', 'opt.txt'} <= set(files_a)

    turbo, wheel = train_vis.turbo_table(), train_vis.color_wheel()
    n_png = 0
    for state, folder_state, epochs in (('train', 'train', (1, 2)), ('val', 'vali', (0, 1, 2))):
        for e in epochs:
            folder = os.path.join(a, 'visualize', 'epoch%04d_%s' % (e, folder_state))
            npzs = sorted(glob.glob(os.path.join(folder, 'rank0000_batch*.npz')))
            assert len(npzs) == (3 if state == 'train' else 2), (folder, npzs)
            for p in npzs:
                bi = int(re.search(r'batch(\d+)', p).group(1))
                with np.load(p) as z:
                    pack = {k: z[k] for k in z.files}
                want = ov.pack_images(pack, turbo, wheel, train_vis.image_kind)
                assert want
                for k, imgs in want.items():
                    for j, w in enumerate(imgs):
                        png = cv2.imread(os.path.join(folder, train_vis.png_name(k, bi + 1000 * e, j)), cv2.IMREAD_COLOR)
                        assert png is not None, (p, k)
                        np.testing.assert_array_equal(png[..., ::-1], w, err_msg='%s %s %d' % (p, k, j))
                        n_png += 1
            assert os.path.isfile(os.path.join(a, 'visualize', '%s_%05d.html' % (state, e)))
    assert n_png == len([f for f in files_a if f.endswith('.png')])
    summary = open(os.path.join(a, 'summary.html')).read()
    pages = re.findall(r'href="([^"]+)"', summary)
    assert len(pages) == 5
    for page in pages:
        path = os.path.join(a, page)
        srcs = re.findall(r'src="([^"]+)"', open(path).read())
        assert srcs
        for s in srcs:
            assert os.path.isfile(os.path.join(os.path.dirname(path), s)), (page, s)
