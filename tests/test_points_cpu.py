"""CPU: the point-cloud oracle (oracle/points.py) on planted cases, the PLY writer / reader and the export CLI's argument
checks (dvd_b200/points.py, dvd_b200/export_points.py)."""
import os

import numpy as np
import pytest

from oracle import points as op


def _flat(H, W, v=2.0, N=1):
    return np.full((N, H, W), v, dtype=np.float32)


def test_depth_threshold_at_1e_2_and_its_fp32_neighbours():
    t = np.float32(1e-2)
    d = _flat(1, 5, float(t))
    d[0, 0, :] = [t, np.nextafter(t, np.float32(1)), np.nextafter(t, np.float32(0)), 0.0, -1.0]
    m = op.select_mask(d, edge_tol=np.inf)
    assert m[0, 0].tolist() == [False, True, False, False, False]


def test_nan_and_inf_depths_and_their_neighbours():
    d = _flat(3, 5)
    d[0, 1, 1] = np.nan
    d[0, 1, 3] = np.inf
    m = op.select_mask(d, edge_tol=0.05)
    bad = {(1, 1), (1, 3), (0, 1), (2, 1), (1, 0), (1, 2), (0, 3), (2, 3), (1, 4)}
    for y in range(3):
        for x in range(5):
            assert m[0, y, x] == ((y, x) not in bad), (y, x)
    # with an infinite tolerance only the pixels themselves go: NaN and inf differences still fail
    m = op.select_mask(d, edge_tol=np.inf)
    assert not m[0, 1, 1] and not m[0, 1, 3] and not m[0, 1, 2]


def test_edge_tol_at_equality():
    # |1 - 1.0625| / 1 = 0.0625 exactly in fp64
    d = _flat(1, 2, 1.0)
    d[0, 0, 1] = 1.0625
    assert op.select_mask(d, 0.0625)[0, 0, 0]
    assert not op.select_mask(d, np.nextafter(0.0625, 0))[0, 0, 0]
    # the other pixel: |1.0625 - 1| / 1.0625 < 0.0625
    assert op.select_mask(d, 0.0625)[0, 0, 1]


def test_border_pixels_have_two_or_three_neighbours():
    d = _flat(3, 3)
    d[0, 1, 1] = 4.0                 # the centre differs from its 4 neighbours
    m = op.select_mask(d, 0.5)
    # edge midpoints (3 neighbours) see the centre: |2 - 4| / 2 > 0.5; corners (2 neighbours) do not; the centre's own ratio
    # |4 - 2| / 4 is 0.5, kept at equality
    assert m[0, 0, 0] and m[0, 0, 2] and m[0, 2, 0] and m[0, 2, 2] and m[0, 1, 1]
    assert not m[0, 0, 1] and not m[0, 1, 0] and not m[0, 1, 2] and not m[0, 2, 1]
    # frames do not neighbour each other
    d2 = np.concatenate([_flat(2, 2, 2.0), _flat(2, 2, 9.0)])
    assert op.select_mask(d2, 0.01).all()


def test_points_on_voxel_faces():
    v = 0.25
    xyz = np.array([[0.0, 0.25, -0.25], [0.2499999, 0.5, -0.2500001], [-1e-30, 1.0, 2.0]], dtype=np.float32)
    k = op.keys(xyz, v, (-8, -8, -8))
    dec = np.stack([(k >> 42) & 0x1FFFFF, (k >> 21) & 0x1FFFFF, k & 0x1FFFFF], 1) - 8
    assert dec.tolist() == [[0, 1, -1], [0, 2, -2], [-1, 4, 8]]
    with pytest.raises(ValueError):
        op.keys(xyz, v, (1, -8, -8))
    with pytest.raises(ValueError):
        op.keys(np.array([[2 ** 21 * v, 0, 0]], np.float32), v, (0, 0, 0))


def test_colours():
    img = np.array([-0.5, 0.0, 0.5, 1.0, 1.5, np.nan, 0.999, 1 / 255.0], dtype=np.float32)
    assert op.colours(img).tolist() == [0, 0, 127, 255, 255, 0, 254, 1]


def test_reduce_means_counts_views_and_min_views():
    hw = 10
    key = np.array([5, 3, 5, 3, 7, 5], dtype=np.int64)
    index = np.array([0, 1, 2, 11, 12, 25], dtype=np.int64)      # frames 0, 0, 0, 1, 1, 2
    xyz = np.arange(18, dtype=np.float32).reshape(6, 3)
    rgb = np.arange(18, dtype=np.uint8).reshape(6, 3) * 10
    r = op.reduce(key, index, xyz, rgb, hw, 1)
    assert r['count'].tolist() == [2, 3, 1] and r['views'].tolist() == [2, 2, 1]
    assert np.array_equal(r['xyz'][0], (xyz[1] + xyz[3]) / 2)
    assert np.array_equal(r['xyz'][1], (xyz[0].astype(np.float64) + xyz[2] + xyz[5]) / 3)
    assert np.array_equal(r['rgb'][2], rgb[4].astype(np.float64))
    r2 = op.reduce(key, index, xyz, rgb, hw, 2)
    assert r2['count'].tolist() == [2, 3]


def test_ply_round_trip(tmp_path):
    from dvd_b200 import points
    rng = np.random.default_rng(0)
    xyz = rng.standard_normal((37, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (37, 3)).astype(np.uint8)
    p = str(tmp_path / 'a.ply')
    points.write_ply(p, xyz, rgb)
    x2, c2 = points.read_ply(p)
    assert np.array_equal(x2, xyz) and np.array_equal(c2, rgb)
    assert os.path.getsize(p) == len(open(p, 'rb').read().split(b'end_header\n')[0]) + 11 + 37 * 15
    points.write_ply(p, np.zeros((0, 3)), np.zeros((0, 3)))
    assert points.read_ply(p)[0].shape == (0, 3)
    assert points.mean_rgb_to_u8([0.49, 0.5, 254.5, 255.0]).tolist() == [0, 1, 255, 255]


def test_camera_block_conventions():
    from dvd_b200 import points
    K = np.array([[[100.0, 0, 31.5], [0, 90.0, 23.5], [0, 0, 1]]], dtype=np.float32)
    c2w = np.eye(4, dtype=np.float32)[None]
    c2w[0, :3, 3] = [1, 2, 3]
    b = points.camera_block(K, c2w)
    assert b.shape == (1, 30) and b.dtype == np.float32
    assert np.array_equal(b[0, :9].reshape(3, 3), K[0].T)
    assert np.array_equal(b[0, 9:18].reshape(3, 3), np.linalg.inv(K[0].astype(np.float64)).T.astype(np.float32))
    assert b[0, 27:].tolist() == [1, 2, 3]
    assert np.array_equal(points.camera_block(K, c2w[:, :3]), b)
    with pytest.raises(ValueError):
        points.camera_block(K, np.zeros((2, 3, 4)))
    assert points.default_origin(c2w, 0.5) == (2 - 2 ** 20, 4 - 2 ** 20, 6 - 2 ** 20)
    with pytest.raises(ValueError):
        points.default_voxel(np.zeros((1, 4, 4)))


def _write_export(d, n=2, H=4, W=6, drop=None, size=None):
    os.makedirs(d, exist_ok=True)
    for i in range(n):
        h, w = size if (size and i == n - 1) else (H, W)
        z = {'depth': np.ones((1, 1, h, w), np.float32), 'img_1': np.zeros((1, 3, h, w), np.float32),
             'K': np.eye(3, dtype=np.float32).reshape(1, 1, 1, 3, 3), 'cam_c2w': np.eye(4, dtype=np.float32)[None]}
        if drop and i == n - 1:
            del z[drop]
        np.savez(os.path.join(d, 'batch%04d.npz' % i), **z)


def test_cli_argument_errors(tmp_path):
    from dvd_b200 import export_points as ep
    base = ['--test_dir', str(tmp_path), '--out', str(tmp_path / 'o.ply')]
    for bad in (['--voxel', '0'], ['--voxel', '-1'], ['--min_views', '0'], ['--chunk', '0'], ['--edge_tol', '-0.1'],
                ['--frames', '3'], ['--frames', 'a:b']):
        with pytest.raises(SystemExit):
            ep.parse_args(base + bad)
    with pytest.raises(SystemExit):
        ep.parse_args(['--out', 'x.ply'])
    a = ep.parse_args(base)
    assert a.voxel is None and a.edge_tol == 0.05 and a.min_views == 2 and a.chunk == 16 and a.frames is None


def test_cli_input_errors(tmp_path):
    from dvd_b200 import export_points as ep
    with pytest.raises(ValueError, match='no batch'):
        ep.list_files(str(tmp_path))
    _write_export(str(tmp_path / 'ok'), n=3)
    files = ep.list_files(str(tmp_path / 'ok'))
    assert [os.path.basename(f) for f in files] == ['batch0000.npz', 'batch0001.npz', 'batch0002.npz']
    fr = ep.Frames(files, '1:')
    assert fr.N == 2 and fr.ids.tolist() == [1, 2] and fr.images(0, 2).shape == (2, 3, 4, 6)
    with pytest.raises(ValueError, match='empty'):
        ep.Frames(files, '5:9')
    _write_export(str(tmp_path / 'size'), size=(4, 8))
    with pytest.raises(ValueError, match='frames of'):
        ep.Frames(ep.list_files(str(tmp_path / 'size')))
    _write_export(str(tmp_path / 'key'), drop='cam_c2w')
    with pytest.raises(ValueError, match='lacks cam_c2w'):
        ep.Frames(ep.list_files(str(tmp_path / 'key')))


def test_cli_help_states_the_default_voxel(capsys):
    from dvd_b200 import export_points as ep
    with pytest.raises(SystemExit):
        ep.parse_args(['--help'])
    assert '0.002 x the median valid depth' in ' '.join(capsys.readouterr().out.split())
