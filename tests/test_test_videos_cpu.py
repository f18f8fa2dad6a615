"""CPU: the test-end canvas oracle (oracle/test_videos.py) on planted values, the turbo table, the slice-row defaults, the
page, and the argument / file checks of dvd_b200/test_videos.py that run before the device is touched."""
import os

import numpy as np
import pytest

from oracle import test_videos as ov


def test_index_rule_on_planted_t():
    one_below = np.nextafter(1.0, 0.0)
    v = np.array([0.0, 1.0, one_below, -1e-300, -3.0, 1.0 + 1e-12, 7.0, np.nan, 0.5, 255 / 256, np.inf, -np.inf])
    assert ov.cmap_index(v, 0.0, 1.0).tolist() == [0, 255, 255, 0, 0, 255, 255, -1, 128, 255, 255, 0]
    # t = (v - vmin) / (vmax - vmin) in fp64, floor(256 t): the first value of each bin opens it
    lo, hi = 0.0, 4.0                                                 # v = 4 t exactly
    v = lo + (hi - lo) * np.array([1 / 256, np.nextafter(1 / 256, 0), 0.25, 17 / 256])
    assert ov.cmap_index(v, lo, hi).tolist() == [1, 0, 64, 17]


def test_constant_panel_maps_to_the_first_colour_and_nan_stays_black():
    assert ov.cmap_index(np.array([3.0, 3.0, -1.0, 9.0, np.nan]), 3.0, 3.0).tolist() == [0, 0, 0, 0, -1]
    lut = ov.turbo_lut()
    c = ov.colour(np.array([3.0, np.nan]), 3.0, 3.0, lut)
    assert c[0].tolist() == lut[0].tolist() and c[1].tolist() == [0, 0, 0]


def test_gt_disparity_at_1e_8_and_its_fp32_neighbours():
    e = np.float32(1e-8)
    up, down = np.nextafter(e, np.float32(1)), np.nextafter(e, np.float32(0))
    g = np.array([0.0, e, up, down, -1.0, -e, 2.0], dtype=np.float32)
    v = ov.gt_disp(g)
    assert v.dtype == np.float64
    assert v[0] == 0.0 and v[1] == 0.0 and v[3] == 0.0               # gt > 1e-8 fails: 0 / (gt + 1e-8)
    assert v[2] == 1.0 / np.float64(np.float32(up + e))              # fp64 division by the fp32 sum
    assert v[4] == 0.0 and np.signbit(v[4])                          # 0 / negative = -0
    assert np.isnan(v[5])                                            # 0 / (-1e-8 + 1e-8) = 0 / 0
    assert v[6] == 1.0 / np.float64(np.float32(2.0) + e)
    # NaN -> black, -0 -> the first colour
    i = ov.cmap_index(v, 0.0, 1.0)
    assert i[5] == -1 and i[4] == 0


def test_rgb_rule_at_0_1_k_over_255_and_nan():
    k = np.arange(256, dtype=np.float32)
    x = k / np.float32(255)
    xs = np.concatenate([x, np.nextafter(x, np.float32(2)), np.nextafter(x, np.float32(-1)),
                         np.array([np.nan, -0.5, 1.5, np.inf, -np.inf], dtype=np.float32)])
    u = ov.rgb_u8(xs)
    expect = np.floor(np.float32(255) * np.clip(np.where(np.isnan(xs), np.float32(0), xs), np.float32(0), np.float32(1)))
    assert np.array_equal(u, expect.astype(np.uint8))
    assert u[0] == 0 and u[255] == 255 and u[-5:].tolist() == [0, 0, 255, 255, 0]
    # k / 255 rounded to fp32 and multiplied by 255 in fp32 lands on k for every k: the frames keep their 8-bit values
    assert np.array_equal(u[:256], k.astype(np.uint8))


def test_cv2_turbo_table_ends_are_googles_turbo():
    lut = ov.turbo_lut()
    assert lut.shape == (256, 3) and lut.dtype == np.uint8
    assert lut[0, ::-1].tolist() == [48, 18, 59] and lut[255, ::-1].tolist() == [122, 4, 3]
    from dvd_b200 import test_videos
    assert np.array_equal(test_videos.turbo_lut(), lut)


def test_slice_row_defaults_and_checks():
    from dvd_b200 import test_videos
    assert test_videos.slice_rows_for(224) == (120, 140) == ov.default_slice_rows(224)
    assert test_videos.slice_rows_for(140) == (120, 140)
    assert test_videos.slice_rows_for(64) == (22, 42) == ov.default_slice_rows(64)
    assert test_videos.slice_rows_for(7) == (0, 7)
    assert test_videos.slice_rows_for(64, '8:12') == (8, 12)
    for bad in ('0:65', '12:8', '5:5', 'a:b', '-1:3'):
        with pytest.raises(ValueError):
            test_videos.slice_rows_for(64, bad)


def test_geometry_and_template_match_the_oracle():
    from dvd_b200 import test_videos
    lut = ov.turbo_lut()
    for k, h, w in ((3, 64, 96), (3, 224, 384), (2, 17, 101), (2, 1, 64)):
        assert test_videos.layout(k, h, w) == ov.layout(k, h, w)
        CH, CW, _ = ov.layout(k, h, w)
        assert CW % 4 == 0 and CH % 2 == 0
        rng = [(np.float32(0.125), np.float32(3.5)), (np.float64(-2.0), np.float64(1e-3)), (0.0, 0.0)][:k]
        titles = ('Refined', 'Initial', 'GT')[:k]
        assert np.array_equal(test_videos.template(titles, h, w, rng, lut), ov.template(titles, h, w, rng, lut))


def _write(d, i, B=2, H=8, W=12, drop=None, depth=None, img_shape=None):
    rng = np.random.default_rng(i)
    z = dict(depth=rng.uniform(1, 4, (B, 1, H, W)).astype(np.float32) if depth is None else depth,
             depth_nn=rng.uniform(1, 4, (B, 1, H, W)).astype(np.float32),
             depth_gt=rng.uniform(0, 4, (B, 1, H, W)).astype(np.float32),
             img_1=rng.uniform(0, 1, img_shape or (B, 3, H, W)).astype(np.float32), K=np.eye(3, dtype=np.float32))
    if drop:
        z.pop(drop)
    np.savez(os.path.join(d, 'batch%04d.npz' % i), **z)


def _main(d, *extra):
    from dvd_b200 import test_videos
    return test_videos.main(['--test_dir', str(d), *extra])


def test_cli_errors_before_the_device(tmp_path):
    d = tmp_path / 'epochbest_test'
    d.mkdir()
    with pytest.raises(ValueError, match='no batch'):
        _main(d)
    _write(d, 0)
    _write(d, 1, drop='depth_nn')
    with pytest.raises(ValueError, match='depth_nn'):
        _main(d)
    _write(d, 1, H=10)
    with pytest.raises(ValueError, match='10x12'):
        _main(d)
    _write(d, 1, img_shape=(2, 3, 8, 11))
    with pytest.raises(ValueError, match='img_1'):
        _main(d)
    _write(d, 1)
    with pytest.raises(ValueError, match='slice rows'):
        _main(d, '--slice_rows', '4:9')
    bad = np.full((2, 1, 8, 12), 2.0, np.float32)
    bad[1, 0, 3, 4] = np.inf
    _write(d, 1, depth=bad)
    with pytest.raises(ValueError, match='frame 3 .*batch0001'):
        _main(d)
    bad[1, 0, 3, 4] = 0.0
    _write(d, 1, depth=bad)
    with pytest.raises(ValueError, match='frame 3'):
        _main(d)
    with pytest.raises(SystemExit):
        _main(d, '--slice_rows', '3-5')
    with pytest.raises(SystemExit):
        _main(d, '--chunk', '0')


def test_page_names_only_the_written_videos():
    from dvd_b200 import test_videos
    page = test_videos._page('epochbest_test', 0.0123, (120, 140))
    import re
    srcs = re.findall(r'src="([^"]+)"', page)
    assert sorted(srcs) == sorted(['epochbest_test.mp4', 'epochbest_test_rgb.mp4', 'epochbest_test_temporal.mp4'])
    assert '<script' not in page and 'http' not in page and 'Disparity loss 0.0123' in page


def test_test_driver_takes_the_video_flags_off_the_reference_command_line():
    from dvd_b200.test import parse_video_flags
    from dvd_b200.options import options_test
    ref = ['--net', 'scene_flow_motion_field', '--dataset', 'synthetic_sequence', '--checkpoint_path', 'LOG', '--epoch', '-1',
           '--output_dir', 'OUT/', '--gpu', '0', '--html_logger']
    assert parse_video_flags(ref) == (False, None, ref)
    videos, rows, rest = parse_video_flags(ref[:4] + ['--videos', '--slice_rows', '8:12'] + ref[4:])
    assert videos and rows == '8:12' and rest == ref
    opt = options_test.parse(rest)
    assert opt.html_logger and not hasattr(opt, 'videos') and not hasattr(opt, 'slice_rows')
    with pytest.raises(SystemExit):
        parse_video_flags(ref + ['--videos', '--slice_rows', '8-12'])
