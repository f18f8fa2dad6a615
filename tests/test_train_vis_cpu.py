"""CPU: the training-page images and pages (dvd_b200/train_vis.py, oracle/train_vis.py) against the reference's own
HTMLVisualizer output recorded in tests/golden/train_vis_golden.pt (oracle/gen_golden_train_vis.py)."""
import json
import os

import numpy as np
import pytest
import torch

from dvd_b200 import train_vis
from oracle import train_vis as ov

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'train_vis_golden.pt')


@pytest.fixture(scope='module')
def golden():
    return torch.load(GOLDEN, weights_only=False)


def _np(pack):
    return {k: (v.numpy() if torch.is_tensor(v) else v) for k, v in pack['inputs'].items()}


def _ref_images(pack, key):
    B = pack['inputs'][key].shape[0]
    return np.stack([pack['images'][train_vis.png_name(key, pack['batch_idx'], b)].numpy() for b in range(B)])


def test_colour_wheel_is_the_reference_wheel(golden):
    np.testing.assert_array_equal(train_vis.color_wheel(), golden['wheel_ref'].numpy())


def test_image_keys_and_file_names_are_the_reference_ones(golden):
    for pack in golden['packs']:
        inp = _np(pack)
        keys = [k for k in sorted(inp) if train_vis.image_kind(k) is not None]
        names = {train_vis.png_name(k, pack['batch_idx'], b) for k in keys for b in range(inp[k].shape[0])}
        assert names == set(pack['images'])
    assert train_vis.image_kind('depth_image_1_2') == 'depth'
    assert train_vis.image_kind('scenef_1_2') is None and train_vis.image_kind('sf_1_2') is None
    with pytest.raises(ValueError):
        train_vis.image_kind('edge_1')


def test_page_header_and_rows_are_the_reference_ones(golden):
    for pack in golden['packs']:
        inp = _np(pack)
        keys = [k for k in sorted(inp) if train_vis.image_kind(k) is not None]
        assert train_vis.page_header(keys) == pack['header']
        assert train_vis.page_rows(keys, pack['batch_idx'], inp['batch_size'], pack['folder']) == pack['rows']


def test_image_pixels_equal_the_reference(golden):
    for pack in golden['packs']:
        inp = _np(pack)
        for k in inp:
            if train_vis.image_kind(k) == 'img':
                np.testing.assert_array_equal(ov.img_images(inp[k]), _ref_images(pack, k), err_msg=k)


def test_depth_heat_inputs_equal_the_reference(golden):
    for pack in golden['packs']:
        inp = _np(pack)
        heats = [ov.depth_heat(d[0]).clip(0, 1) for k in pack['heat_keys'] for d in inp[k]]
        np.testing.assert_array_equal(np.stack(heats), pack['heat'].numpy())


def test_depth_colours_with_the_reference_table_equal_the_reference(golden):
    turbo = golden['turbo_ref'].numpy()
    for pack in golden['packs']:
        inp = _np(pack)
        for k in pack['heat_keys']:
            mine = np.stack([ov.depth_image(d[0], turbo) for d in inp[k]])
            np.testing.assert_array_equal(mine, _ref_images(pack, k), err_msg=k)


def test_depth_colours_with_the_opencv_table_stay_within_the_table_difference(golden):
    """the one deviation of the depth rule: OpenCV's 8-bit turbo over 255 instead of the reference's float table. A colour
    interpolates entries a and b = min(a + 1, 255), so it can move by at most 255 max(|dT[a]|, |dT[b]|) plus one for the
    truncation."""
    ref, cv = golden['turbo_ref'].numpy(), train_vis.turbo_table()
    dT = np.abs(ref - cv) * 255
    for pack in golden['packs']:
        inp = _np(pack)
        for k in pack['heat_keys']:
            for b, d in enumerate(inp[k]):
                x = ov.depth_heat(d[0]).clip(0, 1)
                a = (x * 255).astype(np.int64)
                bound = np.maximum(dT[a], dT[np.minimum(a + 1, 255)]) + 1
                diff = np.abs(ov.depth_image(d[0], cv).astype(np.int64) - _ref_images(pack, k)[b].astype(np.int64))
                assert (diff <= bound).all(), (k, b, diff.max())
    assert dT.max() < 1.0


def test_flow_pixels_equal_the_reference_but_where_the_fp32_angle_moves_a_byte(golden):
    """the flow angle is fp64 atan2 rounded to fp32 here and fp64 in the reference. Everywhere else the rule is the
    reference's, so a pixel may differ only by one per channel. The planted exact sector angles put many bytes on an integer
    boundary, where the fp32 angle moves them most often; they stay a small share of the pixels."""
    wheel = train_vis.color_wheel()
    differing = total = 0
    for pack in golden['packs']:
        inp = _np(pack)
        for k in inp:
            if train_vis.image_kind(k) != 'flow':
                continue
            ref = _ref_images(pack, k).astype(np.int64)
            for b, f in enumerate(inp[k]):
                diff = np.abs(ov.flow_image(f, wheel).astype(np.int64) - ref[b])
                assert diff.max() <= 1, (k, b)
                differing += int((diff.max(-1) > 0).sum())
                total += diff.shape[0] * diff.shape[1]
    assert total > 0 and differing <= total // 20, (differing, total)


def test_oracle_handles_non_finite_depth_and_flow():
    turbo, wheel = train_vis.turbo_table(), train_vis.color_wheel()
    d = np.full((4, 5), 3.0, np.float32)
    d[0, 0], d[1, 1], d[2, 2], d[3, 3] = np.inf, 0.0, -2.0, -1e-6
    img = ov.depth_image(d, turbo)
    assert (img[3, 3] == 0).all()                       # t = inf: (inf - min) / inf is NaN -> black
    assert ov.depth_image(np.full((3, 3), np.nan, np.float32), turbo).max() == 0
    f = np.zeros((2, 3, 2), np.float32)
    assert ov.flow_image(f, wheel).max() == 0           # all-zero flow: NaN after / maxrad -> black


def test_summary_is_extended_on_resume(tmp_path):
    w = train_vis.PageWriter(str(tmp_path))
    w.page = {'id': ('train', 1), 'header': '<th>depth_1</th>\n', 'rows': ''}
    w.flush()
    w.page = {'id': ('val', 1), 'header': '<th>depth</th>\n', 'rows': ''}
    w.close()
    assert json.load(open(tmp_path / 'summary.json')) == {'train': [1], 'val': [1]}
    w = train_vis.PageWriter(str(tmp_path))
    w.page = {'id': ('train', 2), 'header': '', 'rows': ''}
    w.close()
    assert json.load(open(tmp_path / 'summary.json')) == {'train': [1, 2], 'val': [1]}
    html = open(tmp_path / 'summary.html').read()
    for link in ('visualize/train_00001.html', 'visualize/train_00002.html', 'visualize/val_00001.html'):
        assert 'href="%s"' % link in html
        assert (tmp_path / link).is_file()


def test_flush_raises_a_failed_write(tmp_path):
    w = train_vis.PageWriter(str(tmp_path))
    w.futures.append(w.pool.submit(train_vis._write_png, str(tmp_path / 'missing' / 'x.png'), np.zeros((2, 2, 3), np.uint8)))
    with pytest.raises(RuntimeError):
        w.close()


def test_visualize_rejects_an_unknown_folder(tmp_path):
    w = train_vis.PageWriter(str(tmp_path))
    with pytest.raises(ValueError):
        w.visualize({}, 0, str(tmp_path / 'epoch0001_test'))
    w.close()


def test_html_logger_flag_is_parsed():
    from dvd_b200.options import options_train
    base = ['--net', 'scene_flow_motion_field', '--dataset', 'synthetic_sequence']
    assert options_train.parse(base + ['--html_logger'])[0].html_logger is True
    assert options_train.parse(base)[0].html_logger is False


def test_vis_map_layout_matches_the_library():
    import ctypes
    from dvd_b200 import _lib
    assert _lib.load().dvd_struct_size(5) == ctypes.sizeof(_lib.VisMap)
