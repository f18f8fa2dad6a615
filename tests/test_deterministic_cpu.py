"""CPU side of the ordered reductions (DESIGN.md 2.11): the `--deterministic` flag, the step-graph signature of each mode, and
the C ABI of the *_ordered entry points (the arguments of their namesakes, then workspace, bytes, stream)."""
import ctypes
import types

import torch


def test_deterministic_flag_parses():
    from dvd_b200.options import options_train
    base = ['--net', 'scene_flow_motion_field', '--dataset', 'synthetic_sequence', '--midas']
    opt, _ = options_train.parse(base + ['--deterministic'])
    assert opt.deterministic is True
    opt, _ = options_train.parse(base)
    assert opt.deterministic is False


def test_graph_signature_differs_between_modes():
    from dvd_b200.models.scene_flow_motion_field import Model
    fake = types.SimpleNamespace(warm=False)
    b = {'img_1': torch.zeros(8, 3, 224, 384)}
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(False)
        off = Model._graph_sig(fake, b, 8, 1 / 80)
        torch.use_deterministic_algorithms(True)
        on = Model._graph_sig(fake, b, 8, 1 / 80)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert off == (8, (224, 384), 8, False, round(1 / 80, 9))      # the default signature is what it always was
    assert on != off and on[:len(off)] == off


def test_ordered_entry_points_extend_their_namesakes():
    from dvd_b200 import _lib
    sig = _lib.SIGNATURES
    ordered = [n for n in sig if n.endswith('_ordered')]
    assert sorted(ordered) == sorted(['dvd_conv2d_wgrad_ordered', 'dvd_mlp_wgrad_ordered', 'dvd_mlp_dgrad_ordered',
                                      'dvd_reproject_loss_bwd_ordered', 'dvd_relu_bwd_colsum_ordered', 'dvd_bn_act_bwd_ordered',
                                      'dvd_stem_wgrad_ordered', 'dvd_head_bwd_ordered'])
    for n in ordered:
        base = sig[n[:-len('_ordered')]]
        assert sig[n] == base[:-1] + [ctypes.c_void_p, ctypes.c_size_t, base[-1]], n


def test_workspace_sizes():
    from dvd_b200 import _lib
    lib = _lib.load()
    sizes = [lib.dvd_ordered_workspace_bytes(s) for s in range(6)]
    assert all(s > 0 and s % 16 == 0 for s in sizes), sizes
    assert lib.dvd_ordered_workspace_bytes(6) == 0 and lib.dvd_ordered_workspace_bytes(-1) == 0
    assert lib.dvd_reproject_ordered_bytes(0, 224, 384) == 0
