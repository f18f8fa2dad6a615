"""CPU: oracle/raft.py against the fixture written from the reference's RAFT (tests/golden/raft_golden.pt), the parameter names
of dvd_b200.raft.RaftNet, the command-line handling of the RAFT flow source, and the C symbols of csrc/raft_ops.cu."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def rel(a, b, scale=None):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / (scale if scale is not None else max(float(b.abs().max()), 1e-30)))


@pytest.fixture(scope='module')
def gold():
    from oracle.golden_io import load_golden
    return load_golden(GOLDEN, 'raft_golden')


@pytest.fixture(scope='module')
def sd(gold):
    from oracle import raft as oracle_raft
    return oracle_raft.seeded_state_dict(gold['weight_seed'], gold['gain'])


@pytest.mark.parametrize('ci', [0, 1])
def test_oracle_fp64_equals_every_stored_tensor_of_the_reference_run(gold, sd, ci):
    """the reference ran in fp32, the oracle runs in fp64: they agree to fp32 rounding through 20 iterations"""
    from oracle import raft as oracle_raft
    case = gold['cases'][ci]
    im1, im2 = oracle_raft.seeded_pair(case['H'], case['W'], case['seed'])
    assert abs(float(im1.double().sum() + im2.double().sum()) - case['image_checksum']) <= 1e-9 * abs(case['image_checksum'])
    sd64 = oracle_raft.cast(sd, torch.float64)
    tol = 2e-5
    with torch.no_grad():
        for iters in (1, 4, 20):
            tr = {}
            _, up = oracle_raft.raft_forward(sd64, im1.double(), im2.double(), iters, trace=tr)
            fin = case['final'][iters]
            e = float((up - fin['flow_up'].double()).norm(dim=1).mean())
            assert e <= 2 * case['floor_epe'][iters] + 1e-9, (iters, e, case['floor_epe'][iters])
            assert rel(tr['flow_low'], fin['flow_low']) < tol and rel(up, fin['flow_up']) < tol
            if 'up_mask' in fin:
                assert rel(tr['up_mask'], fin['up_mask']) < tol
    for l in range(4):
        assert rel(tr['pyramid'][l], case['pyramid'][l]) < tol, l
    for k in ('fmap1', 'fmap2', 'net0', 'inp'):
        if k in case:
            assert rel(tr[k], case[k]) < tol, k
    pmax = float(case['pyramid'][0].abs().max())
    for i, st in enumerate(tr['iters']):
        assert rel(st['coords1'], case['coords1'][i:i + 1]) < tol and rel(st['delta_flow'], case['delta_flow'][i:i + 1]) < 10 * tol, i
        if i in case['steps']:
            assert rel(st['corr'], case['steps'][i]['corr'], pmax) < tol, i
            if 'net' in case['steps'][i]:
                assert rel(st['net'], case['steps'][i]['net']) < tol, i


def test_lookup_channel_order_on_an_impulse():
    from oracle import raft as oracle_raft
    h, w = 16, 20
    levels = [torch.zeros(h * w, 1, h >> l, w >> l, dtype=torch.float64) for l in range(4)]
    levels[0][:, 0, 9, 12] = 1.0          # q = (y 9, x 12)
    coords = torch.full((1, 2, h, w), 10.0, dtype=torch.float64)
    out = oracle_raft.lookup(levels, coords)
    # offset (x +2, y -1) from the centre (10, 10): the window's slow index moves along x
    assert int(out[0, :, 0, 0].argmax()) == (2 + 4) * 9 + (-1 + 4) and float(out[0, :, 0, 0].sum()) == 1.0


def test_reference_returns_nan_under_128_pixels():
    """why no fixture is smaller: a 1-pixel coarsest level makes the lookup's 2 x / (W - 1) - 1 divide by zero"""
    from oracle import raft as oracle_raft
    sd32 = oracle_raft.seeded_state_dict(0, 0.7)
    a, b = oracle_raft.seeded_pair(64, 96, 1)
    with torch.no_grad():
        assert torch.isnan(oracle_raft.raft_forward(sd32, a, b, 1)[1]).any()


def test_raftnet_parameter_names_equal_the_reference_model(gold, sd):
    from dvd_b200.raft import RaftNet
    net = RaftNet()
    assert sorted(net.state_dict().keys()) == gold['keys']
    net.load_state_dict(sd)
    net.load_state_dict({'module.' + k: v for k, v in sd.items()})
    with pytest.raises(RuntimeError):
        net.load_state_dict({k: v for k, v in sd.items() if k != 'fnet.conv1.bias'})


def test_requests_outside_the_supported_configuration_raise():
    from dvd_b200 import raft
    for kw in (dict(small=True), dict(alternate_corr=True), dict(mixed_precision=True), dict(dropout=0.1)):
        with pytest.raises(ValueError):
            raft.RaftNet(**kw)
    for hw in ((130, 160), (128, 164), (64, 96)):
        with pytest.raises(ValueError):
            raft.check_size(*hw)
    raft.check_size(288, 512)
    with pytest.raises(NotImplementedError):
        raft.RaftNet().train()
    with pytest.raises(RuntimeError):
        raft.RaftNet().plan()             # parameters on the CPU: there is no CPU path


def test_prepare_pairs_arguments(tmp_path, monkeypatch):
    from dvd_b200 import prepare_pairs
    seen = {}

    class Builder:
        raw_pairs, n_frames = 0, 3.0

        def __init__(self, frames, flows, gaps, raft=None, raft_iters=20):
            seen.update(frames=frames, flows=flows, gaps=gaps, raft=raft, raft_iters=raft_iters)

        def write(self, out, flows_out):
            return 0
    monkeypatch.setattr(prepare_pairs, 'PairBuilder', Builder)
    # --flows alone: as before, no RAFT involved
    prepare_pairs.main(['--frames', 'F', '--flows', 'D', '--out', str(tmp_path), '--gaps', '1,2'])
    assert seen == dict(frames='F', flows='D', gaps=[1, 2], raft=None, raft_iters=20)
    # neither or both: an error before any file is read (the frame directory does not exist)
    for extra in ([], ['--flows', 'D', '--raft_ckpt', 'C']):
        with pytest.raises(SystemExit):
            prepare_pairs.main(['--frames', str(tmp_path / 'missing'), '--out', str(tmp_path)] + extra)


def test_pair_builder_and_video_frames_need_a_flow_source(tmp_path):
    from dvd_b200.flow_pairs import PairBuilder
    from dvd_b200.options import options_train
    with pytest.raises(ValueError):
        PairBuilder(str(tmp_path / 'missing'), None, [1])
    opt, _ = options_train.parse(['--net', 'scene_flow_motion_field', '--dataset', 'video_frames', '--raft_ckpt', 'x.pth', '--raft_iters', '12'])
    assert (opt.raft_ckpt, opt.raft_iters) == ('x.pth', 12)
    opt, _ = options_train.parse(['--net', 'scene_flow_motion_field', '--dataset', 'video_frames'])
    assert (opt.raft_ckpt, opt.raft_iters) == (None, 20)


def test_raft_symbols_are_exported_and_bound():
    from dvd_b200 import _lib
    src = open(os.path.join(ROOT, 'include', 'dvd_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    names = sorted(set(re.findall(r'\b(dvd_raft_[a-z0-9_]+)\s*\(', src)))
    assert len(names) == 14, names
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n) and n in _lib.SIGNATURES, n
    lib = _lib.load()
    # 16 x 20 grid: 320 maps of 16x20 + 8x10 + 4x5 + 2x2; a grid under 16 on a side has no 4-level pyramid
    assert lib.dvd_raft_pyramid_floats(1, 16, 20) == 320 * (320 + 80 + 20 + 4)
    assert lib.dvd_raft_pyramid_floats(1, 8, 12) == -1
    assert lib.dvd_raft_instnorm_scratch_bytes(2, 64) == 2 * 64 * 64 * 2 * 8
