"""CPU: oracle/raft_tf32.py, the fp64 emulation of RaftNet's TF32 arithmetic, against oracle/raft.py.

With rounding off the emulation must be oracle/raft.py in fp64 (the structure is the reference's, nothing else is added);
anchors set to the emulation's own values must change nothing (teacher forcing only replaces a value by the one given); with
rounding on it must stay within the TF32 envelope of the fixture written from the reference
(tests/golden/raft_golden.pt), a sanity check of the rounding points only: the GPU test holds RaftNet to the emulation."""
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-30))


@pytest.fixture(scope='module')
def gold():
    from oracle.golden_io import load_golden
    return load_golden(GOLDEN, 'raft_golden')


@pytest.fixture(scope='module')
def sd64(gold):
    from oracle import raft as oracle_raft
    return oracle_raft.cast(oracle_raft.seeded_state_dict(gold['weight_seed'], gold['gain']), torch.float64)


@pytest.fixture(scope='module')
def pair(gold):
    from oracle import raft as oracle_raft
    case = gold['cases'][0]
    im1, im2 = oracle_raft.seeded_pair(case['H'], case['W'], case['seed'])
    return im1.double(), im2.double()


def test_without_rounding_the_encoders_are_the_oracle(sd64, pair):
    from oracle import raft as oracle_raft
    from oracle.raft_tf32 import RaftTF32
    im1, im2 = pair
    with torch.no_grad():
        fmap, cnet = RaftTF32(sd64, rounding=False).encode(torch.cat([im1, im2]))
        for i, im in enumerate((im1, im2)):
            assert rel(fmap[i:i + 1], oracle_raft.encoder(sd64, 'fnet', im, 'instance')) < 1e-12, i
        net, inp = oracle_raft.context(sd64, im1)
        e_net, e_inp = RaftTF32(sd64, rounding=False).context_split(cnet[:1])
    assert rel(e_net, net) < 1e-12 and rel(e_inp, inp) < 1e-12


@pytest.mark.parametrize('it', [0, 3])
def test_without_rounding_an_update_iteration_is_the_oracle(gold, sd64, it):
    from oracle import raft as oracle_raft
    from oracle.raft_tf32 import RaftTF32
    case = gold['cases'][0]
    st = case['steps'][it]
    pyr = [l.double() for l in case['pyramid']]
    coords1 = case['coords1'][it:it + 1].double()
    coords0 = oracle_raft.coords_grid(1, *coords1.shape[-2:], torch.float64, 'cpu')
    net_in, inp = st['net_in'].double(), case['inp'].double()
    with torch.no_grad():
        r_net, r_delta = oracle_raft.update(sd64, net_in, inp, oracle_raft.lookup(pyr, coords1), coords1 - coords0)
        net, net_r, c1, delta = RaftTF32(sd64, rounding=False).update(pyr, net_in, inp, coords1, coords0)
    assert rel(net, r_net) < 1e-12 and rel(delta, r_delta) < 1e-12
    assert torch.equal(net_r, net) and torch.equal(c1, coords1 + delta)


def test_without_rounding_the_mask_head_and_upsampling_are_the_oracle(gold, sd64):
    from oracle import raft as oracle_raft
    from oracle.raft_tf32 import RaftTF32
    case = gold['cases'][0]
    fin = case['final'][1]
    net = case['steps'][3]['net'].double()
    low = fin['flow_low'].double()
    coords0 = oracle_raft.coords_grid(1, *low.shape[-2:], torch.float64, 'cpu')
    emu = RaftTF32(sd64, rounding=False)
    with torch.no_grad():
        mask = emu.up_mask(net)
        assert rel(0.25 * mask, oracle_raft.up_mask(sd64, net)) < 1e-12
        up = emu.upsample(mask, low + coords0, coords0)
    assert rel(up, oracle_raft.upsample(low, 0.25 * mask)) < 1e-12


def test_without_rounding_the_forward_is_the_oracle(sd64, pair):
    from oracle import raft as oracle_raft
    from oracle.raft_tf32 import RaftTF32
    im1, im2 = pair
    with torch.no_grad():
        low, up = RaftTF32(sd64, rounding=False).forward(im1, im2, 3)
        r_low, r_up = oracle_raft.raft_forward(sd64, im1, im2, 3)
    assert rel(low, r_low) < 1e-12 and rel(up, r_up) < 1e-12, (rel(low, r_low), rel(up, r_up))


def test_anchors_at_the_emulations_own_values_change_nothing(sd64, pair):
    from oracle.raft_tf32 import Anchors, RaftTF32, anchor_names
    im1, im2 = pair
    own = {}
    with torch.no_grad():
        low, up = RaftTF32(sd64, trace=own).forward(im1, im2, 2)
        want = set(anchor_names('encoder')) | set(anchor_names('state'))
        want |= {'it%d.%s' % (k, n) for k in range(2) for n in anchor_names('iteration')}
        assert set(own) == want, sorted(want ^ set(own))
        anc = Anchors(own)
        low2, up2 = RaftTF32(sd64, anchors=anc).forward(im1, im2, 2)
    assert torch.equal(low, low2) and torch.equal(up, up2)
    assert set(anc.report) == want
    for name, r in anc.report.items():
        assert r['rel_max'] == 0.0 and r.get('diff', 0.0) == 0.0, (name, r)
    # the rounded anchors are exactly those the table of oracle/raft_tf32.py rounds
    rounded = sorted(n.split('.', 1)[1] if n.startswith('it') else n for n, r in anc.report.items() if r['rounded'])
    assert set(rounded) == {'fnet.stem.out', 'cnet.stem.out', 'inp', 'corr', 'convc1', 'convc2', 'convf1', 'convf2', 'motion',
                            'rh.0', 'rh.1', 'net_r', 'mask0'} | {'%s.%s.%s' % (e, b, s) for e in ('fnet', 'cnet')
                                                               for b in ('layer1.0', 'layer1.1', 'layer2.0', 'layer2.1', 'layer3.0', 'layer3.1')
                                                               for s in ('y', 'out')}


def test_with_rounding_the_emulation_stays_in_the_tf32_envelope(gold, sd64, pair):
    """sanity only: the fixture's TF32 envelope is the eager TF32 on/off spread of DESIGN.md §3 (2.9e-3 px after 4 iterations;
    RaftNet is held to 4 times it) and the encoders' 3 x eager-TF32 bound (about 4e-3 to 1e-2)"""
    from oracle.raft_tf32 import RaftTF32
    case = gold['cases'][0]
    im1, im2 = pair
    tr = {}
    with torch.no_grad():
        _, up = RaftTF32(sd64, trace=tr).forward(im1, im2, 4)
    assert rel(tr['fmap'][:1], case['fmap1']) < 1e-2 and rel(torch.tanh(tr['cnet'][:1, :128]), case['net0']) < 1e-2
    epe = float((up - case['final'][4]['flow_up'].double()).norm(dim=1).mean())
    assert epe < 4 * 2.9e-3, epe
    # and it is not the fp64 oracle: the rounding points are in effect
    assert epe > 10 * case['floor_epe'][4], epe
