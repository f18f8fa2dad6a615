"""TEST INFRASTRUCTURE — writes tests/golden/raft_golden.pt from the UNMODIFIED reference RAFT (third_party/RAFT/core), CPU, fp32.

    python -m oracle.gen_golden_raft

Parameters and images are not stored: `oracle.raft.seeded_state_dict(seed, gain)` and `oracle.raft.seeded_pair(H, W, seed)`
rebuild them (a RAFT checkpoint is 21 MB), and the fixture keeps a checksum of both. One 20-iteration run per case is
traced with a forward hook on the update block (iterations 1 and 4 are its prefixes); the outputs of `iters` = 1, 4 and 20
come from three calls of the reference's forward.

Sizes: the reference's lookup divides by (W - 1) and (H - 1) of every pyramid level, so an image under 128 pixels on a side
(a 1-pixel coarsest level) makes it return NaN; the cases are 128x160 and 136x192 (odd 1/8 grid: the pooling drops a row).

The reference cannot run in fp64 (its lookup casts to float), so the rounding floor stored with each case is the
reference's fp32 `flow_up` against `oracle.raft` in fp64, as mean end-point error in pixels; GAIN was chosen so that the
20-iteration floor stays under 1e-5 px (gain 1.0: 6e-5 px, gain 0.7: 4e-6 px at 128x160).
"""
import argparse
import os
import sys

import torch

from . import golden_io, raft as oracle_raft
from .ref_harness import REF_ROOT

GAIN = 0.7
WEIGHT_SEED = 0
# case 0 keeps every stage; case 1 (the odd grid) only what the pooling, the lookup and the end-to-end result need
CASES = (dict(H=128, W=160, seed=1, full_iters=(0, 3), lean=False), dict(H=136, W=192, seed=2, full_iters=(0,), lean=True))
ITERS = (1, 4, 20)
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')


def import_reference_raft():
    core = os.path.join(REF_ROOT, 'third_party', 'RAFT', 'core')
    if not os.path.isdir(core):
        raise RuntimeError('reference RAFT not found at %s' % core)
    sys.path.insert(0, core)
    import corr
    import raft
    return raft, corr


def epe(a, b):
    return float((a.double() - b.double()).norm(dim=1).mean())


def main():
    torch.manual_seed(0)
    raft, corr = import_reference_raft()
    model = raft.RAFT(argparse.Namespace(small=False, mixed_precision=False, alternate_corr=False, dropout=0)).eval()
    sd = oracle_raft.seeded_state_dict(WEIGHT_SEED, GAIN)
    model.load_state_dict(sd, strict=True)
    sd64 = oracle_raft.cast(sd, torch.float64)
    out = dict(gain=GAIN, weight_seed=WEIGHT_SEED, keys=sorted(model.state_dict().keys()),
               weight_checksum=float(sum(v.double().abs().sum() for v in sd.values())), cases=[])
    for case in CASES:
        im1, im2 = oracle_raft.seeded_pair(case['H'], case['W'], case['seed'])
        steps = []
        hook = model.update_block.register_forward_hook(
            lambda mod, args, res: steps.append(dict(net_in=args[0], corr=args[2], flow=args[3], net=res[0], up_mask=res[1],
                                                     delta_flow=res[2])))
        rec = dict(H=case['H'], W=case['W'], seed=case['seed'], image_checksum=float(im1.double().sum() + im2.double().sum()),
                   final={}, floor_epe={})
        with torch.no_grad():
            for iters in ITERS:
                del steps[:]
                flow_low, flow_up = model(im1, im2, iters=iters, test_mode=True)
                o_up = oracle_raft.raft_forward(sd64, im1.double(), im2.double(), iters)[1]
                rec['final'][iters] = dict(flow_low=flow_low, flow_up=flow_up)
                if iters == ITERS[0] and not case['lean']:
                    rec['final'][iters]['up_mask'] = steps[-1]['up_mask']
                rec['floor_epe'][iters] = epe(flow_up, o_up)
            hook.remove()
            x1, x2 = 2 * (im1 / 255.0) - 1.0, 2 * (im2 / 255.0) - 1.0
            fmap1, fmap2 = model.fnet([x1, x2])
            net0, inp = torch.split(model.cnet(x1), [128, 128], dim=1)
            rec['pyramid'] = list(corr.CorrBlock(fmap1, fmap2, radius=4).corr_pyramid)
            if not case['lean']:
                rec.update(fmap1=fmap1, fmap2=fmap2, net0=torch.tanh(net0), inp=torch.relu(inp))
        h, w = case['H'] // 8, case['W'] // 8
        coords0 = oracle_raft.coords_grid(1, h, w, torch.float32, 'cpu')
        rec['coords1'] = torch.stack([coords0[0] + s['flow'][0] for s in steps])       # the lookup's input, per iteration
        rec['delta_flow'] = torch.stack([s['delta_flow'][0] for s in steps])
        rec['steps'] = {i: (dict(corr=steps[i]['corr']) if case['lean'] else
                            dict(corr=steps[i]['corr'], net_in=steps[i]['net_in'], net=steps[i]['net'])) for i in case['full_iters']}
        out['cases'].append(rec)
        print('%dx%d: floor EPE %s' % (case['H'], case['W'], rec['floor_epe']))
    golden_io.save_golden(out, GOLDEN_DIR, 'raft_golden')


if __name__ == '__main__':
    main()
