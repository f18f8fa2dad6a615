"""Run the scene-flow MLP chain kernels (forward with saved activations, then the data gradient of every evaluation) on
seeded inputs through the raw C ABI and dump everything they write, so that two builds can be compared bit for bit.

    python tools/mlp_kernel_dump.py dump <out_dir> [--root <tree>]   # arrays of the build in <tree> (default: this one)
    python tools/mlp_kernel_dump.py compare <dir_a> <dir_b>         # every array equal bit for bit (g_bias5: see below)

Dumped per case (configuration x size): the forward's acc, s_steps, p_steps, the whole save buffer (saved bf16
activations and ReLU masks of every evaluation), and per evaluation the data gradient's a_out, its dY scratch and
g_bias5. Every output buffer starts zeroed, so bytes a kernel does not write compare equal. Arrays up to 64 MB are written
as .npy; every array's SHA-256 goes to digests.json (the save buffers of 8 pairs at 224 x 384 are gigabytes), and the
comparison is by digest. g_bias5 is summed with atomicAdd across warps in no fixed order; it is compared against the fp32
bound of an n-term sum instead."""
import argparse
import ctypes
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (16, 16, time-dependent) and (16, time-independent) have kernels compiled for their counts; (20, 10, time-dependent) runs
# the generic kernels with a 192-wide first layer (nin = 144).
CONFIGS = {'16-16-T': (16, 16, True), '16-0-F': (16, 0, False), '20-10-T': (20, 10, True)}
# (B, H, W): the benchmark's 8 pairs at 224 x 384, and a pixel count that is not a multiple of the 128-pixel tile
SIZES = {'b8_224x384': (8, 224, 384), 'ragged_3x29x41': (3, 29, 41)}
N_EVAL = 3


def _lib_ops(root):
    if root not in sys.path:
        sys.path.insert(0, root)
    from dvd_b200 import _lib, ops
    return _lib, ops


def make_weights(nin, seed):
    g = torch.Generator().manual_seed(seed)
    dims = [(256, nin)] + [(256, 256)] * 4 + [(3, 256)]
    ws = [(torch.randn(o, i, generator=g) * (2.0 / i) ** 0.5).cuda().contiguous() for o, i in dims]
    bs = [(torch.randn(o, generator=g) * 0.1).cuda().contiguous() for o, _ in dims]
    return ws, bs


def make_inputs(B, H, W, n_eval, seed):
    g = torch.Generator().manual_seed(seed)
    p0 = (torch.randn(B, 3, H, W, generator=g) * 3).cuda()
    t0 = torch.rand(B, 1, H, W, generator=g).cuda()
    g_acc = torch.randn(B, 3, H, W, generator=g).cuda()
    g_steps = [torch.randn(B, 3, H, W, generator=g).cuda() for _ in range(n_eval)]
    return p0, t0, g_acc, g_steps


def run_chain(_lib, ops, pk, p0, t0, g_acc, g_steps, n_eval, n_acc, dt=1 / 80):
    """Forward (training: saved activations) over n_eval Euler steps, then the data gradient of evaluations n_eval - 1 .. 0,
    each reading the previous one's a_out, as the backward pass chains them. Returns a dict of cuda tensors."""
    cfg = pk.cfg
    B, _, H, W = p0.shape
    npx, hw = B * H * W, H * W
    lib = _lib.load()
    P = ctypes.c_void_p
    per = lib.dvd_mlp_save_bytes_per_eval(ctypes.byref(cfg), npx)
    acc = torch.zeros_like(p0)
    s_steps = torch.zeros(n_eval, B, 3, H, W, device='cuda')
    p_steps = torch.zeros(n_eval, B, 3, H, W, device='cuda')
    save = torch.zeros(n_eval * per, dtype=torch.uint8, device='cuda')
    t_ptr = P(t0.data_ptr()) if cfg.time_dependent else P(0)
    _lib.check(lib.dvd_mlp_chain_fwd(ctypes.byref(cfg), P(pk.fwd.data_ptr()), P(pk.bias.data_ptr()), P(p0.data_ptr()), t_ptr,
                                     float(dt), n_eval, n_acc, P(acc.data_ptr()), P(s_steps.data_ptr()), P(p_steps.data_ptr()),
                                     P(save.data_ptr()), npx, hw, ops._stream()), 'dvd_mlp_chain_fwd')
    out = {'acc': acc, 's_steps': s_steps, 'p_steps': p_steps, 'save': save}
    ndy = lib.dvd_mlp_dy_bytes(ctypes.byref(cfg), npx)
    a = None
    for e in range(n_eval - 1, -1, -1):
        a_out = torch.zeros_like(p0)
        dy = torch.zeros(ndy, dtype=torch.uint8, device='cuda')
        gb5 = torch.zeros(3, device='cuda')
        _lib.check(lib.dvd_mlp_dgrad(ctypes.byref(cfg), P(pk.bwd.data_ptr()), P(p_steps[e].data_ptr()), t_ptr, float(dt), e,
                                     int(e < n_acc), P(g_acc.data_ptr()), P(g_steps[e].data_ptr()),
                                     P(a.data_ptr()) if a is not None else P(0), P(a_out.data_ptr()), P(save.data_ptr() + e * per),
                                     P(dy.data_ptr()), P(gb5.data_ptr()), npx, hw, ops._stream()), 'dvd_mlp_dgrad')
        out['a_out_e%d' % e], out['dy_e%d' % e], out['g_bias5_e%d' % e] = a_out, dy, gb5
        gs = g_steps[e].double() + (g_acc.double() if e < n_acc else 0) + (a.double() if a is not None else 0)
        out['g_bias5_abs_e%d' % e] = (gs / cfg.sf_mag_div).abs().sum(dim=(0, 2, 3))    # sum of |terms| per component
        a = a_out
    torch.cuda.synchronize()
    return out


def dump(out_dir, root):
    _lib, ops = _lib_ops(root)
    os.makedirs(out_dir, exist_ok=True)
    digests = {}
    for cname, (fx, ft, td) in CONFIGS.items():
        cfg = ops.make_mlp_cfg(n_freq_xyz=fx, n_freq_t=ft, time_dependent=td)
        ws, bs = make_weights(ops.mlp_n_in(fx, ft, td), seed=11)
        pk = ops.PackedMlp(cfg, 'cuda').refresh(ws, bs)
        for sname, (B, H, W) in SIZES.items():
            p0, t0, g_acc, g_steps = make_inputs(B, H, W, N_EVAL, seed=12)
            res = run_chain(_lib, ops, pk, p0, t0, g_acc, g_steps, N_EVAL, N_EVAL - 1)
            for k, v in res.items():
                name = '%s__%s__%s' % (cname, sname, k)
                arr = v.cpu().numpy()
                digests[name] = {'sha256': hashlib.sha256(arr.tobytes()).hexdigest(), 'shape': list(arr.shape),
                                 'dtype': str(arr.dtype)}
                if arr.nbytes <= 64 << 20:
                    np.save(os.path.join(out_dir, name + '.npy'), arr)
            print('dumped', cname, sname, flush=True)
    with open(os.path.join(out_dir, 'digests.json'), 'w') as f:
        json.dump(digests, f, indent=1)


def compare(dir_a, dir_b):
    da, db = (json.load(open(os.path.join(d, 'digests.json'))) for d in (dir_a, dir_b))
    assert sorted(da) == sorted(db), 'different sets of arrays'
    bad = 0
    for name in sorted(da):
        if '__g_bias5_abs_e' in name:     # the bound's input, computed by torch
            continue
        if '__g_bias5_e' in name:
            # an n-term fp32 sum in any order is within (n - 1) u sum|terms| of the exact sum; two of them within twice that
            a, b = (np.load(os.path.join(d, name + '.npy')).astype(np.float64) for d in (dir_a, dir_b))
            n = int(np.prod(da[name.rsplit('__', 1)[0] + '__acc']['shape'])) // 3
            abs_sum = np.load(os.path.join(dir_a, name.replace('g_bias5_e', 'g_bias5_abs_e') + '.npy'))
            ok = bool(np.all(np.abs(a - b) <= 2 * (n - 1) * 2.0 ** -24 * abs_sum))
        else:
            ok = da[name] == db[name]
        if not ok:
            bad += 1
            print('DIFFERS', name, flush=True)
    print('compared %d arrays: %d differ' % (len(da), bad), flush=True)
    return bad


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest='cmd', required=True)
    d = sub.add_parser('dump')
    d.add_argument('out_dir')
    d.add_argument('--root', default=ROOT, help='tree whose built library runs')
    c = sub.add_parser('compare')
    c.add_argument('dir_a')
    c.add_argument('dir_b')
    a = ap.parse_args()
    if a.cmd == 'dump':
        dump(a.out_dir, os.path.abspath(a.root))
    else:
        sys.exit(1 if compare(a.dir_a, a.dir_b) else 0)


if __name__ == '__main__':
    main()
