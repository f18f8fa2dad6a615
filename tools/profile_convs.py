#!/usr/bin/env python
"""Per-launch table of the tensor-core convolution kernels of one MiDaS training step (16 images, 384x224): CUDA events around
every launch (dvd_b200.conv_ops.PROFILE), grouped by (kind, geometry). Writes gpurun_out/<tag>_conv_table.json and prints the
classes sorted by time."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


def main():
    from dvd_b200 import conv_ops, synthetic
    from dvd_b200.third_party.MiDaS import MidasNet
    tag = sys.argv[1] if len(sys.argv) > 1 else 'r2'
    N = int(os.environ.get('IMAGES', '16'))
    net = synthetic.seed_net_(MidasNet(non_negative=True, normalize_input=True), 0, 2000.0).eval().cuda()
    x = torch.rand(N, 3, 224, 384, device='cuda')
    for _ in range(2):
        d = net(x)
        d.sum().backward()
    torch.cuda.synchronize()
    conv_ops.PROFILE = []
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    d = net(x)
    d.sum().backward()
    b.record()
    torch.cuda.synchronize()
    rec, conv_ops.PROFILE = conv_ops.PROFILE, None
    # un-instrumented timing of the same fwd+bwd
    a2, b2 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a2.record()
    for _ in range(3):
        d = net(x)
        d.sum().backward()
    b2.record()
    torch.cuda.synchronize()
    agg = {}
    for kind, flops, e0, e1, info in rec:
        key = (kind,) + tuple(info)
        g = agg.setdefault(key, [0, 0.0, 0.0])
        g[0] += 1
        g[1] += flops
        g[2] += e0.elapsed_time(e1)
    rows = []
    for key, (n, f, ms) in agg.items():
        kind, Nn, H, W, Cin, OH, OW, Cout, stride, ntaps, kblock = key
        rows.append({'kind': kind, 'N': Nn, 'H': H, 'W': W, 'Cin': Cin, 'OH': OH, 'OW': OW, 'Cout': Cout, 'stride': stride, 'ntaps': ntaps,
                     'kblock': kblock, 'launches': n, 'gflop': f / 1e9, 'ms': ms, 'tflops': f / ms / 1e9 if ms else 0})
    rows.sort(key=lambda r: -r['ms'])
    tot = sum(r['ms'] for r in rows)
    out = {'images': N, 'fwd_bwd_ms_instrumented': a.elapsed_time(b), 'fwd_bwd_ms': a2.elapsed_time(b2) / 3, 'conv_ms': tot, 'rows': rows}
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, 'gpurun_out', tag + '_conv_table.json'), 'w'), indent=0)
    print('fwd+bwd %.2f ms (instrumented %.2f), conv kernels %.2f ms' % (out['fwd_bwd_ms'], out['fwd_bwd_ms_instrumented'], tot))
    for r in rows[:45]:
        print('%-6s %4dx%-4d %5d->%-5d taps %3d s%d kb %3d  x%-3d %8.1f GF %7.3f ms %7.1f TF/s' % (
            r['kind'], r['OH'], r['OW'], r['Cin'], r['Cout'], r['ntaps'], r['stride'], r['kblock'], r['launches'], r['gflop'], r['ms'], r['tflops']))


if __name__ == '__main__':
    main()
