"""Synthetic depth of field of a test export: `python -m dvd_b200.refocus --test_dir OUT/<net>_<dataset>/epochbest_test --out DIR
[--aperture 8] [--max_blur 16] [--focus_point x,y | --focus_depth Z | --focus_pull a:b] [--focus_window 2] [--frames a:b]
[--chunk 16] [--gpu 0]`.

Reads `depth`, `img_1` and, when the files hold it, `depth_nn` (the per-frame initialisation) of the `batch%04d.npz` files with
export_io.Frames (`--frames` as in `export_points`), and blurs every selected frame by each pixel's distance, in
disparity, from the frame's focal plane. With the refined depth the focus holds still; with the initial depth it boils and
hunts, so the two side by side show what consistent depth is for. It writes DIR/dof_%05d.png (the refined-depth render,
numbered like `export_points`' per-frame files), DIR/dof.mp4, DIR/compare.mp4 (frame | initial-depth render | refined-depth
render, 30 fps, `mp4v`; only when `depth_nn` exists) and DIR/refocus.json (the options, the median depths, each frame's
focal disparity and mean blur radius for both sources, and whether the comparison was written).

Each depth source is rendered from its own depths. m is the median valid (finite, > 1e-2) depth of its selected frames; the
blur radius of a pixel is c = min(R, s |disp - phi_t|) pixels, disp = 1/d (0 for an invalid pixel: infinitely far),
R = --max_blur, s = --aperture x m in fp64 rounded to fp32 once: --aperture is the blur radius of a point at half the median
depth when the focus is at the median depth, whatever the export's depth scale. The focal disparity phi_t, computed on the
host in fp64 and rounded to fp32 once per frame, is one of
  --focus_point x,y  1 / the median valid depth in the (2k+1)^2 window at pixel (x, y), clipped to the image (k =
                     --focus_window; default: the image centre). A frame without a valid depth there keeps the previous
                     frame's phi; the first falls back to 1/m;
  --focus_depth Z    1 / (Z m) for every frame;
  --focus_pull a:b   a rack focus, linear in disparity from 1 / (a m) at the first selected frame to 1 / (b m) at the last.
The gather rule (csrc/refocus.cu, include/dvd_b200.h) is exact: the frames are bitwise reproducible and do not depend on
--chunk. Each chunk goes to the device in one copy (depths, images, focal disparities) and its frames come back in one copy.
"""
import argparse
import json
import os
import time

import numpy as np
import torch

from . import ops
from ._lib import DVD_REFOCUS_MAX_RADIUS as MAX_BLUR
from .export_io import Frames, Writer, chunk_size, cuda_device, frame_range, list_files, to_device
from .render_views import median_depth

FPS = 30
F32 = np.float32


def source_median(depth, name):
    """median_depth of one depth source, with a ValueError that names it"""
    d = np.asarray(depth, dtype=F32)
    if not (np.isfinite(d) & (d > F32(1e-2))).any():
        raise ValueError('the %s has no valid depth (finite and > 1e-2) in the selected frames' % name)
    return median_depth(d)


def focus_disparities(depth, m, focus_point=None, focus_window=2, focus_depth=None, focus_pull=None):
    """The focal disparities [N] fp32 of frames depth [N,H,W] whose median valid depth is m (see the module docstring).
    focus_point is (x, y) or None for the image centre; it is used when neither focus_depth nor focus_pull is given."""
    depth = np.asarray(depth, dtype=F32)
    N, H, W = depth.shape
    if focus_depth is not None:
        return np.full(N, 1.0 / (float(focus_depth) * m), dtype=np.float64).astype(F32)
    if focus_pull is not None:
        a, b = (float(v) for v in focus_pull)
        p0, p1 = 1.0 / (a * m), 1.0 / (b * m)
        return (p0 + (p1 - p0) * (np.arange(N, dtype=np.float64) / max(N - 1, 1))).astype(F32)
    x, y = (W // 2, H // 2) if focus_point is None else (int(v) for v in focus_point)
    if not (0 <= x < W and 0 <= y < H):
        raise ValueError('focus point (%d, %d) lies outside the %dx%d frames' % (x, y, W, H))
    k = int(focus_window)
    win = depth[:, max(y - k, 0):min(y + k + 1, H), max(x - k, 0):min(x + k + 1, W)].reshape(N, -1)
    ok = np.isfinite(win) & (win > F32(1e-2))
    out, prev = np.empty(N, dtype=F32), 1.0 / m
    for t in range(N):
        if ok[t].any():
            prev = 1.0 / float(np.median(win[t][ok[t]].astype(np.float64)))
        out[t] = prev
    return out


def mean_blur(depth, phi, scale, R):
    """each frame's mean blur radius c = min(R, s |disp - phi_t|) pixels, c in fp32 as the kernel computes it, the mean in
    fp64"""
    d = np.asarray(depth, dtype=F32)
    ok = np.isfinite(d) & (d > F32(1e-2))
    with np.errstate(all='ignore'):
        disp = np.where(ok, F32(1) / np.where(ok, d, F32(1)), F32(0)).astype(F32)
    c = np.fmin(F32(R), F32(scale) * np.abs(disp - np.asarray(phi, F32)[:, None, None]))
    return c.reshape(c.shape[0], -1).mean(1, dtype=np.float64)


def check_options(aperture, max_blur, focus_point, focus_window, focus_depth, focus_pull, chunk):
    if not (np.isfinite(aperture) and aperture >= 0):
        raise ValueError('aperture must be finite and >= 0, got %r' % aperture)
    if int(max_blur) != max_blur or not 0 <= max_blur <= MAX_BLUR:
        raise ValueError('max_blur must be an integer in [0, %d], got %r' % (MAX_BLUR, max_blur))
    if sum(v is not None for v in (focus_point, focus_depth, focus_pull)) > 1:
        raise ValueError('give at most one of focus_point, focus_depth and focus_pull')
    if int(focus_window) != focus_window or focus_window < 0:
        raise ValueError('focus_window must be an integer >= 0, got %r' % focus_window)
    if focus_depth is not None and not (np.isfinite(focus_depth) and focus_depth > 0):
        raise ValueError('focus_depth must be finite and > 0, got %r' % focus_depth)
    if focus_pull is not None and (len(focus_pull) != 2 or not all(np.isfinite(v) and v > 0 for v in focus_pull)):
        raise ValueError('focus_pull must be two finite values > 0, got %r' % (focus_pull,))
    chunk_size(chunk)


def refocus(test_dir, out, aperture=8.0, max_blur=16, focus_point=None, focus_window=2, focus_depth=None, focus_pull=None,
            frames=None, chunk=16, device=None):
    """Renders the test export in `test_dir` into `out` (see the module docstring) on CUDA device `device` (default: the
    current one). Every argument and file is checked before the device is touched. Returns a dict of the written paths,
    the frame numbers and the record written to refocus.json."""
    check_options(aperture, max_blur, focus_point, focus_window, focus_depth, focus_pull, chunk)
    R, chunk = int(max_blur), int(chunk)
    ex = Frames(list_files(test_dir), frames, optional=('depth_nn',))
    N, H, W = ex.N, ex.H, ex.W
    nn = ex.depth_nn
    if focus_depth is None and focus_pull is None:
        focus_point = (W // 2, H // 2) if focus_point is None else tuple(int(v) for v in focus_point)
    sources = [('refined', ex.depth)] + ([('initial', nn)] if nn is not None else [])
    med, phi, scale = {}, {}, {}
    for name, d in sources:
        med[name] = source_median(d, '%s depth' % name)
        phi[name] = focus_disparities(d, med[name], focus_point, focus_window, focus_depth, focus_pull)
        scale[name] = float(F32(float(aperture) * med[name]))
    order = (['initial'] if nn is not None else []) + ['refined']       # the order of the renders in a chunk's buffer
    depth_of = dict(sources)
    dev = cuda_device(device)

    os.makedirs(out, exist_ok=True)
    mean_c = {name: np.zeros(N) for name, _ in sources}
    written = []
    vids = {'dof': os.path.join(out, 'dof.mp4')}
    if nn is not None:
        vids['compare'] = os.path.join(out, 'compare.mp4')
    with Writer() as wr:
        v_dof = wr.video(vids['dof'], FPS, (H, W))
        v_cmp = wr.video(vids['compare'], FPS, (H, 3 * W)) if nn is not None else None
        for s in range(0, N, chunk):
            e = min(s + chunk, N)
            n = e - s
            g = to_device(dev, *[depth_of[name][s:e] for name in order], ex.images(s, e), *[phi[name][s:e] for name in order])
            depths, img, fphi = g[:len(order)], g[len(order)], g[len(order) + 1:]
            # the frame itself (floor(255 clip(img)): no blur) when a comparison is written, then the renders in `order`
            k = len(order) + (nn is not None)
            buf = torch.empty(k, n, H, W, 3, dtype=torch.uint8, device=dev)
            if nn is not None:
                ops.refocus(depths[0], img, fphi[0], 0.0, 0, out=buf[0])
            for j, name in enumerate(order):
                ops.refocus(depths[j], img, fphi[j], scale[name], R, out=buf[k - len(order) + j])
            for name, d in sources:
                mean_c[name][s:e] = mean_blur(d[s:e], phi[name][s:e], scale[name], R)
            hb = buf.cpu().numpy()                                                       # the chunk's one D2H copy
            for j in range(n):
                p = os.path.join(out, 'dof_%05d.png' % ex.ids[s + j])
                written.append(p)
                wr.png(p, hb[-1, j])
                v_dof.write(hb[-1, j])
                if v_cmp is not None:
                    v_cmp.write(np.concatenate(list(hb[:, j]), 1))
    options = {'aperture': float(aperture), 'max_blur': R, 'focus_point': None if focus_point is None else list(focus_point),
               'focus_window': int(focus_window), 'focus_depth': focus_depth,
               'focus_pull': None if focus_pull is None else [float(v) for v in focus_pull], 'frames': frames, 'chunk': chunk}
    rec = record(test_dir, ex.ids, options, H, W, med, scale, phi, mean_c, nn is not None)
    with open(os.path.join(out, 'refocus.json'), 'w') as f:
        json.dump(rec, f, indent=1)
    return {'frames_written': written, 'videos': vids, 'json': os.path.join(out, 'refocus.json'),
            'frames': [int(i) for i in ex.ids], 'record': rec}


def record(test_dir, ids, options, H, W, med, scale, phi, mean_c, compare):
    """The contents of refocus.json: the options, per depth source its median depth m, its scale s (the fp32 value) and per
    frame its focal disparity (the fp32 value) and mean blur radius; whether compare.mp4 was written."""
    src = lambda name: None if name not in med else {'m': med[name], 'scale': scale[name]}
    return {'test_dir': os.path.abspath(test_dir), 'height': int(H), 'width': int(W), 'options': options,
            'm': med['refined'], 'm_nn': med.get('initial'), 'refined': src('refined'), 'initial': src('initial'),
            'compare_written': bool(compare),
            'frames': [dict({'frame': int(i), 'focus_disp': float(phi['refined'][t]), 'mean_blur': float(mean_c['refined'][t])},
                            **({'focus_disp_nn': float(phi['initial'][t]), 'mean_blur_nn': float(mean_c['initial'][t])}
                               if 'initial' in med else {}))
                       for t, i in enumerate(ids)]}


def _pair(sep, kind):
    def parse(s):
        parts = s.split(sep)
        if len(parts) != 2:
            raise argparse.ArgumentTypeError('expected two values separated by %r, got %r' % (sep, s))
        try:
            return tuple(kind(v) for v in parts)
        except ValueError:
            raise argparse.ArgumentTypeError('expected two %s values separated by %r, got %r' % (kind.__name__, sep, s)) from None
    return parse


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog='python -m dvd_b200.refocus', description=__doc__.split('\n\n')[0])
    p.add_argument('--test_dir', required=True, help='directory of the batch%%04d.npz files the test driver wrote')
    p.add_argument('--out', required=True, help='output directory (dof_%%05d.png, dof.mp4, compare.mp4, refocus.json)')
    p.add_argument('--aperture', type=float, default=8.0, help='blur radius in pixels of a point at half the median depth '
                   'when focused at the median depth')
    p.add_argument('--max_blur', type=int, default=16, help='largest blur radius in pixels (0 to %d)' % MAX_BLUR)
    g = p.add_mutually_exclusive_group()
    g.add_argument('--focus_point', type=_pair(',', int), default=None, metavar='X,Y',
                   help='focus on the median valid depth around pixel (X, Y) of every frame (the default, at the image centre)')
    g.add_argument('--focus_depth', type=float, default=None, metavar='Z', help='focus at Z x the median valid depth')
    g.add_argument('--focus_pull', type=_pair(':', float), default=None, metavar='A:B',
                   help='rack focus from A x to B x the median valid depth, linear in disparity')
    p.add_argument('--focus_window', type=int, default=2, help='--focus_point window half-width k: (2k+1)^2 pixels')
    p.add_argument('--frames', type=frame_range, default=None, help='frames a:b (Python slice of the frames in file order)')
    p.add_argument('--chunk', type=int, default=16, help='frames per device chunk')
    p.add_argument('--gpu', type=int, default=0)
    a = p.parse_args(argv)
    try:
        check_options(a.aperture, a.max_blur, a.focus_point, a.focus_window, a.focus_depth, a.focus_pull, a.chunk)
    except ValueError as e:
        p.error(str(e))
    return a


def main(argv=None):
    a = parse_args(argv)
    t0 = time.perf_counter()
    res = refocus(a.test_dir, a.out, a.aperture, a.max_blur, a.focus_point, a.focus_window, a.focus_depth, a.focus_pull,
                  a.frames, a.chunk, device=a.gpu)
    rec = res['record']
    print('refocused %d frames (m = %.4g%s, comparison %s) into %s in %.2f s'
          % (len(res['frames_written']), rec['m'], '' if rec['m_nn'] is None else ', m_nn = %.4g' % rec['m_nn'],
             'written' if rec['compare_written'] else 'not written: no depth_nn', a.out, time.perf_counter() - t0))
    return res


if __name__ == '__main__':
    main()
