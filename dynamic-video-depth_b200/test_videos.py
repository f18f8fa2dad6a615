"""Disparity videos and temporal slices of a test export, the reference's `on_test_end` (models/video_base.py:157-272):
`python -m dvd_b200.test_videos --test_dir OUT/<net>_<dataset>_<suffix>/epochbest_test [--slice_rows a:b] [--chunk 32]
[--gpu 0]`, or `python -m dvd_b200.test --videos …` after the export.

Reads `depth`, `depth_nn`, `depth_gt` and `img_1` of the `batch%04d.npz` files with export_io.Frames (in index order,
flattened) and writes, with the reference's names (`outdir` = the `epoch*_test` directory, `parent` its parent,
`epoch_string` its name):

* `outdir/compare_%04d.png`: refined, initial (MiDaS) and GT disparity in the turbo colour map, all three over the range of
  the refined disparity of the whole video: vmin = 1 / max(depth), vmax = 1 / min(depth), fp32;
* `outdir/rgb_%04d.png`: the frame, floor(255 · clip(img, 0, 1));
* `outdir/temporal_slice_%04d.png`: for each slice row r, 1 / depth[:, 0, r, :] and 1 / depth_nn[:, 0, r, :] stacked over
  time (one canvas row per frame), each over the min and max of its own finite values (matplotlib's autoscale);
* `parent/<epoch_string>.mp4` (comparison frames, 30 fps), `<epoch_string>_temporal.mp4` (slices, 2 fps),
  `<epoch_string>_rgb.mp4` (RGB frames, 30 fps) and `<epoch_string>.html`, a page with the three videos and no scripts.

The canvases are drawn on the GPU by `dvd_vis_panels` (csrc/test_videos.cu): each starts as a host-drawn template (titles,
one colour bar per panel with its end labels) and every panel pixel is written from the depth maps in place. `depth` and
`depth_nn` stay on the device for the whole run (the slices read every frame); `depth_gt` and `img_1` go up `chunk` frames at a
time, and each chunk's canvases come back in one copy. Disparities: `1 / x` in fp32; GT `np.where(gt > 1e-8, 1, 0) /
(gt + 1e-8)` in numpy's dtypes (fp64). Colour index: floor(256 t), t = (v - vmin) / (vmax - vmin) in fp64, clamped to
[0, 255] (matplotlib's rule for a 256-entry map), vmax == vmin -> 0, NaN -> black. The colour table is OpenCV's
COLORMAP_TURBO (Google's turbo, the table matplotlib's `turbo` holds as floats), read from cv2 at run time.

Geometry (the canvas of k panels of h x w pixels): the panels sit at y0 = TITLE_H and x0 = MARGIN + p (block + MARGIN), block
= w + BAR_GAP + BAR_W + LABEL_GAP + LABEL_W. Each panel's title is centred above it (baseline TITLE_H - 10), its colour bar
(BAR_W wide, max(h, BAR_MIN_H) tall, top = last colour) starts BAR_GAP to its right, and the bar's end values ('%.3g' of vmax
at the top, vmin at the bottom) follow LABEL_GAP further right. The canvas is MARGIN + k (block + MARGIN) wide, rounded up to
a multiple of 4, and TITLE_H + max(h, BAR_MIN_H) + MARGIN tall, rounded up to even. An RGB frame is the h x w frame alone.

Where this differs from the reference:

* videos are MPEG-4 part 2 (`mp4v` through cv2.VideoWriter), not libx264 through ffmpeg; frames of odd size are padded to even
  sizes at the bottom and right with black, as the reference's `pad` filter does;
* panels are drawn at the frames' own resolution in the layout above, not resampled into a matplotlib figure;
* the default slices are rows 120-139 when H >= 140 (the reference's) and the middle min(20, H) rows otherwise (the reference
  raises IndexError); `slice_rows` outside [0, H) raises ValueError;
* the page's "Disparity loss" is the mean over the frames of `ops.disp_vali(depth, depth_gt) / (H W)`, the validation
  metric; the reference prints a `test_loss` that is never updated (always 0);
* a refined depth that is non-finite or <= 0 raises ValueError naming the frame (the reference draws a NaN range); missing
  keys and frames of different sizes raise ValueError.
"""
import argparse
import html
import os
import re
import time

import cv2
import numpy as np
import torch

from . import ops
from .export_io import Frames, Writer, chunk_size, cuda_device, list_files, to_device

KEYS = ('depth', 'depth_nn', 'depth_gt', 'img_1')
MARGIN, TITLE_H, BAR_GAP, BAR_W, LABEL_GAP, LABEL_W, BAR_MIN_H = 8, 32, 6, 14, 4, 72, 48
FONT = cv2.FONT_HERSHEY_SIMPLEX
WHITE = (255, 255, 255)
COMPARE_TITLES = ('Refined', 'Initial', 'GT')
SLICE_TITLES = ('Refined', 'Initial')
DEFAULT_SLICES = (120, 140)
FPS, FPS_SLICES = 30, 2


def turbo_lut():
    """[256,3] uint8 BGR: OpenCV's COLORMAP_TURBO."""
    return cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_TURBO)[:, 0].copy()


def layout(k, h, w):
    """(CH, CW, [(y0, x0)] of the k panels) of a canvas of k colour-mapped h x w panels."""
    bh = max(h, BAR_MIN_H)
    block = w + BAR_GAP + BAR_W + LABEL_GAP + LABEL_W
    CW = MARGIN + k * (block + MARGIN)
    CH = TITLE_H + bh + MARGIN
    return CH + CH % 2, CW + (-CW) % 4, [(TITLE_H, MARGIN + p * (block + MARGIN)) for p in range(k)]


def template(titles, h, w, ranges, lut):
    """[CH,CW,3] uint8: black, each panel's title, colour bar and its end labels; ranges [(vmin, vmax)] per panel."""
    CH, CW, pos = layout(len(titles), h, w)
    t = np.zeros((CH, CW, 3), np.uint8)
    bh = max(h, BAR_MIN_H)
    ramp = lut[(255 * (bh - 1 - np.arange(bh))) // (bh - 1)]
    for title, (y0, x0), (lo, hi) in zip(titles, pos, ranges):
        tw = cv2.getTextSize(title, FONT, 0.6, 1)[0][0]
        cv2.putText(t, title, (x0 + max((w - tw) // 2, 0), TITLE_H - 10), FONT, 0.6, WHITE, 1, cv2.LINE_8)
        bx = x0 + w + BAR_GAP
        t[y0:y0 + bh, bx:bx + BAR_W] = ramp[:, None]
        lx = bx + BAR_W + LABEL_GAP
        cv2.putText(t, '%.3g' % hi, (lx, y0 + 10), FONT, 0.4, WHITE, 1, cv2.LINE_8)
        cv2.putText(t, '%.3g' % lo, (lx, y0 + bh - 1), FONT, 0.4, WHITE, 1, cv2.LINE_8)
    return t


def slice_rows_for(H, rows=None):
    """(a, b) of the temporal slices: `rows` 'a:b' (within [0, H)), else 120:140 when H >= 140, else the middle min(20, H) rows."""
    if rows is None:
        if H >= DEFAULT_SLICES[1]:
            return DEFAULT_SLICES
        k = min(20, H)
        return (H - k) // 2, (H - k) // 2 + k
    if isinstance(rows, str):
        m = re.fullmatch(r'(\d+):(\d+)', rows)
        if not m:
            raise ValueError('slice rows must look like a:b, got %r' % rows)
        rows = int(m.group(1)), int(m.group(2))
    a, b = rows
    if not 0 <= a < b <= H:
        raise ValueError('slice rows %d:%d are not a non-empty range within the %d image rows' % (a, b, H))
    return a, b


def _page(epoch_string, loss, rows):
    videos = (('%s_rgb.mp4' % epoch_string, 'original video'),
              ('%s.mp4' % epoch_string, 'Disparity loss %.6g' % loss),
              ('%s_temporal.mp4' % epoch_string, 'temporal slices, rows %d-%d' % (rows[0], rows[1] - 1)))
    body = ''.join('<h3>%s</h3>\n<video controls loop muted src="%s"></video>\n' % (html.escape(t), html.escape(v)) for v, t in videos)
    return ('<!DOCTYPE html>\n<html>\n<head><meta charset="utf-8"><title>%s</title></head>\n<body style="background:#000;color:#fff">\n'
            '%s</body>\n</html>\n' % (html.escape(epoch_string), body))


def render_test_videos(test_dir, slice_rows=None, chunk=32, device=None):
    """Writes the frames, slices, videos and page of the test export in `test_dir` (see the module docstring) on CUDA device
    `device` (default: the current one). The files are read and checked before the device is touched. Returns a dict of the
    written paths, the frame count, the slice rows and the page's loss."""
    chunk = chunk_size(chunk)
    outdir = os.path.normpath(test_dir)
    parent, epoch_string = os.path.dirname(outdir), os.path.basename(outdir)
    ex = Frames(list_files(outdir), keys=KEYS)
    N, H, W = ex.N, ex.H, ex.W
    a, b = slice_rows_for(H, slice_rows)
    bad = ~(np.isfinite(ex.depth) & (ex.depth > 0)).reshape(N, -1).all(1)
    if bad.any():
        i = int(np.argmax(bad))
        raise ValueError('frame %d (%s) has a refined depth that is not finite and > 0' % (i, ex.file_of[i]))
    dev = cuda_device(device)
    lut_h = turbo_lut()
    lut = torch.from_numpy(lut_h).to(dev)
    # both stay on the device for the whole run
    depth, depth_nn = to_device(dev, ex.depth[:, None], ex.depth_nn[:, None])
    # the global range: vmin = 1 / max, vmax = 1 / min in fp32 (numpy 2: a Python int over a float32 scalar stays float32)
    rng = torch.stack([1 / depth.amax(), 1 / depth.amin()])
    host = rng.cpu().numpy()
    vmin, vmax = rng.double().reshape(2, 1).expand(2, N).contiguous()
    HW = H * W

    CH, CW, pos = layout(3, H, W)
    tmpl = torch.from_numpy(template(COMPARE_TITLES, H, W, [(float(host[0]), float(host[1]))] * 3, lut_h)).to(dev)
    rgb_tmpl = torch.zeros(H, W, 3, dtype=torch.uint8, device=dev)
    sse = torch.empty(N, dtype=torch.float32, device=dev)
    ncmp, nrgb = CH * CW * 3, HW * 3
    written = {'compare': [], 'rgb': [], 'temporal_slice': []}
    vids = {'compare': os.path.join(parent, epoch_string + '.mp4'), 'rgb': os.path.join(parent, epoch_string + '_rgb.mp4'),
            'temporal': os.path.join(parent, epoch_string + '_temporal.mp4')}
    with Writer() as out:
        def png(kind, i, img):
            path = os.path.join(outdir, '%s_%04d.png' % (kind, i))
            written[kind].append(path)
            out.png(path, img)

        v_cmp, v_rgb = out.video(vids['compare'], FPS, (CH, CW)), out.video(vids['rgb'], FPS, (H, W))
        for s in range(0, N, chunk):
            e = min(s + chunk, N)
            n = e - s
            gt, img = to_device(dev, ex.depth_gt[s:e, None], ex.images(s, e))
            ops.disp_vali(depth[s:e], gt, out=sse[s:e])
            buf = torch.empty(n * (ncmp + nrgb), dtype=torch.uint8, device=dev)
            cmp_out, rgb_out = buf[:n * ncmp].view(n, CH, CW, 3), buf[n * ncmp:].view(n, H, W, 3)
            panels = [ops.vis_panel(src, tr, H, W, y0, x0, (HW, W, 1, 0), offset=off, vmin=vmin, vmax=vmax)
                      for (src, tr, off), (y0, x0) in zip(((depth, 'disp', s * HW), (depth_nn, 'disp', s * HW), (gt, 'gt_disp', 0)), pos)]
            ops.vis_panels(tmpl, panels, lut, cmp_out)
            ops.vis_panels(rgb_tmpl, [ops.vis_panel(img, 'rgb', H, W, 0, 0, (3 * HW, W, 1, HW))], None, rgb_out)
            hb = buf.cpu().numpy()                                             # the chunk's one device-to-host copy
            cmp_h, rgb_h = hb[:n * ncmp].reshape(n, CH, CW, 3), hb[n * ncmp:].reshape(n, H, W, 3)
            for j in range(n):
                png('compare', s + j, cmp_h[j])
                png('rgb', s + j, rgb_h[j])
                v_cmp.write(cmp_h[j])
                v_rgb.write(rgb_h[j])

        # temporal slices: panel row = frame, read in place from the resident depth maps; ranges per slice and panel on the device
        S = b - a
        disp = 1 / torch.stack([depth[:, 0, a:b], depth_nn[:, 0, a:b]])      # [2, N, S, W] fp32
        fin = torch.isfinite(disp)
        lo = torch.where(fin, disp, float('inf')).amin(dim=(1, 3))
        hi = torch.where(fin, disp, float('-inf')).amax(dim=(1, 3))
        none = ~fin.any(dim=3).any(dim=1)
        lo, hi = torch.where(none, 0.0, lo).double(), torch.where(none, 0.0, hi).double()   # [2, S]
        lh, hh = lo.cpu().numpy(), hi.cpu().numpy()
        sCH, sCW, spos = layout(2, N, W)
        stmpl = torch.from_numpy(np.stack([template(SLICE_TITLES, N, W, [(lh[0, r], hh[0, r]), (lh[1, r], hh[1, r])], lut_h)
                                           for r in range(S)])).to(dev)
        sl = torch.empty(S, sCH, sCW, 3, dtype=torch.uint8, device=dev)
        panels = [ops.vis_panel(src, 'disp', N, W, y0, x0, (W, HW, 1, 0), offset=a * W, vmin=lo[p], vmax=hi[p])
                  for p, (src, (y0, x0)) in enumerate(zip((depth, depth_nn), spos))]
        ops.vis_panels(stmpl, panels, lut, sl, tmpl_stride=sCH * sCW * 3)
        sl_h = sl.cpu().numpy()
        v_sl = out.video(vids['temporal'], FPS_SLICES, (sCH, sCW))
        for r in range(S):
            png('temporal_slice', r, sl_h[r])
            v_sl.write(sl_h[r])
    loss = float((sse.double() / HW).mean())
    page = os.path.join(parent, epoch_string + '.html')
    with open(page, 'w') as f:
        f.write(_page(epoch_string, loss, (a, b)))
    return dict(written, videos=vids, html=page, frames=N, slice_rows=(a, b), loss=loss)


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog='python -m dvd_b200.test_videos', description=__doc__.split('\n\n')[0])
    p.add_argument('--test_dir', required=True, help='the epoch*_test directory of batch%%04d.npz files the test driver wrote')
    p.add_argument('--slice_rows', default=None,
                   help='image rows a:b of the temporal slices (default 120:140, or the middle 20 rows when H < 140)')
    p.add_argument('--chunk', type=chunk_size, default=32, help='frames per device chunk')
    p.add_argument('--gpu', type=int, default=0)
    a = p.parse_args(argv)
    if a.slice_rows is not None and not re.fullmatch(r'\d+:\d+', a.slice_rows):
        p.error('--slice_rows must look like a:b, got %r' % a.slice_rows)
    return a


def main(argv=None):
    a = parse_args(argv)
    t0 = time.perf_counter()
    res = render_test_videos(a.test_dir, a.slice_rows, a.chunk, device=a.gpu)
    print('wrote %d comparison and RGB frames, %d temporal slices (rows %d:%d), %s in %.2f s'
          % (res['frames'], len(res['temporal_slice']), *res['slice_rows'], res['html'], time.perf_counter() - t0))
    return res


if __name__ == '__main__':
    main()
