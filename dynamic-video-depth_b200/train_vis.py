"""Training and validation pages, the reference's `--html_logger` output (visualize/html_visualizer.py, loggers/loggers.py:376-442).

`train --html_logger` sets `model.visualizer = PageWriter(full_logdir)` on rank 0. For every visualised pack the model passes
the device tensors of the pack, and this module writes, with the reference's names:

* `visualize/epoch%04d_{train,vali}/<key>_%04d_%04d.png` (batch index, pair) for every image key of the pack;
* `visualize/{train,val}_%05d.html`, one table per epoch whose header is the sorted image keys of the epoch's first pack and
  which has one row per pair, linking `epoch%04d_{train,vali}/<png>`;
* `summary.html` and `summary.json` in `full_logdir`: the epochs that have a page, `{'train': [...], 'val': [...]}`. An existing
  `summary.json` is read and extended (a resumed run).

Image keys follow the reference's KEYWORDS (first match wins, so `depth_image_1_2` is a depth). The images of one pack are
rendered on the GPU in two launches (`ops.vis_tiles`, csrc/train_vis.cu holds the rules and their dtypes) and come back in one
copy; the PNG files are encoded on a thread pool while training goes on. `flush()` (the end of every training epoch and of
every validation pass) and `close()` (the end of the run) wait for every outstanding write and raise the first failure.

Where this differs from the reference:

* non-finite data: a NaN reaching the depth colour map makes the reference's worker raise (its pool prints the error and the
  rest of the pack is not written); here that pixel is black and the pack is written in full;
* values outside [0, 255] after scaling are clipped before the conversion to uint8 (numpy's out-of-range cast is
  platform-defined);
* depth colours use OpenCV's 8-bit COLORMAP_TURBO over 255, not the reference's 5-decimal float table; the heat-map input,
  its index and its fraction are the reference's, so a colour differs by at most what the two tables differ by at the two
  entries it interpolates, plus one for the truncation;
* the flow angle is fp64 atan2 rounded to fp32 (the reference's numpy arctan2 is fp64), so that the result does not depend on
  the maths library; a flow colour channel may differ from the reference's by one;
* summary links are relative to `summary.html`, so the log directory can be moved.
"""
import json
import os
import re
from concurrent.futures import ThreadPoolExecutor
from os.path import join

import cv2
import numpy as np
import torch

from . import ops

# util/util_visualize.py's keyword order: the first keyword found in a key names its converter
KEYWORDS = ('depth', 'edgegradient', 'flow', 'img', 'rgb', 'image', 'edge', 'contour', 'softmask')
_KINDS = {'depth': 'depth', 'flow': 'flow', 'img': 'img', 'rgb': 'img', 'image': 'img'}
_FOLDER = re.compile(r'epoch(\d+)_(train|vali)')


def image_kind(key):
    """'depth', 'flow' or 'img' for an image key, None for a key that is not an image. A key whose first keyword has no renderer
    here (edges, contours, soft masks: no pack of this model has one) raises ValueError."""
    for k in KEYWORDS:
        if k in key:
            if k not in _KINDS:
                raise ValueError('image key %r (%s) has no renderer' % (key, k))
            return _KINDS[k]
    return None


def color_wheel():
    """[55,3] fp64 Middlebury flow colour wheel, RGB in 0..255: six ramps (red-yellow 15, yellow-green 6, green-cyan 4,
    cyan-blue 11, blue-magenta 13, magenta-red 6); along a ramp of n steps the changing channel takes floor(255 i / n)."""
    ramps = ((15, 0, 1, +1), (6, 1, 0, -1), (4, 1, 2, +1), (11, 2, 1, -1), (13, 2, 0, +1), (6, 0, 2, -1))
    rows = []
    for n, full, moving, sign in ramps:
        for i in range(n):
            c = [0.0, 0.0, 0.0]
            c[full] = 255.0
            step = np.floor(255 * i / n)
            c[moving] = step if sign > 0 else 255.0 - step
            rows.append(c)
    return np.array(rows, dtype=np.float64)


def turbo_table():
    """[256,3] fp64 RGB in [0, 1]: OpenCV's COLORMAP_TURBO over 255."""
    bgr = cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_TURBO)[:, 0]
    return bgr[:, ::-1].astype(np.float64) / 255.0


def png_name(key, batch_idx, b):
    return '%s_%04d_%04d.png' % (key, batch_idx, b)


def page_header(keys):
    return ''.join('<th>%s</th>\n' % k for k in keys)


def page_rows(keys, batch_idx, n, folder):
    out = ''
    for b in range(n):
        out += '<tr>\n'
        for k in keys:
            out += '<td><img src="%s" style="max-width:100%%;height:auto;"></td>\n' % join(folder, png_name(k, batch_idx, b))
        out += '</tr>\n'
    return out


_PAGE = """<!DOCTYPE html>
<html>
<head>
<meta charset="utf-8">
<title>{title}</title>
<style>
body {{ background: #000; color: #ccc; font-family: sans-serif; }}
table {{ border-collapse: collapse; }}
th, td {{ border: 1px solid #555; padding: 2px; text-align: center; }}
</style>
</head>
<body>
<h3>{title}</h3>
<table>
<thead>
<tr>
{header}</tr>
</thead>
<tbody>
{rows}</tbody>
</table>
</body>
</html>
"""

_SUMMARY = """<!DOCTYPE html>
<html>
<head>
<meta charset="utf-8">
<title>Training summary</title>
<style>
body {{ font-family: sans-serif; }}
table {{ border-collapse: collapse; display: inline-table; vertical-align: top; margin-right: 2em; font-size: x-large; }}
td {{ border: 1px solid #000; padding: 2px 12px; }}
</style>
</head>
<body>
<table><tr><td>Train</td></tr>
{train}</table>
<table><tr><td>Validation</td></tr>
{val}</table>
</body>
</html>
"""


def _write_png(path, rgb):
    if not cv2.imwrite(path, np.ascontiguousarray(rgb[..., ::-1])):
        raise RuntimeError('cv2.imwrite could not write %s' % path)


class PageWriter:
    """The model's `visualizer`: `visualize(pack, batch_idx, outdir)` renders a pack and queues its files; the page of an epoch
    is written by the `flush()` that follows it."""

    def __init__(self, full_logdir, workers=4):
        self.root = full_logdir
        self.summary = join(full_logdir, 'summary')
        if os.path.exists(self.summary + '.json'):
            with open(self.summary + '.json') as f:
                self.progress = json.load(f)
        else:
            self.progress = {'train': [], 'val': []}
        self.pool = ThreadPoolExecutor(max_workers=workers)
        self.futures = []
        self.page = None
        self._tables = None

    def _colour_tables(self, device):
        if self._tables is None or self._tables[0].device != device:
            self._tables = (torch.from_numpy(turbo_table()).to(device),
                            torch.from_numpy(np.ascontiguousarray(color_wheel() / 255)).to(device))
        return self._tables

    def visualize(self, pack, batch_idx, outdir):
        """pack: the reference's pack keys; the image keys hold CUDA tensors ([B,1,H,W] depths, [B,H,W,2] flows, [B,3,H,W]
        images). outdir: `.../visualize/epoch%04d_{train,vali}`, which names the page the rows go to."""
        folder = os.path.basename(os.path.normpath(outdir))
        m = _FOLDER.fullmatch(folder)
        if m is None:
            raise ValueError('outdir must end in epoch%%04d_train or epoch%%04d_vali, got %r' % outdir)
        page = ('train' if m.group(2) == 'train' else 'val', int(m.group(1)))
        if self.page is not None and self.page['id'] != page:
            self._write_page()
        keys = [k for k in sorted(pack) if image_kind(k) is not None]
        if not keys:
            return
        if self.page is None:
            self.page = {'id': page, 'header': page_header(keys), 'rows': ''}
        maps = []
        for k in keys:
            t = pack[k]
            maps.append((image_kind(k), t.permute(0, 3, 1, 2) if image_kind(k) == 'flow' else t))
        n = int(maps[0][1].shape[0])
        if any(int(t.shape[0]) != n for _, t in maps):
            raise ValueError('every image key of a pack holds the same number of images')
        tiles = ops.vis_tiles(maps, *self._colour_tables(maps[0][1].device)).cpu().numpy()
        self.page['rows'] += page_rows(keys, batch_idx, n, folder)
        os.makedirs(outdir, exist_ok=True)
        for q, k in enumerate(keys):
            for b in range(n):
                self.futures.append(self.pool.submit(_write_png, join(outdir, png_name(k, batch_idx, b)), tiles[q * n + b]))

    def _join(self):
        futures, self.futures = self.futures, []
        errors = [f.exception() for f in futures]
        errors = [e for e in errors if e is not None]
        if errors:
            raise errors[0]

    def _write_page(self):
        state, epoch = self.page['id']
        title = '%s epoch %d' % ('Training' if state == 'train' else 'Validation', epoch)
        os.makedirs(join(self.root, 'visualize'), exist_ok=True)
        with open(join(self.root, 'visualize', '%s_%05d.html' % (state, epoch)), 'w') as f:
            f.write(_PAGE.format(title=title, header=self.page['header'], rows=self.page['rows']))
        self.page = None
        self.progress[state].append(epoch)
        with open(self.summary + '.json', 'w') as f:
            json.dump(self.progress, f)
        entry = '<tr><td><a href="visualize/{0}_{1:05d}.html">{1:05d}</a></td></tr>\n'
        with open(self.summary + '.html', 'w') as f:
            f.write(_SUMMARY.format(train=''.join(entry.format('train', e) for e in self.progress['train']),
                                    val=''.join(entry.format('val', e) for e in self.progress['val'])))

    def flush(self):
        """Wait for every queued PNG (raising the first failure) and write the open epoch page and the summary."""
        self._join()
        if self.page is not None:
            self._write_page()

    def close(self):
        try:
            self.flush()
        finally:
            self.pool.shutdown(wait=True)
