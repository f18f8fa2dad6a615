"""TEST INFRASTRUCTURE — CPU oracle, not product code.

numpy restatement of the test-end canvases (dvd_b200/test_videos.py, csrc/test_videos.cu): the disparity transforms, the
ranges, matplotlib's colour-index rule, the look-up in OpenCV's turbo table, the templates and the panel geometry.

The reference's own `on_test_end` cannot run here (it needs matplotlib and ffmpeg), and its figure layout is not reproduced,
so there is no fixture: the canvases are pinned by this restatement.
"""
import cv2
import numpy as np

MARGIN, TITLE_H, BAR_GAP, BAR_W, LABEL_GAP, LABEL_W, BAR_MIN_H = 8, 32, 6, 14, 4, 72, 48


def turbo_lut():
    """[256,3] uint8 BGR, cv2.COLORMAP_TURBO."""
    return cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_TURBO)[:, 0].copy()


def disp(depth):
    """The reference's `1 / depth` on float32 data: float32 (numpy 2 / NEP 50: a Python int is a weak scalar)."""
    with np.errstate(divide='ignore', invalid='ignore'):
        return 1 / np.asarray(depth, dtype=np.float32)


def gt_disp(gt):
    """The reference's `np.where(gt > 1e-8, 1, 0) / (gt + 1e-8)` on float32 data, evaluated as numpy 2 does it (NEP 50): the
    Python float 1e-8 is a weak scalar, so `gt > 1e-8` and `gt + 1e-8` are float32 operations with 1e-8 cast to float32; the
    np.where gives int64, and int64 / float32 promotes both operands to float64 (np.result_type(np.int64, np.float32))."""
    gt = np.asarray(gt, dtype=np.float32)
    with np.errstate(divide='ignore', invalid='ignore'):
        v = np.where(gt > 1e-8, 1, 0) / (gt + 1e-8)
    assert v.dtype == np.float64
    return v


def rgb_u8(img):
    """floor(255 · clip(img, 0, 1)) in float32, NaN -> 0."""
    x = np.clip(np.nan_to_num(np.asarray(img, dtype=np.float32), nan=0.0), np.float32(0), np.float32(1))
    return np.floor(x * np.float32(255)).astype(np.uint8)


def cmap_index(v, vmin, vmax):
    """matplotlib's Colormap.__call__ with N = 256 after Normalize(vmin, vmax) in fp64: t = (v - vmin) / (vmax - vmin), index
    floor(256 t), t >= 1 -> 255 (over = last colour), t < 0 -> 0 (under = first colour), vmax == vmin -> 0 (Normalize gives 0);
    NaN v or t -> -1 (matplotlib's transparent "bad" colour, black on the black figure)."""
    v = np.asarray(v, dtype=np.float64)
    lo, hi = np.float64(vmin), np.float64(vmax)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        t = (v - lo) / (hi - lo)
        f = np.floor(np.nan_to_num(t, nan=0.0, posinf=0.0, neginf=0.0) * 256.0)
    return np.select([np.isnan(v), np.full(v.shape, hi == lo), np.isnan(t), t >= 1, t < 0], [-1, 0, -1, 255, 0], f).astype(np.int64)


def colour(v, vmin, vmax, lut):
    """[..., 3] uint8 BGR of v through the index rule and the table; index -1 is black."""
    i = cmap_index(v, vmin, vmax)
    out = lut[np.maximum(i, 0)].copy()
    out[i < 0] = 0
    return out


def global_range(depth):
    """(vmin, vmax) = (1 / max, 1 / min) of the refined depth of all frames, float32 scalars."""
    d = np.asarray(depth, dtype=np.float32)
    return 1 / d.max(), 1 / d.min()


def slice_range(v):
    """min and max of the finite values (matplotlib's autoscale masks the invalid ones); (0, 0) when there is none."""
    f = v[np.isfinite(v)]
    return (f.min(), f.max()) if f.size else (np.float32(0), np.float32(0))


def default_slice_rows(H):
    if H >= 140:
        return 120, 140
    k = min(20, H)
    return (H - k) // 2, (H - k) // 2 + k


def layout(k, h, w):
    bh = max(h, BAR_MIN_H)
    block = w + BAR_GAP + BAR_W + LABEL_GAP + LABEL_W
    CW, CH = MARGIN + k * (block + MARGIN), TITLE_H + bh + MARGIN
    CW, CH = -(-CW // 4) * 4, -(-CH // 2) * 2
    return CH, CW, [(TITLE_H, MARGIN + p * (block + MARGIN)) for p in range(k)]


def template(titles, h, w, ranges, lut):
    CH, CW, pos = layout(len(titles), h, w)
    t = np.zeros((CH, CW, 3), np.uint8)
    bh = max(h, BAR_MIN_H)
    font, white = cv2.FONT_HERSHEY_SIMPLEX, (255, 255, 255)
    for title, (y0, x0), (lo, hi) in zip(titles, pos, ranges):
        tw = cv2.getTextSize(title, font, 0.6, 1)[0][0]
        cv2.putText(t, title, (x0 + max((w - tw) // 2, 0), TITLE_H - 10), font, 0.6, white, 1, cv2.LINE_8)
        bx = x0 + w + BAR_GAP
        for r in range(bh):                                     # top row = index 255, bottom row = index 0
            t[y0 + r, bx:bx + BAR_W] = lut[255 * (bh - 1 - r) // (bh - 1)]
        cv2.putText(t, '%.3g' % float(hi), (bx + BAR_W + LABEL_GAP, y0 + 10), font, 0.4, white, 1, cv2.LINE_8)
        cv2.putText(t, '%.3g' % float(lo), (bx + BAR_W + LABEL_GAP, y0 + bh - 1), font, 0.4, white, 1, cv2.LINE_8)
    return t


def compare_canvases(depth, depth_nn, depth_gt, lut, rng=None):
    """[N,CH,CW,3] uint8: Refined, Initial and GT disparity of each frame over the global range (depth* [N,1,H,W])."""
    N, _, H, W = depth.shape
    lo, hi = global_range(depth) if rng is None else rng
    t = template(('Refined', 'Initial', 'GT'), H, W, [(lo, hi)] * 3, lut)
    out = np.broadcast_to(t, (N,) + t.shape).copy()
    _, _, pos = layout(3, H, W)
    for v, (y0, x0) in zip((disp(depth[:, 0]), disp(depth_nn[:, 0]), gt_disp(depth_gt[:, 0])), pos):
        out[:, y0:y0 + H, x0:x0 + W] = colour(v, lo, hi, lut)
    return out


def rgb_canvases(img):
    """[N,H,W,3] uint8 BGR of img [N,3,H,W]."""
    return rgb_u8(img)[:, ::-1].transpose(0, 2, 3, 1).copy()


def slice_canvases(depth, depth_nn, rows, lut):
    """[S,CH,CW,3] uint8: for each image row r of rows (a, b), the Refined and Initial disparity of row r of every frame
    (canvas row = frame), each over the finite range of its own values."""
    N, _, H, W = depth.shape
    a, b = rows
    _, _, pos = layout(2, N, W)
    out = []
    for r in range(a, b):
        vs = [disp(depth[:, 0, r]), disp(depth_nn[:, 0, r])]
        rngs = [slice_range(v) for v in vs]
        c = template(('Refined', 'Initial'), N, W, rngs, lut)
        for v, (lo, hi), (y0, x0) in zip(vs, rngs, pos):
            c[y0:y0 + N, x0:x0 + W] = colour(v, lo, hi, lut)
        out.append(c)
    return np.stack(out)

