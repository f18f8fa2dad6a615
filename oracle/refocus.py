"""TEST INFRASTRUCTURE — CPU oracle, not product code.

numpy restatement of the synthetic depth of field (dvd_b200/refocus.py, csrc/refocus.cu): the focal disparities in fp64
rounded to fp32, and the gather rule in float32 with the kernel's operation order. numpy rounds every element-wise float32
operation on its own, so nothing is contracted. The taps are walked in the rule's order, every one of them, with no early
exit: a tap whose q lies outside the image is skipped by giving it weight 0 and colour 0, which adds +0 to every sum.
"""
import numpy as np

F32 = np.float32


def disparity(depth):
    """fp32 1/d where d is finite and > 1e-2, else 0"""
    d = np.asarray(depth, F32)
    ok = np.isfinite(d) & (d > F32(1e-2))
    with np.errstate(all='ignore'):
        return np.where(ok, F32(1) / np.where(ok, d, F32(1)), F32(0)).astype(F32)


def colours(img):
    """clip(img, 0, 1) in fp32 with NaN -> 0"""
    return np.minimum(np.fmax(np.asarray(img, F32), F32(0)), F32(1))


def blur_radius(disp, phi, scale, R):
    """min(R, scale |disp - phi|) in fp32 (fmin: a NaN product gives R, as fminf does)"""
    return np.fmin(F32(R), F32(scale) * np.abs(disp - F32(phi)))


def taps(R):
    """the (dy, dx) offsets with dx^2 + dy^2 <= R^2, dy ascending then dx"""
    return [(dy, dx) for dy in range(-R, R + 1) for dx in range(-R, R + 1) if dx * dx + dy * dy <= R * R]


def median_valid(depth):
    d = np.asarray(depth, F32)
    v = d[np.isfinite(d) & (d > F32(1e-2))]
    if v.size == 0:
        raise ValueError('no valid depth')
    return float(np.median(v))


def focus_point(depth, x, y, k, m):
    """per frame 1 / median of the valid depths in the (2k+1)^2 window at (x, y), clipped to the image, in fp64 rounded to
    fp32; a frame without one keeps the previous frame's value, the first falls back to 1 / m"""
    depth = np.asarray(depth, F32)
    N, H, W = depth.shape
    out, prev = np.empty(N, F32), 1.0 / m
    for t in range(N):
        win = depth[t, max(y - k, 0):min(y + k + 1, H), max(x - k, 0):min(x + k + 1, W)].astype(np.float64).ravel()
        win = win[np.isfinite(win) & (win > np.float64(F32(1e-2)))]
        if win.size:
            prev = 1.0 / float(np.median(win))
        out[t] = F32(prev)
    return out


def focus_depth(N, z, m):
    return np.full(N, F32(1.0 / (z * m)), F32)


def focus_pull(N, a, b, m):
    p0, p1 = 1.0 / (a * m), 1.0 / (b * m)
    t = np.arange(N, dtype=np.float64) / max(N - 1, 1)
    return (p0 + (p1 - p0) * t).astype(F32)


def render_frame(depth, img, phi, scale, R):
    """one frame: depth [H,W], img [3,H,W] fp32 RGB -> BGR [H,W,3] uint8"""
    H, W = np.asarray(depth).shape
    disp = disparity(depth)
    c = blur_radius(disp, phi, scale, R)
    col = colours(img)
    # pad by R: outside the image the weight is forced to 0 and the colour is 0
    P = lambda a: np.pad(a, ((R, R), (R, R)))
    dpad, cpad, inside = P(disp), P(c), P(np.ones((H, W), bool))
    colpad = [P(col[k]) for k in range(3)]
    S = [np.zeros((H, W), F32) for _ in range(3)]
    Wt = np.zeros((H, W), F32)
    for dy, dx in taps(R):
        sl = (slice(R + dy, R + dy + H), slice(R + dx, R + dx + W))
        dq, cq = dpad[sl], cpad[sl]
        ce = np.where(dq < disp, np.minimum(cq, c), cq)
        r = np.sqrt(F32(dx * dx + dy * dy))
        cov = np.minimum(np.maximum((ce - r) + F32(0.5), F32(0)), F32(1))
        w = np.where(inside[sl], cov / np.maximum(ce * ce, F32(0.25)), F32(0))
        for k in range(3):
            S[k] = S[k] + w * colpad[k][sl]
        Wt = Wt + w
    out = [np.minimum(np.floor(F32(255) * (S[k] / Wt)), F32(255)).astype(np.uint8) for k in (2, 1, 0)]
    return np.stack(out, -1)


def render(depth, img, phi, scale, R):
    """frames depth [N,H,W], img [N,3,H,W], focal disparities phi [N] -> BGR [N,H,W,3] uint8"""
    return np.stack([render_frame(depth[t], img[t], phi[t], scale, R) for t in range(np.asarray(depth).shape[0])])
