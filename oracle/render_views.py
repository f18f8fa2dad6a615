"""TEST INFRASTRUCTURE — CPU oracle, not product code.

numpy restatement of the novel-view renderer (dvd_b200/render_views.py, csrc/render_views.cu): the camera paths in fp64, the
world-to-camera blocks, the float32 projection with the kernel's operation order (numpy rounds every element-wise operation
on its own, so no FMA contraction), the splat footprint, the per-pixel key minimum (np.minimum.at, which applies the
candidates in index order; the minimum does not depend on it) and the resolve.
"""
import numpy as np

from . import points as opoints

F32 = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


# ---- camera paths ------------------------------------------------------------------------------------------------------------
def median_depth(depth):
    d = np.asarray(depth, dtype=np.float32)
    return float(np.median(d[np.isfinite(d) & (d > F32(1e-2))]))


def lock_path(K, c2w, j):
    """every view gets the camera of selected frame j"""
    N = K.shape[0]
    return np.repeat(np.asarray(K, F32)[j:j + 1], N, 0), np.repeat(np.asarray(c2w, F32)[j:j + 1, :3], N, 0)


def wiggle_path(K, c2w, frame_ids, amplitude, period, median):
    """c(t) + R(t) (a m cos phi, a m sin phi, 0) in fp64, phi = 2 pi t / period, rounded to fp32; K(t)"""
    out = []
    for c, t in zip(np.asarray(c2w, np.float64)[:, :3], frame_ids):
        phi = 2 * np.pi * float(t) / float(period)
        o = np.array([amplitude * median * np.cos(phi), amplitude * median * np.sin(phi), 0.0])
        m = c.copy()
        m[:, 3] = c[:, 3] + c[:, :3] @ o
        out.append(m)
    return np.asarray(K, F32).copy(), np.asarray(out).astype(F32)


def w2c(c2w):
    """fp32 [3,4] c2w -> fp32 [3,4] (R^T | -R^T c), computed in fp64"""
    c = np.asarray(c2w, np.float64)
    Rt = c[:3, :3].T
    return np.concatenate([Rt, (-Rt @ c[:3, 3])[:, None]], 1).astype(F32)


# ---- projection, splat, resolve ----------------------------------------------------------------------------------------------
def project(xyz, Wc, K):
    """xyz [M,3] fp32, Wc [3,4] fp32, K [3,3] fp32 -> q2, u, v (fp32) and the mask of the points that are not dropped"""
    P = np.asarray(xyz, F32)
    Wc, K = np.asarray(Wc, F32), np.asarray(K, F32)
    with np.errstate(all='ignore'):
        q = [((Wc[i, 0] * P[:, 0] + Wc[i, 1] * P[:, 1]) + Wc[i, 2] * P[:, 2]) + Wc[i, 3] for i in range(3)]
        h = [(K[i, 0] * q[0] + K[i, 1] * q[1]) + K[i, 2] * q[2] for i in range(3)]
        u, v = h[0] / h[2], h[1] / h[2]
    ok = (q[2] > F32(1e-2)) & np.isfinite(q[0]) & np.isfinite(q[1]) & np.isfinite(q[2]) & np.isfinite(u) & np.isfinite(v)
    return q[2], u, v, ok


def splat(keys, xyz, idx, Wc, K, H, W, s):
    """min-accumulates the keys (bits(q2) << 32) | idx of the points into keys [H*W] uint64"""
    q2, u, v, ok = project(xyz, Wc, K)
    q2, u, v, idx = q2[ok], u[ok], v[ok], np.asarray(idx, np.uint64)[ok]
    key = (q2.view(np.uint32).astype(np.uint64) << np.uint64(32)) | idx
    with np.errstate(all='ignore'):
        xf = np.floor(u + F32(0.5)).astype(np.float64)
        yf = np.floor(v + F32(0.5)).astype(np.float64)
    half = (s - 1) // 2
    for dy in range(s):
        for dx in range(s):
            x, y = xf - half + dx, yf - half + dy
            m = (x >= 0) & (x < W) & (y >= 0) & (y < H)
            np.minimum.at(keys, (y[m] * W + x[m]).astype(np.int64), key[m])
    return keys


def resolve(keys, frame_rgb, static_rgb, H, W):
    """keys [H*W] -> BGR [H,W,3] uint8 and the covered pixel count; frame_rgb [H*W,3] uint8 the frame's colours per pixel,
    static_rgb [R,3] uint8 (or None)"""
    out = np.zeros((H * W, 3), np.uint8)
    hit = keys != EMPTY
    i = (keys[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    own = i < H * W
    c = np.empty((i.shape[0], 3), np.uint8)
    c[own] = frame_rgb[i[own]]
    if (~own).any():
        c[~own] = static_rgb[i[~own] - H * W]
    out[hit] = c[:, ::-1]
    return out.reshape(H, W, 3), int(hit.sum())


def static_cloud(fused):
    """the fused cloud of oracle.points.fuse as export_points writes it: fp32 positions, mean colours rounded half up"""
    return (np.asarray(fused['xyz'], np.float64).astype(F32),
            np.clip(np.floor(np.asarray(fused['rgb'], np.float64) + 0.5), 0, 255).astype(np.uint8))


def render(depth, img, P, vK, vc2w, splat_size=1, static=None, edge_tol=0.05):
    """The views of frames depth [N,H,W], img [N,3,H,W] with world points P [N,3,H,W] fp32 from the virtual cameras vK [N,3,3],
    vc2w [N,3,4]; static = (xyz [R,3] fp32, rgb [R,3] uint8) or None -> (views [N,H,W,3] BGR uint8, coverage [N])"""
    N, H, W = np.asarray(depth).shape
    HW = H * W
    if static is not None and HW + static[0].shape[0] >= 2 ** 32:
        raise ValueError('index overflow')
    if not 1 <= splat_size <= 4:
        raise ValueError('splat out of range')
    sel = opoints.select(depth, img, np.asarray(P, F32), edge_tol)
    f_of = sel['index'] // HW
    views, cov = np.zeros((N, H, W, 3), np.uint8), np.zeros(N, np.int64)
    for t in range(N):
        Wc, K = w2c(vc2w[t]), np.asarray(vK[t], F32)
        keys = np.full(HW, EMPTY, np.uint64)
        m = f_of == t
        splat(keys, sel['xyz'][m], sel['index'][m] - t * HW, Wc, K, H, W, splat_size)
        if static is not None and static[0].shape[0]:
            splat(keys, static[0], HW + np.arange(static[0].shape[0], dtype=np.uint64), Wc, K, H, W, splat_size)
        frame_rgb = opoints.colours(np.asarray(img[t], F32).reshape(3, HW).T)
        views[t], cov[t] = resolve(keys, frame_rgb, None if static is None else static[1], H, W)
    return views, cov
