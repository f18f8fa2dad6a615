"""TEST INFRASTRUCTURE — numpy restatement of the scene-flow kernels of csrc/tracks.cu (dvd_b200.tracks), bit for bit.

pair_sums_sf: dvd_pair_consistency_sf. The per-pixel terms are oracle.evaluate's with the scene flow added to the world point
after it is formed (numpy rounds every elementwise operation on its own, as the kernel does), and the sums follow the kernel's
fixed order: each of P * 256 threads adds its pixels in index order, a warp adds its lanes by the xor tree, a block its warps in
order, and the blocks of a pair are added in order.

draw: dvd_draw_tracks. The projection is oracle.render_views.project; candidates are min-accumulated with np.minimum.at, in
an order that may be shuffled (the minimum does not depend on it).
"""
import numpy as np

from .evaluate import _cam, _dot3, valid
from .render_views import project

F32 = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
THREADS, MAX_PARTS, PIXELS_PER_THREAD = 256, 128, 8
HIDE_TOL, HEAD_RADIUS, MAX_SAMPLES = F32(1.05), 1, 1024


# ---- consistency with the scene flow ------------------------------------------------------------------------------------------
def parts_for(hw):
    return int(min(max((hw + THREADS * PIXELS_PER_THREAD - 1) // (THREADS * PIXELS_PER_THREAD), 1), MAX_PARTS))


def fixed_sum(v):
    """v [..., hw] fp64 (0 where a pixel adds nothing) -> [...] summed in the kernels' order"""
    v = np.asarray(v, np.float64)
    hw = v.shape[-1]
    P = parts_for(hw)
    T = P * THREADS
    rows = -(-hw // T)
    pad = np.zeros(v.shape[:-1] + (rows * T,))
    pad[..., :hw] = v
    pad = pad.reshape(v.shape[:-1] + (rows, T))
    acc = np.zeros(v.shape[:-1] + (T,))
    for r in range(rows):                                    # a thread's pixels in index order
        acc = acc + pad[..., r, :]
    lanes = acc.reshape(v.shape[:-1] + (P, THREADS // 32, 32))
    for o in (16, 8, 4, 2, 1):                               # the warp's xor tree: lane l < o takes l + o
        lanes = lanes[..., :o] + lanes[..., o:2 * o]
    warps = lanes[..., 0]
    blocks = np.zeros(v.shape[:-1] + (P,))
    for w in range(THREADS // 32):
        blocks = blocks + warps[..., w]
    out = np.zeros(v.shape[:-1])
    for p in range(P):
        out = out + blocks[..., p]
    return out


def pair_terms_sf(Da, Db, cam_a, cam_b, flow, mask, sf=None):
    """oracle.evaluate.pair_terms with the scene flow sf [3,H,W] fp32 (None: none) added in fp64 to the world point P after it
    is formed: `eval`, `behind`, `good` masks and e_r, e_d, z (NaN where they do not apply)"""
    Da, Db = np.asarray(Da, F32), np.asarray(Db, F32)
    H, W = Da.shape
    flow = np.asarray(flow, F32)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    qx, qy = x + flow[..., 0].astype(np.float64), y + flow[..., 1].astype(np.float64)
    fin = np.isfinite(qx) & np.isfinite(qy)
    qxs, qys = np.where(fin, qx, 0.0), np.where(fin, qy, 0.0)
    ix, iy = np.minimum(np.maximum(qxs, 0.0), W - 1.0), np.minimum(np.maximum(qys, 0.0), H - 1.0)
    x0f, y0f = np.floor(ix), np.floor(iy)
    x0, y0 = x0f.astype(np.int64), y0f.astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    wx1, wy1 = ix - x0f, iy - y0f
    wx0, wy0 = 1.0 - wx1, 1.0 - wy1
    t00, t01, t10, t11 = Db[y0, x0], Db[y0, x1], Db[y1, x0], Db[y1, x1]
    ev = (np.asarray(mask) == 0) & fin & valid(Da) & valid(t00) & valid(t01) & valid(t10) & valid(t11)
    db = (((wy0 * wx0) * t00.astype(np.float64) + (wy0 * wx1) * t01.astype(np.float64)) + (wy1 * wx0) * t10.astype(np.float64)) \
        + (wy1 * wx1) * t11.astype(np.float64)
    Ka, Kia, Ra, ta = _cam(cam_a)
    Kb, _, Rb, tb = _cam(cam_b)
    da = Da.astype(np.float64)
    with np.errstate(all='ignore'):
        cv = [da * _dot3(Kia[r], x, y, 1.0) for r in range(3)]
        P = [_dot3(Ra[r], *cv) + ta[r] for r in range(3)]
        if sf is not None:
            sf = np.asarray(sf, F32)
            P = [P[r] + sf[r].astype(np.float64) for r in range(3)]
        pw = [P[r] - tb[r] for r in range(3)]
        c = [_dot3(Rb[:, r], *pw) for r in range(3)]
        z = c[2]
        behind = ev & ~(z > 1e-3)
        good = ev & (z > 1e-3)
        px, py = _dot3(Kb[0], *c) / z, _dot3(Kb[1], *c) / z
        ex, ey = px - qx, py - qy
        er = np.sqrt(ex * ex + ey * ey)
        ed = np.abs(z - db) / db
    nan = np.full((H, W), np.nan)
    return {'eval': ev, 'behind': behind, 'good': good, 'e_r': np.where(good, er, nan), 'e_d': np.where(good, ed, nan),
            'z': np.where(ev, z, nan)}


def region_sums(t, sel):
    """the six sums of one pair's terms t over the pixels `sel` [H,W] bool, in the kernel's order"""
    g, b = (t['good'] & sel).reshape(-1), (t['behind'] & sel).reshape(-1)
    er, ed = np.where(g, t['e_r'].reshape(-1), 0.0), np.where(g, t['e_d'].reshape(-1), 0.0)
    terms = np.stack([g.astype(np.float64), b.astype(np.float64), er, ed, (g & (er < 1.0)).astype(np.float64),
                      (g & (er < 3.0)).astype(np.float64)])
    return fixed_sum(terms)


def pair_sums_sf(depth, cam, ia, ib, flow, mask, sf, motion_seg=None):
    """dvd_pair_consistency_sf -> sums [P,3,6] fp64 (regions all, static, moving), bit for bit"""
    P = len(ia)
    out = np.zeros((P, 3, 6))
    for p in range(P):
        a, b = int(ia[p]), int(ib[p])
        t = pair_terms_sf(depth[a], depth[b], cam[a], cam[b], flow[p], mask[p], None if sf is None else sf[p])
        out[p, 0] = region_sums(t, np.ones_like(t['good']))
        if motion_seg is not None:
            moving = np.asarray(motion_seg[a]) != 0
            out[p, 1] = region_sums(t, ~moving)
            out[p, 2] = region_sums(t, moving)
    return out


# ---- drawing ------------------------------------------------------------------------------------------------------------------
def _project(cam, xyz):
    cam = np.asarray(cam, F32)
    z, u, v, ok = project(np.asarray(xyz, F32).reshape(-1, 3), cam[:12].reshape(3, 4), cam[12:].reshape(3, 3))
    return u, v, z, ok


def _pixel(u):
    with np.errstate(all='ignore'):
        return np.floor(np.asarray(u, F32) + F32(0.5))


def _plot(D, H, W, xf, yf, z, dx=0, dy=0):
    """(pixel index, plotted) of samples at (xf + dx, yf + dy) with depth z: in the image and not hidden"""
    x, y = xf.astype(np.float64) + dx, yf.astype(np.float64) + dy
    inside = (x >= 0) & (x <= W - 1) & (y >= 0) & (y <= H - 1)
    o = np.where(inside, np.where(inside, y, 0) * W + np.where(inside, x, 0), 0).astype(np.int64)
    d = np.asarray(D, F32).reshape(-1)[o]
    with np.errstate(all='ignore'):
        hidden = valid(d) & (np.asarray(z, F32) > d * HIDE_TOL)
    return o, inside & ~hidden


def draw(X, first, length, rgb, cams, depth, img, number, tail, rng=None):
    """dvd_draw_tracks -> (out [F,H,W,3] uint8 BGR, proj [M,L1,3] fp32, vis [M,L1] uint8; NaN / 0 where no frame drew the
    step). rng: a numpy Generator that shuffles the order in which each frame's candidates are applied."""
    X = np.asarray(X, F32)
    M, L1 = X.shape[:2]
    depth = np.asarray(depth, F32)
    F, H, W = depth.shape
    first, length = np.asarray(first, np.int64), np.asarray(length, np.int64)
    rgb = np.asarray(rgb, np.uint8)
    proj = np.full((M, L1, 3), np.nan, F32)
    vis = np.zeros((M, L1), np.uint8)
    out = np.empty((F, H, W, 3), np.uint8)
    with np.errstate(invalid='ignore'):
        base = (np.minimum(np.fmax(np.asarray(img, F32), F32(0)), F32(1)) * F32(255)).astype(np.uint8)
    for f in range(F):
        keys = np.full(H * W, EMPTY, np.uint64)
        k = int(number[f]) - first
        alive = np.nonzero((k >= 0) & (k < length))[0]
        ka = k[alive]
        pix, key = [], []
        u, v, z, ok = _project(cams[f], X[alive, ka])
        xf, yf = _pixel(u), _pixel(v)
        for dy in range(-HEAD_RADIUS, HEAD_RADIUS + 1):
            for dx in range(-HEAD_RADIUS, HEAD_RADIUS + 1):
                o, hit = _plot(depth[f], H, W, xf, yf, z, dx, dy)
                hit &= ok
                pix.append(o[hit])
                key.append(alive[hit].astype(np.uint64))
                if dx == 0 and dy == 0:
                    vis[alive, ka] = hit
        proj[alive, ka] = np.where(ok[:, None], np.stack([u, v, z], 1), F32(np.nan))
        for r in range(1, tail + 1):
            sel = ka >= r
            i, j = alive[sel], ka[sel] - r
            u0, v0, z0, ok0 = _project(cams[f], X[i, j])
            u1, v1, z1, ok1 = _project(cams[f], X[i, j + 1])
            good = ok0 & ok1
            i, u0, v0, z0, u1, v1, z1 = i[good], u0[good], v0[good], z0[good], u1[good], v1[good], z1[good]
            du, dv, dz = u1 - u0, v1 - v0, z1 - z0
            with np.errstate(all='ignore'):
                n = np.fmin(np.ceil(np.fmax(np.abs(du), np.abs(dv))), F32(MAX_SAMPLES))
            S = np.where(n >= 1, np.where(n >= 1, n, 1), 1).astype(np.int64)
            rep = np.repeat(np.arange(len(i)), S + 1)
            s = np.arange(rep.shape[0]) - np.repeat(np.cumsum(S + 1) - (S + 1), S + 1)
            t = s.astype(F32) / S[rep].astype(F32)
            us, vs, zs = u0[rep] + t * du[rep], v0[rep] + t * dv[rep], z0[rep] + t * dz[rep]
            o, hit = _plot(depth[f], H, W, _pixel(us), _pixel(vs), zs)
            pix.append(o[hit])
            key.append((np.uint64(r) << np.uint64(32)) | i[rep][hit].astype(np.uint64))
        pix, key = np.concatenate(pix), np.concatenate(key)
        if rng is not None:
            perm = rng.permutation(pix.shape[0])
            pix, key = pix[perm], key[perm]
        np.minimum.at(keys, pix, key)
        b = base[f].reshape(3, -1).T.astype(np.int64)                  # [HW, 3] RGB
        o = b.copy()
        hit = keys != EMPTY
        rank = (keys[hit] >> np.uint64(32)).astype(np.int64)
        c = rgb[(keys[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)].astype(np.int64)
        w = (256 * (tail + 1 - rank) // (tail + 1))[:, None]
        o[hit] = (c * w + b[hit] * (256 - w) + 128) >> 8
        out[f] = o[:, ::-1].reshape(H, W, 3).astype(np.uint8)
    return out, proj, vis
