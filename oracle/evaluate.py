"""TEST INFRASTRUCTURE — numpy fp64 restatement of the evaluation kernels (csrc/depth_metrics.cu, dvd_b200.evaluate).

Every per-pixel term is formed with the operations, in the order, that include/dvd_b200.h states for dvd_masked_select,
dvd_depth_metrics and dvd_pair_consistency; numpy rounds each elementwise operation on its own, as the kernels do, so the
terms agree bit for bit (ln aside, which both sides round to within an ulp). The sums here are numpy's, in another order
than the kernels' fixed one.
"""
import numpy as np

F32 = np.float32
DELTAS = (1.25, 1.25 ** 2, 1.25 ** 3)


def valid(a):
    """finite and > 1e-2 (compared in fp32, as depth2disp does)"""
    a = np.asarray(a, dtype=F32)
    return np.isfinite(a) & (a > F32(1e-2))


def lower_median(x):
    """the element of 0-based rank (n - 1) // 2 of a 1-d array, NaN when it is empty"""
    x = np.asarray(x).reshape(-1)
    if x.size == 0:
        return np.float32(np.nan)
    k = (x.size - 1) // 2
    return np.partition(x, k)[k]


def masked_select_median(values, other=None):
    """dvd_masked_select: values [N,H,W] fp32 -> (median [N+1] fp32, count [N+1] int64), per frame and then pooled"""
    v = np.asarray(values, dtype=F32)
    ok = valid(v) if other is None else valid(v) & valid(other)
    med = [lower_median(v[n][ok[n]]) for n in range(v.shape[0])] + [lower_median(v[ok])]
    cnt = [int(ok[n].sum()) for n in range(v.shape[0])] + [int(ok.sum())]
    return np.asarray(med, dtype=F32), np.asarray(cnt, dtype=np.int64)


def accuracy_terms(d, g, s):
    """per-pixel terms of one frame and source at scale s (fp64): a dict of arrays over the valid pixels (g, d valid), with
    d' = s d: abs_rel, sq_rel, sq, sq_log, ratio = max(d'/g, g/d')"""
    d, g = np.asarray(d, F32), np.asarray(g, F32)
    ok = valid(d) & valid(g)
    dv, gv = d[ok].astype(np.float64), g[ok].astype(np.float64)
    dp = np.float64(s) * dv
    diff = dp - gv
    sq = diff * diff
    lgd = np.log(dp) - np.log(gv)
    return {'abs_rel': np.abs(diff) / gv, 'sq_rel': sq / gv, 'sq': sq, 'sq_log': lgd * lgd,
            'ratio': np.maximum(dp / gv, gv / dp)}


def accuracy_sums(depth, depth_nn, depth_gt, scales):
    """dvd_depth_metrics: [N,H,W] fp32 maps and scales [N,2,3] -> sums [N,2,22] fp64"""
    N = np.asarray(depth).shape[0]
    out = np.zeros((N, 2, 22))
    for n in range(N):
        for j, d in enumerate((depth, depth_nn)):
            for a in range(3):
                t = accuracy_terms(d[n], depth_gt[n], scales[n][j][a])
                out[n, j, 0] = t['sq'].size
                out[n, j, 1 + 7 * a:5 + 7 * a] = [t['abs_rel'].sum(), t['sq_rel'].sum(), t['sq'].sum(), t['sq_log'].sum()]
                out[n, j, 5 + 7 * a:8 + 7 * a] = [(t['ratio'] < th).sum() for th in DELTAS]
    return out


def _cam(c):
    """camera_block row [30] -> K, Kinv, R [3,3], t [3] in fp64"""
    c = np.asarray(c, F32).astype(np.float64)
    return c[0:9].reshape(3, 3).T, c[9:18].reshape(3, 3).T, c[18:27].reshape(3, 3), c[27:30]


def _dot3(row, x, y, z):
    return (row[0] * x + row[1] * y) + row[2] * z


def pair_terms(Da, Db, cam_a, cam_b, flow, mask):
    """per-pixel terms of one pair and one depth source: a dict of [H,W] arrays: `eval` (evaluated), `behind`, and where
    evaluated and not behind: e_r, e_d, z (fp64); NaN elsewhere"""
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
        pw = [(_dot3(Ra[r], *cv) + ta[r]) - tb[r] for r in range(3)]
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


def pair_sums(depth, depth_nn, cam, ia, ib, flow, mask, motion_seg=None):
    """dvd_pair_consistency: -> sums [P,2,2,6] fp64 (count, behind, sum e_r, sum e_d, #e_r < 1, #e_r < 3)"""
    P = len(ia)
    out = np.zeros((P, 2, 2, 6))
    for p in range(P):
        a, b = int(ia[p]), int(ib[p])
        stat = None if motion_seg is None else (np.asarray(motion_seg[a]) == 0)
        for j, D in enumerate((depth, depth_nn)):
            t = pair_terms(D[a], D[b], cam[a], cam[b], flow[p], mask[p])
            for r, region in enumerate((None, stat)):
                if r == 1 and stat is None:
                    continue
                sel = np.ones_like(t['good']) if region is None else region
                g, er = t['good'] & sel, t['e_r']
                out[p, j, r] = [g.sum(), (t['behind'] & sel).sum(), er[g].sum(), t['e_d'][g].sum(), (er[g] < 1.0).sum(),
                                (er[g] < 3.0).sum()]
    return out
