"""numpy restatement of the training-page images (csrc/train_vis.cu): util/util_visualize.py's depth and image converters,
third_party/util_colormap.py's heatmap_to_pseudo_color and util/util_flow.py's flow2img, in numpy 2's dtypes, with the
project's three deviations (non-finite depth colours black, bytes clipped before the uint8 conversion, the flow angle fp64
arctan2 rounded to fp32). The tables are parameters, so the reference's own turbo table can be fed in."""
import numpy as np

EPS64 = np.finfo(float).eps


def _bytes(v):
    """clip to [0, 255] (NaN -> 0), then truncate to uint8"""
    v = np.clip(v, 0, 255)
    return np.where(np.isnan(v), 0, v).astype(np.uint8)


def depth_heat(d):
    """[H,W] fp32 depth -> the heat-map input x of heatmap_to_pseudo_color (fp32, before its clip)"""
    d = np.asarray(d, dtype=np.float32)
    t = 1 / (d + 1e-6)
    return (t - np.min(t)) / (np.max(t) - np.min(t) + 1e-6)


def depth_image(d, turbo):
    """[H,W] fp32 depth -> [H,W,3] uint8 through the [256,3] fp64 table `turbo`"""
    h = depth_heat(d)
    x = h.clip(0, 1)
    p = x * 255                                       # fp32
    bad = np.isnan(p)
    a = np.where(bad, 0, p).astype(np.int64)
    b = np.minimum(a + 1, 255)
    f = np.where(bad, 0, p) - a                       # fp32 - int64 -> fp64
    c = turbo[a] + (turbo[b] - turbo[a]) * f[..., None]
    c[h < 0.0] = 0.0
    c[h > 1.0] = 1.0
    c[bad] = 0.0
    return _bytes(c * 255)


def flow_image(flow, wheel):
    """[H,W,2] fp32 flow -> [H,W,3] uint8; wheel: [55,3] fp64 in 0..255"""
    u = np.array(flow[..., 0], dtype=np.float32)
    v = np.array(flow[..., 1], dtype=np.float32)
    unknown = (abs(u) > 1e7) | (abs(v) > 1e7)
    u[unknown] = v[unknown] = 0
    rad = np.sqrt(u ** 2 + v ** 2)
    maxrad = np.max(rad)
    maxrad = np.float32(-1) if np.isnan(maxrad) else maxrad
    U = (u / maxrad).astype(np.float64) + EPS64
    V = (v / maxrad).astype(np.float64) + EPS64
    bad = np.isnan(U) | np.isnan(V)
    U[bad] = V[bad] = 0
    r = np.sqrt(U ** 2 + V ** 2)
    r = np.where(r > 1, 1, r)
    ang = np.arctan2(-V, -U).astype(np.float32).astype(np.float64)
    fk = (ang / np.pi + 1) / 2 * (len(wheel) - 1) + 1
    k0 = np.floor(fk).astype(np.int64)
    k1 = k0 + 1
    k1[k1 == len(wheel) + 1] = 1
    f = fk - k0
    img = np.zeros(u.shape + (3,))
    for i in range(3):
        col0 = wheel[k0 - 1, i] / 255
        col1 = wheel[k1 - 1, i] / 255
        col = (1 - f) * col0 + f * col1
        col = np.where(r <= 1, 1 - r * (1 - col), col * 0.75)
        img[..., i] = np.floor(255 * col * (1 - bad))
    img[unknown] = 0
    return _bytes(img / 255 * 255)


def fk_of(flow):
    """the fp64 wheel position fk of every pixel of a [H,W,2] flow, as flow_image computes it"""
    u = np.array(flow[..., 0], dtype=np.float32)
    v = np.array(flow[..., 1], dtype=np.float32)
    unknown = (abs(u) > 1e7) | (abs(v) > 1e7)
    u[unknown] = v[unknown] = 0
    maxrad = np.max(np.sqrt(u ** 2 + v ** 2))
    maxrad = np.float32(-1) if np.isnan(maxrad) else maxrad
    U = (u / maxrad).astype(np.float64) + EPS64
    V = (v / maxrad).astype(np.float64) + EPS64
    bad = np.isnan(U) | np.isnan(V)
    U[bad] = V[bad] = 0
    ang = np.arctan2(-V, -U).astype(np.float32).astype(np.float64)
    return (ang / np.pi + 1) / 2 * 54 + 1


def img_images(arr):
    """[B,3,H,W] fp32 -> [B,H,W,3] uint8; the rescale is decided on the whole array"""
    t = np.asarray(arr, dtype=np.float32)
    if np.min(t) < -0.1:
        t = (t + 1) / 2
    elif np.max(t) > 1.5:
        t = t / 255
    return _bytes(np.transpose(t, (0, 2, 3, 1)) * 255)


def pack_images(pack, turbo, wheel, kind_of):
    """{image key: [B,H,W,3] uint8} of a pack of numpy arrays; kind_of(key) -> 'depth' / 'flow' / 'img' / None"""
    out = {}
    for k in sorted(pack):
        kind = kind_of(k)
        if kind == 'depth':
            out[k] = np.stack([depth_image(d[0], turbo) for d in pack[k]])
        elif kind == 'flow':
            out[k] = np.stack([flow_image(f, wheel) for f in pack[k]])
        elif kind == 'img':
            out[k] = img_images(pack[k])
    return out
