"""CPU restatement of the flow-pair preprocessing kernels (csrc/flow_pairs.cu), in their operation order.

  resize_flow_cubic   cv2.resize(flow, (W, H), INTER_CUBIC) on float32 followed by the x / y rescale of the reference's
                      `resize_flow` (scripts/preprocess/davis/generate_flows.py:44-54): half-pixel centres, A = -0.75,
                      clamped source taps, the horizontal pass first, then the vertical one.
  pair_masks          the forward / backward consistency masks of generate_flows.py:57-82,139-148: grid_sample
                      (bilinear, zeros, align_corners=True) of one flow at p + the other flow, L2 error > 1, or the target
                      out of the image.

Every fp32 operation is rounded on its own (numpy float32 arithmetic), as the kernels do with __fmul_rn / __fadd_rn; the
bilinear taps are accumulated with fused multiply-adds, as ATen's CPU grid_sample does. cv2 sums the vertical pass with
SIMD lanes (b0 r0 + (b1 r1 + (b2 r2 + b3 r3))) and the last few elements of a row that do not fill a vector left to right;
the restatement takes the SIMD order everywhere, which agrees bitwise except on those tail elements (~1 ulp).
"""
import numpy as np

f32 = np.float32
_A = f32(-0.75)


def cubic_coeffs(x):
    """OpenCV's interpolateCubic for an array of fractions x (fp32), -> [..., 4]."""
    x = x.astype(f32)
    x1 = x + f32(1)
    c0 = ((_A * x1 - f32(5) * _A) * x1 + f32(8) * _A) * x1 - f32(4) * _A
    c1 = (((_A + f32(2)) * x - (_A + f32(3))) * x) * x + f32(1)
    y = f32(1) - x
    c2 = (((_A + f32(2)) * y - (_A + f32(3))) * y) * y + f32(1)
    c3 = ((f32(1) - c0) - c1) - c2
    return np.stack([c0, c1, c2, c3], -1)


def cubic_taps(dst, src):
    """(clamped source indices [dst, 4], coefficients [dst, 4]) of one axis."""
    scale = 1.0 / (float(dst) / float(src))
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(f32)
    s = np.floor(f)
    frac = (f - s).astype(f32)
    idx = np.clip(s.astype(np.int64)[:, None] - 1 + np.arange(4)[None, :], 0, src - 1)
    return idx, cubic_coeffs(frac)


def resize_flow_cubic(flow, H, W):
    """flow [..., h, w, 2] fp32 -> [..., H, W, 2] fp32."""
    flow = np.asarray(flow, dtype=f32)
    h, w = flow.shape[-3:-1]
    xi, xc = cubic_taps(W, w)
    yi, yc = cubic_taps(H, h)
    # horizontal pass on every source row: v = ((c0 s0 + c1 s1) + c2 s2) + c3 s3
    g = flow[..., :, xi, :]                                  # [..., h, W, 4, 2]
    hp = g[..., 0, :] * xc[:, 0, None]
    for k in range(1, 4):
        hp = hp + g[..., k, :] * xc[:, k, None]
    # vertical pass: b0 r0 + (b1 r1 + (b2 r2 + b3 r3))
    r = hp[..., yi, :, :]                                    # [..., H, 4, W, 2]
    c = yc[:, :, None, None]
    out = r[..., 3, :, :] * c[:, 3]
    for k in (2, 1, 0):
        out = r[..., k, :, :] * c[:, k] + out
    mul = np.array([W / float(w), H / float(h)], dtype=np.float64)
    return (out.astype(np.float64) * mul).astype(f32)


def _bad(field, fl):
    """[..., H, W] bool: p + fl(p) leaves the image, or |field(p + fl(p)) + fl(p)| > 1 (grid_sample bilinear, zeros)."""
    H, W = fl.shape[-3:-1]
    ys, xs = np.meshgrid(np.arange(H, dtype=f32), np.arange(W, dtype=f32), indexing='ij')
    qx, qy = xs + fl[..., 0], ys + fl[..., 1]
    oob = (qx < 0) | (qx > f32(W - 1)) | (qy < 0) | (qy > f32(H - 1))
    sx, sy = f32((W - 1) / 2), f32((H - 1) / 2)
    ix = ((qx / sx - f32(1)) + f32(1)) * sx
    iy = ((qy / sy - f32(1)) + f32(1)) * sy
    x0, y0 = np.floor(ix), np.floor(iy)
    w, n = ix - x0, iy - y0
    e, s = f32(1) - w, f32(1) - n
    wts = (s * e, s * w, n * e, n * w)
    x0 = np.clip(np.nan_to_num(x0, nan=-2.0), -2, W + 1).astype(np.int64)
    y0 = np.clip(np.nan_to_num(y0, nan=-2.0), -2, H + 1).astype(np.int64)
    acc = None
    for (dy, dx), wt in zip(((0, 0), (0, 1), (1, 0), (1, 1)), wts):
        tx, ty = x0 + dx, y0 + dy
        ok = (tx >= 0) & (tx < W) & (ty >= 0) & (ty < H)
        txc, tyc = np.clip(tx, 0, W - 1), np.clip(ty, 0, H - 1)
        v = field[tyc, txc] if fl.ndim == 3 else field[np.arange(field.shape[0]).reshape(-1, 1, 1), tyc, txc]
        v = np.where(ok[..., None], v, f32(0)).astype(f32)
        # ATen's CPU kernel accumulates the four taps with fused multiply-adds: the fp64 product is exact, so one
        # rounding of product + acc to fp32 restates fmaf (bar a double-rounding tie)
        t = v.astype(np.float64) * wt[..., None]
        acc = t.astype(f32) if acc is None else (t + acc).astype(f32)
    d = acc + fl
    err = np.sqrt(d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1])
    return oob | (err > f32(1)), err


def pair_masks(flow_1_2, flow_2_1, convention='flowpair'):
    """flows [B, H, W, 2] (or [H, W, 2]) fp32 -> (mask_1, mask_2):
    'flowpair'  uint8 [.., H, W], 1 = inconsistent or out of bounds (the flowpair_*.npz masks);
    'pair_file' fp32 [.., H, W, 1, 1], 1 - ceil(mask): 1 = valid (the sequence .pt files)."""
    f12, f21 = np.asarray(flow_1_2, dtype=f32), np.asarray(flow_2_1, dtype=f32)
    bad_1, _ = _bad(f12, f21)        # on frame 2's grid: sample flow_1_2 at p + flow_2_1(p)
    bad_2, _ = _bad(f21, f12)
    if convention == 'flowpair':
        return bad_1.astype(np.uint8), bad_2.astype(np.uint8)
    if convention == 'pair_file':
        return ((~bad_1).astype(f32)[..., None, None], (~bad_2).astype(f32)[..., None, None])
    raise ValueError('convention must be "flowpair" or "pair_file", got %r' % (convention,))


def consistency_error(flow_1_2, flow_2_1):
    """(err_1, err_2) [.., H, W] fp32: the L2 round-trip errors the masks threshold."""
    f12, f21 = np.asarray(flow_1_2, dtype=f32), np.asarray(flow_2_1, dtype=f32)
    return _bad(f12, f21)[1], _bad(f21, f12)[1]


def digest(t):
    """compact bitwise fingerprint of a tensor: SHA-256 of its dtype, shape and bytes (first 20 hex digits)"""
    import hashlib
    import torch
    t = torch.as_tensor(t).contiguous()
    h = hashlib.sha256(('%s%s' % (t.dtype, tuple(t.shape))).encode())
    h.update(t.numpy().tobytes())
    return h.hexdigest()[:20]


def digest_item(item):
    """dataset item -> {key: digest} for tensors, the value for plain scalars, the basename for pair_path"""
    import os
    import torch
    out = {}
    for k, v in item.items():
        if torch.is_tensor(v):
            out[k] = digest(v)
        elif k == 'pair_path':
            out[k] = os.path.basename(str(v))
        else:
            out[k] = v
    return out


def unpack_band(bits, shape):
    """the fixture's band flags (np.packbits, row-major) -> bool array of `shape`"""
    n = int(np.prod(shape))
    return np.unpackbits(np.asarray(bits, dtype=np.uint8))[:n].reshape(shape).astype(bool)
