"""The flat Adam update's fp32 contract (`csrc/adam.cu`), as a checker.

`dvd_adam_flat_dev` ticks a device-side counter {t as int bits, fp32(1 - b1^t), fp32(sqrt(1 - b2^t))} and then updates, per
element and in fp32 (the compiler may contract the products into fmaf):

    gk = g * gscale
    m' = b1 * m + (1 - b1) * gk
    v' = b2 * v + (1 - b2) * gk * gk
    p' = p - (lr / bc1) * (m' / (sqrtf(v') / bc2_sqrt + eps))

with b1, b2, lr, eps the fp32 values the kernel receives and 1 - b evaluated in fp32. `check_adam` restates this in fp64 and
bounds the kernel's result by its rounding: m' and v' within `k_mv` units of 2^-24 of the magnitude of their two terms, p'
within 2^-24 |p| + 2^-21 |update| of p minus the update computed from the kernel's own m' and v' (a handful of correctly
rounded fp32 operations), and, per parameter tensor, the slope of (p - p') against the exact update within 1e-4 plus what
the element bound allows. The slope is what sees a bias correction or learning rate that is off by a few per cent on
tensors whose weights are so large that one update is below their ulp. The constants matter: fp32(0.9) is not 0.9, and
1 - 0.9 differs from 1 - fp32(0.9) by 2.4e-7 relatively, four units of 2^-24, which the step-1 bound on v' sees.
"""
import math

import numpy as np
import torch

U = 2.0 ** -24          # unit roundoff of fp32
TINY = 2.0 ** -149      # smallest fp32 subnormal: the absolute floor of one rounding


def f32(x):
    return float(np.float32(x))


def expected_state(t, betas):
    """The device counter after t ticks, as the kernel computes it from the fp32 betas (pow in double, then fp32)."""
    b1, b2 = f32(betas[0]), f32(betas[1])
    return t, f32(1.0 - b1 ** t), f32(math.sqrt(1.0 - b2 ** t))


def state_matches(state, t, betas):
    """`state` = the 4-float step_state tensor: step bits, bc1 and bc2_sqrt must be exactly what `t` ticks give."""
    s = state.detach().cpu()
    step = int(s[:1].view(torch.int32)[0])
    _, bc1, bc2s = expected_state(t, betas)
    return step == t and float(s[1]) == bc1 and float(s[2]) == bc2s


def check_adam(p0, m0, v0, g, p1, m1, v1, *, t, lr, betas, eps=1e-8, gscale=1.0, segments=None, k_mv=3.0, slope_tol=1e-4):
    """Flat fp32 tensors before (p0, m0, v0) and after (p1, m1, v1) one update with gradient buffer g at step t (the counter
    after the tick). `segments` = [(offset, numel), ...] of the parameter tensors; every element outside them (alignment
    padding) must be exactly 0 in all seven buffers. Returns a report dict; `report['fail']` lists what broke."""
    b1, b2 = f32(betas[0]), f32(betas[1])
    omb1, omb2 = float(np.float32(1.0) - np.float32(b1)), float(np.float32(1.0) - np.float32(b2))
    lrf, epsf, gs = f32(lr), f32(eps), f32(gscale)
    _, bc1, bc2s = expected_state(t, betas)
    d = lambda x: x.detach().reshape(-1).double()   # noqa: E731
    P0, M0, V0, P1, M1, V1 = d(p0), d(m0), d(v0), d(p1), d(m1), d(v1)
    gk = (d(g) * gs).float().double()               # the kernel rounds g * gscale to fp32
    fail, rep = [], {}
    if not (torch.isfinite(P1).all() and torch.isfinite(M1).all() and torch.isfinite(V1).all()):
        fail.append('non-finite p/m/v after the update')
        return {'fail': fail}

    tm1, tm2 = b1 * M0, omb1 * gk
    rm = (M1 - (tm1 + tm2)).abs() / (U * (tm1.abs() + tm2.abs()) + TINY)
    tv1, tv2 = b2 * V0, omb2 * gk * gk
    rv = (V1 - (tv1 + tv2)).abs() / (U * (tv1.abs() + tv2.abs()) + TINY)
    rep['m_units'], rep['v_units'] = float(rm.max()), float(rv.max())
    if rep['m_units'] > k_mv:
        fail.append("m' off by %.2f units of 2^-24 of its terms (bound %g)" % (rep['m_units'], k_mv))
    if rep['v_units'] > k_mv:
        fail.append("v' off by %.2f units of 2^-24 of its terms (bound %g)" % (rep['v_units'], k_mv))
    del rm, rv, tm1, tm2, tv1, tv2

    step_size = lrf / bc1
    u_own = step_size * M1 / (V1.sqrt() / bc2s + epsf)          # from the kernel's own m', v'
    bound = U * P0.abs() + 8 * U * u_own.abs() + TINY
    rp = (P1 - (P0 - u_own)).abs() / bound
    rep['p_ratio'] = float(rp.max())
    if rep['p_ratio'] > 1.0:
        i = int(rp.argmax())
        fail.append("p' outside 2^-24|p| + 2^-21|update| by %.3gx at element %d (p %.9g -> %.9g, update %.6g)"
                    % (rep['p_ratio'], i, float(P0[i]), float(P1[i]), float(u_own[i])))
    del rp, u_own

    m_ex = b1 * M0 + omb1 * gk
    v_ex = b2 * V0 + omb2 * gk * gk
    u_ex = step_size * m_ex / (v_ex.sqrt() / bc2s + epsf)
    del m_ex, v_ex
    step = P0 - P1
    rep['slope_ratio'] = 0.0       # worst |slope - 1| / tolerance over the tensors
    if segments is not None:
        covered = torch.zeros(P0.numel(), dtype=torch.bool, device=P0.device)
        for i, (o, n) in enumerate(segments):
            covered[o:o + n] = True
            uu = u_ex[o:o + n]
            den = float((uu * uu).sum())
            if den == 0.0:
                if bool((step[o:o + n] != 0).any()):
                    fail.append('tensor %d moved without an update' % i)
                continue
            slope = float((step[o:o + n] * uu).sum()) / den
            tol = slope_tol + float((bound[o:o + n] * uu.abs()).sum()) / den
            rep['slope_ratio'] = max(rep['slope_ratio'], abs(slope - 1.0) / tol)
            if abs(slope - 1.0) > tol:
                fail.append('tensor %d: slope of the step against the exact update %.8f (tolerance %.2e)' % (i, slope, tol))
        pad = ~covered
        for name, x in (('p', p0), ('m', m0), ('v', v0), ('g', g), ("p'", p1), ("m'", m1), ("v'", v1)):
            if bool((x.detach().reshape(-1)[pad] != 0).any()):
                fail.append('alignment padding of %s is not 0' % name)
    rep['fail'] = fail
    return rep


def adam_fp32_numpy(p, g, m, v, t, lr, betas, eps=1e-8, gscale=1.0, *, bc_step=None, lr_scale=1.0, use_gscale=True,
                    fp64_betas=None):
    """The kernel's arithmetic in numpy fp32 (no contraction), with switches that plant the defects the checker must see:
    bias correction at `bc_step` instead of t, lr scaled by `lr_scale`, `gscale` ignored, and 1 - b taken from the double
    betas `fp64_betas` (1 - 0.9 rounded to fp32) instead of from fp32(beta). Returns (p', m', v')."""
    F = np.float32
    b1, b2 = F(betas[0]), F(betas[1])
    if fp64_betas is not None:
        omb1, omb2 = F(1.0 - float(fp64_betas[0])), F(1.0 - float(fp64_betas[1]))
    else:
        omb1, omb2 = F(1) - b1, F(1) - b2
    s = t if bc_step is None else bc_step
    bc1 = F(1.0 - float(b1) ** s)
    bc2s = F(math.sqrt(1.0 - float(b2) ** s))
    gk = g * F(gscale) if use_gscale else g.copy()
    m1 = b1 * m + omb1 * gk
    v1 = b2 * v + omb2 * gk * gk
    step_size = F(F(lr) * F(lr_scale)) / bc1
    with np.errstate(divide='ignore', invalid='ignore'):
        p1 = p - step_size * (m1 / (np.sqrt(v1) / bc2s + F(eps)))
    return p1.astype(np.float32), m1.astype(np.float32), v1.astype(np.float32)
