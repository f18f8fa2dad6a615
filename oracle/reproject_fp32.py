"""TEST INFRASTRUCTURE — CPU emulation, not product code.

Bit-faithful fp32 restatement of the re-projection kernels (dynamic-video-depth_b200/csrc/reproject.cu): `derive_pose`,
`row_terms`, `pixel_forward`, `sf_residual`, the loss terms of `add_losses`, the hand-written `pixel_backward` and
`tap_grads`, the materialise kernel and `unproject_fwd` / `unproject_bwd`, each in the kernels' operation order and
vectorised over the pixels of a [B, H, W] batch (numpy).

Every step of the kernels' per-pixel chain is an `fmaf`, an explicitly rounded multiply or add, a min / max / floor, an
IEEE division or a sign-bit operation, so with `Fp32(round=True)` the per-pixel results are expected to match the kernels
bit for bit. The one operation whose rounding is not specified by IEEE is `rcp.approx.ftz.f32`: `Fp32.rcp` is pluggable
(the GPU tests supply the hardware instruction; the CPU default is the correctly rounded 1/x). `Fp32(round=False)` turns
every primitive into plain fp64 arithmetic, which must then equal `oracle.geometry` in fp64: that is what pins the
emulation's algebra, including the hand backward, to the reference's.

The reference's normalise / un-normalise round trip of the bilinear sample coordinate is not reproduced: the kernels skip
it (see `pixel_forward`).
"""
import numpy as np

F32, F64 = np.float32, np.float64


def fma_f32(a, b, c):
    """Correctly rounded fp32 fused multiply-add of fp32 operands (the product is exact in fp64; TwoSum gives the exact
    sum as s + e; s is rounded to fp32, except that an s sitting exactly on an fp32 midpoint with e != 0 is rounded
    toward e, which removes the double-rounding case)."""
    a64, b64, c64 = (np.asarray(v, dtype=F32).astype(F64) for v in (a, b, c))
    p = a64 * b64
    s = p + c64
    bp = s - p
    e = (p - (s - bp)) + (c64 - bp)
    r = s.astype(F32)
    d = s - r.astype(F64)
    nb = np.nextafter(r, np.where(d > 0, F32(np.inf), F32(-np.inf)).astype(F32))
    mid = (d != 0) & (r.astype(F64) + nb.astype(F64) == 2.0 * s)
    take_nb = mid & (e != 0) & ((e > 0) == (d > 0))
    return np.where(take_nb, nb, r).astype(F32)


def rcp_rn(x):
    """Correctly rounded 1/x (the CPU stand-in for rcp.approx.ftz.f32)."""
    return (F32(1.0) / np.asarray(x, dtype=F32)).astype(F32)


class Fp32:
    """The kernels' rounding primitives. round=False: every one is plain fp64 arithmetic."""

    def __init__(self, round=True, rcp=None):
        self.round = round
        self.dt = F32 if round else F64
        self._rcp = rcp if rcp is not None else rcp_rn

    def f(self, x):
        return np.asarray(x, dtype=self.dt)

    def mul(self, a, b):
        return self.f(a) * self.f(b)

    def add(self, a, b):
        return self.f(a) + self.f(b)

    def fma(self, a, b, c):
        if not self.round:
            return self.f(a) * self.f(b) + self.f(c)
        return fma_f32(a, b, c)

    def div(self, a, b):
        return self.f(a) / self.f(b)

    def rcp(self, x):
        return self._rcp(x) if self.round else 1.0 / self.f(x)

    @staticmethod
    def fmax(a, b):
        """fmaxf: max(-0, +0) = +0"""
        r = np.maximum(a, b)
        return np.where((a == 0) & (b == 0), a + b, r)

    @staticmethod
    def fmin(a, b):
        """fminf: min(-0, +0) = -0"""
        r = np.minimum(a, b)
        return np.where((a == 0) & (b == 0), -((-a) + (-b)), r)

    def sgn_scale(self, v, c):
        """c * sign(v), 0 at v == 0: the sign bit of v XORed into c (signed zeros included)."""
        v, c = self.f(v), self.f(c)
        return np.where(v == 0, self.f(0.0), np.where(np.signbit(v), -c, c)).astype(self.dt)


# ---------------------------------------------------------------------------------------------------------------------
# poses

def derive_pose(A, poses):
    """PoseC of every pair from the [B, 48] pose blocks; each field is a list of [B, 1, 1] arrays (broadcast over pixels)."""
    p = A.f(np.asarray(poses, dtype=F32))
    col = lambda i: p[:, i][:, None, None]  # noqa: E731
    Kinv = [col(i) for i in range(9)]
    K = [col(9 + i) for i in range(9)]
    R1 = [col(18 + i) for i in range(9)]
    R2 = [col(27 + i) for i in range(9)]
    t1 = [col(36 + i) for i in range(3)]
    t2 = [col(39 + i) for i in range(3)]

    def mm3(X, Y, xt):
        Z = []
        for i in range(3):
            for j in range(3):
                a = A.f(np.zeros_like(X[0]))
                for k in range(3):
                    a = A.fma(X[k * 3 + i] if xt else X[i * 3 + k], Y[k * 3 + j], a)
                Z.append(a)
        return Z
    M1 = mm3(R1, Kinv, False)
    Am = mm3(R2, M1, True)
    dx, dy, dz = A.add(t1[0], -t2[0]), A.add(t1[1], -t2[1]), A.add(t1[2], -t2[2])
    cv = [A.fma(R2[6 + i], dz, A.fma(R2[3 + i], dy, A.mul(R2[i], dx))) for i in range(3)]
    return dict(Kinv=Kinv, K=K, R1=R1, R2=R2, nM1=[-m for m in M1], A=Am, cv=cv,
                t21=[A.add(t2[i], -t1[i]) for i in range(3)], t1=t1, t2=t2)


def mv(A, M, x, y, z):
    return (A.fma(M[2], z, A.fma(M[1], y, A.mul(M[0], x))),
            A.fma(M[5], z, A.fma(M[4], y, A.mul(M[3], x))),
            A.fma(M[8], z, A.fma(M[7], y, A.mul(M[6], x))))


def mtv(A, M, x, y, z):
    return (A.fma(M[6], z, A.fma(M[3], y, A.mul(M[0], x))),
            A.fma(M[7], z, A.fma(M[4], y, A.mul(M[1], x))),
            A.fma(M[8], z, A.fma(M[5], y, A.mul(M[2], x))))


def ray_of(A, M, x, y):
    """M (x, y, 1): `fmaf(M1, y, M0 * x) + M2` per row"""
    return tuple(A.add(A.fma(M[3 * r + 1], y, A.mul(M[3 * r], x)), M[3 * r + 2]) for r in range(3))


def pixel_coords(A, B, H, W):
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing='ij')
    return A.f(np.broadcast_to(xs, (B, H, W))), A.f(np.broadcast_to(ys, (B, H, W)))


# ---------------------------------------------------------------------------------------------------------------------
# per-pixel chain

def pixel_forward(A, ps, d2, flow, d1, sf):
    """pixel_forward + sf_residual over every pixel. d2, d1 [B, H, W]; flow [B, H, W, 2]; sf [B, 3, H, W] (or None: zero
    scene flow, the static flow of the materialise kernel)."""
    d2, d1 = A.f(d2), A.f(d1)
    B, H, W = d1.shape
    x, y = pixel_coords(A, B, H, W)
    fx, fy = A.f(flow[..., 0]), A.f(flow[..., 1])
    sfk = [A.f(sf[:, k]) for k in range(3)] if sf is not None else [A.f(np.zeros_like(d1))] * 3
    o = {}
    ra = [A.fma(ps['A'][3 * k + 1], y, ps['A'][3 * k + 2]) for k in range(3)]
    rn = [A.fma(ps['nM1'][3 * k + 1], y, ps['nM1'][3 * k + 2]) for k in range(3)]
    hw, hh = A.f(W - 1), A.f(H - 1)
    nx = -x
    nqx = A.fma(fx, -1.0, nx)
    nqy = A.fma(fy, -1.0, -y)
    ix = A.fmin(hw, A.fmax(-nqx, A.f(0.0)))
    iy = A.fmin(hh, A.fmax(-nqy, A.f(0.0)))
    x0f, y0f = np.floor(ix), np.floor(iy)
    xi, yi = x0f.astype(np.int64), y0f.astype(np.int64)
    i00 = yi * W + xi
    sx1 = (xi < W - 1).astype(np.int64)
    sy1 = np.where(yi < H - 1, W, 0)
    flat = d2.reshape(B, H * W)
    tap = lambda idx: np.take_along_axis(flat, idx.reshape(B, -1), 1).reshape(B, H, W)  # noqa: E731
    dk = [tap(i00), tap(i00 + sx1), tap(i00 + sy1), tap(i00 + sy1 + sx1)]
    p12 = []
    for k in range(3):
        ac = A.fma(-ps['A'][3 * k], nx, ra[k])
        t = A.fma(d1, ac, ps['cv'][k])
        t = A.fma(ps['R2'][k], sfk[0], t)
        t = A.fma(ps['R2'][3 + k], sfk[1], t)
        p12.append(A.fma(ps['R2'][6 + k], sfk[2], t))
    i12 = mv(A, ps['K'], *p12)
    rz = A.rcp(A.add(i12[2], A.f(1e-8)))
    zok = ~(i12[2] < A.f(1e-3))
    ex = np.where(zok, A.fma(i12[0], rz, nqx), -fx)
    ey = np.where(zok, A.fma(i12[1], rz, nqy), -fy)
    wx1, wy1 = A.fma(x0f, -1.0, ix), A.fma(y0f, -1.0, iy)
    wx0, wy0 = A.fma(wx1, -1.0, 1.0), A.fma(wy1, -1.0, 1.0)
    w = [A.mul(wx0, wy0), A.mul(wx1, wy0), A.mul(wx0, wy1), A.mul(wx1, wy1)]
    wd = [A.mul(w[k], dk[k]) for k in range(4)]
    eb, sb = A.add(wd[1], wd[3]), A.add(wd[2], wd[3])
    s1 = A.add(A.add(wd[0], wd[1]), sb)
    su, sv = A.fma(x0f, s1, eb), A.fma(y0f, s1, sb)
    wpc = mv(A, ps['Kinv'], su, sv, s1)
    e = []
    for k in range(3):
        nr = A.fma(-ps['nM1'][3 * k], -x, rn[k])
        t = A.fma(sfk[k], -1.0, A.fma(d1, nr, ps['t21'][k]))
        e.append(A.fma(ps['R2'][3 * k + 2], wpc[2], A.fma(ps['R2'][3 * k + 1], wpc[1], A.fma(ps['R2'][3 * k], wpc[0], t))))
    o.update(x=x, y=y, d1=d1, i00=i00, sx1=sx1, sy1=sy1, w=w, x0f=x0f, y0f=y0f, s1=s1, wpc=wpc, p12=p12, i12=i12, rz=rz,
             zok=zok, ex=ex, ey=ey, e=e)
    return o


def mask_of(A, cfg, m2, o):
    m2 = A.f(m2)
    if not cfg['midas']:
        return m2
    return np.where((o['d1'] < A.f(100.0)) & (o['wpc'][2] < A.f(100.0)), m2, A.f(0.0))


def loss_terms(A, cfg, o):
    """The unmasked per-pixel terms (fl, dl, sl) of add_losses."""
    ex, ey = o['ex'], o['ey']
    fl = A.fma(ex, ex, A.mul(ey, ey)) if cfg['warm'] else A.add(np.abs(ex), np.abs(ey))
    za, zb = o['p12'][2], o['wpc'][2]
    if cfg['disp_mode'] == 0:
        a, b = A.fmax(za, A.f(1e-3)), A.fmax(zb, A.f(1e-3))
        dl = A.mul(A.f(100.0), np.abs(A.add(A.rcp(a), -A.rcp(b))))
    elif cfg['disp_mode'] == 1:
        a, b = A.fmax(za, A.f(1e-3)), A.fmax(zb, A.f(1e-3))
        dl = A.add(A.div(A.fmax(a, b), A.fmin(a, b)), A.f(-1.0))
    else:
        dl = np.abs(A.add(za, -zb))
    e = o['e']
    sl = A.add(A.add(np.abs(e[0]), np.abs(e[1])), np.abs(e[2]))
    return fl, dl, sl


def finalize(A, cfg, sums):
    """reproject_finalize_kernel on the exact (fp64) sums (flow, disp, sf, mask) → dict of the scalars."""
    t = [F64(s) for s in sums]
    if A.round:
        n = F32(F32(t[3]) + F32(1e-8))
        fl, dl, sl = (F32(F32(v) / n) for v in t[:3])
        cf, cd = F32(F32(cfg['flow_mul']) / n), F32(F32(cfg['disp_mul']) / n)
    else:
        n = t[3] + 1e-8
        fl, dl, sl = (v / n for v in t[:3])
        cf, cd = cfg['flow_mul'] / n, cfg['disp_mul'] / n
    second = dl if cfg['second_is_disp'] else sl
    return dict(flow=fl, disp=dl, sf=sl, loss=cfg['flow_mul'] * fl + cfg['disp_mul'] * second, masksum=t[3], cf=cf, cd=cd)


def loss_forward(A, cfg, ps, d1, d2, flow, mask, sf, o=None):
    """Masked per-pixel terms (m, m·fl, m·dl, m·sl) and the finalised scalars."""
    o = pixel_forward(A, ps, d2, flow, d1, sf) if o is None else o
    m = mask_of(A, cfg, np.asarray(mask).reshape(o['d1'].shape), o)
    fl, dl, sl = loss_terms(A, cfg, o)
    terms = [A.mul(m, fl), A.mul(m, dl), A.mul(m, sl)]   # fmaf(m, t, acc) with m in {0, 1} adds exactly m·t
    sums = [np.sum(t.astype(F64)) for t in terms] + [np.sum(m.astype(F64))]
    return dict(o=o, m=m, terms=terms, scalars=finalize(A, cfg, sums))


def tap_grads(A, o, hu, hv, h1):
    base = A.fma(hu, o['x0f'], A.fma(hv, o['y0f'], h1))
    bx = A.add(base, hu)
    w = o['w']
    return [A.mul(w[0], base), A.mul(w[1], bx), A.mul(w[2], A.add(base, hv)), A.mul(w[3], A.add(bx, hv))]


def pixel_backward(A, cfg, ps, o, m, cf, cd):
    """pixel_backward → (g_sf as a list of three [B, H, W] arrays, h = Kinv^T g_wpc as three arrays); tap_grads(A, o, *h)
    gives the four tap gradients."""
    cf, cd = A.f(cf), A.f(cd)
    mcf = np.where(o['zok'], A.mul(m, cf), A.f(0.0))
    if cfg['warm']:
        t2 = A.add(mcf, mcf)
        gux, guy = A.mul(t2, o['ex']), A.mul(t2, o['ey'])
    else:
        gux, guy = A.sgn_scale(o['ex'], mcf), A.sgn_scale(o['ey'], mcf)
    rz, i12 = o['rz'], o['i12']
    gi0, gi1 = A.mul(gux, rz), A.mul(guy, rz)
    tt = A.fma(gux, i12[0], A.mul(guy, i12[1]))
    gi2 = A.mul(A.mul(tt, rz), A.mul(rz, -1.0))
    gp0, gp1, gp2 = mtv(A, ps['K'], gi0, gi1, gi2)
    zero = A.f(np.zeros_like(gp0))
    ge = [zero, zero, zero]
    mc = A.mul(m, cd)
    Kinv = ps['Kinv']
    if cfg['second_is_disp']:
        za, zb = o['p12'][2], o['wpc'][2]
        lo = A.f(1e-3)
        if cfg['disp_mode'] == 0:
            ra, rb = A.rcp(A.fmax(za, lo)), A.rcp(A.fmax(zb, lo))
            s = A.sgn_scale(A.fma(rb, -1.0, ra), A.mul(mc, 100.0))
            sa, sb = np.where(za >= lo, s, A.f(0.0)), np.where(zb >= lo, s, A.f(0.0))
            gp2 = A.fma(A.mul(sa, ra), A.mul(ra, -1.0), gp2)
            gwc2 = A.mul(A.mul(sb, rb), rb)
        elif cfg['disp_mode'] == 1:
            a, bb = A.fmax(za, lo), A.fmax(zb, lo)
            ra, rb = A.rcp(a), A.rcp(bb)
            ge_ab = a >= bb
            ga = np.where(ge_ab, rb, A.mul(A.mul(-bb, ra), ra))
            gb = np.where(ge_ab, A.mul(A.mul(-a, rb), rb), ra)
            gp2 = A.add(gp2, np.where(za >= lo, A.mul(ga, mc), A.f(0.0)))
            gwc2 = np.where(zb >= lo, A.mul(gb, mc), A.f(0.0))
        else:
            s = A.sgn_scale(A.fma(zb, -1.0, za), mc)
            gp2 = A.add(gp2, s)
            gwc2 = A.mul(s, -1.0)
        hu, hv, h1 = A.mul(Kinv[6], gwc2), A.mul(Kinv[7], gwc2), A.mul(Kinv[8], gwc2)
    else:
        ge = [A.sgn_scale(o['e'][k], mc) for k in range(3)]
        a0, a1, a2 = mtv(A, ps['R2'], *ge)
        hu, hv, h1 = mtv(A, Kinv, a0, a1, a2)
    gv = mv(A, ps['R2'], gp0, gp1, gp2)
    gv = [A.fma(ge[k], -1.0, gv[k]) for k in range(3)]
    return gv, (hu, hv, h1)


def tap_index(o):
    """Flat (per pair) element index of the four taps of every pixel: nw, ne, sw, se (a clamped tap shares its neighbour's)."""
    i00, sx1, sy1 = o['i00'], o['sx1'], o['sy1']
    return [i00, i00 + sx1, i00 + sy1, i00 + sy1 + sx1]


def scatter(o, g, B, HW):
    """fp64 sum, absolute sum and contribution count (non-zero contributions) of g_depth_2 per element."""
    tot, ab, cnt = (np.zeros((B, HW)) for _ in range(3))
    bidx = np.broadcast_to(np.arange(B)[:, None, None], o['i00'].shape)
    for idx, gk in zip(tap_index(o), g):
        gk = gk.astype(F64)
        nz = gk != 0
        np.add.at(tot, (bidx[nz], idx[nz]), gk[nz])
        np.add.at(ab, (bidx[nz], idx[nz]), np.abs(gk[nz]))
        np.add.at(cnt, (bidx[nz], idx[nz]), 1.0)
    return tot, ab, cnt


# ---------------------------------------------------------------------------------------------------------------------
# un-projection and materialisation

def unproject_fwd(A, depth, poses, which=1):
    """unproject_fwd_kernel: P = R (d · ray) + t, depth [B, H, W] → [B, 3, H, W]."""
    p = A.f(np.asarray(poses, dtype=F32))
    d = A.f(depth)
    B, H, W = d.shape
    col = lambda i: p[:, i][:, None, None]  # noqa: E731
    Kinv = [col(i) for i in range(9)]
    R = [col((18 if which == 1 else 27) + i) for i in range(9)]
    t = [col((36 if which == 1 else 39) + i) for i in range(3)]
    x, y = pixel_coords(A, B, H, W)
    rx, ry, rz = ray_of(A, Kinv, x, y)
    o = mv(A, R, A.mul(d, rx), A.mul(d, ry), A.mul(d, rz))
    return np.stack([A.add(o[k], t[k]) for k in range(3)], 1)


def unproject_bwd(A, gP, poses, which=1):
    """unproject_bwd_kernel: gd = <gP, R ray>, gP [B, 3, H, W] → [B, H, W]."""
    p = A.f(np.asarray(poses, dtype=F32))
    g = A.f(gP)
    B, _, H, W = g.shape
    col = lambda i: p[:, i][:, None, None]  # noqa: E731
    Kinv = [col(i) for i in range(9)]
    R = [col((18 if which == 1 else 27) + i) for i in range(9)]
    x, y = pixel_coords(A, B, H, W)
    wx, wy, wz = mv(A, R, *ray_of(A, Kinv, x, y))
    return A.fma(g[:, 2], wz, A.fma(g[:, 1], wy, A.mul(g[:, 0], wx)))


def materialize(A, ps, d1, d2, flow, sf):
    """reproject_materialize_kernel: the nine per-pixel tensors, channel-planar."""
    o = pixel_forward(A, ps, d2, flow, d1, sf)
    x, y = o['x'], o['y']
    n = ray_of(A, ps['nM1'], x, y)
    wP2 = mv(A, ps['R2'], *o['wpc'])
    P1 = [A.fma(-o['d1'], n[k], ps['t1'][k]) for k in range(3)]
    wP2 = [A.add(wP2[k], ps['t2'][k]) for k in range(3)]
    os_ = pixel_forward(A, ps, d2, flow, d1, None)

    def proj(q, c, k):
        return np.where(q['zok'], A.fma(q['i12'][k], q['rz'], -c), A.f(0.0))
    st = lambda v: np.stack(v, 1)  # noqa: E731
    return {'global_p1': st(P1), 'sf_by_depth': st([A.add(wP2[k], -P1[k]) for k in range(3)]),
            'warped_global_p2': st(wP2), 'warped_p2_camera_2': st(o['wpc']), 'p1_camera_2': st(o['p12']),
            'dflow_1_2': st([proj(o, x, 0), proj(o, y, 1)]), 'staticflow_1_2': st([proj(os_, x, 0), proj(os_, y, 1)]),
            'depth_image_1_2': o['i12'][2][:, None], 'depth_warp_1_2': o['s1'][:, None]}


def materialize_bwd(A, ps, d1, d2, flow, sf, G):
    """reproject_materialize_bwd_kernel for cotangents G (dict of the nine keys, channel-planar) → (g_d1, g_d2, g_sf).
    The kernel writes this adjoint with plain * and +, which the compiler may contract: it is a model to a few ulps, not
    bit for bit."""
    o = pixel_forward(A, ps, d2, flow, d1, sf)
    Gc = {k: [A.f(v[:, c]) for c in range(v.shape[1])] for k, v in G.items()}
    gP = [A.add(Gc['global_p1'][k], -Gc['sf_by_depth'][k]) for k in range(3)]
    gW = [A.add(Gc['warped_global_p2'][k], Gc['sf_by_depth'][k]) for k in range(3)]
    a = mtv(A, ps['R2'], *gW)
    gC = [A.add(Gc['warped_p2_camera_2'][k], a[k]) for k in range(3)]
    gp = list(Gc['p1_camera_2'])
    gu, gvv = Gc['dflow_1_2']
    rz, i12 = o['rz'], o['i12']
    gi0 = np.where(o['zok'], A.mul(gu, rz), A.f(0.0))
    gi1 = np.where(o['zok'], A.mul(gvv, rz), A.f(0.0))
    gi2 = A.add(Gc['depth_image_1_2'][0], np.where(o['zok'], -A.mul(A.mul(
        A.add(A.mul(gu, i12[0]), A.mul(gvv, i12[1])), rz), rz), A.f(0.0)))
    a = mtv(A, ps['K'], gi0, gi1, gi2)
    gp = [A.add(gp[k], a[k]) for k in range(3)]
    b = mv(A, ps['R2'], *gp)
    g_sf = np.stack(b, 1)
    gP = [A.add(gP[k], b[k]) for k in range(3)]
    os_ = pixel_forward(A, ps, d2, flow, d1, None)
    su, sv = Gc['staticflow_1_2']
    s0, s1 = A.mul(su, os_['rz']), A.mul(sv, os_['rz'])
    s2 = -A.mul(A.mul(A.add(A.mul(su, os_['i12'][0]), A.mul(sv, os_['i12'][1])), os_['rz']), os_['rz'])
    b = mv(A, ps['R2'], *mtv(A, ps['K'], s0, s1, s2))
    gP = [np.where(os_['zok'], A.add(gP[k], b[k]), gP[k]) for k in range(3)]
    rx, ry, rzz = ray_of(A, ps['nM1'], o['x'], o['y'])
    g_d1 = -A.fma(gP[2], rzz, A.fma(gP[1], ry, A.mul(gP[0], rx)))
    hu, hv, h1 = mtv(A, ps['Kinv'], *gC)
    h1 = A.add(h1, Gc['depth_warp_1_2'][0])
    B, H, W = o['d1'].shape
    tot, ab, cnt = scatter(o, tap_grads(A, o, hu, hv, h1), B, H * W)
    return g_d1, tot.reshape(B, H, W), g_sf


# ---------------------------------------------------------------------------------------------------------------------
# inputs and configurations

def edge_inputs(B, H, W, seed=0, sigma=3.0):
    """CPU fp32 inputs of B synthetic pairs with the edges of the chain planted in every pair: a depth_1 patch >= 100
    and a depth_2 patch >= 100 (midas mask), a depth_2 patch at 1e-4 (disparity clamp of the warped depth), a column of
    scene flow that pushes p12 behind camera 2 (rejected projection, clamped za), and flows that leave the image to the
    right and at the bottom (border clamps)."""
    import torch
    from dvd_b200 import ops, synthetic
    pairs = [(k % 40, k % 40 + 1 + (k % 5)) for k in range(B)]
    batch = synthetic.make_batch(pairs, H=H, W=W, seed=seed, leading_dim=False, flow_sigma=sigma)
    d1 = synthetic.make_depths(B, H, W, seed=seed + 1)
    d2 = synthetic.make_depths(B, H, W, seed=seed + 2)
    sf = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(seed + 3)) * 0.05
    flow = batch['flow_1_2']
    h4, w4 = max(H // 4, 1), max(W // 4, 1)
    d1[:, :, :h4, :w4] = 150.0
    d2[:, :, h4:2 * h4, w4:2 * w4] = 120.0
    d2[:, :, 2 * h4:3 * h4, :w4] = 1e-4
    sf[:, 2, :, W // 2] = -3.0 * d1[:, 0, :, W // 2]
    flow[:, H // 3, :, 0] = 2.0 * W
    flow[:, :, W // 3, 1] = 2.0 * H
    batch['flow_1_2'] = flow.contiguous()
    return dict(d1=d1, d2=d2, sf=sf, flow=batch['flow_1_2'], mask=batch['mask_2'].reshape(B, H, W).contiguous(),
                poses=ops.pack_poses_from_batch(batch), batch=batch)

def cfg_dict(midas, warm, disp_mode, second_is_disp, flow_mul=1.0, disp_mul=1.0):
    return dict(midas=int(midas), warm=int(warm), disp_mode=int(disp_mode), second_is_disp=int(second_is_disp),
                flow_mul=float(np.float32(flow_mul)), disp_mul=float(np.float32(disp_mul)))


def all_cfgs(flow_mul=1.0, disp_mul=1.0):
    """Every raw dvd_loss_cfg: midas, warm, disp_mode in {0, 1, 2}, second_is_disp."""
    return [cfg_dict(mi, wa, dm, sd, flow_mul, disp_mul) for mi in (0, 1) for wa in (0, 1) for dm in (0, 1, 2)
            for sd in (0, 1)]


def reference_kw(cfg):
    """The reference's flags of a cfg that make_loss_cfg builds (disp_mode 0 <=> second_is_disp), else None."""
    if (cfg['disp_mode'] == 0) != bool(cfg['second_is_disp']):
        return None
    return dict(midas=bool(cfg['midas']), warm=bool(cfg['warm']), use_disp=cfg['disp_mode'] == 0,
                use_disp_ratio=cfg['disp_mode'] == 1, flow_mul=cfg['flow_mul'], disp_mul=cfg['disp_mul'])
