"""TEST INFRASTRUCTURE — fp64 emulation of the scene-flow MLP kernels' arithmetic (csrc/sf_mlp_tc.cu).

The STRUCTURE is the reference's (oracle/sf_mlp.py: feature order with t first, LeakyReLU 0.2, ÷ sf_mag_div, Euler update); the
PRECISION MODEL is the kernels':

  * split2 (tc_common.cuh): hi = bf16_rne(x), lo = bf16_rne(fp32(x − hi)), so x ≈ hi + lo to 2^-17 |x|;
  * a layer is acc = Σ_k (A_hi W_hi + A_lo W_hi + A_hi W_lo) — here in fp64, where the tensor cores accumulate in fp32 — then
    y = fp32(fp32(acc) + b), the mask bit y > 0, fmaxf(y, 0.2f·y) and split2 of that for the next layer. The output layer is
    s = fp32(fp32(acc) + b5) / sf_mag_div (an IEEE divide); the Euler update p += s, t += dt is fp32;
  * the embedding takes the argument fp32(f_k · x) the kernel forms and evaluates sin / cos in fp64. The kernel's fast_sincos
    (Cody-Waite reduction + MUFU) is about 5e-7 absolute away from that: the expected residual of every embedded feature;
  * the data gradient of one eval: gs = a_in + g_acc + g_step (the kernel's order, fp32), d5 = gs / sf_mag_div, then through
    split2 and the same three-product model on the transposed weights; at each hidden layer ×1 or ×0.2f by the saved mask
    bit, then split2. The layer-0 result is contracted with d(embedding)/dxyz (identity features included): a_out = a_in + that;
  * the weight gradient is g_w[l] = Σ_px dYhi_l ⊗ Xhi_l and g_b[l] = Σ_px dYhi_l (l < 5) on the bf16 `hi` planes the kernels
    save (sf_mlp_layout.cuh: kSavePlanes = 1). The products are exact in fp64, so against the kernel only the fp32 accumulation
    order is left. g_b[5] is the sum of d5 (accumulated by the data-gradient kernel).

Layout decoders restate make_layout (sf_mlp_layout.cuh) and sw128_offset / mn128_offset (tc_common.cuh): the packed weight
images, the per-eval `save` buffer (X_l hi planes and the 5 × 256-bit LeakyReLU masks per pixel) and the dY scratch. They
return raw bf16 bit patterns (int16); `bits_to_f64` turns them into values.

Teacher forcing: the caller starts each eval from the kernel's own p_steps[e] and feeds the data gradient of eval e the kernel's
a_in and mask bits, so rounding flips cannot accumulate across evals or across the forward -> backward boundary.

With rounding=False (split2 -> (x, 0), no fp32 rounding, exact sin / cos, plain weights) the emulation is
oracle.sf_mlp.sf_multi_step + autograd in fp64 (tests/test_sf_mlp_bf16_oracle_cpu.py).
"""
import torch

from oracle.sf_mlp import freqs

WIDTH, LAYERS, TILE_M, CHUNK = 256, 6, 128, 64
C02 = 0.20000000298023224       # 0.2f, the LeakyReLU slope as the kernels hold it


# ---- rounding ---------------------------------------------------------------------------------------------------------------
def f32(x, rounding=True):
    """x rounded to fp32 (kept in x's dtype); identity without rounding"""
    return x.float().to(x.dtype) if rounding else x


def split2(x, rounding=True):
    """(hi, lo) in fp64 of the fp32 value x: hi = bf16_rne(x), lo = bf16_rne(fp32(x - hi)); (x, None) without rounding"""
    if not rounding:
        return x, None
    x32 = x.float()
    hi = x32.to(torch.bfloat16).float()
    lo = (x32 - hi).to(torch.bfloat16)
    return hi.double(), lo.double()


def bf16_bits(x):
    """bit pattern (int16) of bf16_rne(fp32(x))"""
    return x.float().to(torch.bfloat16).view(torch.int16)


def bits_to_f64(bits):
    return bits.view(torch.bfloat16).double()


# ---- layout (sf_mlp_layout.cuh: make_layout) --------------------------------------------------------------------------------
def n_in(n_freq_xyz, n_freq_t, time_dependent):
    return (1 + 2 * n_freq_t if time_dependent else 0) + 3 + 6 * n_freq_xyz


def specialised(n_freq_xyz, n_freq_t, time_dependent):
    """the two configurations with kernels compiled for their counts (layer 0 padded to a multiple of 16, not 64)"""
    return n_freq_xyz == 16 and (not time_dependent or n_freq_t == 16)


def blk_bytes(rows):
    return (rows + 63) // 64 * 8192


class Layout:
    def __init__(self, n_freq_xyz, n_freq_t, time_dependent, npx):
        self.nin = n_in(n_freq_xyz, n_freq_t, time_dependent)
        q = 16 if specialised(n_freq_xyz, n_freq_t, time_dependent) else 64
        self.kpad0 = (self.nin + q - 1) // q * q
        self.k0_chunks = (self.kpad0 + 63) // 64
        self.npx = npx
        self.ntiles = (npx + TILE_M - 1) // TILE_M
        self.nq = 2 * self.ntiles
        self.wf_off, o = [], 0
        for l in range(LAYERS):
            self.wf_off.append(o)
            o += self.nkc_f(l) * 2 * self.rows_f(l) * 128
        self.wf_total = o
        self.wb_off, o = [], 0
        for l in range(LAYERS):
            self.wb_off.append(o)
            o += self.nkc_b(l) * 2 * self.rows_b(l) * 128
        self.wb_total = o
        self.xs_off, o = [], 0
        for l in range(LAYERS):
            self.xs_off.append(o)
            o += self.nq * blk_bytes(self.rows_x(l))
        self.mask_off = o
        o += 5 * self.ntiles * TILE_M * 32
        self.save_total = (o + 255) & ~255
        self.dy_off, o = [], 0
        for l in range(LAYERS):
            self.dy_off.append(o)
            o += self.nq * blk_bytes(self.rows_dy(l))
        self.dy_total = (o + 255) & ~255

    def rows_f(self, l):
        return WIDTH if l < 5 else 16

    def rows_b(self, l):
        return self.kpad0 if l == 0 else WIDTH

    def nkc_f(self, l):
        return self.k0_chunks if l == 0 else 4

    def nkc_b(self, l):
        return 1 if l == 5 else 4

    def rows_x(self, l):
        return self.kpad0 if l == 0 else WIDTH

    def rows_dy(self, l):
        return 16 if l == 5 else WIDTH

    def layer_in(self, l):
        return self.nin if l == 0 else WIDTH

    def layer_out(self, l):
        return 3 if l == 5 else WIDTH

    def packed_weights_bytes(self):
        """dvd_mlp_packed_weights_bytes: the larger of the two images (computed for 128 pixels there; independent of npx)"""
        return max(self.wf_total, self.wb_total)


def sw128_offset(row, k):
    """byte offset of element (row, k) in one [rows x 64] K-major SWIZZLE_128B block (ints or int64 tensors)"""
    return (row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 3) ^ row) & 7) << 4) + (k & 7) * 2


def mn128_offset(mn, k):
    """byte offset of element (mn, k) in one MN-major SWIZZLE_128B block of 64 K rows (ints or int64 tensors)"""
    return (mn >> 6) * 8192 + (k >> 3) * 1024 + (k & 7) * 128 + ((((mn & 63) >> 3) ^ k) & 7) * 16 + (mn & 7) * 2


def _gather(buf, byte_idx):
    return buf.view(torch.int16)[byte_idx // 2]


def decode_image(buf, L, l, fwd):
    """(hi, lo) bit planes [rows, nkc * 64] of layer l's packed weight block: forward image B[n = out][k = in], data-gradient
    image B[n = in][k = out], padding included"""
    rows, nkc = (L.rows_f(l), L.nkc_f(l)) if fwd else (L.rows_b(l), L.nkc_b(l))
    base = L.wf_off[l] if fwd else L.wb_off[l]
    r = torch.arange(rows, device=buf.device).view(-1, 1)
    col = torch.arange(nkc * 64, device=buf.device).view(1, -1)
    idx = base + (col >> 6) * 2 * rows * 128 + sw128_offset(r, col & 63)
    return _gather(buf, idx), _gather(buf, idx + rows * 128)


def decode_blocks(buf, off, rows, nq):
    """bit plane [nq * 64 pixels, rows] of an MN-major activation / dY array (64-pixel blocks of blk_bytes(rows) bytes)"""
    g = torch.arange(nq * 64, device=buf.device).view(-1, 1)
    c = torch.arange(rows, device=buf.device).view(1, -1)
    return _gather(buf, off + (g >> 6) * blk_bytes(rows) + mn128_offset(c, g & 63))


def decode_x(save_e, L, l):
    """saved X_l hi plane [nq * 64, rows_x(l)] of one eval's save buffer (pixel g = b * hw + i, pad pixels included)"""
    return decode_blocks(save_e, L.xs_off[l], L.rows_x(l), L.nq)


def decode_dy(dy, L, l):
    """dY_l hi plane [nq * 64, rows_dy(l)] of a dY scratch buffer"""
    return decode_blocks(dy, L.dy_off[l], L.rows_dy(l), L.nq)


def decode_masks(save_e, L):
    """LeakyReLU masks [5, ntiles * 128, 256] (bool, pre-activation > 0): 8 little-endian 32-bit words per layer and pixel, so
    channel c is bit c % 8 of byte c / 8"""
    n = 5 * L.ntiles * TILE_M
    by = save_e[L.mask_off:L.mask_off + n * 32].view(5, L.ntiles * TILE_M, 32).long()
    c = torch.arange(WIDTH, device=save_e.device)
    return ((by[..., c >> 3] >> (c & 7)) & 1).bool()


# ---- the net ----------------------------------------------------------------------------------------------------------------
class Net:
    """Weights in the emulation's form. fwd[l] = (hi, lo) of W_l [out, in], bwd[l] = (hi, lo) of W_l^T [in, out] (lo None
    without rounding), b[l] the fp32 bias (fp64 tensor)."""

    def __init__(self, fwd, bwd, b, n_freq_xyz, n_freq_t, time_dependent, sf_mag_div=100.0, rounding=True):
        self.fwd, self.bwd, self.b = fwd, bwd, b
        self.fx, self.td = n_freq_xyz, bool(time_dependent)
        self.ft = n_freq_t if time_dependent else 0
        self.nt = 1 + 2 * self.ft if self.td else 0
        self.div, self.rounding = float(sf_mag_div), rounding

    @classmethod
    def from_weights(cls, layers, cfg_kw, sf_mag_div=100.0, rounding=True):
        """layers [(W [out, in], b)] (fp32 values); the weights split here as pack_weights_kernel does"""
        fwd = [split2(w.double(), rounding) for w, _ in layers]
        bwd = [split2(w.double().t().contiguous(), rounding) for w, _ in layers]
        return cls(fwd, bwd, [b.double() for _, b in layers], sf_mag_div=sf_mag_div, rounding=rounding, **cfg_kw)

    @classmethod
    def from_images(cls, wf, wb, biases, L, cfg_kw, sf_mag_div=100.0):
        """weights decoded from the kernels' packed images (uint8 buffers of dvd_mlp_pack_weights)"""
        fwd, bwd = [], []
        for l in range(LAYERS):
            o, i = L.layer_out(l), L.layer_in(l)
            hi, lo = decode_image(wf, L, l, True)
            fwd.append((bits_to_f64(hi[:o, :i]), bits_to_f64(lo[:o, :i])))
            hi, lo = decode_image(wb, L, l, False)
            bwd.append((bits_to_f64(hi[:i, :o]), bits_to_f64(lo[:i, :o])))
        return cls(fwd, bwd, [b.double() for b in biases], sf_mag_div=sf_mag_div, **cfg_kw)


def _mm(a, w, terms):
    """A [N, K] (hi, lo) times B [rows, K]^T (hi, lo): A_hi B_hi + A_lo B_hi (+ A_hi B_lo with terms = 3), fp64"""
    ah, al = a
    wh, wl = w
    acc = ah @ wh.t()
    if al is not None:
        acc = acc + al @ wh.t()
    if wl is not None and terms == 3:
        acc = acc + ah @ wl.t()
    return acc


def _sincos_args(net, p):
    """fp32(f_k * x_d) [N, fx, 3] and the frequencies [fx] (fp64 values of the fp32 linspace)"""
    f = freqs(net.fx, torch.float64).to(p.device)
    return f32(f.view(1, -1, 1) * p.view(-1, 1, 3), net.rounding), f


def embed(net, p, t):
    """features [N, nin] in the reference's order: [t, cos(ft t), sin(ft t)] (time-dependent), x, y, z, cos(f_k x_d), sin(f_k x_d)
    (k major, d minor); p [N, 3], t [N] (fp32 values, fp64)"""
    r = net.rounding
    out = []
    if net.td:
        out.append(t.view(-1, 1))
        if net.ft:
            a = f32(freqs(net.ft, torch.float64).to(t.device).view(1, -1) * t.view(-1, 1), r)
            out += [f32(torch.cos(a), r), f32(torch.sin(a), r)]
    out.append(p)
    if net.fx:
        a, _ = _sincos_args(net, p)
        out += [f32(torch.cos(a), r).reshape(len(p), -1), f32(torch.sin(a), r).reshape(len(p), -1)]
    return torch.cat(out, 1)


def forward_eval(net, p, t, terms=3):
    """one evaluation of the field on p [N, 3], t [N] or None -> dict: x [X_0 .. X_5] as (hi, lo), y [Y_0 .. Y_4] (hidden
    pre-activations), mask [Y_l > 0], s [N, 3] (= raw output / sf_mag_div)"""
    r = net.rounding
    x = split2(embed(net, p, t), r)
    X, Y, M = [x], [], []
    for l in range(5):
        y = f32(f32(_mm(x, net.fwd[l], terms), r) + net.b[l], r)
        a = torch.maximum(y, f32(y * (C02 if r else 0.2), r))
        x = split2(a, r)
        X.append(x), Y.append(y), M.append(y > 0)
    o = f32(f32(_mm(x, net.fwd[5], terms), r) + net.b[5], r)
    return {'x': X, 'y': Y, 'mask': M, 's': f32(o / net.div, r)}


def dgrad_eval(net, p, masks, a_in=None, g_acc=None, g_step=None, terms=3):
    """backward of one eval: masks [M_0 .. M_4] ([N, 256] bool), p the eval's input points; a_in / g_acc / g_step [N, 3] or None
    (pass g_acc only where the eval is accumulated) -> dict: dy [dY_0 .. dY_5] as (hi, lo), a_out [N, 3], gb5 [3]"""
    r = net.rounding
    gs = torch.zeros_like(p) if a_in is None else a_in
    for g in (g_acc, g_step):
        if g is not None:
            gs = f32(gs + g, r)
    d5 = f32(gs / net.div, r)
    dy = split2(d5, r)
    DY = [None] * 5 + [dy]
    for l in range(5, 0, -1):
        v = f32(_mm(dy, net.bwd[l], terms), r)
        v = torch.where(masks[l - 1], v, f32(v * (C02 if r else 0.2), r))
        dy = split2(v, r)
        DY[l - 1] = dy
    g0 = f32(_mm(dy, net.bwd[0], terms), r)
    # contraction with d(embedding)/dxyz: identity features, d cos(f x)/dx = -f sin(f x), d sin(f x)/dx = f cos(f x)
    c = net.nt
    gp = g0[:, c:c + 3]
    if net.fx:
        a, f = _sincos_args(net, p)
        n = len(p)
        gc = g0[:, c + 3:c + 3 + 3 * net.fx].reshape(n, net.fx, 3)
        gsn = g0[:, c + 3 + 3 * net.fx:c + 3 + 6 * net.fx].reshape(n, net.fx, 3)
        fv = f.view(1, -1, 1)
        gp = gp + (-fv * f32(torch.sin(a), r) * gc + fv * f32(torch.cos(a), r) * gsn).sum(1)
    a_out = f32((a_in if a_in is not None else 0.0) + gp, r)
    return {'dy': DY, 'a_out': a_out, 'gb5': d5.sum(0)}


def wgrad(x_hi, dy_hi):
    """g_w[l] = dY_l^T X_l [out, in], g_b[l] = Σ dY_l (l < 5; None for l = 5) from per-pixel operands [N, ·] (fp64)"""
    g_w = [dy_hi[l].t() @ x_hi[l] for l in range(LAYERS)]
    g_b = [dy_hi[l].sum(0) for l in range(5)] + [None]
    return g_w, g_b


def chain(net, p0, t0, dt, n_eval, n_acc, g_acc=None, g_steps=None, terms=3):
    """The whole Euler chain and its backward without teacher forcing (the rounding-free structure check):
    p0 [N, 3], t0 [N] or None -> dict(acc, s [n_eval], g_p, g_w, g_b)"""
    r = net.rounding
    dt = f32(torch.tensor(float(dt), dtype=torch.float64), r).item()      # the kernels take dt as a float
    p, t = p0, t0
    P, F = [], []
    acc = torch.zeros_like(p0)
    for e in range(n_eval):
        f = forward_eval(net, p, t, terms)
        P.append(p), F.append(f)
        if e < n_acc:
            acc = f32(acc + f['s'], r)
        p = f32(p + f['s'], r)
        t = f32(t + dt, r) if t is not None else None
    a = None
    g_w = [0.0] * LAYERS
    g_b = [0.0] * LAYERS
    for e in range(n_eval - 1, -1, -1):
        d = dgrad_eval(net, P[e], F[e]['mask'], a, g_acc if e < n_acc else None,
                       g_steps[e] if g_steps is not None else None, terms)
        a = d['a_out']
        w, b = wgrad([x[0] for x in F[e]['x']], [y[0] for y in d['dy']])
        g_w = [g_w[l] + w[l] for l in range(LAYERS)]
        g_b = [g_b[l] + (b[l] if l < 5 else d['gb5']) for l in range(LAYERS)]
    return {'acc': acc, 's': [f['s'] for f in F], 'g_p': a, 'g_w': g_w, 'g_b': g_b}


def to_px(x):
    """[B, C, H, W] -> [B * H * W, C] in the kernels' pixel order (g = b * hw + i)"""
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1])


def from_px(x, B, H, W):
    return x.reshape(B, H, W, -1).permute(0, 3, 1, 2).contiguous()


# ---- metrics ----------------------------------------------------------------------------------------------------------------
def plane_agreement(k_bits, emu):
    """kernel bf16 bit plane vs the emulated value (fp64, rounded here): share of elements that differ, share more than one
    bf16 step off, and the largest error of those relative to the plane's maximum"""
    e_bits = bf16_bits(emu)
    kv, ev = bits_to_f64(k_bits), bits_to_f64(e_bits)
    d = (k_bits.int() - e_bits.int()).abs()
    diff = (d != 0) & (kv != ev)
    far = diff & (d > 1)
    n = max(k_bits.numel(), 1)
    scale = max(float(ev.abs().max()), 1e-30) if ev.numel() else 1.0
    far_rel = float(((kv - ev).abs() * far).max()) / scale if far.any() else 0.0
    return float(diff.sum()) / n, float(far.sum()) / n, far_rel


def rel_max(a, b):
    """max |a - b| / max |b|"""
    a, b = a.double(), b.double()
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)


def chunk_effect(x_hi, dy_hi, g_w, valid):
    """the least change of g_w (max-norm, relative to its maximum) that dropping one 64-pixel chunk with at least one valid pixel
    makes: min over chunks of max |Σ_chunk dY ⊗ X| / max |g_w|"""
    n = x_hi.shape[0] // CHUNK
    part = torch.einsum('qpo,qpi->qoi', dy_hi.reshape(n, CHUNK, -1), x_hi.reshape(n, CHUNK, -1))
    eff = part.abs().amax((1, 2)) / max(float(g_w.abs().max()), 1e-30)
    keep = valid.reshape(n, CHUNK).any(1)
    return float(eff[keep].min())
