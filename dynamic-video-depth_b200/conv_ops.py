"""Python face of the depth-net kernels (csrc/conv2d_tc.cu, csrc/depth_ops.cu): descriptors, output allocation, checks.

Everything here works on channels-last fp32 CUDA tensors (logical [N,C,H,W], memory NHWC) under the ROUNDED-OPERAND
CONTRACT of the tensor-core convolutions: the operands of a convolution (activations forward, gradients backward)
must already hold TF32-rounded values; every producer below has a `round_out` switch and `round_tf32` admits foreign
tensors. No autograd here — the MiDaS engine (depth_engine.py) schedules forward and backward explicitly.
"""
import ctypes

import torch

from . import _lib
from ._lib import ConvDesc, DVD_CONV_MAX_TAPS
from .ops import LAUNCHES, _ptr, _stream, _ws, ordered, ordered_workspace

GROUP_BLOCK = 64     # grouped convolutions run as block-diagonal GEMM blocks of this many channels

# bench.py's live roofline probe: when a list, every tensor-core launch is bracketed by CUDA events on the launching stream and
# appended as (kind, algorithmic FLOPs, start event, end event); None (the default) adds nothing to the launch path
PROFILE = None


def _prof(kind, flops, desc=None):
    if PROFILE is None:
        return None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    info = (desc.N, desc.H, desc.W, desc.Cin, desc.OH, desc.OW, desc.Cout, desc.stride, desc.ntaps, desc.kblock) if desc is not None else None
    PROFILE.append((kind, flops, e0, e1, info))
    return e1


def _cl(t, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32):
        raise ValueError('%s must be a float32 CUDA tensor (dvd_b200 has no CPU path)' % name)
    if t.dim() != 4 or not t.is_contiguous(memory_format=torch.channels_last):
        raise ValueError('%s must be a channels-last [N,C,H,W] tensor' % name)
    return t


def empty_cl(N, C, H, W, device):
    return torch.empty((N, C, H, W), dtype=torch.float32, device=device, memory_format=torch.channels_last)


def round_tf32(x, out=None):
    out = torch.empty_like(x) if out is None else out
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_round_tf32(_ptr(x), _ptr(out), x.numel(), _stream()), 'dvd_round_tf32')
    return out


# ------------------------------------------------------------------------------------------------
# tap tables

def fwd_taps(k, pad):
    return [(ky - pad, kx - pad, ky * k + kx) for ky in range(k) for kx in range(k)]


def dgrad_taps_s1(k, pad):
    """gx[y, x] = sum_{ky,kx} gy[y + pad - ky, x + pad - kx] * W[.., ky, kx]"""
    return [(pad - ky, pad - kx, ky * k + kx) for ky in range(k) for kx in range(k)]


def dgrad_phase_taps_s2(k, pad, a, b):
    """stride-2 data gradient, sub-pixel phase (a, b): output pixels (2i + a, 2j + b) read gy[i + dy, j + dx] for the taps
    whose parity matches: (2i + a + pad - ky) even."""
    out = []
    for ky in range(k):
        if (a + pad - ky) % 2:
            continue
        for kx in range(k):
            if (b + pad - kx) % 2:
                continue
            out.append(((a + pad - ky) // 2, (b + pad - kx) // 2, ky * k + kx))
    return out


def make_desc(N, H, W, Cin, OH, OW, Cout, taps, stride=1, kblock=0, YH=None, YW=None, out_map=(1, 0, 1, 0), relu=False,
              round_out=True, bn_eps=0.0):
    if not 1 <= len(taps) <= DVD_CONV_MAX_TAPS:
        raise ValueError('1..%d taps' % DVD_CONV_MAX_TAPS)
    d = ConvDesc()
    d.N, d.H, d.W, d.Cin, d.OH, d.OW, d.Cout = N, H, W, Cin, OH, OW, Cout
    d.stride, d.ntaps, d.kblock = stride, len(taps), kblock
    d.YH, d.YW = (OH if YH is None else YH), (OW if YW is None else YW)
    d.oy_mul, d.oy_add, d.ox_mul, d.ox_add = out_map
    d.relu, d.round_out, d.bn_eps = int(bool(relu)), int(bool(round_out)), float(bn_eps)
    for i, (dy, dx, wt) in enumerate(taps):
        d.dy[i], d.dx[i], d.wt[i] = dy, dx, wt
    return d


# ------------------------------------------------------------------------------------------------
# raw launches

_WORKSPACE = {}     # device index -> zero-initialised exchange area of the stream-K schedule (dvd_conv2d_nhwc_ws)


def conv_workspace(device):
    """The exchange area of the convolution kernel's stream-K schedule on this device, one for every caller that passes it to
    conv2d_launch. Never allocated during a graph capture (the eager warm-up steps before a capture allocate it)."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    ws = _WORKSPACE.get(idx)
    if ws is None:
        if torch.cuda.is_current_stream_capturing():
            return None
        ws = torch.zeros(_lib.load().dvd_conv2d_workspace_bytes() // 4, dtype=torch.float32, device=torch.device('cuda', idx))
        torch.cuda.current_stream(idx).synchronize()
        _WORKSPACE[idx] = ws
    return ws


def conv2d_launch(desc, x, w_img, y, bias=None, bn=None, res=None, res2=None, mask=None, flops=0.0, kind='conv', workspace=None):
    """One tensor-core convolution. workspace=None runs whole tiles only, so a pixel's sum order does not depend on the other
    pixels of the launch. With conv_workspace(device) the layers whose whole tiles would leave much of the machine idle take the
    stream-K schedule instead. The caller must guarantee that launches sharing an exchange area are ordered on one stream, and a
    caller that runs convolutions concurrently on several streams passes none: a stream-K launch spins in its finishing CTAs until
    the CTAs holding the rest of their tiles have run, which is only deadlock-free when no other spinning launch can occupy the SMs
    those CTAs wait for."""
    g, b, m, v = bn if bn is not None else (None, None, None, None)
    LAUNCHES['n'] += 1
    ev = _prof(kind, flops, desc)
    ws_bytes = workspace.numel() * 4 if workspace is not None else 0
    _lib.check(_lib.load().dvd_conv2d_nhwc_ws(ctypes.byref(desc), _ptr(x), _ptr(w_img), _ptr(bias), _ptr(g), _ptr(b), _ptr(m), _ptr(v),
                                              _ptr(res), _ptr(res2), _ptr(mask), _ptr(y), _ptr(workspace), ws_bytes, _stream()),
               'dvd_conv2d_nhwc_ws')
    if ev is not None:
        ev.record()
    return y


def pack_weight(weight, groups=1, bn=None, out_fwd=None, out_bwd=None, want_fwd=True, want_bwd=True):
    """weight [Cout, Cin/groups, k, k] (any strides) -> TF32-rounded images (see dvd_conv2d_pack), both from one launch:
    forward [k*k][Cout][cols] and data gradient [k*k][Cin][cols] (scaled by the eval-BatchNorm factor of `bn` = (gamma, var, eps)).
    Returns (fwd, bwd); an image that is not wanted is None."""
    co, cil, kh, kw = weight.shape
    ci = cil * groups
    kblock = GROUP_BLOCK if groups > 1 else 0
    if want_fwd and out_fwd is None:
        out_fwd = torch.empty(kh * kw, co, kblock if kblock else ci, dtype=torch.float32, device=weight.device)
    if want_bwd and out_bwd is None:
        out_bwd = torch.empty(kh * kw, ci, kblock if kblock else co, dtype=torch.float32, device=weight.device)
    st = weight.stride()
    g, v, eps = bn if bn is not None else (None, None, 0.0)
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_conv2d_pack(_ptr(weight), st[0], st[1], st[2], st[3], _ptr(out_fwd if want_fwd else None),
                                           _ptr(out_bwd if want_bwd else None), co, ci, kh, groups, kblock, _ptr(g), _ptr(v), float(eps),
                                           _stream()), 'dvd_conv2d_pack')
    return (out_fwd if want_fwd else None), (out_bwd if want_bwd else None)


class PackTable:
    """Every convolution of a net packed by ONE launch per step (dvd_conv2d_pack_batch): a device-resident table of
    dvd_pack_item, rebuilt only when a parameter, BatchNorm buffer or image tensor has moved."""

    def __init__(self, convs):
        self.convs = list(convs)
        self.key = None
        self.table = None
        self.total = 0

    def _key(self):
        k = []
        for c in self.convs:
            k.append(c.conv.weight.data_ptr())
            k.append(c.w_fwd.data_ptr() if c.w_fwd is not None else 0)
            k.append(c.w_bwd.data_ptr() if c.w_bwd is not None else 0)
            if c.bn is not None:
                k.append(c.bn.weight.data_ptr())
                k.append(c.bn.running_var.data_ptr())
        return tuple(k)

    def _build(self, need_bwd):
        lib = _lib.load()
        items = (_lib.PackItem * len(self.convs))()
        blk = 0
        for it, c in zip(items, self.convs):
            w = c.conv.weight
            co, cil, kh, kw = w.shape
            ci = cil * c.groups
            dev = w.device
            if c.w_fwd is None:
                c.w_fwd = torch.empty(kh * kw, co, c.kblock if c.kblock else ci, dtype=torch.float32, device=dev)
            if need_bwd and c.w_bwd is None:
                c.w_bwd = torch.empty(kh * kw, ci, c.kblock if c.kblock else co, dtype=torch.float32, device=dev)
            st = w.stride()
            it.weight, it.w_fwd, it.w_bwd = w.data_ptr(), c.w_fwd.data_ptr(), (c.w_bwd.data_ptr() if c.w_bwd is not None else None)
            if c.bn is not None:
                it.bn_gamma, it.bn_var, it.bn_eps = c.bn.weight.data_ptr(), c.bn.running_var.data_ptr(), float(c.bn.eps)
            it.s_co, it.s_ci, it.s_ky, it.s_kx = st
            it.Cout, it.Cin, it.ksize, it.groups, it.kblock = co, ci, kh, c.groups, c.kblock
            it.blk0 = blk
            nb = lib.dvd_conv2d_pack_blocks(co, ci, kh, c.groups, c.kblock)
            if nb < 1:
                raise ValueError('dvd_conv2d_pack_batch works on 32 x 32 channel tiles: Cout, Cin (and kblock) must be multiples of 32')
            blk += nb
        raw = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8)
        self.table = raw.to(self.convs[0].conv.weight.device)
        self.total = blk

    def pack(self, need_bwd=True):
        if not self.convs[0].conv.weight.is_cuda:
            raise ValueError('dvd_b200 has no CPU path: the depth net must live on a CUDA device')
        if need_bwd and any(c.w_bwd is None for c in self.convs):
            self.key = None
        if self.key is None or self.key != self._key():
            self._build(need_bwd)
            self.key = self._key()
        LAUNCHES['n'] += 1
        _lib.check(_lib.load().dvd_conv2d_pack_batch(_ptr(self.table), len(self.convs), self.total, int(bool(need_bwd)), _stream()),
                   'dvd_conv2d_pack_batch')


def wgrad_launch(desc, x, gy, dweight, ksize, groups=1, weight=None, bn=None, dgamma=None, flops=0.0, colsum=None, bn_mean=None):
    st = dweight.stride()
    if weight is not None and weight.stride() != st:
        raise ValueError('parameter and gradient must share their strides')
    g, v = bn if bn is not None else (None, None)
    LAUNCHES['n'] += 1
    ev = _prof('wgrad', flops, desc)
    if ordered():
        LAUNCHES['n'] += 2
        ws = _ws(ordered_workspace(dweight.device, _lib.DVD_ORD_CONV_WGRAD))
        _lib.check(_lib.load().dvd_conv2d_wgrad_ordered(ctypes.byref(desc), _ptr(x), _ptr(gy), _ptr(dweight), _ptr(weight), st[0], st[1],
                                                        st[2], st[3], int(ksize), int(groups), _ptr(g), _ptr(v), _ptr(dgamma),
                                                        _ptr(colsum), _ptr(bn_mean), *ws, _stream()), 'dvd_conv2d_wgrad_ordered')
    else:
        _lib.check(_lib.load().dvd_conv2d_wgrad(ctypes.byref(desc), _ptr(x), _ptr(gy), _ptr(dweight), _ptr(weight), st[0], st[1], st[2],
                                                st[3], int(ksize), int(groups), _ptr(g), _ptr(v), _ptr(dgamma), _ptr(colsum),
                                                _ptr(bn_mean), _stream()), 'dvd_conv2d_wgrad')
    if ev is not None:
        ev.record()


def relu_bwd_colsum(g, y=None, gm=None, colsum=None, bn=None, dgamma=None, round_out=True):
    """gm = g * [y > 0] (rounded); colsum += per-channel sums; dgamma -= mean * rstd * sums. bn = (mean, var, eps)."""
    N, C, H, W = g.shape
    m, v, eps = bn if bn is not None else (None, None, 0.0)
    LAUNCHES['n'] += 1
    if ordered() and (colsum is not None or dgamma is not None):
        LAUNCHES['n'] += 1
        ws = _ws(ordered_workspace(g.device, _lib.DVD_ORD_CHANNEL_SUMS))
        _lib.check(_lib.load().dvd_relu_bwd_colsum_ordered(_ptr(g), _ptr(y), _ptr(gm), _ptr(colsum), _ptr(m), _ptr(v), float(eps),
                                                           _ptr(dgamma), N * H * W, C, int(bool(round_out)), *ws, _stream()),
                   'dvd_relu_bwd_colsum_ordered')
        return gm
    _lib.check(_lib.load().dvd_relu_bwd_colsum(_ptr(g), _ptr(y), _ptr(gm), _ptr(colsum), _ptr(m), _ptr(v), float(eps), _ptr(dgamma),
                                               N * H * W, C, int(bool(round_out)), _stream()), 'dvd_relu_bwd_colsum')
    return gm


def maxpool_fwd(x):
    N, C, H, W = _cl(x, 'x').shape
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = empty_cl(N, C, OH, OW, x.device)
    idx = torch.empty((N, OH, OW, C), dtype=torch.uint8, device=x.device)
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_maxpool3x3s2_fwd(_ptr(x), _ptr(y), _ptr(idx), N, H, W, C, _stream()), 'dvd_maxpool3x3s2_fwd')
    return y, idx


def maxpool_bwd(g, idx, H, W):
    N, C, OH, OW = _cl(g, 'g').shape
    gx = empty_cl(N, C, H, W, g.device)
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_maxpool3x3s2_bwd(_ptr(g), _ptr(idx), _ptr(gx), N, H, W, C, _stream()), 'dvd_maxpool3x3s2_bwd')
    return gx


def _f3(v):
    return (ctypes.c_float * 3)(*[float(a) for a in v]) if v is not None else None


def stem_fwd(x_nchw, conv, bn, norm_mean=None, norm_std=None, round_out=True):
    """relu(bn(conv7x7/2((x - mean) / std))) on the raw NCHW image -> channels-last [N,64,OH,OW]."""
    if not (x_nchw.is_cuda and x_nchw.dtype == torch.float32 and x_nchw.is_contiguous() and x_nchw.shape[1] == 3):
        raise ValueError('the stem needs a contiguous float32 CUDA image [N,3,H,W]')
    N, _, H, W = x_nchw.shape
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = empty_cl(N, 64, OH, OW, x_nchw.device)
    st = conv.weight.stride()
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_stem_fwd(_ptr(x_nchw), _ptr(conv.weight), st[0], st[1], st[2], st[3], _ptr(bn.weight), _ptr(bn.bias),
                                        _ptr(bn.running_mean), _ptr(bn.running_var), float(bn.eps), _f3(norm_mean), _f3(norm_std),
                                        _ptr(y), N, H, W, int(bool(round_out)), _stream()), 'dvd_stem_fwd')
    return y


def stem_wgrad(x_nchw, g, a0, conv, bn, norm_mean=None, norm_std=None):
    N, _, H, W = x_nchw.shape
    st = conv.weight.stride()
    if conv.weight.grad.stride() != st:
        raise ValueError('parameter and gradient must share their strides')
    scratch = torch.empty(147 * 64 + 64, dtype=torch.float32, device=g.device)
    LAUNCHES['n'] += 3
    args = (_ptr(x_nchw), _ptr(g), _ptr(a0), _ptr(conv.weight), _ptr(conv.weight.grad), st[0], st[1], st[2], st[3], _ptr(bn.weight),
            _ptr(bn.running_mean), _ptr(bn.running_var), float(bn.eps), _ptr(bn.weight.grad), _ptr(bn.bias.grad), _f3(norm_mean),
            _f3(norm_std), _ptr(scratch), N, H, W)
    if ordered():
        LAUNCHES['n'] += 1
        ws = _ws(ordered_workspace(g.device, _lib.DVD_ORD_STEM))
        _lib.check(_lib.load().dvd_stem_wgrad_ordered(*args, *ws, _stream()), 'dvd_stem_wgrad_ordered')
    else:
        _lib.check(_lib.load().dvd_stem_wgrad(*args, _stream()), 'dvd_stem_wgrad')


def head_fwd(x, weight, bias):
    """depth = 10000 / max(relu(conv1x1_{32->1}(x) + b), 1e-2): x channels-last [N,32,H,W] -> [N,1,H,W]."""
    N, C, H, W = _cl(x, 'x').shape
    if C != 32:
        raise ValueError('the head takes 32 channels')
    d = torch.empty((N, 1, H, W), dtype=torch.float32, device=x.device)
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_head_fwd(_ptr(x), _ptr(weight), _ptr(bias), _ptr(d), N * H * W, _stream()), 'dvd_head_fwd')
    return d


def head_bwd(x, weight, bias, g_depth, gw, gb, relu_mask=True, round_out=True):
    N, C, H, W = x.shape
    gx = torch.empty_like(x)
    LAUNCHES['n'] += 1
    args = (_ptr(x), _ptr(weight), _ptr(bias), _ptr(g_depth), _ptr(gx), _ptr(gw), _ptr(gb), N * H * W, int(bool(relu_mask)),
            int(bool(round_out)))
    if ordered():
        LAUNCHES['n'] += 1
        ws = _ws(ordered_workspace(x.device, _lib.DVD_ORD_HEAD))
        _lib.check(_lib.load().dvd_head_bwd_ordered(*args, *ws, _stream()), 'dvd_head_bwd_ordered')
    else:
        _lib.check(_lib.load().dvd_head_bwd(*args, _stream()), 'dvd_head_bwd')
    return gx


def upsample2x_fwd(x, align_corners, round_out=True):
    N, C, H, W = _cl(x, 'x').shape
    y = empty_cl(N, C, 2 * H, 2 * W, x.device)
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_upsample2x_fwd(_ptr(x), _ptr(y), N, H, W, C, int(bool(align_corners)), int(bool(round_out)), _stream()),
               'dvd_upsample2x_fwd')
    return y


def upsample2x_bwd(g, align_corners, round_out=True):
    N, C, OH, OW = _cl(g, 'g').shape
    H, W = OH // 2, OW // 2
    gx = empty_cl(N, C, H, W, g.device)
    LAUNCHES['n'] += 1
    _lib.check(_lib.load().dvd_upsample2x_bwd(_ptr(g), _ptr(gx), N, H, W, C, int(bool(align_corners)), int(bool(round_out)), _stream()),
               'dvd_upsample2x_bwd')
    return gx


# ------------------------------------------------------------------------------------------------
class Conv:
    """One convolution of the depth net (nn.Conv2d parameters, optionally followed by an eval-mode nn.BatchNorm2d) and its
    three tensor-core passes. Weight images are re-packed by `pack()` (once per optimisation step)."""

    def __init__(self, conv, bn=None):
        self.conv, self.bn = conv, bn
        self.k = conv.kernel_size[0]
        self.stride = conv.stride[0]
        self.pad = conv.padding[0]
        self.groups = conv.groups
        self.cin, self.cout = conv.in_channels, conv.out_channels
        if conv.kernel_size[0] != conv.kernel_size[1] or conv.stride[0] != conv.stride[1] or conv.dilation != (1, 1):
            raise ValueError('square, undilated convolutions only')
        if self.stride not in (1, 2):
            raise ValueError('stride 1 or 2')
        self.kblock = GROUP_BLOCK if self.groups > 1 else 0
        self.w_fwd = self.w_bwd = None

    # -- parameters ---------------------------------------------------------------------------------
    def _bn_fwd(self):
        b = self.bn
        return (b.weight, b.bias, b.running_mean, b.running_var) if b is not None else None

    def pack(self, need_bwd=True):
        w = self.conv.weight.detach()
        bn = (self.bn.weight.detach(), self.bn.running_var, self.bn.eps) if self.bn is not None else None
        f, b = pack_weight(w, self.groups, bn=bn, out_fwd=self.w_fwd, out_bwd=self.w_bwd, want_bwd=need_bwd)
        self.w_fwd = f
        if need_bwd:
            self.w_bwd = b

    def flops(self, N, OH, OW):
        """algorithmic FLOPs of one pass (forward = data gradient = weight gradient) over N x OH x OW output pixels"""
        return 2.0 * N * OH * OW * self.cout * (self.cin // self.groups) * self.k * self.k

    def out_hw(self, H, W):
        return (H + 2 * self.pad - self.k) // self.stride + 1, (W + 2 * self.pad - self.k) // self.stride + 1

    # -- forward: y = relu(bn(conv(x) + bias) + res + res2) ----------------------------------------------
    def fwd(self, x, res=None, res2=None, relu=False, round_out=True):
        N, C, H, W = x.shape
        OH, OW = self.out_hw(H, W)
        d = make_desc(N, H, W, self.cin, OH, OW, self.cout, fwd_taps(self.k, self.pad), self.stride, self.kblock, relu=relu,
                      round_out=round_out, bn_eps=self.bn.eps if self.bn is not None else 0.0)
        y = empty_cl(N, self.cout, OH, OW, x.device)
        return conv2d_launch(d, x, self.w_fwd, y, self.conv.bias, self._bn_fwd(), res, res2, flops=self.flops(N, OH, OW), kind='fwd',
                             workspace=conv_workspace(x.device))

    # -- data gradient: gx = [mask > 0] * (conv^T(gy) + res + res2);  gy must be the gradient w.r.t. the convolution's
    #    BatchNorm OUTPUT (the scale is folded into the weight image) -------------------------------------------------
    def dgrad(self, gy, H, W, res=None, res2=None, mask=None, round_out=True):
        N, Co, OH, OW = gy.shape
        gx = empty_cl(N, self.cin, H, W, gy.device)
        ws = conv_workspace(gy.device)
        if self.stride == 1:
            d = make_desc(N, OH, OW, self.cout, H, W, self.cin, dgrad_taps_s1(self.k, self.pad), 1, self.kblock, round_out=round_out)
            return conv2d_launch(d, gy, self.w_bwd, gx, res=res, res2=res2, mask=mask, flops=self.flops(N, OH, OW), kind='dgrad',
                                 workspace=ws)
        phases = [(a, b, dgrad_phase_taps_s2(self.k, self.pad, a, b)) for a in (0, 1) for b in (0, 1)]
        if any(not t for _, _, t in phases):
            if res is not None or res2 is not None or mask is not None:
                raise ValueError('epilogue fusion is not available for a strided data gradient with empty phases')
            gx.zero_()
        for a, b, taps in phases:
            if not taps:
                continue
            ph, pw = (H - a + 1) // 2, (W - b + 1) // 2
            if ph <= 0 or pw <= 0:
                continue
            d = make_desc(N, OH, OW, self.cout, ph, pw, self.cin, taps, 1, self.kblock, YH=H, YW=W, out_map=(2, a, 2, b),
                          round_out=round_out)
            conv2d_launch(d, gy, self.w_bwd, gx, res=res, res2=res2, mask=mask, kind='dgrad',
                          flops=self.flops(N, OH, OW) * len(taps) / (self.k * self.k), workspace=ws)
        return gx

    # -- weight gradient (accumulates into conv.weight.grad; BatchNorm: gy un-scaled, dgamma gets the <W, dW> term). With
    #    `sums` the same launch reduces gy over the pixels: conv-bias gradient, or BatchNorm beta + the mean term of gamma ------
    def can_fuse_sums(self):
        return self.groups > 1 or self.cout % 128 == 0

    def wgrad(self, x, gy, sums=False):
        N, C, H, W = x.shape
        _, Co, OH, OW = gy.shape
        w = self.conv.weight
        d = make_desc(N, H, W, self.cin, OH, OW, self.cout, fwd_taps(self.k, self.pad), self.stride,
                      bn_eps=self.bn.eps if self.bn is not None else 0.0)
        fuse = sums and self.can_fuse_sums() and (self.bn is not None or self.conv.bias is not None)
        if sums and not fuse:
            self.bias_or_bn_grad(gy)
        if self.bn is not None:
            wgrad_launch(d, x, gy, w.grad, self.k, self.groups, weight=w.detach(), bn=(self.bn.weight.detach(), self.bn.running_var),
                         dgamma=self.bn.weight.grad, flops=self.flops(N, OH, OW), colsum=self.bn.bias.grad if fuse else None,
                         bn_mean=self.bn.running_mean if fuse else None)
        else:
            wgrad_launch(d, x, gy, w.grad, self.k, self.groups, flops=self.flops(N, OH, OW),
                         colsum=self.conv.bias.grad if fuse else None)

    def bias_or_bn_grad(self, gm):
        """per-channel sums of the masked gradient in a kernel of their own (layers whose weight-gradient launch cannot carry them):
        conv bias gradient, or BatchNorm beta gradient + the mean term of gamma's."""
        if self.bn is not None:
            relu_bwd_colsum(gm, colsum=self.bn.bias.grad, bn=(self.bn.running_mean, self.bn.running_var, self.bn.eps),
                            dgamma=self.bn.weight.grad, round_out=False)
        elif self.conv.bias is not None:
            relu_bwd_colsum(gm, colsum=self.conv.bias.grad, round_out=False)
