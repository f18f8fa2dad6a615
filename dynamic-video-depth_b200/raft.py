"""RAFT optical flow (forward only) on the kernels of libdvd_b200.so, for the configuration the reference's flow stage
uses and no other (scripts/preprocess/davis/generate_flows.py: third_party/RAFT/core, large model, all-pairs correlation, 4 levels,
radius 4, hidden = context = 128, no warm start, test_mode).

`RaftNet` holds the parameters under the reference's names, so `raft-sintel.pth` loads (a leading `module.` is accepted).
Both encoders work per image (InstanceNorm normalises every sample on its own, the context encoder's BatchNorm is in eval
mode), so `encode()` runs them once per frame and `flow()` reuses the features for every pair the frame takes part in;
the reference re-runs both encoders for every pair. `forward(image1, image2)` is the drop-in for RAFT.forward(test_mode=True).

Convolutions with tensor-core shapes run on dvd_conv2d_nhwc (TF32, rounded-operand contract, whole tiles only so that a
pixel's result does not depend on the batch it is computed in); everything else is csrc/raft_ops.cu. CUDA only.
"""
import torch
import torch.nn as nn

from . import _lib, conv_ops
from .conv_ops import conv2d_launch, make_desc, pack_weight
from .ops import LAUNCHES, _ptr, _stream

LOOKUP_CHANNELS = 352          # 4 levels x 81 samples = 324, zero-padded to a multiple of 32 for the 1x1 convolution behind it
MIN_SIDE = 128                 # the coarsest of the four pyramid levels must be at least 2 x 2 (the reference's lookup returns NaN below)


def check_size(H, W):
    if H % 8 or W % 8:
        raise ValueError('RAFT images must have height and width divisible by 8 (the reference feeds 288x512 and does not pad), '
                         'got %dx%d' % (H, W))
    if H < MIN_SIDE or W < MIN_SIDE:
        raise ValueError('RAFT images must be at least %dx%d: the lookup of the coarsest correlation level divides by its size '
                         'minus one, got %dx%d' % (MIN_SIDE, MIN_SIDE, H, W))


# ------------------------------------------------------------------------------------------------
# parameters, under the reference's names

class _Block(nn.Module):
    def __init__(self, cin, dim, stride, batch_norm):
        super().__init__()
        self.stride = stride
        self.conv1 = nn.Conv2d(cin, dim, 3, padding=1, stride=stride)
        self.conv2 = nn.Conv2d(dim, dim, 3, padding=1)
        if batch_norm:
            self.norm1, self.norm2 = nn.BatchNorm2d(dim), nn.BatchNorm2d(dim)
        if stride != 1:
            ds = [nn.Conv2d(cin, dim, 1, stride=stride)]
            if batch_norm:
                self.norm3 = nn.BatchNorm2d(dim)
                ds.append(self.norm3)          # one module under two names, as in the reference's checkpoint
            self.downsample = nn.Sequential(*ds)


class _Encoder(nn.Module):
    def __init__(self, batch_norm):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3)
        if batch_norm:
            self.norm1 = nn.BatchNorm2d(64)
        self.layer1 = nn.Sequential(_Block(64, 64, 1, batch_norm), _Block(64, 64, 1, batch_norm))
        self.layer2 = nn.Sequential(_Block(64, 96, 2, batch_norm), _Block(96, 96, 1, batch_norm))
        self.layer3 = nn.Sequential(_Block(96, 128, 2, batch_norm), _Block(128, 128, 1, batch_norm))
        self.conv2 = nn.Conv2d(128, 256, 1)

    def blocks(self):
        return list(self.layer1) + list(self.layer2) + list(self.layer3)


BLOCK_NAMES = ('layer1.0', 'layer1.1', 'layer2.0', 'layer2.1', 'layer3.0', 'layer3.1')     # _Encoder.blocks(), the reference's names


class _MotionEncoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.convc1 = nn.Conv2d(324, 256, 1)
        self.convc2 = nn.Conv2d(256, 192, 3, padding=1)
        self.convf1 = nn.Conv2d(2, 128, 7, padding=3)
        self.convf2 = nn.Conv2d(128, 64, 3, padding=1)
        self.conv = nn.Conv2d(256, 126, 3, padding=1)


class _Gru(nn.Module):
    def __init__(self):
        super().__init__()
        for g in 'zrq':
            setattr(self, 'conv%s1' % g, nn.Conv2d(384, 128, (1, 5), padding=(0, 2)))
        for g in 'zrq':
            setattr(self, 'conv%s2' % g, nn.Conv2d(384, 128, (5, 1), padding=(2, 0)))


class _FlowHead(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(128, 256, 3, padding=1)
        self.conv2 = nn.Conv2d(256, 2, 3, padding=1)


class _UpdateBlock(nn.Module):
    def __init__(self):
        super().__init__()
        self.encoder, self.gru, self.flow_head = _MotionEncoder(), _Gru(), _FlowHead()
        self.mask = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 576, 1))


# ------------------------------------------------------------------------------------------------
# launches. Activations are plain contiguous [N,H,W,C] fp32 tensors.

def _raft(name, *args):
    LAUNCHES['n'] += 1
    _lib.check(getattr(_lib.load(), name)(*args, _stream()), name)


class _TC:
    """One dvd_conv2d_nhwc launch: weight [Cout,Cin,kh,kw] packed once (TF32-rounded, tap-major), bias and eval BatchNorm in
    the epilogue."""

    def __init__(self, weight, bias, stride=1, padding=(0, 0), bn=None, relu=False, round_out=True):
        weight = weight.detach()
        co, ci, kh, kw = weight.shape
        if kh == kw:
            self.image, _ = pack_weight(weight, want_bwd=False)
        else:                                   # 1x5 / 5x1: the pack kernel takes square kernels, so one 1x1 slice per tap
            self.image = torch.empty(kh * kw, co, ci, dtype=torch.float32, device=weight.device)
            for ky in range(kh):
                for kx in range(kw):
                    t = ky * kw + kx
                    pack_weight(weight[:, :, ky:ky + 1, kx:kx + 1], out_fwd=self.image[t:t + 1], want_bwd=False)
        self.taps = [(ky - padding[0], kx - padding[1], ky * kw + kx) for ky in range(kh) for kx in range(kw)]
        self.cin, self.cout, self.k, self.stride, self.padding = ci, co, (kh, kw), stride, padding
        self.bias = bias.detach().contiguous() if bias is not None else None
        self.bn = tuple(t.detach() for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var)) if bn is not None else None
        self.bn_eps = bn.eps if bn is not None else 0.0
        self.relu, self.round_out = relu, round_out

    def flops(self, npx_out):
        return 2.0 * npx_out * self.cout * self.cin * self.k[0] * self.k[1]

    def __call__(self, x, res=None):
        N, H, W, C = x.shape
        assert C == self.cin and x.is_contiguous()
        OH = (H + 2 * self.padding[0] - self.k[0]) // self.stride + 1
        OW = (W + 2 * self.padding[1] - self.k[1]) // self.stride + 1
        d = make_desc(N, H, W, self.cin, OH, OW, self.cout, self.taps, self.stride, relu=self.relu, round_out=self.round_out,
                      bn_eps=self.bn_eps)
        y = torch.empty(N, OH, OW, self.cout, dtype=torch.float32, device=x.device)
        return conv2d_launch(d, x, self.image, y, self.bias, self.bn, res, flops=self.flops(N * OH * OW), kind='raft')


def instnorm_stats(x):
    """x [N,H,W,C] -> stats [N,C,2] = (mean, 1 / sqrt(var + 1e-5)) per image and channel (biased variance)"""
    N, H, W, C = x.shape
    stats = torch.empty(N, C, 2, dtype=torch.float32, device=x.device)
    nbytes = _lib.load().dvd_raft_instnorm_scratch_bytes(N, C)
    scratch = torch.empty(nbytes // 8, dtype=torch.float64, device=x.device)
    _raft('dvd_raft_instnorm_stats', _ptr(x), _ptr(stats), _ptr(scratch), nbytes, N, H * W, C, 1e-5)
    return stats


def norm_act(x, stats=None, res=None, relu_inner=False, relu_outer=False, round_out=True):
    N, H, W, C = x.shape
    y = torch.empty_like(x)
    _raft('dvd_raft_norm_act', _ptr(x), _ptr(stats), _ptr(res), _ptr(y), N, H * W, C, int(relu_inner), int(relu_outer), int(round_out))
    return y


def raft_stem(images, weight, bias):
    """[N,3,H,W] in 0..255 -> conv7x7/2(2 (x / 255) - 1) + bias, [N,H/2,W/2,64]"""
    N, _, H, W = images.shape
    y = torch.empty(N, H // 2, W // 2, 64, dtype=torch.float32, device=images.device)
    _raft('dvd_raft_stem_fwd', _ptr(images), _ptr(weight), _ptr(bias), _ptr(y), y.numel() * 4, N, H, W)
    return y


def corr_pyramid(fmap1, fmap2):
    """fmaps [B,h,w,C] -> the four correlation levels in one flat buffer (see dvd_raft_corr_pyramid)"""
    B, h, w, C = fmap1.shape
    n = _lib.load().dvd_raft_pyramid_floats(B, h, w)
    if n < 0:
        raise ValueError('a %dx%d feature grid leaves a correlation level under 2x2' % (h, w))
    pyr = torch.empty(n, dtype=torch.float32, device=fmap1.device)
    LAUNCHES['n'] += 3
    _raft('dvd_raft_corr_pyramid', _ptr(fmap1), _ptr(fmap2), _ptr(pyr), n * 4, B, h, w, C)
    return pyr


def pyramid_levels(pyr, B, h, w):
    """views [B*h*w, h_l, w_l] of the flat pyramid buffer"""
    out, off = [], 0
    P = B * h * w
    hl, wl = h, w
    for _ in range(4):
        out.append(pyr[off:off + P * hl * wl].view(P, hl, wl))
        off += P * hl * wl
        hl, wl = hl // 2, wl // 2
    return out


def lookup(pyr, coords1, round_out=True):
    B, h, w, _ = coords1.shape
    out = torch.empty(B, h, w, LOOKUP_CHANNELS, dtype=torch.float32, device=coords1.device)
    _raft('dvd_raft_lookup', _ptr(pyr), pyr.numel() * 4, _ptr(coords1), _ptr(out), out.numel() * 4, B, h, w, int(round_out))
    return out


def upsample(masks, coords1, mask_scale=0.25):
    """masks: three [B,h,w,192] tensors (channels 0..191, 192..383, 384..575 of the mask head) -> flow [B,8h,8w,2]"""
    B, h, w, _ = coords1.shape
    flow = torch.empty(B, 8 * h, 8 * w, 2, dtype=torch.float32, device=coords1.device)
    _raft('dvd_raft_upsample', _ptr(masks[0]), _ptr(masks[1]), _ptr(masks[2]), _ptr(coords1), _ptr(flow), flow.numel() * 4, B, h, w,
          float(mask_scale))
    return flow


def _keep(trace, name, t):
    """trace[name] = a copy of t as it is now: X, XR, net and coords1 are overwritten in place later in the same iteration"""
    if trace is not None:
        trace[name] = t.clone()


def coords_grid(B, h, w, device):
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32, device=device), torch.arange(w, dtype=torch.float32, device=device),
                            indexing='ij')
    return torch.stack([xs, ys], -1)[None].repeat(B, 1, 1, 1).contiguous()


# ------------------------------------------------------------------------------------------------
class FrameFeatures:
    """Per-frame encoder outputs on the device: fmap [N,h,w,256] (feature encoder) and cnet [N,h,w,256] (context encoder,
    before its tanh / relu split), NHWC fp32."""

    def __init__(self, fmap, cnet):
        self.fmap, self.cnet = fmap, cnet

    def __len__(self):
        return self.fmap.shape[0]

    def index(self, idx):
        idx = torch.as_tensor(idx, dtype=torch.long, device=self.fmap.device)
        return FrameFeatures(self.fmap.index_select(0, idx), self.cnet.index_select(0, idx))


class _Plan:
    """Everything derived from the parameters once per checkpoint: packed weight images and the merged / padded / split layers."""

    def __init__(self, net):
        self.f_blocks = [self._block(b, False) for b in net.fnet.blocks()]
        self.c_blocks = [self._block(b, True) for b in net.cnet.blocks()]
        self.f_out = _TC(net.fnet.conv2.weight, net.fnet.conv2.bias, round_out=False)
        self.c_out = _TC(net.cnet.conv2.weight, net.cnet.conv2.bias, round_out=False)
        # dvd_stem_fwd has no convolution bias: (conv + b - mean) * scale + beta = (conv - (mean - b)) * scale + beta
        self.c_stem_mean = (net.cnet.norm1.running_mean - net.cnet.conv1.bias).detach().contiguous()
        u, e, g = net.update_block, net.update_block.encoder, net.update_block.gru
        dev = e.convc1.weight.device
        w = torch.zeros(256, LOOKUP_CHANNELS, 1, 1, device=dev)
        w[:, :324] = e.convc1.weight.detach()
        self.convc1 = _TC(w, e.convc1.bias, relu=True)
        self.convc2 = _TC(e.convc2.weight, e.convc2.bias, padding=(1, 1), relu=True)
        self.convf2 = _TC(e.convf2.weight, e.convf2.bias, padding=(1, 1), relu=True)
        # conv(cat[cor 192 | flo 64]) as two launches, the second adding the first: no concatenated operand is built. 126 outputs are
        # padded to 128 with zero rows; the two flow channels take their place in the GRU operand, which is the reference's cat
        w = torch.zeros(128, 256, 3, 3, device=dev)
        w[:126] = e.conv.weight.detach()
        b = torch.zeros(128, device=dev)
        b[:126] = e.conv.bias.detach()
        self.conv_flo = _TC(w[:, 192:].contiguous(), None, padding=(1, 1), round_out=False)
        self.conv_cor = _TC(w[:, :192].contiguous(), b, padding=(1, 1), relu=True)
        self.gru = []
        for tag, pad in (('1', (0, 2)), ('2', (2, 0))):
            cz, cr, cq = (getattr(g, 'conv%s%s' % (k, tag)) for k in 'zrq')
            zr = _TC(torch.cat([cz.weight.detach(), cr.weight.detach()], 0), torch.cat([cz.bias.detach(), cr.bias.detach()], 0), padding=pad,
                     round_out=False)
            self.gru.append((zr, _TC(cq.weight, cq.bias, padding=pad, round_out=False)))
        self.fh1 = _TC(u.flow_head.conv1.weight, u.flow_head.conv1.bias, padding=(1, 1), relu=True, round_out=False)
        self.mask0 = _TC(u.mask[0].weight, u.mask[0].bias, padding=(1, 1), relu=True)
        # 576 outputs are neither <= 256 nor a multiple of 256: three launches of 192
        self.mask2 = [_TC(u.mask[2].weight[i * 192:(i + 1) * 192], u.mask[2].bias[i * 192:(i + 1) * 192], round_out=False) for i in range(3)]

    @staticmethod
    def _block(b, batch_norm):
        bn = (lambda name: getattr(b, name)) if batch_norm else (lambda name: None)
        c1 = _TC(b.conv1.weight, b.conv1.bias, stride=b.stride, padding=(1, 1), bn=bn('norm1'), relu=batch_norm, round_out=batch_norm)
        c2 = _TC(b.conv2.weight, b.conv2.bias, padding=(1, 1), bn=bn('norm2'), relu=batch_norm, round_out=False)
        ds = None
        if b.stride != 1:
            ds = _TC(b.downsample[0].weight, b.downsample[0].bias, stride=b.stride, bn=bn('norm3'), relu=batch_norm, round_out=batch_norm)
        return c1, c2, ds


class RaftNet(nn.Module):
    def __init__(self, small=False, alternate_corr=False, mixed_precision=False, dropout=0.0):
        super().__init__()
        if small or alternate_corr or mixed_precision or dropout:
            raise ValueError('RaftNet runs the reference flow stage\'s configuration only: small=False, alternate_corr=False, '
                             'mixed_precision=False, dropout=0')
        self.fnet, self.cnet, self.update_block = _Encoder(False), _Encoder(True), _UpdateBlock()
        self.eval()
        self._plan, self._plan_key = None, None

    def load_state_dict(self, state_dict, strict=True, **kw):
        sd = {(k[7:] if k.startswith('module.') else k): v for k, v in state_dict.items()}
        return super().load_state_dict(sd, strict=strict, **kw)

    def train(self, mode=True):
        if mode:
            raise NotImplementedError('RaftNet is inference only (BatchNorm in eval mode, no backward pass)')
        return super().train(False)

    def plan(self):
        key = tuple((t.data_ptr(), t._version) for t in list(self.parameters()) + list(self.buffers()))
        if self._plan is None or key != self._plan_key:
            if not next(self.parameters()).is_cuda:
                raise RuntimeError('RaftNet runs on the CUDA kernels of libdvd_b200.so only: dvd_b200 has no CPU path')
            with torch.no_grad():
                self._plan, self._plan_key = _Plan(self), key
        return self._plan

    # -- encoders -------------------------------------------------------------------------------------
    @staticmethod
    def _check_images(images):
        if not (torch.is_tensor(images) and images.is_cuda and images.dtype == torch.float32 and images.dim() == 4 and images.shape[1] == 3):
            raise ValueError('RAFT images must be a float32 CUDA tensor [N,3,H,W] holding 0..255 (dvd_b200 has no CPU path)')
        check_size(images.shape[2], images.shape[3])
        return images.contiguous()

    def feature_stem(self, images, trace=None):
        """relu(InstanceNorm(conv1(2 (x / 255) - 1))) of the feature encoder, [N,H/2,W/2,64]"""
        s = raft_stem(images, self.fnet.conv1.weight.detach().contiguous(), self.fnet.conv1.bias.detach())
        _keep(trace, 'fnet.stem', s)
        return norm_act(s, instnorm_stats(s), relu_inner=True)

    def context_stem(self, images):
        c, n = self.cnet.conv1, self.cnet.norm1
        y = conv_ops.stem_fwd(images, c, _Norm(n.weight.detach(), n.bias.detach(), self.plan().c_stem_mean, n.running_var, n.eps),
                              norm_mean=(127.5,) * 3, norm_std=(127.5,) * 3)
        return y.permute(0, 2, 3, 1)          # channels-last memory: a contiguous [N,H/2,W/2,64] view

    @torch.no_grad()
    def encode(self, images, trace=None):
        """images [N,3,H,W] fp32 in 0..255 on the device -> FrameFeatures of the N frames. trace: None, or a dict that receives
        a copy of every intermediate tensor under the names of oracle/raft_tf32.py (NHWC)"""
        images = self._check_images(images)
        P = self.plan()
        prev = conv_ops.set_workspace_lane(-1)
        try:
            x = self.feature_stem(images, trace)
            _keep(trace, 'fnet.stem.out', x)
            for name, (c1, c2, ds) in zip(BLOCK_NAMES, P.f_blocks):
                p = 'fnet.' + name + '.'
                a = c1(x)
                y = norm_act(a, instnorm_stats(a), relu_inner=True)
                b = c2(y)
                _keep(trace, p + 'a', a)
                _keep(trace, p + 'y', y)
                _keep(trace, p + 'b', b)
                if ds is None:
                    x = norm_act(b, instnorm_stats(b), res=x, relu_inner=True, relu_outer=True)
                else:
                    yb = norm_act(b, instnorm_stats(b), relu_inner=True, round_out=False)
                    d = ds(x)
                    x = norm_act(d, instnorm_stats(d), res=yb, relu_outer=True)
                    _keep(trace, p + 'yb', yb)
                    _keep(trace, p + 'd', d)
                _keep(trace, p + 'out', x)
            fmap = P.f_out(x)
            _keep(trace, 'fmap', fmap)
            x = self.context_stem(images)
            _keep(trace, 'cnet.stem.out', x)
            for name, (c1, c2, ds) in zip(BLOCK_NAMES, P.c_blocks):
                p = 'cnet.' + name + '.'
                y = c1(x)
                b = c2(y)
                # relu(x + relu(bn2(conv2))): the shortcut is added after the branch's own ReLU, so it is not the convolution's residual
                x = norm_act(b, res=x, relu_outer=True) if ds is None else ds(x, res=b)
                _keep(trace, p + 'y', y)
                _keep(trace, p + 'b', b)
                _keep(trace, p + 'out', x)
            cnet = P.c_out(x)
            _keep(trace, 'cnet', cnet)
            return FrameFeatures(fmap, cnet)
        finally:
            conv_ops.set_workspace_lane(prev)

    # -- update iterations ----------------------------------------------------------------------------
    def update_step(self, P, pyr, coords1, net, X, XR, net_r, want_delta=False, trace=None):
        """one iteration in place: coords1, net, X, XR, net_r are overwritten; returns (lookup output, delta_flow or None).
        trace: None, or a dict that receives a copy of every tensor of the iteration (names of oracle/raft_tf32.py, NHWC; the
        operand buffers as 'X.<stage>' / 'XR.<stage>' after each kernel that writes them)"""
        B, h, w, _ = coords1.shape
        npx = B * h * w
        e = self.update_block.encoder
        corr = lookup(pyr, coords1)
        c1 = P.convc1(corr)
        cor = P.convc2(c1)
        flo = torch.empty(B, h, w, 128, dtype=torch.float32, device=coords1.device)
        _raft('dvd_raft_convf1', _ptr(coords1), _ptr(e.convf1.weight.detach().contiguous()), _ptr(e.convf1.bias.detach()), _ptr(flo), B, h, w, 1)
        f2 = P.convf2(flo)
        m = P.conv_cor(cor, res=P.conv_flo(f2))
        _raft('dvd_raft_motion_pack', _ptr(m), _ptr(coords1), _ptr(X), _ptr(XR), B, h, w)
        if trace is not None:
            for name, t in (('corr', corr), ('convc1', c1), ('convc2', cor), ('convf1', flo), ('convf2', f2), ('motion', m),
                            ('X.pack', X), ('XR.pack', XR)):
                _keep(trace, name, t)
        for i, (zr_conv, q_conv) in enumerate(P.gru):
            zr = zr_conv(X)
            _raft('dvd_raft_gru_rh', _ptr(zr), _ptr(net), _ptr(XR), npx)
            _keep(trace, 'XR.rh.%d' % i, XR)
            q = q_conv(XR)
            _raft('dvd_raft_gru_update', _ptr(zr), _ptr(q), _ptr(net), _ptr(X), _ptr(net_r if i == 1 else None), npx)
            if trace is not None:
                for name, t in (('zr', zr), ('q', q), ('net', net), ('X.gru', X)):
                    _keep(trace, '%s.%d' % (name, i), t)
        fh = P.fh1(net_r)
        fhc = self.update_block.flow_head.conv2
        delta = torch.empty(B, h, w, 2, dtype=torch.float32, device=coords1.device) if want_delta or trace is not None else None
        _raft('dvd_raft_flow_head', _ptr(fh), _ptr(fhc.weight.detach().contiguous()), _ptr(fhc.bias.detach()), _ptr(coords1), _ptr(delta), B, h, w)
        if trace is not None:
            for name, t in (('net_r', net_r), ('fh', fh), ('delta', delta), ('coords1', coords1)):
                _keep(trace, name, t)
        return corr, delta

    def init_state(self, cnet, trace=None):
        """cnet [B,h,w,256] -> (net [B,h,w,128], X, XR [B,h,w,384], net_r [B,h,w,128]) with the tanh / relu halves in place"""
        B, h, w, _ = cnet.shape
        dev = cnet.device
        net, net_r = (torch.empty(B, h, w, 128, dtype=torch.float32, device=dev) for _ in range(2))
        X, XR = (torch.empty(B, h, w, 384, dtype=torch.float32, device=dev) for _ in range(2))
        _raft('dvd_raft_context_split', _ptr(cnet), _ptr(net), _ptr(X), _ptr(XR), B * h * w)
        if trace is not None:
            for name, t in (('net', net), ('X', X), ('XR', XR)):
                _keep(trace, name, t)
        return net, X, XR, net_r

    def mask_parts(self, P, net_r, trace=None):
        mk = P.mask0(net_r)
        parts = [c(mk) for c in P.mask2]
        if trace is not None:
            _keep(trace, 'mask0', mk)
            trace['mask'] = [t.clone() for t in parts]
        return parts

    @torch.no_grad()
    def flow(self, feat_a, feat_b, iters=20, return_low=False, trace=None):
        """flow from the frames of feat_a to those of feat_b, pair by pair: [B,H,W,2] fp32 (x, y), the layout of the flow-pair kernels.
        trace: None, or a dict that receives 'pyramid' (the flat buffer), the initial state ('net', 'X', 'XR'), one dict per
        iteration under 'iters' (see update_step), the mask head ('mask0', 'mask': the three parts) and 'flow_up'"""
        iters = int(iters)
        if iters < 1:
            raise ValueError('iters must be at least 1')
        if len(feat_a) != len(feat_b) or feat_a.fmap.shape != feat_b.fmap.shape:
            raise ValueError('feat_a and feat_b must hold the same number of frames of one size')
        P = self.plan()
        prev = conv_ops.set_workspace_lane(-1)
        try:
            fa, fb, cn = feat_a.fmap.contiguous(), feat_b.fmap.contiguous(), feat_a.cnet.contiguous()
            B, h, w, _ = fa.shape
            pyr = corr_pyramid(fa, fb)
            _keep(trace, 'pyramid', pyr)
            net, X, XR, net_r = self.init_state(cn, trace)
            coords1 = coords_grid(B, h, w, fa.device)
            for _ in range(iters):
                it = None
                if trace is not None:
                    it = {}
                    trace.setdefault('iters', []).append(it)
                self.update_step(P, pyr, coords1, net, X, XR, net_r, trace=it)
            up = upsample(self.mask_parts(P, net_r, trace), coords1)
            _keep(trace, 'flow_up', up)
            return (up, coords1 - coords_grid(B, h, w, fa.device)) if return_low else up
        finally:
            conv_ops.set_workspace_lane(prev)

    def forward(self, image1, image2, iters=20, flow_init=None, upsample=True, test_mode=True):
        """RAFT.forward(image1, image2, iters, test_mode=True) -> (flow_low [B,2,H/8,W/8], flow_up [B,2,H,W])"""
        if flow_init is not None or not test_mode or not upsample:
            raise ValueError('RaftNet.forward is the reference\'s test_mode=True call without a warm start')
        up, low = self.flow(self.encode(image1), self.encode(image2), iters, return_low=True)
        return low.permute(0, 3, 1, 2), up.permute(0, 3, 1, 2)


class _Norm:
    """the BatchNorm fields dvd_b200.conv_ops.stem_fwd reads"""

    def __init__(self, weight, bias, running_mean, running_var, eps):
        self.weight, self.bias, self.running_mean, self.running_var, self.eps = weight, bias, running_mean, running_var, eps


def load_raft(path, device='cuda'):
    """RaftNet with the parameters of a RAFT checkpoint (raft-sintel.pth as the reference uses it, or any state dict with its keys)"""
    net = RaftNet()
    net.load_state_dict(torch.load(path, map_location='cpu'))
    return net.to(device)
