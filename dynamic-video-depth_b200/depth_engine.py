"""MiDaS depth net (D1 + D1' of SURVEY.md 8(a)) on the repo's own kernels, forward AND backward, scheduled explicitly.

Replaces `MidasNet.forward` of the reference (third_party/MiDaS.py:206-246, third_party/midas_blocks.py:48-68,102-168, the
torchvision ResNeXt101-32x8d behind torch.hub) and the autograd graph PyTorch would build for it: no cuDNN, no ATen
elementwise kernels. Every convolution is a wgmma TF32 launch of csrc/conv2d_tc.cu with its neighbours folded into the
epilogue; the schedule below is written once per direction:

  forward   stem (CUDA cores: Cin = 3) -> max-pool -> 33 bottlenecks [conv1+bn1+relu | grouped conv2+bn2+relu |
            conv3+bn3+identity+relu] -> layerN_rn (+ the in-place ReLU of the first RCU) -> 4 fusion blocks
            [RCU = conv+bias+relu | conv+bias+skip(+other path)(+relu of the next RCU)], x2 bilinear -> head.
  backward  the mirror image: each data-gradient launch adds the skip gradient and applies the ReLU mask of the tensor it
            differentiates in its epilogue, so the only elementwise kernels left are per-channel sums (bias / BatchNorm
            gradients), the x2 bilinear adjoint, max-pool and the CUDA-core stem / head.
  BatchNorm is in eval mode on this path (models/scene_flow_motion_field.py:157,168) with trainable gamma / beta:
            d beta = sum gm, d gamma = rstd * (<W, sum gm x> - mean * sum gm) needs no saved pre-BN activation.

Parameter gradients are ACCUMULATED into `p.grad` (the flat gradient buffer of dvd_b200.flat.FlatParams; created on demand
otherwise) — the engine is the owner of the depth net's backward, autograd only sees one node (`MidasFunction`).
Activations handed between convolutions are stored TF32-rounded (rounded-operand contract, conv_ops.py).
"""
import os

import torch

from . import conv_ops as co
from .conv_ops import Conv

_NORM_MEAN = (0.485, 0.456, 0.406)
_NORM_STD = (0.229, 0.224, 0.225)


class _Block:
    """torchvision Bottleneck (ResNeXt): conv1/bn1, conv2/bn2 (32 groups, stride), conv3/bn3, optional downsample."""

    def __init__(self, m):
        self.c1, self.c2, self.c3 = Conv(m.conv1, m.bn1), Conv(m.conv2, m.bn2), Conv(m.conv3, m.bn3)
        self.ds = Conv(m.downsample[0], m.downsample[1]) if m.downsample is not None else None

    def convs(self):
        return [c for c in (self.c1, self.c2, self.c3, self.ds) if c is not None]


class _RCU:
    def __init__(self, m):
        self.c1, self.c2 = Conv(m.conv1), Conv(m.conv2)


class MidasEngine:
    def __init__(self, net):
        p, s = net.pretrained, net.scratch
        self.net = net
        self.normalize = bool(net.normalize_input)
        self.stem_conv, self.stem_bn = p.layer1[0], p.layer1[1]
        self.stages = [[_Block(b) for b in p.layer1[4]], [_Block(b) for b in p.layer2], [_Block(b) for b in p.layer3],
                       [_Block(b) for b in p.layer4]]
        self.rn = [Conv(s.layer1_rn), Conv(s.layer2_rn), Conv(s.layer3_rn), Conv(s.layer4_rn)]
        self.rcu_a = [_RCU(getattr(s, 'refinenet%d' % i).resConfUnit1) for i in (1, 2, 3, 4)]   # on layerN_rn (unused for 4)
        self.rcu_b = [_RCU(getattr(s, 'refinenet%d' % i).resConfUnit2) for i in (1, 2, 3, 4)]
        self.oc0, self.oc2, self.oc4 = Conv(s.output_conv[0]), Conv(s.output_conv[2]), s.output_conv[4]
        self._all = [c for st in self.stages for b in st for c in b.convs()] + self.rn
        self._all += [c for r in self.rcu_a[:3] + self.rcu_b for c in (r.c1, r.c2)] + [self.oc0, self.oc2]
        self.saved = None           # what backward() needs, kept by a training forward
        self._table = None
        self._sides = {}            # device index -> side stream of the two-stream backward
        self._side = None           # the side stream of the backward in progress
        self._keep = []
        # called as grad_hook(stage) at the points of backward() where a contiguous block of parameter gradients is final:
        # 'decoder+layer4', 'layer3', 'rest' - the data-parallel path all-reduces that block while the backward goes on
        self.grad_hook = None

    # ---------------------------------------------------------------------------------------------------
    # Two-stream backward: the weight gradient of a layer depends only on tensors the data-gradient chain has already produced
    # (the layer's input activation and the masked gradient of its output): it is issued on a SIDE stream behind an event, while
    # the main stream goes on with the data gradient. Both kernels are persistent one-CTA-per-SM grids, so the hardware fills the
    # SMs a finishing grid leaves idle (its last, partly empty wave; launch latency; prologue) with CTAs of the other stream.
    # Tensors handed to the side stream are kept alive until the next join (the caching allocator would otherwise hand their
    # memory to the main stream while the side stream still reads it). The weight-gradient launches take no stream-K exchange
    # area, so the data-gradient launches on the main stream keep theirs to themselves.
    def _on_side(self, fn, *keep):
        if os.environ.get('DVD_BWD_OVERLAP', '1') == '0':
            fn()
            return
        ev = torch.cuda.Event()
        ev.record()
        self._side.wait_event(ev)
        with torch.cuda.stream(self._side):
            fn()
        self._keep.extend(keep)

    def _stage_done(self, stage):
        """the parameter gradients of `stage` are final once the main stream has joined the side stream: hand them to grad_hook"""
        ev = torch.cuda.Event()
        ev.record(self._side)
        torch.cuda.current_stream().wait_event(ev)
        self._keep.clear()
        if self.grad_hook is not None:
            self.grad_hook(stage)

    # ---------------------------------------------------------------------------------------------------
    def pack(self, need_bwd=True):
        if self._table is None:
            self._table = co.PackTable(self._all)
        self._table.pack(need_bwd)

    def _ensure_grads(self):
        for p in self.net.parameters():
            if p.grad is None:
                p.grad = torch.zeros_like(p)

    # ---------------------------------------------------------------------------------------------------
    def forward(self, x, train):
        """x [N,3,H,W] raw image in [0,1] (contiguous fp32 CUDA) -> depth [N,1,H,W]. train=True keeps what backward needs.
        H and W must be positive multiples of 32: layer4 runs at 1/32 of the image, and at any other size the x2 up-sampled
        decoder path no longer matches the skip tensor it is added to (the convolution epilogue would read it with the wrong
        strides). Checked before any launch."""
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError('the MiDaS engine takes an image batch [N,3,H,W], got %s' % (tuple(x.shape),))
        N, _, H, W = x.shape
        if N < 1 or H < 32 or W < 32 or H % 32 or W % 32:
            raise ValueError('the MiDaS engine runs at sizes whose height and width are positive multiples of 32, got %d x %d '
                             '(batch %d)' % (H, W, N))
        self.pack(need_bwd=train)
        x = x.contiguous()
        nm, ns = (_NORM_MEAN, _NORM_STD) if self.normalize else (None, None)
        a0 = co.stem_fwd(x, self.stem_conv, self.stem_bn, nm, ns)
        a1, pool_idx = co.maxpool_fwd(a0)
        S = {'x': x, 'a0': a0, 'pool_idx': pool_idx, 'blocks': []} if train else None
        cur = a1
        feats = []
        for st in self.stages:
            for b in st:
                idt = b.ds.fwd(cur, round_out=False) if b.ds is not None else cur
                y1 = b.c1.fwd(cur, relu=True)
                y2 = b.c2.fwd(y1, relu=True)
                y3 = b.c3.fwd(y2, res=idt, relu=True)
                if train:
                    S['blocks'].append((cur, y1, y2))
                cur = y3
            feats.append(cur)
        l1, l2, l3, l4 = feats
        # the first RCU of every fusion block applies its ReLU in place to layerN_rn's output (midas_blocks.py:121): fused here
        lr = [self.rn[i].fwd(feats[i], relu=True) for i in range(4)]
        dec = []
        path = None
        for K in (3, 2, 1, 0):              # refinenet4 .. refinenet1
            if path is None:
                t, c1a = lr[K], None
            else:
                ra = self.rcu_a[K]
                c1a = ra.c1.fwd(lr[K], relu=True)
                t = ra.c2.fwd(c1a, res=lr[K], res2=path, relu=True)     # relu(path + RCU1(layerK_rn)): the ReLU is RCU2's
            rb = self.rcu_b[K]
            c1b = rb.c1.fwd(t, relu=True)
            o = rb.c2.fwd(c1b, res=t)
            path = co.upsample2x_fwd(o, True)
            dec.append((c1a, t, c1b))
        h0 = self.oc0.fwd(path, round_out=False)
        h1 = co.upsample2x_fwd(h0, False)
        h2 = self.oc2.fwd(h1, relu=True, round_out=False)
        depth = co.head_fwd(h2, self.oc4.weight, self.oc4.bias)
        if train:
            S.update(feats=feats, lr=lr, dec=dec, p1=path, h1=h1, h2=h2)
        self.saved = S
        return depth

    # ---------------------------------------------------------------------------------------------------
    def backward(self, g_depth):
        """Accumulates dL/dparam into .grad for every parameter of the net, given dL/ddepth [N,1,H,W]."""
        S, self.saved = self.saved, None
        if S is None:
            raise RuntimeError('MidasEngine.backward without a training forward')
        self._ensure_grads()
        g_depth = g_depth.contiguous()
        dev = torch.cuda.current_device()
        if dev not in self._sides:
            self._sides[dev] = torch.cuda.Stream(device=dev)
        self._side = self._sides[dev]
        oc4 = self.oc4
        gm_h2 = co.head_bwd(S['h2'], oc4.weight, oc4.bias, g_depth, oc4.weight.grad, oc4.bias.grad, relu_mask=True)
        H1, W1 = S['h1'].shape[2:]
        self._on_side(lambda x_=S['h1'], g_=gm_h2: self.oc2.wgrad(x_, g_, sums=True), S['h1'], gm_h2)
        g_h1 = self.oc2.dgrad(gm_h2, H1, W1, round_out=False)
        g_h0 = co.upsample2x_bwd(g_h1, False)
        self._on_side(lambda x_=S['p1'], g_=g_h0: self.oc0.wgrad(x_, g_, sums=True), S['p1'], g_h0)
        g_path = self.oc0.dgrad(g_h0, H1 // 2, W1 // 2, round_out=False)
        g_feat = [None] * 4
        for j, K in enumerate((0, 1, 2, 3)):      # refinenet1 .. refinenet4
            c1a, t, c1b = S['dec'][3 - j]
            lrK = S['lr'][K]
            g_o = co.upsample2x_bwd(g_path, True)
            Hk, Wk = g_o.shape[2:]
            rb = self.rcu_b[K]
            self._on_side(lambda x_=c1b, g_=g_o: rb.c2.wgrad(x_, g_, sums=True), c1b, g_o)
            g_c1b = rb.c2.dgrad(g_o, Hk, Wk, mask=c1b)
            self._on_side(lambda x_=t, g_=g_c1b: rb.c1.wgrad(x_, g_, sums=True), t, g_c1b)
            g_t = rb.c1.dgrad(g_c1b, Hk, Wk, res=g_o, mask=t)       # w.r.t. the pre-ReLU sum (t itself for refinenet4)
            if c1a is not None:
                ra = self.rcu_a[K]
                g_path = g_t                                         # the other fusion input: previous path
                self._on_side(lambda x_=c1a, g_=g_t: ra.c2.wgrad(x_, g_, sums=True), c1a, g_t)
                g_c1a = ra.c2.dgrad(g_t, Hk, Wk, mask=c1a)
                self._on_side(lambda x_=lrK, g_=g_c1a: ra.c1.wgrad(x_, g_, sums=True), lrK, g_c1a)
                g_lr = ra.c1.dgrad(g_c1a, Hk, Wk, res=g_t, mask=lrK)
            else:
                g_lr = g_t
            self._on_side(lambda x_=S['feats'][K], g_=g_lr: self.rn[K].wgrad(x_, g_), S['feats'][K], g_lr)
            g_feat[K] = self.rn[K].dgrad(g_lr, Hk, Wk, round_out=False)
        # encoder: gm3 = masked gradient w.r.t. the pre-ReLU output of the block being differentiated
        l4 = S['feats'][3]
        gm3 = co.relu_bwd_colsum(g_feat[3], y=l4, gm=torch.empty_like(l4))
        bi = len(S['blocks'])
        g_in = None
        for si in (3, 2, 1, 0):
            st = self.stages[si]
            for k in range(len(st) - 1, -1, -1):
                bi -= 1
                b = st[k]
                x_in, y1, y2 = S['blocks'][bi]
                Hi, Wi = x_in.shape[2:]
                Ho, Wo = y2.shape[2:]
                self._on_side(lambda x_=y2, g_=gm3: b.c3.wgrad(x_, g_, sums=True), y2, gm3)
                gm2 = b.c3.dgrad(gm3, Ho, Wo, mask=y2)
                self._on_side(lambda x_=y1, g_=gm2: b.c2.wgrad(x_, g_, sums=True), y1, gm2)
                gm1 = b.c2.dgrad(gm2, Hi, Wi, mask=y1)
                self._on_side(lambda x_=x_in, g_=gm1: b.c1.wgrad(x_, g_, sums=True), x_in, gm1)
                first = si == 0 and k == 0
                # the block input is the previous block's ReLU output (mask) - and, at a stage boundary, also a decoder input
                extra = g_feat[si - 1] if (k == 0 and si > 0) else None
                if b.ds is not None:
                    self._on_side(lambda x_=x_in, g_=gm3: b.ds.wgrad(x_, g_, sums=True), x_in, gm3)
                    g_ds = b.ds.dgrad(gm3, Hi, Wi, round_out=False)
                    g_in = b.c1.dgrad(gm1, Hi, Wi, res=g_ds, res2=extra, mask=None if first else x_in, round_out=not first)
                else:
                    g_in = b.c1.dgrad(gm1, Hi, Wi, res=gm3, res2=extra, mask=x_in)
                gm3 = g_in
            if si in (3, 2):
                self._stage_done('decoder+layer4' if si == 3 else 'layer3')
        a0 = S['a0']
        g_a0 = co.maxpool_bwd(g_in, S['pool_idx'], a0.shape[2], a0.shape[3])
        # issued while the last weight gradients are still running on the side stream
        nm, ns = (_NORM_MEAN, _NORM_STD) if self.normalize else (None, None)
        co.stem_wgrad(S['x'], g_a0, a0, self.stem_conv, self.stem_bn, nm, ns)
        self._stage_done('rest')


class MidasFunction(torch.autograd.Function):
    """depth = MiDaS(x) as ONE autograd node; its backward runs the engine's explicit schedule and deposits the parameter
    gradients in `.grad` (the image itself gets no gradient: it is data)."""

    @staticmethod
    def forward(ctx, x, token, engine):
        ctx.engine = engine
        return engine.forward(x, train=True)

    @staticmethod
    def backward(ctx, g):
        ctx.engine.backward(g)
        return None, None, None
