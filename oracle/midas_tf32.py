"""TEST INFRASTRUCTURE — fp64 emulation of the MiDaS engine's arithmetic (dvd_b200.depth_engine.MidasEngine).

The STRUCTURE is the reference's (the functional, state-dict-driven form of oracle.depth_nets.midas_forward); the PRECISION
MODEL is the engine's rounded-operand contract (DESIGN.md §2.1):

  * every tensor a tensor-core convolution consumes is rounded to TF32 where it is produced (fp64 -> fp32 -> cvt.rna), and every
    consumer sees the rounded value. Not rounded, as in the engine: the down-sample branch outputs (the residual of conv3),
    output_conv.0 / output_conv.2 outputs (h0, h2) and the depth map;
  * in the backward, the gradient w.r.t. every convolution's output sum (post-BatchNorm / post-bias, plus residuals, before the
    ReLU) is rounded to TF32: that is the operand of the layer's data- and weight-gradient launches. The stem's gradient is not
    (CUDA-core fp32 in the engine);
  * convolutions use the engine's packed weight images: the forward image (tf32(W)) forward, the data-gradient image
    (tf32(W * gamma * rsqrt(var + eps)), the BatchNorm scale folded in) for the data gradient; the weight gradient uses the plain
    fp32 weight where the engine does (BatchNorm gamma: rstd * (<W, sum gm x> - mean * sum gm));
  * stem, max-pool, x2 bilinear up-sampling and the head follow their CUDA-core fp32 definitions (plain weights, no rounding
    except the stem output).

Each convolution is one autograd node (`_ConvLayer`) because its data gradient runs through an image autograd cannot derive from
the forward; everything around it (BatchNorm-free sums, ReLU masks, up-sampling, max-pool, stem, head) is torch autograd.

Teacher forcing: with `anchors` (the tensors the engine saves for its backward) the emulation re-synchronises at each of them:
the anchor records how far the emulated value is from the engine's, then continues with the engine's value; gradients pass
straight through. ReLU masks and max-pool argmaxes come from the engine's activations, so a flip near zero or a near-tie cannot
make the emulated backward drift from the engine's.

With rounding=False and images=None the emulation is midas_forward + autograd in fp64 (tests/test_midas_tf32_oracle_cpu.py).
"""
import torch
import torch.nn.functional as F

_BN_EPS = 1e-5
_MEAN = (0.485, 0.456, 0.406)
_STD = (0.229, 0.224, 0.225)
GROUP_BLOCK = 64        # block width of the block-diagonal image of a grouped convolution (conv_ops.GROUP_BLOCK)
STAGES = (('layer1.4', 3, 1), ('layer2', 4, 2), ('layer3', 23, 2), ('layer4', 3, 2))


def round_tf32(t):
    """t (any float dtype) -> the TF32 value cvt.rna.tf32.f32 makes of fp32(t), in t's dtype (round to nearest, ties away)"""
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32).to(t.dtype)


# ---- packed weight images (csrc/conv2d_tc.cu, conv_pack_kernel) -------------------------------------------------------------
def _group_index(Cout, Cin, groups, device):
    cpg, opg = Cin // groups, Cout // groups
    co = torch.arange(Cout, device=device).view(-1, 1).expand(Cout, cpg)
    ci = (co // opg) * cpg + torch.arange(cpg, device=device).view(1, -1)
    return co, ci


def image_index(Cout, Cin, groups, mode, device):
    """(row, column) of weight[co, j] in the forward (mode 0, [t][co][c]) or data-gradient (mode 1, [t][ci][c]) image, both
    [Cout, Cin / groups]. Grouped layers store one GROUP_BLOCK-wide block-diagonal block per row."""
    co, ci = _group_index(Cout, Cin, groups, device)
    kb = GROUP_BLOCK if groups > 1 else 0
    if mode == 0:
        return co, (ci - (co // kb) * kb if kb else ci)
    return ci, (co - (ci // kb) * kb if kb else co)


def unpack_image(img, Cout, Cin, k, groups, mode):
    """packed image [k*k][rows][cols] -> weight layout [Cout, Cin / groups, k, k]"""
    r, c = image_index(Cout, Cin, groups, mode, img.device)
    return img[:, r, c].permute(1, 2, 0).reshape(Cout, Cin // groups, k, k)


def off_group_entries(img, Cout, Cin, groups, mode):
    """the image with every entry that belongs to a weight zeroed: what is left must be zero (block-diagonal padding)"""
    r, c = image_index(Cout, Cin, groups, mode, img.device)
    out = img.clone()
    out[:, r, c] = 0
    return out


# ---- autograd pieces --------------------------------------------------------------------------------------------------------
class _RoundValue(torch.autograd.Function):
    """forward: TF32-round the value (an activation a convolution will read); backward: identity"""

    @staticmethod
    def forward(ctx, x):
        return round_tf32(x)

    @staticmethod
    def backward(ctx, g):
        return g


class _RoundGrad(torch.autograd.Function):
    """forward: identity; backward: TF32-round the gradient (it is a data- / weight-gradient operand)"""

    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return round_tf32(g)


class _MaskedRelu(torch.autograd.Function):
    """relu(x) whose backward mask is given (the engine's activation > 0) instead of derived from x"""

    @staticmethod
    def forward(ctx, x, mask):
        ctx.save_for_backward(mask)
        return x.clamp(min=0)

    @staticmethod
    def backward(ctx, g):
        mask, = ctx.saved_tensors
        return g * mask, None


class _Anchor(torch.autograd.Function):
    """forward: the engine's value; backward: the gradient passes to the emulated value unchanged"""

    @staticmethod
    def forward(ctx, emu, ref):
        return ref.clone()

    @staticmethod
    def backward(ctx, g):
        return g, None


class _ConvLayer(torch.autograd.Function):
    """y = conv(x, wf) * sc + sh with sc = gamma * rstd, sh = beta - mean * sc (eval BatchNorm), or + bias, or plain.
    Backward (gm = dL/dy): dx = conv^T(gm, wb) with wb the data-gradient image (BatchNorm scale folded in); dW = sc * (x * gm);
    dgamma = rstd * (<W, x * gm> - mean * sum gm); dbeta = dbias = sum gm. Identical to autograd of the unfused layer when
    wf = W and wb = W * sc."""

    @staticmethod
    def forward(ctx, x, w, gamma, beta, bias, wf, wb, mean, var, stride, pad, groups):
        ctx.conf = (stride, pad, groups, gamma is not None, bias is not None)
        z = F.conv2d(x, wf, None, stride, pad, 1, groups)
        if gamma is not None:
            rstd = (var + _BN_EPS).rsqrt()
            sc = gamma * rstd
            z = z * sc.view(1, -1, 1, 1) + (beta - mean * sc).view(1, -1, 1, 1)
        elif bias is not None:
            z = z + bias.view(1, -1, 1, 1)
        ctx.save_for_backward(x, w, gamma, wb, mean, var)
        return z

    @staticmethod
    def backward(ctx, gm):
        x, w, gamma, wb, mean, var = ctx.saved_tensors
        stride, pad, groups, has_bn, has_bias = ctx.conf
        dx = dw = dgamma = dbeta = dbias = None
        if ctx.needs_input_grad[0]:
            dx = torch.nn.grad.conv2d_input(x.shape, wb, gm, stride, pad, 1, groups)
        dwu = torch.nn.grad.conv2d_weight(x, w.shape, gm, stride, pad, 1, groups)
        s = gm.sum((0, 2, 3))
        if has_bn:
            rstd = (var + _BN_EPS).rsqrt()
            dw = dwu * (gamma * rstd).view(-1, 1, 1, 1)
            dgamma = rstd * ((w * dwu).sum((1, 2, 3)) - mean * s)
            dbeta = s
        else:
            dw = dwu
            dbias = s if has_bias else None
        return dx, dw, dgamma, dbeta, dbias, None, None, None, None, None, None, None


# ---- anchors ----------------------------------------------------------------------------------------------------------------
def anchor_names(n_blocks=33):
    """names of the tensors the engine saves for its backward, in forward order (pool_idx is used, not compared)"""
    names = ['a0']
    bi = 0
    for si, (_, n, _) in enumerate(STAGES):
        for i in range(n):
            # the input of a stage's first block is the previous stage's output: checked as feat<si - 1>
            names += (['block%d.cur' % bi] if (i > 0 or si == 0) else []) + ['block%d.y1' % bi, 'block%d.y2' % bi]
            bi += 1
        names.append('feat%d' % si)
    names += ['lr%d' % i for i in range(4)]
    for K in (3, 2, 1, 0):
        names += (['refinenet%d.c1a' % (K + 1), 'refinenet%d.t' % (K + 1)] if K < 3 else []) + ['refinenet%d.c1b' % (K + 1)]
    return names + ['p1', 'h1', 'h2']


def engine_anchors(S):
    """a lane's saved dict of MidasEngine._forward_one -> {anchor name: tensor}"""
    A = {'a0': S['a0'], 'pool_idx': S['pool_idx']}
    for bi, (cur, y1, y2) in enumerate(S['blocks']):
        A['block%d.cur' % bi], A['block%d.y1' % bi], A['block%d.y2' % bi] = cur, y1, y2
    for i in range(4):
        A['feat%d' % i], A['lr%d' % i] = S['feats'][i], S['lr'][i]
    for j, K in enumerate((3, 2, 1, 0)):
        c1a, t, c1b = S['dec'][j]
        if c1a is not None:
            A['refinenet%d.c1a' % (K + 1)], A['refinenet%d.t' % (K + 1)] = c1a, t
        A['refinenet%d.c1b' % (K + 1)] = c1b
    A['p1'], A['h1'], A['h2'] = S['p1'], S['h1'], S['h2']
    return A


class Anchors:
    """teacher forcing at the engine's tensors (name -> fp32 tensor, any memory format; pool_idx [N,OH,OW,C] uint8) and the
    record of how far each emulated value was from it: for TF32-rounded tensors the share of elements that differ, the share
    that differ by more than one TF32 step (a neighbouring TF32 value), and the max-norm error relative to the tensor's max."""

    def __init__(self, tensors, dtype=torch.float64):
        self.t, self.dtype = tensors, dtype
        self.report = {}

    def __contains__(self, name):
        return name in self.t

    def value(self, name):
        return self.t[name].to(self.dtype).contiguous()

    def pool_idx(self):
        return self.t['pool_idx'].permute(0, 3, 1, 2).long()

    def record(self, name, emu, ref, rounded):
        e32, r32 = emu.detach().float().contiguous(), ref.float().contiguous()
        err = float((emu.detach() - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)
        rec = {'n': emu.numel(), 'rel_max': err, 'rounded': rounded}
        if rounded:
            d = (e32.view(torch.int32).long() - r32.view(torch.int32).long()).abs()
            rec['diff'] = float((d != 0).double().mean())
            rec['far'] = float(((d != 0) & (d != 0x2000)).double().mean())
            rec['far_rel_max'] = float(((emu.detach() - ref).abs() * ((d != 0) & (d != 0x2000))).max()) / max(float(ref.abs().max()), 1e-30)
        self.report[name] = rec


# ---- the net ----------------------------------------------------------------------------------------------------------------
class _Emu:
    def __init__(self, sd, images, rounding, anchors):
        self.sd, self.images, self.rounding, self.A = sd, images, rounding, anchors

    def rv(self, t):
        return _RoundValue.apply(t) if self.rounding else t

    def rg(self, t):
        return _RoundGrad.apply(t) if self.rounding else t

    def anchor(self, name, emu, rounded):
        if self.A is None or name is None or name not in self.A:
            return emu
        ref = self.A.value(name)
        self.A.record(name, emu, ref, rounded)
        return _Anchor.apply(emu, ref)

    def conv(self, pre, x, stride=1, pad=0, groups=1, bn=None):
        sd = self.sd
        w = sd[pre + '.weight']
        gamma = beta = mean = var = None
        if bn is not None:
            gamma, beta, mean, var = (sd[bn + s] for s in ('.weight', '.bias', '.running_mean', '.running_var'))
        if self.images is not None:
            wf, wb = self.images[pre]
        else:
            wf = w.detach()
            wb = (w * (gamma * (var + _BN_EPS).rsqrt()).view(-1, 1, 1, 1)).detach() if bn is not None else w.detach()
        return _ConvLayer.apply(x, w, gamma, beta, sd.get(pre + '.bias'), wf, wb, mean, var, stride, pad, groups)

    def act(self, s, name, relu=True, round_value=True, round_grad=True):
        """s = a layer's output sum -> (gradient rounded) -> ReLU -> (value rounded) -> anchor"""
        if round_grad:
            s = self.rg(s)
        if relu:
            if self.A is not None and name in self.A:
                s = _MaskedRelu.apply(s, (self.A.t[name] > 0).contiguous())
            else:
                s = F.relu(s)
        if round_value:
            s = self.rv(s)
        return self.anchor(name, s, round_value and self.rounding)

    def maxpool(self, a0):
        if self.A is None or 'pool_idx' not in self.A:
            return F.max_pool2d(a0, 3, stride=2, padding=1)
        N, C, H, W = a0.shape
        OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        win = F.unfold(F.pad(a0, (1, 1, 1, 1), value=float('-inf')), 3, stride=2).view(N, C, 9, OH, OW)
        idx = self.A.pool_idx()
        self.A.report['pool_idx'] = {'n': idx.numel(), 'flips': float((win.detach().argmax(2) != idx).double().mean())}
        return win.gather(2, idx.unsqueeze(2)).squeeze(2)

    def forward(self, x, normalize_input=True):
        sd = self.sd
        if normalize_input:
            x = (x - torch.tensor(_MEAN, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)) / \
                torch.tensor(_STD, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
        p = 'pretrained.'
        # stem: CUDA cores, plain fp32 weights; the output is a convolution operand (rounded), its gradient is not
        z = F.conv2d(x, sd[p + 'layer1.0.weight'], None, 2, 3)
        z = F.batch_norm(z, sd[p + 'layer1.1.running_mean'], sd[p + 'layer1.1.running_var'], sd[p + 'layer1.1.weight'],
                         sd[p + 'layer1.1.bias'], training=False, eps=_BN_EPS)
        a0 = self.act(z, 'a0', round_grad=False)
        cur = self.anchor('block0.cur', self.maxpool(a0), self.rounding)
        feats = []
        bi = 0
        for si, (stage, n, stride) in enumerate(STAGES):
            for i in range(n):
                b = '%s%s.%d' % (p, stage, i)
                s = stride if i == 0 else 1
                y1 = self.act(self.conv(b + '.conv1', cur, bn=b + '.bn1'), 'block%d.y1' % bi)
                y2 = self.act(self.conv(b + '.conv2', y1, s, 1, 32, bn=b + '.bn2'), 'block%d.y2' % bi)
                idt = cur
                if (b + '.downsample.0.weight') in sd:
                    idt = self.conv(b + '.downsample.0', cur, s, bn=b + '.downsample.1')
                    idt = self.anchor('block%d.ds' % bi, idt, False)
                y3 = self.conv(b + '.conv3', y2, bn=b + '.bn3') + idt
                cur = self.act(y3, ('feat%d' % si) if i == n - 1 else ('block%d.cur' % (bi + 1)))
                bi += 1
            feats.append(cur)
        s_ = 'scratch.'
        lr = [self.act(self.conv(s_ + 'layer%d_rn' % (i + 1), feats[i], pad=1), 'lr%d' % i) for i in range(4)]
        path = None
        for K in (3, 2, 1, 0):
            rn = s_ + 'refinenet%d' % (K + 1)
            if path is None:
                t = lr[K]
            else:
                c1a = self.act(self.conv(rn + '.resConfUnit1.conv1', lr[K], pad=1), rn[len(s_):] + '.c1a')
                t = self.act(self.conv(rn + '.resConfUnit1.conv2', c1a, pad=1) + lr[K] + path, rn[len(s_):] + '.t')
            c1b = self.act(self.conv(rn + '.resConfUnit2.conv1', t, pad=1), rn[len(s_):] + '.c1b')
            o = self.act(self.conv(rn + '.resConfUnit2.conv2', c1b, pad=1) + t, None, relu=False)
            path = self.rv(F.interpolate(o, scale_factor=2, mode='bilinear', align_corners=True))
        path = self.anchor('p1', path, self.rounding)
        h0 = self.act(self.conv(s_ + 'output_conv.0', path, pad=1), None, relu=False, round_value=False)
        h1 = self.anchor('h1', self.rv(F.interpolate(h0, scale_factor=2, mode='bilinear', align_corners=False)), self.rounding)
        h2 = self.act(self.conv(s_ + 'output_conv.2', h1, pad=1), 'h2', round_value=False)
        # head: CUDA cores, plain weights
        o = F.relu(F.conv2d(h2, sd[s_ + 'output_conv.4.weight'], sd[s_ + 'output_conv.4.bias']))
        return 10000.0 / torch.clamp(o, min=1e-2)


def midas_tf32_forward(sd, x, images=None, rounding=True, anchors=None, normalize_input=True):
    """depth [N,1,H,W] of MiDaS under the engine's precision model. sd: state dict (floating leaves may require grad; use fp64);
    images: {conv name: (forward image, data-gradient image)} in weight layout (unpack_image), None = the plain weights;
    rounding: TF32 rounding of operands and operand gradients; anchors: Anchors of the engine's saved tensors, or None."""
    return _Emu(sd, images, rounding, anchors).forward(x, normalize_input)
