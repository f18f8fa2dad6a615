"""TEST INFRASTRUCTURE — fp64 emulation of the RAFT forward's arithmetic (dvd_b200.raft.RaftNet).

The STRUCTURE is the reference's, through the functions of oracle/raft.py (NCHW, the reference's parameter names, its
layers in its order). It never reads RaftNet's plan: the plan's merged, split and padded layers (convc1 over 352 channels,
the motion encoder's last convolution as two launches with 126 outputs padded to 128, z and r in one 256-output launch, the
1x5 / 5x1 kernels as five 1x1 slices, the mask head as three launches of 192, the context stem's bias folded into the
BatchNorm mean, the flow written into channels 382/383 of the GRU operand) have no counterpart here, so a wiring error in
any of them is a distance between RaftNet and this emulation.

The PRECISION MODEL is RaftNet's. A tensor-core convolution (csrc/conv2d_tc.cu, rounded-operand contract) is an fp64
convolution of its operand, already rounded where it was produced, with round_tf32(W), followed by bias / eval BatchNorm /
residual / ReLU as in the kernel's epilogue. The CUDA-core stages (the stems, InstanceNorm, correlation and pooling, lookup,
convf1, the GRU gates, the flow head's last convolution, convex up-sampling) follow their fp32 definitions in fp64 with the
plain weights. TF32 rounding (fp64 -> fp32 -> cvt.rna) happens exactly where RaftNet rounds, and nowhere else:

  tensor (anchor name)       producer                                       rounded  consumer
  fnet.stem                  dvd_raft_stem_fwd, conv 7x7/2 + bias            no      InstanceNorm
  fnet.stem.out              norm_act relu(IN)                               yes     layer1.0 conv1, its shortcut
  fnet.<blk>.a               conv1                                           no      InstanceNorm
  fnet.<blk>.y               norm_act relu(IN(a))                            yes     conv2
  fnet.<blk>.b               conv2                                           no      InstanceNorm
  fnet.<blk>.yb              norm_act relu(IN(b)) (down-sampling blocks)     no      residual of the shortcut's norm_act
  fnet.<blk>.d               downsample conv (down-sampling blocks)          no      InstanceNorm
  fnet.<blk>.out             norm_act relu(relu(IN(b)) + x), relu(IN(d) + yb) yes    next block, fnet.conv2
  fmap                       fnet.conv2 1x1                                  no      correlation (CUDA cores)
  cnet.stem.out              dvd_stem_fwd relu(bn(conv))                     yes     layer1.0 conv1, its shortcut
  cnet.<blk>.y               conv1 + bn1 + relu                              yes     conv2
  cnet.<blk>.b               conv2 + bn2 + relu                              no      norm_act / downsample residual
  cnet.<blk>.out             relu(b + x), or downsample + bn3 + b + relu     yes     next block, cnet.conv2
  cnet                       cnet.conv2 1x1                                  no      context split
  net                        tanh(cnet[:, :128]), the hidden state           no      GRU (X[:, :128] holds round(net))
  inp                        relu(cnet[:, 128:])                             yes     X / XR[:, 128:256]
  pyramid.<l>                correlation / 2x2 pooling, fp32 FMA             no      lookup
  corr                       lookup, 324 channels + zero tail to 352         yes     convc1
  convc1, convc2             relu(conv)                                      yes     convc2, motion conv
  convf1                     dvd_raft_convf1 relu(conv 7x7 of the flow)      yes     convf2
  convf2                     relu(conv)                                      yes     motion conv
  motion                     relu(conv(cat[convc2, convf2])), 126 channels   yes     X / XR[:, 256:382]
  (flow)                     coords1 - coords0                               yes     X / XR[:, 382:384] as (x, y)
  z.<i>, r.<i>               convz / convr of GRU half i                     no      sigmoid
  rh.<i>                     sigmoid(r) * net                                yes     XR[:, :128], convq
  q.<i>                      convq                                           no      tanh
  net.<i>                    (1 - z) net + z tanh(q)                         no      next half (X[:, :128] holds round(net))
  net_r                      round(net) after the second half                yes     flow_head.conv1, mask.0
  fh                         relu(flow_head.conv1)                           no      flow_head.conv2 (CUDA cores)
  delta                      flow_head.conv2                                 no      coords1 += delta
  coords1                    coords1 + delta                                 no      next iteration
  mask0                      relu(mask.0)                                    yes     mask.2
  mask                       mask.2, 576 channels                            no      up-sampling (scaled by 0.25 there)
  flow_up                    softmax over 9 + convex 8x up-sampling          no      the caller

Teacher forcing: with `anchors` (an oracle.midas_tf32.Anchors of RaftNet's traced tensors in this module's names and layout,
see `encoder_anchors`, `state_anchors` and `iteration_anchors`) the emulation records its distance from RaftNet's tensor at each anchor and continues from RaftNet's
value, so every stage is checked on RaftNet's own inputs. Names of an update iteration carry the prefix given to `update`.

With rounding=False the emulation is oracle/raft.py in fp64 (tests/test_raft_tf32_oracle_cpu.py).
"""
import torch
import torch.nn.functional as F

from oracle import raft as ref
from oracle.midas_tf32 import Anchors, round_tf32  # noqa: F401  (Anchors: the record the tests read)

HDIM = ref.HDIM
LOOKUP_CHANNELS = ref.LEVELS * ref.WINDOW * ref.WINDOW
BLOCKS = (('layer1.0', 1), ('layer1.1', 1), ('layer2.0', 2), ('layer2.1', 1), ('layer3.0', 2), ('layer3.1', 1))   # (name, stride)


def lookup(pyr, coords1):
    """oracle.raft.lookup in pixel coordinates, as dvd_raft_lookup defines it: bilinear between the four neighbours of
    (x / 2^l + i - 4, y / 2^l + j - 4), zero outside. grid_sample's normalised-coordinate round trip would leave weights of
    about 1e-16 on neighbours an integer coordinate does not touch, which read as far-off TF32 values next to RaftNet's zeros"""
    N, _, h, w = coords1.shape
    P = N * h * w
    c = coords1.permute(0, 2, 3, 1).reshape(P, 1, 1, 2)
    off = ref.window_offsets(coords1.dtype, coords1.device)[None]
    out = []
    for l, corr in enumerate(pyr):
        H, W = corr.shape[-2:]
        m = corr.reshape(P, H * W)
        p = c / 2 ** l + off
        x0, y0 = torch.floor(p[..., 0]), torch.floor(p[..., 1])
        ax, ay = p[..., 0] - x0, p[..., 1] - y0

        def tap(x, y):
            inside = (x >= 0) & (x < W) & (y >= 0) & (y < H)
            idx = (y.clamp(0, H - 1) * W + x.clamp(0, W - 1)).long().reshape(P, -1)
            return torch.where(inside, m.gather(1, idx).reshape(x.shape), torch.zeros((), dtype=m.dtype, device=m.device))
        v = (1 - ay) * ((1 - ax) * tap(x0, y0) + ax * tap(x0 + 1, y0)) + ay * ((1 - ax) * tap(x0, y0 + 1) + ax * tap(x0 + 1, y0 + 1))
        out.append(v.reshape(N, h, w, ref.WINDOW * ref.WINDOW))
    return torch.cat(out, -1).permute(0, 3, 1, 2)


class RaftTF32:
    """sd: the reference's state dict in fp64 (oracle.raft.cast); rounding: RaftNet's TF32 rounding of operands and weights;
    anchors: Anchors of RaftNet's tensors, or None; trace: None, or a dict that receives every anchor-named value this
    emulation computes (before teacher forcing replaces it)."""

    def __init__(self, sd, rounding=True, anchors=None, trace=None):
        self.sd, self.rounding, self.A, self.trace = sd, rounding, anchors, trace
        self.prefix = ''
        self._w = {}

    # -- rounding points and anchors ------------------------------------------------------------------
    def rv(self, t):
        return round_tf32(t) if self.rounding else t

    def anchor(self, name, emu, rounded):
        name = self.prefix + name
        if self.trace is not None:
            self.trace[name] = emu
        if self.A is None or name not in self.A:
            return emu
        engine = self.A.value(name)
        self.A.record(name, emu, engine, rounded and self.rounding)
        return engine

    def tc(self, name, x, stride=1, padding=0):
        """a tensor-core convolution: fp64 sums of the (rounded) operand times round_tf32(W), plus the bias"""
        if name not in self._w:
            w = self.sd[name + '.weight']
            self._w[name] = round_tf32(w) if self.rounding else w
        return F.conv2d(x, self._w[name], self.sd.get(name + '.bias'), stride=stride, padding=padding)

    # -- encoders -------------------------------------------------------------------------------------
    def _block(self, p, x, kind, stride):
        sd = self.sd
        if kind == 'instance':
            a = self.anchor(p + '.a', self.tc(p + '.conv1', x, stride, 1), False)
            y = self.anchor(p + '.y', self.rv(F.relu(ref._norm(sd, None, a, kind))), True)
            b = self.anchor(p + '.b', self.tc(p + '.conv2', y, 1, 1), False)
            yb = F.relu(ref._norm(sd, None, b, kind))
            if stride == 1:
                return self.anchor(p + '.out', self.rv(F.relu(x + yb)), True)
            yb = self.anchor(p + '.yb', yb, False)
            d = self.anchor(p + '.d', self.tc(p + '.downsample.0', x, stride, 0), False)
            return self.anchor(p + '.out', self.rv(F.relu(ref._norm(sd, None, d, kind) + yb)), True)
        # eval BatchNorm: each convolution's epilogue
        y = self.anchor(p + '.y', self.rv(F.relu(ref._norm(sd, p + '.norm1', self.tc(p + '.conv1', x, stride, 1), kind))), True)
        b = self.anchor(p + '.b', F.relu(ref._norm(sd, p + '.norm2', self.tc(p + '.conv2', y, 1, 1), kind)), False)
        if stride != 1:
            x = ref._norm(sd, p + '.norm3', self.tc(p + '.downsample.0', x, stride, 0), kind)
        return self.anchor(p + '.out', self.rv(F.relu(x + b)), True)

    def encoder(self, prefix, images, kind):
        """oracle.raft.encoder: [N,3,H,W] in 0..255 -> [N,256,H/8,W/8]"""
        z = ref._conv(self.sd, prefix + '.conv1', 2 * (images / 255.0) - 1.0, 2, 3)       # CUDA cores, plain weights
        if kind == 'instance':
            z = self.anchor(prefix + '.stem', z, False)
        x = self.anchor(prefix + '.stem.out', self.rv(F.relu(ref._norm(self.sd, prefix + '.norm1', z, kind))), True)
        for name, stride in BLOCKS:
            x = self._block('%s.%s' % (prefix, name), x, kind, stride)
        return self.anchor('fmap' if prefix == 'fnet' else 'cnet', self.tc(prefix + '.conv2', x), False)

    def encode(self, images):
        """both encoders of every image: (fmap, cnet before its tanh / relu split)"""
        return self.encoder('fnet', images, 'instance'), self.encoder('cnet', images, 'batch')

    def context_split(self, cnet):
        """oracle.raft.context: -> (net, inp); the operand copy round(net) is made where the GRU reads it"""
        net = self.anchor('net', torch.tanh(cnet[:, :HDIM]), False)
        return net, self.anchor('inp', self.rv(F.relu(cnet[:, HDIM:])), True)

    def pyramid(self, fmap1, fmap2):
        return [self.anchor('pyramid.%d' % l, p, False) for l, p in enumerate(ref.corr_pyramid(fmap1, fmap2))]

    # -- one update iteration -------------------------------------------------------------------------
    def _gru(self, h, x):
        """oracle.raft.sep_conv_gru; the operands [round(h) | x] and [round(r h) | x]"""
        p = 'update_block.gru.'
        for i, (tag, pad) in enumerate((('1', (0, 2)), ('2', (2, 0)))):
            hx = torch.cat([self.rv(h), x], 1)
            z = torch.sigmoid(self.anchor('z.%d' % i, self.tc(p + 'convz' + tag, hx, 1, pad), False))
            r = torch.sigmoid(self.anchor('r.%d' % i, self.tc(p + 'convr' + tag, hx, 1, pad), False))
            rh = self.anchor('rh.%d' % i, self.rv(r * h), True)
            q = torch.tanh(self.anchor('q.%d' % i, self.tc(p + 'convq' + tag, torch.cat([rh, x], 1), 1, pad), False))
            h = self.anchor('net.%d' % i, (1 - z) * h + z * q, False)
        return h

    def update(self, pyr, net, inp, coords1, coords0, prefix=''):
        """lookup (oracle.raft.lookup) + oracle.raft.update from the iteration's input state -> (net, net_r, coords1, delta_flow)"""
        self.prefix = prefix
        try:
            sd, p = self.sd, 'update_block.encoder.'
            corr = self.anchor('corr', self.rv(lookup(pyr, coords1)), True)
            flow = coords1 - coords0
            cor = self.anchor('convc1', self.rv(F.relu(self.tc(p + 'convc1', corr))), True)
            cor = self.anchor('convc2', self.rv(F.relu(self.tc(p + 'convc2', cor, 1, 1))), True)
            flo = self.anchor('convf1', self.rv(F.relu(ref._conv(sd, p + 'convf1', flow, 1, 3))), True)     # CUDA cores, plain weights
            flo = self.anchor('convf2', self.rv(F.relu(self.tc(p + 'convf2', flo, 1, 1))), True)
            out = self.anchor('motion', self.rv(F.relu(self.tc(p + 'conv', torch.cat([cor, flo], 1), 1, 1))), True)
            net = self._gru(net, torch.cat([inp, out, self.rv(flow)], 1))
            net_r = self.anchor('net_r', self.rv(net), True)
            fh = self.anchor('fh', F.relu(self.tc('update_block.flow_head.conv1', net_r, 1, 1)), False)
            delta = self.anchor('delta', ref._conv(sd, 'update_block.flow_head.conv2', fh, 1, 1), False)    # CUDA cores
            coords1 = self.anchor('coords1', coords1 + delta, False)
            return net, net_r, coords1, delta
        finally:
            self.prefix = ''

    # -- mask head and up-sampling --------------------------------------------------------------------
    def up_mask(self, net_r):
        """the mask head's logits, before the 0.25 of oracle.raft.up_mask"""
        mk = self.anchor('mask0', self.rv(F.relu(self.tc('update_block.mask.0', net_r, 1, 1))), True)
        return self.anchor('mask', self.tc('update_block.mask.2', mk), False)

    def upsample(self, mask, coords1, coords0):
        return self.anchor('flow_up', ref.upsample(coords1 - coords0, 0.25 * mask), False)

    # -- the whole forward ----------------------------------------------------------------------------
    def forward(self, image1, image2, iters=20):
        """oracle.raft.raft_forward -> (flow_low, flow_up); iteration k's anchors are named 'it<k>.<name>'"""
        N = image1.shape[0]
        fmap, cnet = self.encode(torch.cat([image1, image2]))
        pyr = self.pyramid(fmap[:N], fmap[N:])
        net, inp = self.context_split(cnet[:N])
        _, _, h, w = fmap.shape
        coords0 = ref.coords_grid(N, h, w, fmap.dtype, fmap.device)
        coords1 = coords0.clone()
        net_r = None
        for k in range(iters):
            net, net_r, coords1, _ = self.update(pyr, net, inp, coords1, coords0, 'it%d.' % k)
        flow_up = self.upsample(self.up_mask(net_r), coords1, coords0)
        return coords1 - coords0, flow_up


# ------------------------------------------------------------------------------------------------
def _nchw(t):
    return t.permute(0, 3, 1, 2)


def encoder_anchors(trace):
    """RaftNet.encode's trace -> {anchor name: tensor in this module's layout}"""
    return {k: _nchw(v) for k, v in trace.items()}


def state_anchors(trace, B, h, w):
    """RaftNet.flow's trace, without its iterations -> anchors of the initial state, the pyramid and the mask head"""
    A = {'net': _nchw(trace['net']), 'inp': _nchw(trace['X'][..., HDIM:2 * HDIM])}
    P, off, hl, wl = B * h * w, 0, h, w
    for l in range(ref.LEVELS):          # the flat buffer holds level l as [B*h*w, h >> l, w >> l] after the levels before it
        A['pyramid.%d' % l] = trace['pyramid'][off:off + P * hl * wl].view(P, 1, hl, wl)
        off += P * hl * wl
        hl, wl = hl // 2, wl // 2
    A['mask0'] = _nchw(trace['mask0'])
    A['mask'] = _nchw(torch.cat(trace['mask'], -1))
    A['flow_up'] = _nchw(trace['flow_up'])
    return A


def iteration_anchors(it, prefix=''):
    """one iteration of RaftNet.flow's trace -> anchors named prefix + name: the merged z|r output split into z and r, the
    lookup without its zero tail, the motion output without its two pad channels, r h from the operand buffer"""
    A = {'corr': it['corr'][..., :LOOKUP_CHANNELS], 'motion': it['motion'][..., :126]}
    for k in ('convc1', 'convc2', 'convf1', 'convf2', 'net_r', 'fh', 'delta', 'coords1'):
        A[k] = it[k]
    for i in (0, 1):
        A['z.%d' % i], A['r.%d' % i] = it['zr.%d' % i][..., :HDIM], it['zr.%d' % i][..., HDIM:]
        A['rh.%d' % i] = it['XR.rh.%d' % i][..., :HDIM]
        A['q.%d' % i], A['net.%d' % i] = it['q.%d' % i], it['net.%d' % i]
    return {prefix + k: _nchw(v) for k, v in A.items()}


def anchor_names(kind):
    """the anchors one emulation stage records: 'encoder', 'iteration', or 'state' (initial state, pyramid, mask head)"""
    if kind == 'encoder':
        names = ['fnet.stem', 'fnet.stem.out', 'fmap', 'cnet.stem.out', 'cnet']
        for name, stride in BLOCKS:
            names += ['fnet.%s.%s' % (name, s) for s in ('a', 'y', 'b', 'out') + (('yb', 'd') if stride != 1 else ())]
            names += ['cnet.%s.%s' % (name, s) for s in ('y', 'b', 'out')]
        return names
    if kind == 'iteration':
        names = ['corr', 'convc1', 'convc2', 'convf1', 'convf2', 'motion', 'net_r', 'fh', 'delta', 'coords1']
        return names + ['%s.%d' % (s, i) for i in (0, 1) for s in ('z', 'r', 'rh', 'q', 'net')]
    return ['net', 'inp', 'mask0', 'mask', 'flow_up'] + ['pyramid.%d' % l for l in range(ref.LEVELS)]
