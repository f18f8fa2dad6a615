"""TEST INFRASTRUCTURE — plain-torch restatement of RAFT inference as the reference's flow stage runs it
(third_party/RAFT/core: raft.py, extractor.py, update.py, corr.py, utils/utils.py; large model, all-pairs correlation,
4 levels, radius 4, hidden = context = 128, no warm start, test mode).

Functional over a state dict with the reference's parameter names (a leading `module.` is stripped), in the dtype and on
the device of the inputs, so that the same code gives the fp64 truth on the CPU and an eager fp32 baseline on a GPU.
`trace`, when a dict, receives every intermediate tensor the fixtures pin.
"""
import torch
import torch.nn.functional as F

LEVELS, RADIUS, HDIM = 4, 4, 128
WINDOW = 2 * RADIUS + 1


def strip_module(sd):
    return {(k[7:] if k.startswith('module.') else k): v for k, v in sd.items()}


def cast(sd, dtype, device=None):
    return {k: (v.to(device=device, dtype=dtype) if v.is_floating_point() else v.to(device=device))
            for k, v in strip_module(sd).items()}


def _conv(sd, name, x, stride=1, padding=0):
    return F.conv2d(x, sd[name + '.weight'], sd[name + '.bias'], stride=stride, padding=padding)


def _norm(sd, name, x, kind):
    if kind == 'instance':
        return F.instance_norm(x, eps=1e-5)
    return F.batch_norm(x, sd[name + '.running_mean'], sd[name + '.running_var'], sd[name + '.weight'], sd[name + '.bias'],
                        False, 0.0, 1e-5)


def _res_block(sd, p, x, kind, stride):
    y = F.relu(_norm(sd, p + '.norm1', _conv(sd, p + '.conv1', x, stride, 1), kind))
    y = F.relu(_norm(sd, p + '.norm2', _conv(sd, p + '.conv2', y, 1, 1), kind))
    if stride != 1:
        # the block registers the same norm as `norm3` and as `downsample.1`
        x = _norm(sd, p + '.norm3', _conv(sd, p + '.downsample.0', x, stride, 0), kind)
    return F.relu(x + y)


def stem(sd, prefix, image, kind):
    """conv1 on 2 (x / 255) - 1, its norm and ReLU: [N,3,H,W] in 0..255 -> [N,64,H/2,W/2]"""
    x = 2 * (image / 255.0) - 1.0
    return F.relu(_norm(sd, prefix + '.norm1', _conv(sd, prefix + '.conv1', x, 2, 3), kind))


def encoder(sd, prefix, image, kind):
    x = stem(sd, prefix, image, kind)
    for layer, stride in (('layer1', 1), ('layer2', 2), ('layer3', 2)):
        x = _res_block(sd, '%s.%s.0' % (prefix, layer), x, kind, stride)
        x = _res_block(sd, '%s.%s.1' % (prefix, layer), x, kind, 1)
    return _conv(sd, prefix + '.conv2', x)


def context(sd, image):
    c = encoder(sd, 'cnet', image, 'batch')
    return torch.tanh(c[:, :HDIM]), F.relu(c[:, HDIM:])


def corr_pyramid(fmap1, fmap2):
    """levels of [N*h*w, 1, h / 2^l, w / 2^l]: <fmap1[p], fmap2[q]> / sqrt(C), averaged 2x2 over q level by level"""
    N, C, h, w = fmap1.shape
    corr = torch.matmul(fmap1.reshape(N, C, h * w).transpose(1, 2), fmap2.reshape(N, C, h * w))
    corr = corr.reshape(N * h * w, 1, h, w) / torch.sqrt(torch.tensor(float(C), dtype=fmap1.dtype, device=fmap1.device))
    pyr = [corr]
    for _ in range(LEVELS - 1):
        corr = F.avg_pool2d(corr, 2, stride=2)
        pyr.append(corr)
    return pyr


def window_offsets(dtype=torch.float32, device=None):
    """channel k of a level reads the offset (x, y) = (k // 9 - 4, k % 9 - 4): the reference adds meshgrid(dy, dx) pairs to
    (x, y) coordinates, so the slow index of the 9 x 9 window moves along x"""
    r = torch.arange(-RADIUS, RADIUS + 1, dtype=dtype, device=device)
    return torch.stack(torch.meshgrid(r, r, indexing='ij'), dim=-1)       # [9, 9, 2]: [..., 0] -> x, [..., 1] -> y


def lookup(pyr, coords1):
    """coords1 [N,2,h,w] (x, y) -> [N, 4*81, h, w]; bilinear, zeros outside, pixel coordinates"""
    N, _, h, w = coords1.shape
    c = coords1.permute(0, 2, 3, 1).reshape(N * h * w, 1, 1, 2)
    off = window_offsets(coords1.dtype, coords1.device)[None]
    out = []
    for l, corr in enumerate(pyr):
        H, W = corr.shape[-2:]
        p = c / 2 ** l + off
        grid = torch.cat([2 * p[..., :1] / (W - 1) - 1, 2 * p[..., 1:] / (H - 1) - 1], dim=-1)
        out.append(F.grid_sample(corr, grid, align_corners=True).reshape(N, h, w, WINDOW * WINDOW))
    return torch.cat(out, dim=-1).permute(0, 3, 1, 2).contiguous()


def motion_encoder(sd, flow, corr):
    p = 'update_block.encoder.'
    cor = F.relu(_conv(sd, p + 'convc1', corr))
    cor = F.relu(_conv(sd, p + 'convc2', cor, 1, 1))
    flo = F.relu(_conv(sd, p + 'convf1', flow, 1, 3))
    flo = F.relu(_conv(sd, p + 'convf2', flo, 1, 1))
    out = F.relu(_conv(sd, p + 'conv', torch.cat([cor, flo], 1), 1, 1))
    return torch.cat([out, flow], 1)


def sep_conv_gru(sd, h, x):
    p = 'update_block.gru.'
    for tag, pad in (('1', (0, 2)), ('2', (2, 0))):
        hx = torch.cat([h, x], 1)
        z = torch.sigmoid(_conv(sd, p + 'convz' + tag, hx, 1, pad))
        r = torch.sigmoid(_conv(sd, p + 'convr' + tag, hx, 1, pad))
        q = torch.tanh(_conv(sd, p + 'convq' + tag, torch.cat([r * h, x], 1), 1, pad))
        h = (1 - z) * h + z * q
    return h


def update(sd, net, inp, corr, flow):
    """one iteration of BasicUpdateBlock without its mask head: -> (net, delta_flow)"""
    x = torch.cat([inp, motion_encoder(sd, flow, corr)], 1)
    net = sep_conv_gru(sd, net, x)
    p = 'update_block.flow_head.'
    return net, _conv(sd, p + 'conv2', F.relu(_conv(sd, p + 'conv1', net, 1, 1)), 1, 1)


def up_mask(sd, net):
    return 0.25 * _conv(sd, 'update_block.mask.2', F.relu(_conv(sd, 'update_block.mask.0', net, 1, 1)))


def upsample(flow, mask):
    """convex 8x up-sampling: flow [N,2,h,w], mask [N,576,h,w] -> [N,2,8h,8w]"""
    N, _, h, w = flow.shape
    m = torch.softmax(mask.reshape(N, 1, 9, 8, 8, h, w), dim=2)
    u = F.unfold(8 * flow, [3, 3], padding=1).reshape(N, 2, 9, 1, 1, h, w)
    return torch.sum(m * u, dim=2).permute(0, 1, 4, 2, 5, 3).reshape(N, 2, 8 * h, 8 * w)


def coords_grid(N, h, w, dtype, device):
    ys, xs = torch.meshgrid(torch.arange(h, dtype=dtype, device=device), torch.arange(w, dtype=dtype, device=device), indexing='ij')
    return torch.stack([xs, ys], 0)[None].repeat(N, 1, 1, 1)


def raft_forward(sd, image1, image2, iters=20, trace=None):
    """-> (flow_low [N,2,H/8,W/8], flow_up [N,2,H,W]); images [N,3,H,W] in 0..255; sd already in the images' dtype"""
    if image1.shape[-2] % 8 or image1.shape[-1] % 8:
        raise ValueError('image height and width must be multiples of 8')
    fmap1 = encoder(sd, 'fnet', image1, 'instance')
    fmap2 = encoder(sd, 'fnet', image2, 'instance')
    pyr = corr_pyramid(fmap1, fmap2)
    net, inp = context(sd, image1)
    N, _, h, w = fmap1.shape
    coords0 = coords_grid(N, h, w, image1.dtype, image1.device)
    coords1 = coords0.clone()
    if trace is not None:
        trace.update(fmap1=fmap1, fmap2=fmap2, net0=net, inp=inp, pyramid=pyr, iters=[])
    for _ in range(iters):
        corr = lookup(pyr, coords1)
        net, delta = update(sd, net, inp, corr, coords1 - coords0)
        if trace is not None:
            trace['iters'].append(dict(coords1=coords1, corr=corr, net=net, delta_flow=delta))
        coords1 = coords1 + delta
    mask = up_mask(sd, net)
    flow_low = coords1 - coords0
    flow_up = upsample(flow_low, mask)
    if trace is not None:
        trace.update(up_mask=mask, flow_low=flow_low, flow_up=flow_up)
    return flow_low, flow_up


# ------------------------------------------------------------------------------------------------
# seeded parameters (a real checkpoint is 21 MB; fixtures and tests rebuild these from the seed instead)

def _encoder_shapes(prefix, out_dim, batch_norm):
    convs, norms = [(prefix + '.conv1', 64, 3, 7, 7)], [(prefix + '.norm1', 64)]
    cin = 64
    for layer, dim, stride in (('layer1', 64, 1), ('layer2', 96, 2), ('layer3', 128, 2)):
        for blk in (0, 1):
            p = '%s.%s.%d' % (prefix, layer, blk)
            convs += [(p + '.conv1', dim, cin, 3, 3), (p + '.conv2', dim, dim, 3, 3)]
            norms += [(p + '.norm1', dim), (p + '.norm2', dim)]
            if blk == 0 and stride != 1:
                convs.append((p + '.downsample.0', dim, cin, 1, 1))
                norms += [(p + '.downsample.1', dim), (p + '.norm3', dim)]     # one module under two names
            cin = dim
    convs.append((prefix + '.conv2', out_dim, 128, 1, 1))
    return convs, (norms if batch_norm else [])


def conv_shapes():
    """[(name, Cout, Cin, kh, kw)] of every convolution, and [(name, C)] of every BatchNorm2d (cnet only)"""
    fc, _ = _encoder_shapes('fnet', 256, False)
    cc, cn = _encoder_shapes('cnet', 256, True)
    u = 'update_block.'
    upd = [(u + 'encoder.convc1', 256, LEVELS * WINDOW * WINDOW, 1, 1), (u + 'encoder.convc2', 192, 256, 3, 3),
           (u + 'encoder.convf1', 128, 2, 7, 7), (u + 'encoder.convf2', 64, 128, 3, 3), (u + 'encoder.conv', 126, 256, 3, 3)]
    upd += [(u + 'gru.conv%s1' % g, 128, 384, 1, 5) for g in 'zrq'] + [(u + 'gru.conv%s2' % g, 128, 384, 5, 1) for g in 'zrq']
    upd += [(u + 'flow_head.conv1', 256, 128, 3, 3), (u + 'flow_head.conv2', 2, 256, 3, 3),
            (u + 'mask.0', 256, 128, 3, 3), (u + 'mask.2', 576, 256, 1, 1)]
    return fc + cc + upd, cn


def seeded_state_dict(seed=0, gain=1.0, flow_gain=0.25):
    """fp32 parameters under the reference's names from one CPU generator. Convolutions: N(0, gain^2 * 2 / fan_in) (the
    last flow-head convolution additionally times flow_gain, so that an iteration moves a pixel by a fraction of a pixel),
    biases U(-0.1, 0.1); BatchNorm with non-trivial statistics."""
    g = torch.Generator().manual_seed(seed)
    convs, norms = conv_shapes()
    sd = {}
    for name, co, ci, kh, kw in convs:
        std = gain * (2.0 / (ci * kh * kw)) ** 0.5 * (flow_gain if name.endswith('flow_head.conv2') else 1.0)
        sd[name + '.weight'] = torch.randn(co, ci, kh, kw, generator=g) * std
        sd[name + '.bias'] = (torch.rand(co, generator=g) - 0.5) * 0.2
    shared = {}
    for name, c in norms:
        twin = name.replace('.downsample.1', '.norm3')
        if twin in shared:
            vals = shared[twin]
        else:
            vals = shared[twin] = (0.5 + torch.rand(c, generator=g), (torch.rand(c, generator=g) - 0.5) * 0.4,
                                   torch.randn(c, generator=g) * 0.1, 0.5 + torch.rand(c, generator=g))
        for k, v in zip(('weight', 'bias', 'running_mean', 'running_var'), vals):
            sd['%s.%s' % (name, k)] = v.clone()
        sd[name + '.num_batches_tracked'] = torch.zeros((), dtype=torch.long)
    return sd


def seeded_pair(H, W, seed=0, shift=2.0):
    """a smooth random texture and a warped copy of it, [1,3,H,W] fp32 in 0..255"""
    g = torch.Generator().manual_seed(seed)
    tex = F.interpolate(torch.rand(1, 3, H // 4 + 2, W // 4 + 2, generator=g), size=(H, W), mode='bicubic', align_corners=True)
    tex = tex.clamp(0, 1)
    disp = F.interpolate(torch.randn(1, 2, 4, 5, generator=g), size=(H, W), mode='bicubic', align_corners=True) * shift
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing='ij')
    gx = 2 * (xs + disp[0, 0]) / (W - 1) - 1
    gy = 2 * (ys + disp[0, 1]) / (H - 1) - 1
    warped = F.grid_sample(tex, torch.stack([gx, gy], -1)[None], mode='bilinear', padding_mode='border', align_corners=True)
    return (tex * 255).contiguous(), (warped * 255).contiguous()
