"""Deterministic synthetic frame-pair batches of the reference's pair-file format.

Format follows what `datasets/davis_sequence.py:86-113` hands to the Model (after the DataLoader's
leading batch dim of 1) and the packing of `scripts/preprocess/davis/generate_sequence_midas.py:61-76,
146-147,179,187`: pose / intrinsic tensors hold TRANSPOSES so that `row @ M` works
(R_i = R_c2w_i^T, R_i_T = R_c2w_i, K = K^T, K_inv = (K^-1)^T). Distributions: SURVEY.md §8(d).
"""
import math

import torch

GAPS = (1, 2, 4, 6, 8)


def pair_list(n_frames=80, gaps=GAPS):
    """All (f, f+g) with f < n_frames-1-g — the reference's rule
    (scripts/preprocess/davis/generate_sequence_midas.py:187): 374 pairs for 80 frames."""
    out = []
    for g in gaps:
        for f in range(0, n_frames - 1 - g):
            out.append((f, f + g))
    return out


def _rot_y(a):
    c, s = math.cos(a), math.sin(a)
    return torch.tensor([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]], dtype=torch.float64)


def camera(frame_id, H, W):
    """c2w rotation, translation and intrinsics of one synthetic frame (float64)."""
    R = _rot_y(0.01 + 0.005 * frame_id)
    t = torch.tensor([0.05 * frame_id, 0.0, 0.0], dtype=torch.float64)
    f = 300.0 * W / 384.0
    K = torch.tensor([[f, 0.0, (W - 1) / 2.0], [0.0, f, (H - 1) / 2.0], [0.0, 0.0, 1.0]],
                     dtype=torch.float64)
    return R, t, K


def make_batch(pairs, H=224, W=384, n_frames=80, seed=0, smooth_flow=False, dtype=torch.float32,
               leading_dim=True, mask_p=0.9, flow_sigma=3.0):
    """Build one batch dict for `pairs` = [(frame_id_1, frame_id_2), ...] (B pairs).

    Returned tensors live on the CPU; `leading_dim` adds the DataLoader's batch dim of 1 that
    `Model._train_on_batch` squeezes (models/scene_flow_motion_field.py:177-179)."""
    B = len(pairs)
    g = torch.Generator().manual_seed(seed)

    def rnd(*shape):
        return torch.rand(*shape, generator=g, dtype=torch.float64)

    def nrm(*shape):
        return torch.randn(*shape, generator=g, dtype=torch.float64)

    def flow():
        if smooth_flow:
            lo = nrm(B, 2, (H + 7) // 8 + 1, (W + 7) // 8 + 1) * flow_sigma
            f = torch.nn.functional.interpolate(lo, size=(H, W), mode='bilinear', align_corners=True)
            return f.permute(0, 2, 3, 1).contiguous()
        return nrm(B, H, W, 2) * flow_sigma

    b = {}
    b['img_1'] = rnd(B, 3, H, W)
    b['img_2'] = rnd(B, 3, H, W)
    b['flow_1_2'] = flow()
    b['flow_2_1'] = flow()
    b['mask_1'] = (rnd(B, H, W, 1, 1) < mask_p).double()
    b['mask_2'] = (rnd(B, H, W, 1, 1) < mask_p).double()
    b['motion_seg_1'] = torch.ones(B, H, W, 1, 1, dtype=torch.float64)
    R1, R2, t1, t2, Ks, Kinvs = [], [], [], [], [], []
    for (f1, f2) in pairs:
        Ra, ta, K = camera(f1, H, W)
        Rb, tb, _ = camera(f2, H, W)
        R1.append(Ra), R2.append(Rb), t1.append(ta), t2.append(tb)
        Ks.append(K), Kinvs.append(torch.linalg.inv(K))
    R1, R2 = torch.stack(R1), torch.stack(R2)
    b['R_1'] = R1.transpose(1, 2).reshape(B, 1, 1, 3, 3).contiguous()
    b['R_1_T'] = R1.reshape(B, 1, 1, 3, 3).contiguous()
    b['R_2'] = R2.transpose(1, 2).reshape(B, 1, 1, 3, 3).contiguous()
    b['R_2_T'] = R2.reshape(B, 1, 1, 3, 3).contiguous()
    b['t_1'] = torch.stack(t1).reshape(B, 1, 1, 1, 3)
    b['t_2'] = torch.stack(t2).reshape(B, 1, 1, 1, 3)
    b['K'] = torch.stack(Ks).transpose(1, 2).reshape(B, 1, 1, 3, 3).contiguous()
    b['K_inv'] = torch.stack(Kinvs).transpose(1, 2).reshape(B, 1, 1, 3, 3).contiguous()
    fid1 = torch.tensor([p[0] for p in pairs], dtype=torch.float64)
    fid2 = torch.tensor([p[1] for p in pairs], dtype=torch.float64)
    b['time_stamp_1'] = (fid1 / n_frames).reshape(B, 1, 1, 1).expand(B, 1, H, W).contiguous()
    b['time_stamp_2'] = (fid2 / n_frames).reshape(B, 1, 1, 1).expand(B, 1, H, W).contiguous()
    b['frame_id_1'] = fid1.clone()
    b['frame_id_2'] = fid2.clone()
    b['depth_pred_1'] = torch.ones(B, 1, H, W, dtype=torch.float64)
    out = {}
    for k, v in b.items():
        v = v.to(dtype)
        out[k] = v.unsqueeze(0) if leading_dim else v
    out['time_step'] = torch.tensor([1.0 / n_frames], dtype=dtype)
    out['pair_path'] = ['synthetic_%03d_%03d' % p for p in pairs]
    return out


def make_frame(idx, H=224, W=384, n_frames=80, invalid_p=0.1):
    """One per-frame `vali` item of frame `idx` with the keys and layouts of datasets/davis_sequence.py:117-152 (pose tensors
    hold transposes as in make_batch; cam_c2w is the 4x4 camera-to-world matrix). `depth_mvs` is a seeded smooth depth map in
    [2, 8] with a share `invalid_p` of its pixels set to 0 (invalid); `depth_pred` another one in [1.5, 9]."""
    g = torch.Generator().manual_seed(100003 + idx)
    R, t, K = camera(idx, H, W)
    c2w = torch.eye(4, dtype=torch.float64)
    c2w[:3, :3], c2w[:3, 3] = R, t
    gt = make_depths(1, H, W, seed=200003 + idx)[0]
    gt = gt * (torch.rand(1, H, W, generator=g, dtype=torch.float64) >= invalid_p).float()
    s = {'time_stamp_1': torch.full((1, H, W), idx / n_frames, dtype=torch.float64),
         'img': torch.rand(3, H, W, generator=g, dtype=torch.float64), 'frame_id_1': idx, 'time_step': 1.0 / n_frames,
         'depth_pred': make_depths(1, H, W, seed=300003 + idx, lo=1.5, hi=9.0)[0], 'cam_c2w': c2w, 'depth_mvs': gt,
         'R_1': R.t().reshape(1, 1, 3, 3), 'R_1_T': R.reshape(1, 1, 3, 3), 't_1': t.reshape(1, 1, 1, 3),
         'K': K.t().reshape(1, 1, 3, 3), 'K_inv': torch.linalg.inv(K).t().reshape(1, 1, 3, 3)}
    s = {k: (v.float().contiguous() if torch.is_tensor(v) else v) for k, v in s.items()}
    s['pair_path'] = 'synthetic_frame_%03d' % idx
    return s


def make_depths(B, H, W, seed=1, lo=2.0, hi=8.0, dtype=torch.float32):
    """Smooth positive depth maps for op-level tests (the depth nets are tested separately)."""
    g = torch.Generator().manual_seed(seed)
    lo_res = torch.rand(B, 1, (H + 15) // 16 + 1, (W + 15) // 16 + 1, generator=g, dtype=torch.float64)
    d = torch.nn.functional.interpolate(lo_res, size=(H, W), mode='bilinear', align_corners=True)
    return (lo + (hi - lo) * d).to(dtype).contiguous()


def default_opt(**over):
    """argparse.Namespace with the flags of experiments/davis/train_sequence.sh:24-63 (the configuration
    BASELINE.json's metric is quoted on): joint phase needs epoch > warm_sf."""
    import argparse
    d = dict(optim='adam', lr=1e-6, adam_beta1=0.5, adam_beta2=0.9, full_logdir=None, global_rank=0,
             dataset='davis_sequence', batch_size=1, epoch_batches=2000, vis_every_train=0, vis_at_start=True,
             vis_batches_train=0, multiprocess_distributed=False,
             l1_mul=0.0, disp_mul=1.0, one_way=True, loss_type='l1', scene_lr_mul=1000.0, n_down=3,
             weight_steps=False, sf_min_mul=0, sf_quantile=0.5, static=False, static_mul=1, flow_mul=1.0,
             acc_mul=1.0, si_mul=0, cos_mul=0, motion_seg_hard=False, warm_mul=1, interp_steps=5,
             warm_static=False, use_disp=True, use_disp_ratio=False, time_dependent=True, use_cnn=False,
             use_embedding=False, use_motion_seg=False, warm_reg=False, warm_sf=5, n_freq_xyz=16, n_freq_t=16,
             sf_mag_div=100.0, midas=True)
    d.update(over)
    return argparse.Namespace(**d)


def seed_net_(net, seed=0, head_bias=None, head_gain=40.0):
    """Deterministic weights that depend only on parameter NAMES (not on construction order), so the
    reference net and the dvd_b200 mirror get bit-identical values. Variance-preserving: weights
    N(0, 1/fan_in); the last BN of every residual branch is damped (x0.25) so that a 101-layer random
    ResNeXt does not blow up; BN running stats randomised around (0, 1). For MiDaS the 1-channel head
    gets `head_bias` (SURVEY.md §8(d): depth = 10000/out must land in the valid < 100 range) and its
    weights `head_gain` x larger so that the synthetic depth map varies spatially (~ +-20 %)."""
    import hashlib
    with torch.no_grad():
        for name, t in list(net.named_parameters()) + list(net.named_buffers()):
            if not t.dtype.is_floating_point:
                continue
            h = int(hashlib.sha1(('%d:%s' % (seed, name)).encode()).hexdigest()[:8], 16)
            g = torch.Generator().manual_seed(h)
            leaf = name.split('.')[-1]
            if leaf == 'running_var':
                v = 0.75 + 0.5 * torch.rand(t.shape, generator=g)
            elif leaf == 'running_mean':
                v = 0.05 * torch.randn(t.shape, generator=g)
            elif t.dim() >= 2:
                v = torch.randn(t.shape, generator=g) * math.sqrt(1.0 / t[0].numel())
            elif leaf == 'weight':   # BN affine scale
                v = 1.0 + 0.1 * (torch.rand(t.shape, generator=g) - 0.5)
                if '.bn3.' in name:
                    v = 0.25 * v
            else:
                v = 0.02 * (torch.rand(t.shape, generator=g) - 0.5)
            t.copy_(v.to(t.dtype))
        if head_bias is not None:
            head = net.scratch.output_conv[4]
            head.weight.mul_(head_gain)
            head.bias.fill_(head_bias)
    return net
