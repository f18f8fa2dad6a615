"""TEST INFRASTRUCTURE — CPU restatement of `dvd_disp_vali` (csrc/eval_ops.cu).

`terms_fp32` evaluates the kernel's per-pixel term in its operation order with numpy float32 scalars-by-array arithmetic, where
every operation is rounded on its own (numpy never contracts), so it must equal both the kernel's terms and torch CPU's
elementwise terms of the reference formula bit for bit. `reference_terms` is that formula itself (models/video_base.py:66-74),
`frame_sse_fp64` the per-frame sums in fp64 and `sum_bound` the γ_n·Σ|t| bound a fixed-order fp32 sum of n terms meets.
"""
import numpy as np
import torch

U32 = 2.0 ** -24


def _disp(x):
    v = (x > np.float32(1e-2)).astype(np.float32)
    den = x + (np.float32(1.0) - v) * np.float32(1e-8)
    return (np.float32(1.0) / den) * v, v


def terms_fp32(depth, depth_gt):
    """[N,1,H,W] float32 (numpy or torch) -> the per-pixel terms, float32 numpy."""
    d = np.asarray(depth.numpy() if torch.is_tensor(depth) else depth, dtype=np.float32)
    g = np.asarray(depth_gt.numpy() if torch.is_tensor(depth_gt) else depth_gt, dtype=np.float32)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        rd, _ = _disp(d)
        rg, vg = _disp(g)
        diff = rd * vg - rg * vg
        return diff * diff


def reference_terms(depth, depth_gt):
    """torch's elementwise terms of `mse_loss(depth2disp(d) * vali, depth2disp(g) * vali)` (video_base.py:66-74)."""
    def depth2disp(x):
        valid = (x > 1e-2).float()
        return (1 / (x + (1 - valid) * 1e-8)) * valid
    vali = depth_gt > 1e-2
    return torch.nn.functional.mse_loss(depth2disp(depth) * vali, depth2disp(depth_gt) * vali, reduction='none')


def reference_mse(depth, depth_gt):
    """the reference's own value for one batch (mean over every pixel of the batch)."""
    def depth2disp(x):
        valid = (x > 1e-2).float()
        return (1 / (x + (1 - valid) * 1e-8)) * valid
    vali = depth_gt > 1e-2
    return torch.nn.functional.mse_loss(depth2disp(depth) * vali, depth2disp(depth_gt) * vali)


def frame_sse_fp64(terms):
    t = np.asarray(terms, dtype=np.float64)
    return t.reshape(t.shape[0], -1).sum(1), np.abs(t).reshape(t.shape[0], -1).sum(1)


def gamma(n):
    return n * U32 / (1.0 - n * U32)


def sum_depth(H, W, parts_per_frame, threads=256):
    """Longest chain of fp32 additions behind one frame_sse of the kernel: a thread's own terms (at most ceil(H·W / (P·T)) + 3
    with the float4 path), the warp tree (5), the block's warps (7) in pass 1, and the same two stages (5 + 3) in pass 2."""
    per_thread = -(-(H * W) // (parts_per_frame * threads)) + 3
    return per_thread + 5 + 7 + 5 + 3


def sum_bound(abs_sum, H, W, parts_per_frame):
    return gamma(sum_depth(H, W, parts_per_frame)) * abs_sum
