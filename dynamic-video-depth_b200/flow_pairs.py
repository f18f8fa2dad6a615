"""Training pairs of one video, built from the per-frame files and the optical flows, without per-pair files.

The reference prepares a video in three steps: `generate_flows.py` resizes each RAFT flow with cv2 and builds the
consistency masks on the CPU one pair at a time, `generate_sequence_midas.py` writes one `.pt` file per pair (2 MB each at
384x224), and `datasets/davis_sequence.py` `torch.load`s one of them per step. `PairBuilder` does the same work once:

  input   <frames>/frame_%05d.npz       img [H,W,3], pose_c2w, intrinsics, depth_mvs, depth_pred, optional motion_seg (absent
                                        or None: motion_seg_1 is then mask_2, as the ShutterStock generate_sequence_midas.py does)
          <flows>/flowpair_%05d_%05d.npz flow_1_2, flow_2_1 [h,w,2] and, when generate_flows.py wrote it, mask_1 / mask_2
  flows   a file that holds masks and flows at the frames' resolution is used as it is (it is exactly the reference's
          output); any other file is treated as raw flows at any resolution: all such pairs of one gap go through
          ops.flow_resize_cubic and ops.flow_pair_masks in one launch each, on the GPU
  output  item i = the dict davis_sequence.Dataset.__getitem__ returns for the pair file generate_sequence_midas.py writes
          (datadict_from_pair, generate_sequence_midas.py:117-170, then davis_sequence.py:98-115), bitwise

Pairs follow the reference's rule, (f, f + g) for f < n - 1 - g, gap by gap. Frames are kept once, the per-pair tensors once
per pair, all on the host (pinned when CUDA is available), so the builder is a map-style dataset that works under a DataLoader
with workers and that `ResidentSequence(builder, device)` moves to the GPU unchanged. `write()` emits the reference's own
files (flowpair_*.npz and shuffle_False_gap_XX_sequence_XXXXX.pt) for its train.py / datasets.
"""
import glob
import os

import numpy as np
import torch

FRAME_FMT = 'frame_%05d.npz'
FLOW_FMT = 'flowpair_%05d_%05d.npz'
SEQ_FMT = 'shuffle_False_gap_%02d_sequence_%05d.pt'


def pair_list(n_frames, gaps):
    """[(f, f + g)] for every gap g and f < n_frames - 1 - g (generate_sequence_midas.py:186-193 with bs = 1)."""
    return [(f, f + g) for g in gaps for f in range(n_frames - 1 - g)]


def read_npz(path):
    """The arrays of an .npz file. An entry stored as None (a 0-d object array: the ShutterStock frame files write
    motion_seg=None) is left out, so it reads as absent."""
    with np.load(path, allow_pickle=True) as d:
        out = {k: d[k] for k in d.keys()}
    return {k: v for k, v in out.items() if not (v.dtype == object and v.shape == () and v.item() is None)}


def pose_tensors(im1, im2):
    """prepare_pose_dict_one_way (generate_sequence_midas.py:49-87): transposed rotations, K^T and (K^-1)^T, fp32."""
    def t(a, shape):
        return torch.from_numpy(np.ascontiguousarray(a)).float().reshape(shape)
    p1, p2, K = im1['pose_c2w'], im2['pose_c2w'], im1['intrinsics']
    m33, v3 = (1, 1, 1, 3, 3), (1, 1, 1, 1, 3)
    return {'R_1': t(p1[:3, :3].T, m33), 'R_2': t(p2[:3, :3].T, m33), 'R_1_T': t(p1[:3, :3], m33), 'R_2_T': t(p2[:3, :3], m33),
            't_1': t(p1[:3, 3], v3), 't_2': t(p2[:3, 3], v3), 'K': t(K.T, m33), 'K_inv': t(np.linalg.inv(K).T, m33)}


def pair_file_masks(mask):
    """uint8 flowpair mask [.., H, W] (1 = bad) -> the pair file's fp32 1 - ceil(mask), [.., H, W, 1, 1] (1 = valid)."""
    return 1 - torch.ceil(torch.as_tensor(mask).float())[..., None, None]


def to_dataset_item(pf, n_frames, unit=1.0):
    """davis_sequence.Dataset.__getitem__ (train mode, davis_sequence.py:98-115) on a loaded pair file `pf`."""
    _, H, W, _ = pf['img_1'].shape
    out = {k: v.float() for k, v in pf.items() if not isinstance(v, list)}
    out['img_1'] = pf['img_1'].permute([0, 3, 1, 2]).float()
    out['img_2'] = pf['img_2'].permute([0, 3, 1, 2]).float()
    out['time_step'] = unit / n_frames
    out['time_stamp_1'] = (pf['fid_1'].reshape([-1, 1, 1, 1]).expand(-1, -1, H, W) / n_frames).float()
    out['time_stamp_2'] = (pf['fid_2'].reshape([-1, 1, 1, 1]).expand(-1, -1, H, W) / n_frames).float()
    out['frame_id_1'] = torch.from_numpy(np.asarray(pf['fid_1'])).float()
    out['frame_id_2'] = torch.from_numpy(np.asarray(pf['fid_2'])).float()
    return out


def process_raw_flows(flow_1_2, flow_2_1, H, W, device=None):
    """raw flows [B,h,w,2] (host arrays or tensors, one gap) -> host tensors (flow_1_2, flow_2_1 [B,H,W,2] fp32, mask_1,
    mask_2 [B,H,W] uint8, 1 = bad): one resize launch per direction when (h, w) != (H, W), then one mask launch."""
    device = torch.device(device if device is not None else 'cuda')
    if device.type != 'cuda':
        raise RuntimeError('raw flows are resized and masked by the CUDA kernels of dvd_b200; a CUDA device is needed')
    f12 = torch.as_tensor(flow_1_2, dtype=torch.float32).to(device, non_blocking=True).contiguous()
    f21 = torch.as_tensor(flow_2_1, dtype=torch.float32).to(device, non_blocking=True).contiguous()
    return tuple(t.cpu() for t in finish_flows(f12, f21, H, W))


def finish_flows(f12, f21, H, W):
    """device flows [B,h,w,2] -> (flow_1_2, flow_2_1 [B,H,W,2], mask_1, mask_2 [B,H,W] uint8), still on the device"""
    from . import ops
    if tuple(f12.shape[1:3]) != (H, W):
        f12, f21 = ops.flow_resize_cubic(f12, H, W), ops.flow_resize_cubic(f21, H, W)
    m1, m2 = ops.flow_pair_masks(f12, f21, convention='flowpair')
    return f12, f21, m1, m2


RAFT_SIZE = (288, 512)      # generate_flows.py:121-122


def raft_images(frames, size=RAFT_SIZE):
    """The frames' colour images at RAFT's resolution, [n,3,h,w] fp32 in 0..255 (generate_flows.py:119-126). The reference
    resizes with skimage.transform.resize(anti_aliasing=True); this is cv2.resize with INTER_AREA (INTER_LINEAR when
    enlarging), a different filter: flows of a video whose frames are not already `size` differ from the reference's by
    what the filter changes."""
    import cv2
    h, w = size
    out = []
    for d in frames:
        im = np.asarray(d['img_orig'] if 'img_orig' in d else d['img'], np.float32) * 255
        if im.shape[:2] != (h, w):
            shrink = im.shape[0] >= h and im.shape[1] >= w
            im = cv2.resize(im, (w, h), interpolation=cv2.INTER_AREA if shrink else cv2.INTER_LINEAR)
        out.append(torch.from_numpy(np.ascontiguousarray(im.transpose(2, 0, 1))))
    return torch.stack(out)


class PairBuilder(torch.utils.data.Dataset):
    def __init__(self, frames_dir, flows_dir, gaps, unit=1.0, device=None, name=None, raft=None, raft_iters=20, images=None,
                 raft_chunk=16):
        """frames_dir: frames_midas/<track>; flows_dir: flow_pairs/<track>; gaps: iterable of frame gaps; unit: 2.0 for a
        subsampled video (davis_sequence.py:93-96); device: where raw flows are processed (default cuda if available).
        With flows_dir None the flows are estimated here: raft is a dvd_b200.raft.RaftNet on the device, images the frames at
        RAFT's resolution ([n,3,h,w] in 0..255, one per frame file in order; default raft_images() of the frame files), and
        raft_chunk the number of pairs per launch."""
        if flows_dir is None and raft is None:
            raise ValueError('PairBuilder needs optical flows: a directory of flowpair_*.npz or a RaftNet to estimate them')
        if flows_dir is not None and raft is not None:
            raise ValueError('give either a flow directory or a RaftNet, not both')
        files = sorted(glob.glob(os.path.join(frames_dir, 'frame_*.npz')))
        if not files:
            raise FileNotFoundError('no frame_*.npz under %s' % frames_dir)
        self.n_frames = len(files) + 0.0
        self.unit = float(unit)
        self.name = name or os.path.basename(os.path.normpath(frames_dir))
        self.gaps = [int(g) for g in gaps]
        self.pairs = pair_list(len(files), self.gaps)
        if not self.pairs:
            raise ValueError('%d frames give no pair for gaps %s' % (len(files), self.gaps))
        pin = torch.cuda.is_available()
        used = sorted({f for p in self.pairs for f in p})
        frames = {f: read_npz(os.path.join(frames_dir, FRAME_FMT % f)) for f in used}
        self.H, self.W = frames[used[0]]['img'].shape[:2]
        self.frames = {}
        for f, d in frames.items():
            fr = {'img': torch.from_numpy(d['img']).float()[None, ...],
                  'depth_mvs': torch.from_numpy(d['depth_mvs']).float().reshape(1, 1, self.H, self.W),
                  'depth_pred': torch.from_numpy(d['depth_pred']).float().reshape(1, 1, self.H, self.W)}
            if 'motion_seg' in d:
                fr['motion_seg'] = torch.from_numpy(d['motion_seg'])[None, ..., None, None].float()
            self.frames[f] = {k: (v.pin_memory() if pin else v) for k, v in fr.items()}
        self.poses = [pose_tensors(frames[a], frames[b]) for a, b in self.pairs]
        # per pair: flow_1_2, flow_2_1 [H,W,2] fp32 and mask_1, mask_2 [H,W] uint8 (1 = bad), as in flowpair_*.npz
        self.flows = [None] * len(self.pairs)
        self.raw_pairs = 0
        raw = {}
        if raft is not None:
            if images is None:
                images = raft_images([frames[f] for f in used])
            elif len(images) == len(files):
                images = images[used]
            self._estimate_flows(raft, images, used, int(raft_iters), int(raft_chunk))
        for i, (a, b) in enumerate(self.pairs if raft is None else ()):
            d = read_npz(os.path.join(flows_dir, FLOW_FMT % (a, b)))
            f12, f21 = np.asarray(d['flow_1_2'], np.float32), np.asarray(d['flow_2_1'], np.float32)
            if f12.shape != f21.shape or f12.ndim != 3 or f12.shape[-1] != 2:
                raise ValueError('%s: flows must be [h,w,2], got %s and %s' % (FLOW_FMT % (a, b), f12.shape, f21.shape))
            if 'mask_1' in d and 'mask_2' in d and f12.shape[:2] == (self.H, self.W):
                self.flows[i] = tuple(torch.from_numpy(np.ascontiguousarray(x)) for x in
                                      (f12, f21, np.asarray(d['mask_1'], np.uint8), np.asarray(d['mask_2'], np.uint8)))
            else:
                raw.setdefault((b - a, f12.shape), []).append((i, f12, f21))
        if raw:
            self._process_raw(raw, device)
        if pin:
            self.flows = [tuple(t.pin_memory() for t in fl) for fl in self.flows]
        counter = {}
        self.seq_names = []
        for a, b in self.pairs:
            c = counter.get(b - a, 0)
            counter[b - a] = c + 1
            self.seq_names.append(SEQ_FMT % (b - a, c))

    def _process_raw(self, raw, device):
        for (_, (h, w, _)), items in sorted(raw.items(), key=lambda kv: kv[0][0]):
            f12, f21, m1, m2 = process_raw_flows(np.stack([it[1] for it in items]), np.stack([it[2] for it in items]),
                                                 self.H, self.W, device)
            for j, (i, _, _) in enumerate(items):
                self.flows[i] = (f12[j].clone(), f21[j].clone(), m1[j].clone(), m2[j].clone())
            self.raw_pairs += len(items)

    def _estimate_flows(self, raft, images, used, iters, chunk):
        """RAFT on the device: every frame encoded once, then both directions of all pairs of a gap in chunks, handed to the
        resize and mask kernels without leaving the device; only the finished flows and masks are copied to the host."""
        if len(images) != len(used):
            raise ValueError('%d RAFT images for %d frames' % (len(images), len(used)))
        dev = next(raft.parameters()).device
        images = torch.as_tensor(images, dtype=torch.float32)
        feats = [raft.encode(images[i:i + chunk].to(dev)) for i in range(0, len(images), chunk)]
        feats = type(feats[0])(torch.cat([f.fmap for f in feats]), torch.cat([f.cnet for f in feats]))
        slot = {f: k for k, f in enumerate(used)}
        for i0 in range(0, len(self.pairs), chunk):
            ids = list(range(i0, min(i0 + chunk, len(self.pairs))))
            fa, fb = feats.index([slot[self.pairs[i][0]] for i in ids]), feats.index([slot[self.pairs[i][1]] for i in ids])
            out = finish_flows(raft.flow(fa, fb, iters), raft.flow(fb, fa, iters), self.H, self.W)
            f12, f21, m1, m2 = (t.cpu() for t in out)
            for j, i in enumerate(ids):
                self.flows[i] = (f12[j].clone(), f21[j].clone(), m1[j].clone(), m2[j].clone())
        self.raw_pairs = len(self.pairs)

    def __len__(self):
        return len(self.pairs)

    def flowpair(self, i):
        """The flowpair_%05d_%05d.npz content of pair i (generate_flows.py:149-155)."""
        (a, b), (f12, f21, m1, m2) = self.pairs[i], self.flows[i]
        return {'flow_1_2': f12.numpy(), 'flow_2_1': f21.numpy(), 'mask_1': m1.numpy(), 'mask_2': m2.numpy(),
                'frame_id_1': a, 'frame_id_2': b}

    def pair_file(self, i):
        """The sequence .pt dict of pair i (generate_sequence_midas.collate_sequence_fix_gap with one pair)."""
        (a, b), (f12, f21, m1, m2) = self.pairs[i], self.flows[i]
        fa, fb = self.frames[a], self.frames[b]
        mask_1, mask_2 = pair_file_masks(m1[None]), pair_file_masks(m2[None])
        d = dict(self.poses[i])
        d.update(img_1=fa['img'], img_2=fb['img'], depth_1=fa['depth_mvs'], flow_1_2=f12[None], flow_2_1=f21[None],
                 mask_1=mask_1, mask_2=mask_2, motion_seg_1=fa.get('motion_seg', mask_2), depth_pred_1=fa['depth_pred'],
                 fid_1=torch.FloatTensor([a]), fid_2=torch.FloatTensor([b]))
        return d

    def __getitem__(self, i):
        out = to_dataset_item(self.pair_file(i), self.n_frames, self.unit)
        out['pair_path'] = os.path.join(self.name, self.seq_names[i])
        return out

    def write(self, out_dir, flows_out=None):
        """Write the reference's files: flowpair_*.npz under `flows_out` (if given) and the sequence .pt files under
        `out_dir` (sequences_select_pairs_midas/<track>/001 for davis_sequence). Returns the number of pairs."""
        os.makedirs(out_dir, exist_ok=True)
        if flows_out:
            os.makedirs(flows_out, exist_ok=True)
        for i, (a, b) in enumerate(self.pairs):
            if flows_out:
                np.savez(os.path.join(flows_out, FLOW_FMT % (a, b)), **self.flowpair(i))
            pf = {k: v.clone() for k, v in self.pair_file(i).items()}
            torch.save(pf, os.path.join(out_dir, self.seq_names[i]))
        return len(self.pairs)
