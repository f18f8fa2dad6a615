"""Host-side mirror of networks/sceneflow_field.py: `SceneFlowFieldNet` (M1+M2) as a thin shell over the
wgmma kernels. Same ctor signature, same state-dict names (`convs.{0..5}.conv.{weight,bias}`), same
`forward(x[B,3,H,W], t[B,1,H,W]) -> [B,3,H,W]` (raw network output, before `/ sf_mag_div`).
"""
from torch import nn

from .blocks import Conv2dBlock, PeriodicEmbed
from .. import ops


class SceneFlowFieldNet(nn.Module):
    def __init__(self, time_dependent=True, N_freq_xyz=0, N_freq_t=0, output_dim=3, net_width=32, n_layers=3,
                 activation='lrelu', norm='none'):
        super().__init__()
        if output_dim != 3 or net_width != 256 or n_layers != 4 or activation != 'lrelu' or norm != 'none':
            raise NotImplementedError(
                'dvd_b200 implements the configuration the reference Model instantiates '
                '(net_width=256, n_layers=4, lrelu, no norm; models/scene_flow_motion_field.py:107)')
        ops.check_mlp_counts(N_freq_xyz, N_freq_t, time_dependent)   # fail at construction, not at the first step
        n_xyz = 3 + 6 * N_freq_xyz
        n_t = 1 + 2 * N_freq_t
        n_in = n_xyz + n_t if time_dependent else n_xyz
        convs = [Conv2dBlock(n_in, net_width, 1, 1, norm=norm, activation=activation)]
        convs += [Conv2dBlock(net_width, net_width, 1, 1, norm=norm, activation=activation) for _ in range(n_layers)]
        convs.append(Conv2dBlock(net_width, output_dim, 1, 1, norm='none', activation='none'))
        self.convs = nn.Sequential(*convs)
        self.t_embed = PeriodicEmbed(max_freq=N_freq_t, N_freq=N_freq_t) if N_freq_t > 0 else nn.Identity()
        self.xyz_embed = PeriodicEmbed(max_freq=N_freq_xyz, N_freq=N_freq_xyz) if N_freq_xyz > 0 else nn.Identity()
        self.time_dependent = time_dependent
        self.n_freq_xyz, self.n_freq_t = N_freq_xyz, N_freq_t
        self._packed = None
        self._packed_version = None

    # ---- kernel-facing helpers ----------------------------------------------------------------------
    def weights(self):
        return [c.conv.weight for c in self.convs]

    def biases(self):
        return [c.conv.bias for c in self.convs]

    def mlp_cfg(self, sf_mag_div=1.0):
        return ops.make_mlp_cfg(self.n_freq_xyz, self.n_freq_t if self.time_dependent else 0,
                                self.time_dependent, sf_mag_div)

    def packed(self, sf_mag_div=1.0, force=False):
        """bf16 (hi,lo) wgmma images of the weights; re-packed whenever a parameter changed
        (tracked through the tensors' in-place version counters) or `force`."""
        ver = (float(sf_mag_div),) + tuple(p._version for p in self.parameters()) + tuple(p.data_ptr() for p in self.parameters())
        if force or self._packed is None or self._packed_version != ver:
            dev = self.convs[0].conv.weight.device
            if self._packed is None or self._packed.cfg.sf_mag_div != float(sf_mag_div) or self._packed.fwd.device != dev:
                self._packed = ops.PackedMlp(self.mlp_cfg(sf_mag_div), dev)
            ws = [w.reshape(w.shape[0], -1) for w in self.weights()]
            self._packed.refresh(ws, self.biases())
            self._packed_version = ver
        return self._packed

    def chain(self, p0, t0, dt, n_eval, n_acc, sf_mag_div):
        """Euler chain (Model.forward_sf_net_multi_step) → (acc, s_steps)."""
        pk = self.packed(sf_mag_div)
        ws = [w.reshape(w.shape[0], -1) for w in self.weights()]
        return ops.scene_flow_chain(p0, t0, pk, dt, n_eval, n_acc, ws, self.biases())

    def forward(self, x, t=None):
        if t is None and self.time_dependent:
            raise ValueError
        acc, _ = self.chain(x.contiguous(), t.contiguous() if t is not None else None, 0.0, 1, 1, 1.0)
        return acc
