"""GeneralRenderingNetwork + SingleVarianceNetwork parameter holders for the fused blend kernel.

Mirror of reference reconstruction/models/rendering_network.py:26-129 (state-dict keys
s, ray_dir_fc.{0,2}, base_fc.{0,2}, vis_fc.{0,2}, vis_fc2.{0,2}, rgb_fc.{0,2,4}) and
reconstruction/models/fields.py:179-185.  The arithmetic of forward() lives in csrc/render_tc.cu
(render_blend_tc_kernel: the per-(sample, view) MLPs as mma.sync chains, default) and csrc/render.cu
(render_blend_kernel: fp32 FMA, O2345_BLEND_FP32, the reference of the parity tests), fused with the Projector's
per-view feature fetch, so the [n_views, n_rays, n_samples, 59] tensors the reference materialises never exist.  Both
kernels share the per-sample front end and the weight-pack layout in csrc/blend_common.cuh.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib as L


class GeneralRenderingNetwork(nn.Module):
    def __init__(self, in_geometry_feat_ch=8, in_rendering_feat_ch=56, anti_alias_pooling=True):
        super().__init__()
        if (in_geometry_feat_ch, in_rendering_feat_ch, anti_alias_pooling) != (16, 56, True):
            raise NotImplementedError("blend kernel is specialised for 16 geometry / 56 rendering channels with pooling")
        self.in_geometry_feat_ch, self.in_rendering_feat_ch = in_geometry_feat_ch, in_rendering_feat_ch
        self.anti_alias_pooling = anti_alias_pooling
        self.s = nn.Parameter(torch.tensor(0.2))
        act = nn.ELU(inplace=True)
        c = in_rendering_feat_ch + 3
        self.ray_dir_fc = nn.Sequential(nn.Linear(4, 16), act, nn.Linear(16, c), act)
        self.base_fc = nn.Sequential(nn.Linear(c * 3 + in_geometry_feat_ch, 64), act, nn.Linear(64, 32), act)
        self.vis_fc = nn.Sequential(nn.Linear(32, 32), act, nn.Linear(32, 33), act)
        self.vis_fc2 = nn.Sequential(nn.Linear(32, 32), act, nn.Linear(32, 1), nn.Sigmoid())
        self.rgb_fc = nn.Sequential(nn.Linear(32 + 1 + 4, 16), act, nn.Linear(16, 8), act, nn.Linear(8, 1))
        self._pack, self._pack_key = None, None

    def packed(self):
        """Weights in the [in][out] layout documented in csrc/blend_common.cuh (O2345_RNET_PACK_FLOATS floats)."""
        key = tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._pack is not None and key == self._pack_key:
            return self._pack
        f = lambda t: t.detach().float()
        dev = self.s.device

        def wt(lin, pad_out=None):  # [out,in] -> [in][out(+pad)]
            w = f(lin.weight).t().contiguous()
            if pad_out and w.shape[1] < pad_out:
                w = torch.cat([w, torch.zeros(w.shape[0], pad_out - w.shape[1], device=dev)], 1)
            return w.reshape(-1)

        def pad(v, n):
            v = f(v).reshape(-1)
            return torch.cat([v, torch.zeros(n - v.numel(), device=dev)])

        b0 = f(self.base_fc[0].weight).t().contiguous()      # [193][64], rows: geo 16 | mean 59 | var 59 | feat 59
        v1 = self.vis_fc[2]
        parts = [
            wt(self.ray_dir_fc[0]), f(self.ray_dir_fc[0].bias),
            wt(self.ray_dir_fc[2], 64), pad(self.ray_dir_fc[2].bias, 64),
            b0.reshape(-1), f(self.base_fc[0].bias),
            wt(self.base_fc[2]), f(self.base_fc[2].bias),
            wt(self.vis_fc[0]), f(self.vis_fc[0].bias),
            f(v1.weight)[:32].t().contiguous().reshape(-1), f(v1.bias)[:32],
            f(v1.weight)[32], pad(v1.bias[32:33], 4),
            wt(self.vis_fc2[0]), f(self.vis_fc2[0].bias),
            f(self.vis_fc2[2].weight).reshape(-1), pad(self.vis_fc2[2].bias, 4),
            wt(self.rgb_fc[0]), f(self.rgb_fc[0].bias),
            wt(self.rgb_fc[2]), f(self.rgb_fc[2].bias),
            f(self.rgb_fc[4].weight).reshape(-1), pad(self.rgb_fc[4].bias, 4),
            pad(f(self.s).abs(), 4),
        ]
        pack = torch.cat([p.reshape(-1) for p in parts]).contiguous()
        assert pack.numel() == L.RNET_PACK_FLOATS, pack.numel()
        self._pack, self._pack_key = pack, key
        return pack

    def forward(self, geometry_feat, rgb_feat, ray_diff, mask):
        raise NotImplementedError(
            "the o2345 path fuses the Projector fetch with this network (SparseNeuSRenderer.render / "
            "blend_points); pre-gathered [V,R,S,59] inputs are never materialised")


class SingleVarianceNetwork(nn.Module):
    def __init__(self, init_val=1.0):
        super().__init__()
        self.register_parameter('variance', nn.Parameter(torch.tensor(init_val)))

    def forward(self, x):
        return torch.ones([len(x), 1], device=x.device) * torch.exp(self.variance * 10.0)

    def inv_s(self):
        """exp(10 * variance) clipped like render_core (reference sparse_neus_renderer.py:340)."""
        return float(torch.exp(self.variance.detach() * 10.0).clip(1e-6, 1e6))
