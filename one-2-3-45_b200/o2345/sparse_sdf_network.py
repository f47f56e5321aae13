"""SparseSdfNetwork on the o2345 CUDA kernels.

Mirror of reference reconstruction/models/sparse_sdf_network.py:139-499: same constructor
arguments, same state-dict keys (compress_layer.*, sparse_costreg_net.conv{0..11}.net.{0,1}.*,
sdf_layer.lin{0,1,2}.{bias,weight_g,weight_v}), same method signatures and return-dict keys.
Inference only: the analytic gradient replaces autograd (reference :476-499).  `sdf` / `gradient` run
csrc/sdf_mlp_tc.cu (split-fp16 tensor-core GEMMs, fp32-grade values; `ops.SDF_PRECISION`) or csrc/sdf_mlp.cu (fp32 FMA).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ._lib import inference_only
from . import ops
from .featurenet import ConvBnReLU
from .synthetic import costreg_channels


class _SparseConvParams(nn.Module):
    """spnn.Conv3d parameter holder: `kernel` [27, Cin, Cout]."""

    def __init__(self, cin, cout):
        super().__init__()
        self.kernel = nn.Parameter(torch.zeros(27, cin, cout))


class _SparseBlock(nn.Module):
    """BasicSparse(De)ConvolutionBlock: net.0 = conv, net.1 = BatchNorm (reference tsparse/modules.py:94-124)."""

    def __init__(self, cin, cout):
        super().__init__()
        self.net = nn.Sequential(_SparseConvParams(cin, cout), nn.BatchNorm1d(cout), nn.Identity())


class SparseCostRegNet(nn.Module):
    """3-level sparse U-Net (reference tsparse/modules.py:259-304) executed on index lattices."""

    def __init__(self, d_in, d_out=8):
        super().__init__()
        self.d_in, self.d_out = d_in, d_out
        for name, cin, cout in costreg_channels(d_in, d_out):
            setattr(self, name, _SparseBlock(cin, cout))

    def _block(self, name, x, lin, lout, mode, skip=None):
        blk = getattr(self, name).net
        return ops.sp_conv_bn_relu(x, lin, lout, mode, ops.cf32(blk[0].kernel), ops.cf32(blk[1].weight),
                                   ops.cf32(blk[1].bias), skip=skip, eps=blk[1].eps)

    @torch.no_grad()
    def forward(self, feats, level0: ops.SparseLevel):
        l0 = level0
        l1 = ops.sp_coarsen(l0)
        l2 = ops.sp_coarsen(l1)
        l3 = ops.sp_coarsen(l2)
        conv0 = self._block("conv0", feats, l0, l0, 0)
        conv2 = self._block("conv2", self._block("conv1", conv0, l0, l1, 1), l1, l1, 0)
        conv4 = self._block("conv4", self._block("conv3", conv2, l1, l2, 1), l2, l2, 0)
        x = self._block("conv6", self._block("conv5", conv4, l2, l3, 1), l3, l3, 0)
        x = self._block("conv7", x, l3, l2, 2, skip=conv4)
        x = self._block("conv9", x, l2, l1, 2, skip=conv2)
        x = self._block("conv11", x, l1, l0, 2, skip=conv0)
        return x


class _WeightNormLinear(nn.Module):
    """nn.utils.weight_norm(nn.Linear) parameter holder: bias, weight_g [out,1], weight_v [out,in]."""

    def __init__(self, din, dout):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(dout))
        self.weight_g = nn.Parameter(torch.ones(dout, 1))
        self.weight_v = nn.Parameter(torch.zeros(dout, din))

    def effective(self):
        v = self.weight_v.detach().float()
        return v * (self.weight_g.detach().float() / v.norm(dim=1, keepdim=True))


class LatentSDFLayer(nn.Module):
    """39 -> 128 -> (+16) 128 -> (+16) 128 weight-normed MLP (reference sparse_sdf_network.py:35-136)."""

    def __init__(self, d_in=3, d_out=129, d_hidden=128, n_layers=4, multires=6, d_conditional_feature=16, **_):
        super().__init__()
        if (d_hidden, n_layers, multires, d_conditional_feature) != (128, 4, 6, 16):
            raise NotImplementedError("the sm_90a SDF kernel is specialised for hidden 128, 4 layers, multires 6, latent 16")
        d_pe = d_in * (2 * multires + 1)
        self.lin0 = _WeightNormLinear(d_pe, d_hidden)
        self.lin1 = _WeightNormLinear(d_hidden + d_conditional_feature, d_hidden)
        self.lin2 = _WeightNormLinear(d_hidden + d_conditional_feature, d_hidden)
        self._pack, self._pack_key = None, None

    def packed(self):
        key = tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._pack is None or key != self._pack_key:
            self._pack = ops.sdf_pack_weights(self.lin0.effective(), self.lin0.bias, self.lin1.effective(),
                                              self.lin1.bias, self.lin2.effective(), self.lin2.bias)
            self._pack_key = key
        return self._pack


def channel_last_volume(conditional_volume):
    """[1,16,X,Y,Z] -> cached channel-last [X,Y,Z,16] copy used by the gather kernels."""
    cl = getattr(conditional_volume, "_o2345_cl", None)
    key = (conditional_volume.data_ptr(), conditional_volume._version)
    if cl is None or cl[0] != key:
        v = conditional_volume.detach().float()
        if v.dim() == 5:
            v = v[0]
        cl = (key, v.permute(1, 2, 3, 0).contiguous())
        try:
            conditional_volume._o2345_cl = cl
        except Exception:
            pass
    return cl[1]


class SparseSdfNetwork(nn.Module):
    def __init__(self, lod, ch_in, voxel_size, vol_dims, hidden_dim=128, activation='softplus',
                 cost_type='variance_mean', d_pyramid_feature_compress=16, regnet_d_out=8, num_sdf_layers=4,
                 multires=6):
        super().__init__()
        if lod not in (0, 1):
            raise NotImplementedError("lod 0 and lod 1 (num_lods <= 2) are on the accelerated path")
        if d_pyramid_feature_compress not in ((16,) if lod == 0 else (8, 16)) or regnet_d_out != 16 or activation != 'softplus':
            raise NotImplementedError("kernels are specialised for 16 (lod 0) or 8 / 16 (lod 1) compressed channels, "
                                      "16 latent channels and softplus")
        self.lod, self.ch_in, self.voxel_size = lod, ch_in, voxel_size
        self.vol_dims = torch.tensor(vol_dims)
        self.hidden_dim, self.cost_type = hidden_dim, cost_type
        self.d_pyramid_feature_compress, self.regnet_d_out, self.multires = d_pyramid_feature_compress, regnet_d_out, multires
        self.compress_layer = ConvBnReLU(ch_in, d_pyramid_feature_compress, 3, 1, 1)
        # lod > 0: the parent's 16 features join the variance / mean cost (reference :174-178)
        d_in = 2 * d_pyramid_feature_compress + (16 if lod > 0 else 0)
        self.sparse_costreg_net = SparseCostRegNet(d_in=d_in, d_out=regnet_d_out)
        self.sdf_layer = LatentSDFLayer(d_in=3, d_out=hidden_dim + 1, d_hidden=hidden_dim, n_layers=num_sdf_layers,
                                        multires=multires, d_conditional_feature=16)
        self._coords = None

    # ------------------------------------------------------------------ B2-B7
    @inference_only
    def get_conditional_volume(self, feature_maps, partial_vol_origin, proj_mats, sizeH=None, sizeW=None, lod=0,
                               pre_coords=None, pre_feats=None):
        """feature_maps [1,V,C,H,W], partial_vol_origin [1,3], proj_mats [1,V,4,4] -> dict with
        dense_volume_scale{lod} [1,16,D,D,D], valid_mask_volume_scale{lod} / visible_mask_scale{lod} [1,1,D,D,D],
        coords_scale{lod} [1,3,D,D,D] (reference sparse_sdf_network.py:286-400).  With lod 1 (the network's own lod,
        as in the reference) the voxels are the 8 children of every row of pre_coords [N,4] (batch, x, y, z in this
        lattice's units) seen by more than one view, and pre_feats [N,16] are their parents' features."""
        assert feature_maps.shape[0] == 1, "batch size 1 is assumed (as in the reference, :263)"
        dev = proj_mats.device
        D = int(self.vol_dims[0])
        V, _, H, W = feature_maps.shape[1:]
        sizeH = H if sizeH is None else int(sizeH)
        sizeW = W if sizeW is None else int(sizeW)
        C = self.d_pyramid_feature_compress
        feats = torch.empty(V, H, W, C, dtype=torch.float32, device=dev)
        self.compress_layer.run(feature_maps[0], out=feats, layout="nhwc")
        proj = ops.cf32(proj_mats[0])
        origin = ops.cf32(partial_vol_origin[0])
        n0 = D ** 3
        extra = {}
        if self.lod == 0:
            min_views = min(1, V - 1)
            bits, keep = ops.frustum_mask(proj, origin, self.voxel_size, D, sizeH, sizeW, min_views)
            rows, index, count = ops.compact(keep)
            max_rows = n0
            cost = ops.costvol_gather(feats, proj, origin, self.voxel_size, D, sizeH, sizeW, rows, count, bits, max_rows)
        else:
            if pre_coords is None or pre_feats is None:
                raise ValueError("lod > 0 needs pre_coords and pre_feats (the pruned voxels of the previous lod)")
            pre_coords, pre_feats = ops.cf32(pre_coords), ops.cf32(pre_feats)
            if pre_coords.dim() != 2 or pre_coords.shape[1] != 4 or pre_feats.shape != (pre_coords.shape[0], 16):
                raise ValueError(f"pre_coords must be [N,4] and pre_feats [N,16], got {tuple(pre_coords.shape)} / "
                                 f"{tuple(pre_feats.shape)}")
            if pre_coords.shape[0] == 0:
                raise ValueError("no voxels survived the previous lod's pruning")
            # `> 1` views, fixed (reference :355): the frustum test with min_views = 1 at this lattice
            bits, fkeep = ops.frustum_mask(proj, origin, self.voxel_size, D, sizeH, sizeW, 1)
            keep, parent = ops.lod_children(pre_coords, D, fkeep)
            rows, index, count = ops.compact(keep)
            max_rows = min(8 * pre_coords.shape[0], n0)
            cost = ops.costvol_gather_lod(feats, proj, origin, self.voxel_size, D, sizeH, sizeW, rows, count, bits, max_rows,
                                          parent, pre_feats)
            extra = {"parent": parent, "frustum_keep": fkeep}
        level0 = ops.SparseLevel(D, rows, index, count, max_rows)
        reg = self.sparse_costreg_net(cost, level0)
        vol_cl, vol_cf, occ = ops.dense_scatter(reg, rows, count, D, max_rows)
        vol_cf._o2345_cl = ((vol_cf.data_ptr(), vol_cf._version), vol_cl)
        if self._coords is None or self._coords.device != dev:
            r = torch.arange(D, dtype=torch.float32, device=dev)
            self._coords = torch.stack(torch.meshgrid(r, r, r, indexing="ij"))[None]
        self._last = {"mask_bits": bits, "keep": keep, "rows": rows, "index": index, "count": count, "cost": cost, "reg": reg,
                      "feats_nhwc": feats, **extra}
        return {"dense_volume_scale%d" % self.lod: vol_cf, "valid_mask_volume_scale%d" % self.lod: occ,
                "visible_mask_scale%d" % self.lod: occ, "coords_scale%d" % self.lod: self._coords}

    # ------------------------------------------------------------------ B8
    @inference_only
    def sdf(self, pts, conditional_volume, lod):
        """pts [n,3] -> {'sdf_pts_scale0' [n,1], 'sdf_features_pts_scale0' [n,127], 'sampled_latent_scale0' [n,16]}."""
        out = ops.sdf_query(ops.PointSource.explicit(pts), channel_last_volume(conditional_volume),
                            self.sdf_layer.packed(), want_feat=True, want_latent=True)
        return {"sdf_pts_scale%d" % lod: out["sdf"], "sdf_features_pts_scale%d" % lod: out["feat"],
                "sampled_latent_scale%d" % lod: out["latent"]}

    # ------------------------------------------------------------------ B9
    @inference_only
    def gradient(self, x, conditional_volume, lod):
        """Analytic d sdf / d x, shape [n,1,3] (the reference differentiates with autograd, :476-499)."""
        out = ops.sdf_query(ops.PointSource.explicit(x), channel_last_volume(conditional_volume),
                            self.sdf_layer.packed(), want_grad=True)
        return out["grad"].unsqueeze(1)

    @inference_only
    def get_sdf_volume(self, conditional_volume, mask_volume, coords_volume, partial_origin):
        """[1,1,D,D,D]: the SDF MLP at every voxel with mask_volume > 0, at coords * voxel_size + partial_origin with
        that voxel's own latent row, 1.0 elsewhere (reference :441-474).  coords_volume must be the lattice
        (coords_scale* of get_conditional_volume): the kernel derives each voxel's coordinates from its index."""
        vol_cl = channel_last_volume(conditional_volume)
        D = vol_cl.shape[0]
        if tuple(coords_volume.shape[-3:]) != (D, D, D) or mask_volume.numel() != D ** 3:
            raise ValueError("conditional_volume, mask_volume and coords_volume must describe the same D^3 lattice")
        sdf = ops.sdf_voxels(ops.cf32(mask_volume).view(-1), vol_cl, ops.cf32(partial_origin).view(-1), self.voxel_size,
                             self.sdf_layer.packed())
        return sdf.view(1, 1, D, D, D)
