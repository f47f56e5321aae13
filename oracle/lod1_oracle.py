"""CPU restatement of the lod-1 refinement path (num_lods = 2) on top of recon_oracle.py.

  sdf_volume           SparseSdfNetwork.get_sdf_volume          reference sparse_sdf_network.py:441-474
  prune                get_valid_sparse_coords_by_sdf           reference sparse_neus_renderer.py:822-879
  conditional_volume   get_conditional_volume, lod > 0 branch   reference sparse_sdf_network.py:198-219,336-400

Written the way the reference computes (avg_pool3d dilation, the threshold loop, np.random.choice on numpy's global
generator, children in parent order), not the way the kernels do, so that the tests compare two formulations.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from . import recon_oracle as O

# upsample(): child k of a parent adds these offsets to (x, y, z) (pos_list = [1, 2, 3, [1, 2], [1, 3], [2, 3], [1, 2, 3]])
CHILD_OFFSETS = torch.tensor([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [1, 0, 1], [0, 1, 1], [1, 1, 1]],
                             dtype=torch.float32)


def sdf_volume(dense, occ, origin, voxel_size, sd):
    """[1,1,D,D,D]: the SDF MLP at coords * voxel_size + origin with each occupied voxel's own latent, 1.0 elsewhere."""
    C, D = dense.shape[1], dense.shape[2]
    vol = dense.reshape(C, -1).t()
    m = occ.reshape(-1) > 0
    pts = O.lattice_coords(D) * voxel_size + origin.reshape(1, 3)
    out = torch.ones(D ** 3, 1)
    out[m] = O.sdf_mlp(pts[m], vol[m], sd)[:, :1]
    return out.reshape(1, 1, D, D, D)


def prune(sdf_vol, occ, feature_volume, threshold=0.02, maximum_pts=110000):
    """-> coords [N,4] (0, x, y, z), feats [N,C], the final mask [D^3] and the threshold used."""
    C, D = feature_volume.shape[0], feature_volume.shape[1]
    coords = O.lattice_coords(D)
    mask = occ.reshape(-1, 1) > 0
    feats = feature_volume.reshape(C, -1).t()

    def run(t):
        m = (torch.abs(sdf_vol.reshape(-1, 1)) < t).float().reshape(1, 1, D, D, D)
        m = F.avg_pool3d(m, kernel_size=7, stride=1, padding=3).reshape(-1, 1) > 0
        final = torch.logical_and(mask, m)[:, 0]
        return final, torch.sum(final.float())

    final, n = run(threshold)
    while n > maximum_pts and threshold > 0.003:
        threshold = threshold - 0.002
        final, n = run(threshold)
    vc = torch.cat([torch.zeros(int(final.sum()), 1), coords[final]], 1)
    vf = feats[final]
    if n > maximum_pts:
        n = n.long()
        keep = torch.ones([int(n)]) > 0
        choice = np.random.choice(n.numpy(), n.numpy() - maximum_pts, replace=False)
        keep[torch.nonzero(keep)[choice]] = False
        vc, vf = vc[keep], vf[keep]
        idx = torch.nonzero(final)[:, 0][keep]
        final = torch.zeros_like(final)
        final[idx] = True
    return vc, vf, final, threshold


def conditional_volume(fmaps, origin, proj, sd, dim, voxel_size, H, W, pre_coords, pre_feats):
    """lod-1 conditional volume from the doubled pre_coords [N,4] and pre_feats [N,16].  Returns dict(dense, occ, xyz, cost,
    rows) with the kept children xyz / cost / U-Net rows in the reference's (parent-major) order."""
    feats = O.compress_features(fmaps, sd)
    up = (pre_coords[:, None, 1:] + CHILD_OFFSETS[None]).reshape(-1, 3)
    up_feat = pre_feats.repeat_interleave(8, 0)
    mv, mm = O.backproject_features(up, origin, voxel_size, feats, proj, H, W)
    keep = mm.sum(-1) > 1
    xyz = up[keep]
    cost = torch.cat([O.variance_mean(mv[keep], mm[keep]), up_feat[keep]], 1)
    rows = O.cost_reg_net(cost, xyz, sd)
    dense, occ = O.sparse_to_dense(xyz, rows, dim)
    return {"dense": dense, "occ": occ, "xyz": xyz, "cost": cost, "rows": rows}
