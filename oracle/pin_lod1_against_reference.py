"""Pin oracle/lod1_oracle.py against the REAL reference and freeze tests/golden/lod1_mini.npz.

Runs only where the reference tree is present (it is imported with the stubs of oracle/_refimport.py, as
pin_against_reference.py does):

    python -m oracle.pin_lod1_against_reference

Mini configuration of pin_against_reference.py (6 views of 64^2, D0 = 24 -> D1 = 48, R = 32), seeded weights
(o2345.synthetic.all_states(0) + lod1_states(0)).  Rows, each the reference against the CPU restatement:
  get_sdf_volume                          the lod-0 SDF volume (stored whole: the GPU prune is fed exactly these values)
  get_valid_sparse_coords_by_sdf x 3      the default budget, one that stops the threshold ladder part-way, one that
                                          forces the subsample (numpy seeded with PRUNE_SEED before each call)
  lod-1 get_conditional_volume            children keep flags, cost rows (lattice order), dense volume, occupancy
  lod-1 sdf / -sdf grid / vertex colours  on the mini points, the R^3 lattice, the mini vertices (lod-0 feature maps)
Float arrays are stored subsampled, flags as packed bits (np.packbits of the lattice mask).
"""
from __future__ import annotations

import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "one-2-3-45_b200"))
sys.path.insert(0, ROOT)

from o2345 import synthetic as S  # noqa: E402
from oracle import _refimport  # noqa: E402
from oracle import lod1_oracle as L1  # noqa: E402
from oracle import recon_oracle as O  # noqa: E402
from oracle.pin_against_reference import GOLD, MINI, mini_points, mini_scene, report, t  # noqa: E402

PRUNE_SEED = 11
PRUNE_CASES = ("default", "ladder", "subsample")


def lattice_mask(coords, D):
    """[N,4] (b, x, y, z) float coordinates -> bool [D^3] lattice mask."""
    c = coords[:, 1:].long()
    m = torch.zeros(D ** 3, dtype=torch.bool)
    m[(c[:, 0] * D + c[:, 1]) * D + c[:, 2]] = True
    return m


def lattice_order(xyz, D):
    c = xyz.long()
    return torch.argsort((c[:, 0] * D + c[:, 1]) * D + c[:, 2])


def prune_budgets(renderer, sdf0, coords0, occ0, vol0):
    """maximum_pts of the three cases, from the reference's own survivor counts per threshold."""
    counts = []
    for k in range(10):
        c, _ = renderer.get_valid_sparse_coords_by_sdf(sdf0, coords0, occ0, vol0, threshold=0.02 - 0.002 * k,
                                                       maximum_pts=10 ** 9)
        counts.append(c.shape[0])
    assert counts[0] > counts[2] and counts[-1] > 10, counts
    return {"default": 110000, "ladder": counts[2], "subsample": counts[-1] - 7}


def main():
    ref = _refimport.import_reference()
    torch.manual_seed(0)
    states = {k: O.to_torch_state(v) for k, v in {**S.all_states(0), **S.lod1_states(0)}.items()}
    D0, V, H, W = MINI["D"], MINI["V"], MINI["H"], MINI["W"]
    D1 = 2 * D0
    vs0, vs1 = 2.0 / (D0 - 1), 2.0 / (D1 - 1)
    ok = True
    gold = {}
    conf = _refimport.Conf({"general.base_exp_dir": tempfile.gettempdir()})

    def sdf_network(lod, D, vs, C, key):
        net = ref.sparse_sdf_network.SparseSdfNetwork(lod=lod, ch_in=56, voxel_size=vs, vol_dims=[D, D, D], hidden_dim=128,
                                                      d_pyramid_feature_compress=C, regnet_d_out=16, num_sdf_layers=4,
                                                      multires=6)
        res = net.load_state_dict(states[key], strict=False)
        assert not res.unexpected_keys and all("num_batches_tracked" in k for k in res.missing_keys), res
        return net

    def parts(fkey, rkey, vkey, sdf_net):
        fnet = ref.featurenet.FeatureNet()
        assert not fnet.load_state_dict(states[fkey], strict=False).unexpected_keys
        rnet = ref.rendering_network.GeneralRenderingNetwork(in_geometry_feat_ch=16, in_rendering_feat_ch=56)
        rnet.load_state_dict(states[rkey])
        vnet = ref.fields.SingleVarianceNetwork(0.3)
        vnet.load_state_dict(states[vkey])
        renderer = ref.sparse_neus_renderer.SparseNeuSRenderer(None, sdf_net, vnet, rnet, 64, 64, 0, 1.0, alpha_type="div",
                                                               conf=conf)
        return fnet, rnet, renderer

    def fused(fnet, imgs):
        pyr = fnet(imgs)
        up = torch.nn.functional.interpolate
        return torch.cat([up(pyr[0], scale_factor=4, mode="bilinear", align_corners=True),
                          up(pyr[1], scale_factor=2, mode="bilinear", align_corners=True), pyr[2]], 1)

    sdf0_net = sdf_network(0, D0, vs0, 16, "sdf_network_lod0")
    sdf1_net = sdf_network(1, D1, vs1, 8, "sdf_network_lod1")
    fnet0, _, renderer0 = parts("pyramid_feature_network", "rendering_network_lod0", "variance_network_lod0", sdf0_net)
    fnet1, rnet1, renderer1 = parts("pyramid_feature_network_lod1", "rendering_network_lod1", "variance_network_lod1",
                                    sdf1_net)

    cams, imgs_np = mini_scene()
    imgs, proj, origin = t(imgs_np), t(cams["affine_mats"]), t(cams["partial_vol_origin"])
    w2cs, intr, qc2w = t(cams["w2cs"]), t(cams["intrinsics"]), t(cams["query_c2w"])[None]

    with torch.no_grad():
        fm0 = fused(fnet0, imgs)
        out0 = sdf0_net.get_conditional_volume(fm0[None], origin[None], proj[None], sizeH=H, sizeW=W, lod=0)
        vol0, occ0, coords0 = out0["dense_volume_scale0"], out0["valid_mask_volume_scale0"], out0["coords_scale0"]

        # ---- get_sdf_volume (trainer_generic.py:898-900)
        sdf0 = sdf0_net.get_sdf_volume(vol0, occ0, coords0, origin[None])
        ok &= report("lod-0 sdf volume", sdf0, L1.sdf_volume(vol0, occ0, origin, vs0, states["sdf_network_lod0"]), 2e-5)
        gold["sdf0"] = sdf0.reshape(-1).numpy()

        # ---- get_valid_sparse_coords_by_sdf at three budgets (trainer_generic.py:915-918)
        budgets = prune_budgets(renderer0, sdf0[0], coords0[0], occ0[0], vol0[0])
        gold["prune_max_pts"] = np.array([budgets[c] for c in PRUNE_CASES], np.int64)
        survivors = {}
        for case in PRUNE_CASES:
            np.random.seed(PRUNE_SEED)
            c_ref, f_ref = renderer0.get_valid_sparse_coords_by_sdf(sdf0[0], coords0[0], occ0[0], vol0[0],
                                                                    maximum_pts=budgets[case])
            np.random.seed(PRUNE_SEED)
            c_o, f_o, _, _ = L1.prune(sdf0[0], occ0[0], vol0[0], maximum_pts=budgets[case])
            same = c_ref.shape == c_o.shape and torch.equal(c_ref, c_o)
            print(f"[{'ok ' if same else 'BAD'}] prune[{case}] survivors ({c_ref.shape[0]}) identical")
            ok &= same and report(f"prune[{case}] features", f_ref, f_o, 0)
            gold[f"prune_{case}_mask"] = np.packbits(lattice_mask(c_ref, D0).numpy())
            gold[f"prune_{case}_feat_s"] = f_ref.flatten()[::7].numpy()
            survivors[case] = (c_ref, f_ref)

        # ---- lod-1 conditional volume (trainer_generic.py:905-932)
        pre_c, pre_f = survivors["default"]
        pre_c = pre_c.clone()
        pre_c[:, 1:] = pre_c[:, 1:] * 2
        fm1 = fused(fnet1, imgs)
        out1 = sdf1_net.get_conditional_volume(fm1[None], origin[None], proj[None], sizeH=H, sizeW=W, pre_coords=pre_c,
                                               pre_feats=pre_f)
        vol1, occ1 = out1["dense_volume_scale1"], out1["valid_mask_volume_scale1"]
        # the intermediate rows of that call, through the reference's own functions (sparse_sdf_network.py:340-372)
        up_feat, up_coords = sdf1_net.upsample(pre_f, pre_c, 1)
        comp1 = sdf1_net.compress_layer(fm1)
        mv, mm = ref.back_project.back_project_sparse_type(up_coords, origin[None], vs1, comp1[:, None], proj[:, None],
                                                           sizeH=H, sizeW=W)
        keep = mm.sum(-1) > 1
        cost_ref = torch.cat([sdf1_net.aggregate_multiview_features(mv[keep], mm[keep]), up_feat[keep]], 1)
        xyz = up_coords[keep][:, 1:]
        o1 = L1.conditional_volume(O.pyramid_feature_maps(imgs, states["pyramid_feature_network_lod1"]), origin, proj,
                                   states["sdf_network_lod1"], D1, vs1, H, W, pre_c, pre_f)
        same = torch.equal(xyz, o1["xyz"])
        print(f"[{'ok ' if same else 'BAD'}] lod-1 children kept ({xyz.shape[0]} of {up_coords.shape[0]}) identical")
        ok &= same
        order = lattice_order(xyz, D1)
        ok &= report("lod-1 cost rows", cost_ref, o1["cost"], 2e-4)
        ok &= report("lod-1 dense volume (stub torchsparse)", vol1, o1["dense"], 5e-5)
        ok &= report("lod-1 occupancy", occ1, o1["occ"], 0)
        gold.update(lod1_keep=np.packbits(lattice_mask(up_coords[keep], D1).numpy()),
                    lod1_cost_s=cost_ref[order].flatten()[::11].numpy(), lod1_dense_s=vol1.flatten()[::13].numpy(),
                    lod1_occ=np.packbits(occ1.reshape(-1).numpy() > 0))

        # ---- lod-1 sdf on the mini points
        pts = t(mini_points(MINI["n_pts"]))
        s1 = sdf1_net.sdf(pts, vol1, 1)["sdf_pts_scale1"]
        ok &= report("lod-1 sdf", s1, O.sdf_query(pts, vol1, states["sdf_network_lod1"])[0], 2e-5)
        gold["lod1_sdf"] = s1.numpy()

        # ---- lod-1 -sdf grid (extract_fields of sdf_renderer_lod1)
        u1 = renderer1.extract_fields(torch.tensor([-1.0] * 3), torch.tensor([1.0] * 3), MINI["R"],
                                      lambda p, **kw: sdf1_net.sdf(p, **kw), "cpu", conditional_volume=vol1, lod=1)
        ok &= report("lod-1 -sdf grid", u1, O.sdf_grid(vol1, states["sdf_network_lod1"], MINI["R"]), 2e-5)
        gold["lod1_u_grid"] = u1.astype(np.float32)

    # ---- lod-1 vertex colours: rendering_network_lod1 with the lod-0 feature maps (trainer_generic.py:959-978)
    vp = t(np.random.default_rng(9).uniform(-0.7, 0.7, size=(MINI["n_verts"], 3)).astype(np.float32))
    feats = renderer1.rendering_projector.compute_view_independent(
        vp, lod=1, geometryVolume=vol1[0], geometryVolumeMask=occ1[0], sdf_network=sdf1_net, rendering_feature_maps=fm0,
        color_maps=imgs, w2cs=w2cs, target_candidate_w2cs=None, intrinsics=intr, img_wh=[W, H], query_img_idx=0,
        query_c2w=qc2w)
    with torch.no_grad():
        col_ref, _ = rnet1(feats[0], feats[1], feats[2], feats[3])
    col_o, _ = O.vertex_colors(vp, vol1, occ1, O.pyramid_feature_maps(imgs, states["pyramid_feature_network"]), imgs, w2cs,
                               intr, states["sdf_network_lod1"], states["rendering_network_lod1"], W=W, H=H)
    ok &= report("lod-1 vertex colours", col_ref[0].detach(), col_o, 2e-4)
    gold["lod1_vert_color"] = col_ref[0].detach().numpy()

    path = os.path.join(GOLD, "lod1_mini.npz")
    np.savez_compressed(path, **gold)
    print("golden vectors written to", path)
    print("ALL PINNED" if ok else "SOME CHECKS FAILED")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
