"""Pin the any-camera rendering (synthetic.normalise_cameras, GenericTrainer.render_cameras) against the REAL reference
and freeze tests/golden/views_mini.npz.

Runs only where the reference tree is (oracle/_refimport.py):

    python -m oracle.pin_views_against_reference

1. The reference's own BlenderPerView.__getitem__ on files written from synthetic.pose_json(60): the normalised w2c of
   the 8 stage-1 views (target_candidate_w2cs, data/One2345_eval_new_data.py:291-306), query_c2w and query_near_far.
2. The reference's SparseNeuSRenderer.render of stage-1 view 3 at the mini configuration of pin_against_reference.py
   (24^3 volume, 6 source views of 64^2, perturb 0, white background, alpha_inter_ratio 1): its camera is normalised
   with the dataset's arithmetic (view-0-relative w2c, K w2c scale_mat decomposed by the dataset's load_K_Rt_from_P,
   near / far = 0.95 (d - 1), 1.05 (d + 1)) in the mini scene's frame, its rays come from the reference's
   gen_rays_from_single_image, and 48 of them are rendered.
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "one-2-3-45_b200"))
sys.path.insert(0, ROOT)

from o2345 import synthetic as S  # noqa: E402
from oracle import recon_oracle as O  # noqa: E402
from oracle import _refimport  # noqa: E402
from oracle.pin_against_reference import MINI, mini_scene, report, t  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
NOVEL_VIEW = 3          # stage-1 view rendered at the mini configuration
BLENDER2OPENCV = np.diag([1.0, -1.0, -1.0, 1.0])


def stage1_cameras(gold):
    """target_candidate_w2cs / query_c2w / query_near_far of the reference dataset at the demo configuration."""
    import types
    from PIL import Image
    sys.modules.setdefault("kornia", types.ModuleType("kornia"))
    import data.One2345_eval_new_data as ds
    d = tempfile.mkdtemp()
    meta = S.pose_json(60.0)
    json.dump(meta, open(os.path.join(d, "pose.json"), "w"))
    os.makedirs(os.path.join(d, "stage1_8")), os.makedirs(os.path.join(d, "stage2_8"))
    img = Image.fromarray(np.full((256, 256, 3), 200, np.uint8))
    names = list(meta["c2ws"].keys())
    img.save(os.path.join(d, "stage1_8", names[0]))
    for n in names[8:40]:
        img.save(os.path.join(d, "stage2_8", n))
    smp = ds.BlenderPerView(root_dir="/", split="test", specific_dataset_name=d)[0]
    cams = S.scene_cameras(meta)
    poses = np.array(list(meta["c2ws"].values()))
    c2w, _, nf = S.normalise_cameras(cams, poses[:8], meta["intrinsics"])
    ok = report("stage-1 w2cs", smp["target_candidate_w2cs"], np.linalg.inv(c2w.astype(np.float64)), 1e-5)
    ok &= report("query_c2w", smp["query_c2w"], c2w[0], 1e-5)
    ok &= report("query_near_far", smp["query_near_far"], nf[0], 1e-5)
    gold.update(target_candidate_w2cs=smp["target_candidate_w2cs"].numpy(), query_c2w=smp["query_c2w"].numpy(),
                query_near_far=smp["query_near_far"].numpy())
    return ok, ds


def mini_meta():
    meta = S.pose_json(60.0)
    k = np.array(meta["intrinsics"])
    k[:2] *= MINI["W"] / 256.0
    meta["intrinsics"] = k.tolist()
    return meta


def main():
    ref = _refimport.import_reference()
    torch.manual_seed(0)
    gold = {}
    ok, ds = stage1_cameras(gold)

    states = {k: O.to_torch_state(v) for k, v in S.all_states(0).items()}
    D, H, W = MINI["D"], MINI["H"], MINI["W"]
    sdf_net = ref.sparse_sdf_network.SparseSdfNetwork(lod=0, ch_in=56, voxel_size=2.0 / (D - 1), vol_dims=[D, D, D],
                                                     hidden_dim=128, d_pyramid_feature_compress=16,
                                                     regnet_d_out=16, num_sdf_layers=4, multires=6)
    sdf_net.load_state_dict(states["sdf_network_lod0"], strict=False)
    fnet = ref.featurenet.FeatureNet()
    fnet.load_state_dict(states["pyramid_feature_network"], strict=False)
    rnet = ref.rendering_network.GeneralRenderingNetwork(in_geometry_feat_ch=16, in_rendering_feat_ch=56)
    rnet.load_state_dict(states["rendering_network_lod0"])
    vnet = ref.fields.SingleVarianceNetwork(0.3)
    vnet.load_state_dict(states["variance_network_lod0"])
    renderer = ref.sparse_neus_renderer.SparseNeuSRenderer(
        None, sdf_net, vnet, rnet, 64, 64, 0, 1.0, alpha_type="div",
        conf=_refimport.Conf({"general.base_exp_dir": tempfile.gettempdir()}))
    cams, imgs_np = mini_scene()
    imgs = t(imgs_np)

    # the novel camera, normalised the way the dataset normalises its views
    meta = mini_meta()
    poses = np.array(list(meta["c2ws"].values()))
    w2c_ref_inv = np.linalg.inv(np.linalg.inv(poses[0] @ BLENDER2OPENCV))
    K4 = np.eye(4)
    K4[:3, :3] = np.array(meta["intrinsics"])
    P = (K4 @ (np.linalg.inv(poses[NOVEL_VIEW] @ BLENDER2OPENCV) @ w2c_ref_inv) @ cams["scale_mat"])[:3, :4]
    c2w = ds.load_K_Rt_from_P(None, P)[1]
    dist = np.sqrt(np.sum(c2w[:3, 3] ** 2))
    near_far = np.array([0.95 * (dist - 1), 1.05 * (dist + 1)], np.float32)
    c2w_o, _, nf_o = S.normalise_cameras(cams, poses[NOVEL_VIEW], meta["intrinsics"])
    ok &= report(f"view {NOVEL_VIEW} c2w (mini frame)", c2w, c2w_o[0], 1e-5)
    ok &= report(f"view {NOVEL_VIEW} near/far", near_far, nf_o[0], 1e-5)

    with torch.no_grad():
        pyr = fnet(imgs)
        up = torch.nn.functional.interpolate
        fm = torch.cat([up(pyr[0], scale_factor=4, mode="bilinear", align_corners=True),
                        up(pyr[1], scale_factor=2, mode="bilinear", align_corners=True), pyr[2]], 1)
        out = sdf_net.get_conditional_volume(fm[None], t(cams["partial_vol_origin"])[None], t(cams["affine_mats"])[None],
                                             sizeH=H, sizeW=W, lod=0)
        rays = ref.rays.gen_rays_from_single_image(H, W, torch.zeros(3, H, W), t(meta["intrinsics"]), t(c2w))
        o, v = S.query_rays(np.array(meta["intrinsics"], np.float32), c2w_o[0], H, W)
        ok &= report("rays_o", rays["rays_o"], o, 1e-5)
        ok &= report("rays_v", rays["rays_v"], v, 1e-5)
        sel = np.linspace(0, H * W - 1, MINI["n_rays"]).astype(np.int64)
    res = renderer.render(rays["rays_o"][sel], rays["rays_v"][sel], t(near_far[:1]), t(near_far[1:]), sdf_net, rnet,
                          perturb_overwrite=0, background_rgb=1.0, alpha_inter_ratio=1.0, lod=0,
                          conditional_volume=out["dense_volume_scale0"],
                          conditional_valid_mask_volume=out["valid_mask_volume_scale0"], feature_maps=fm, color_maps=imgs,
                          w2cs=t(cams["w2cs"]), intrinsics=t(cams["intrinsics"]), img_wh=[W, H], query_c2w=t(c2w)[None],
                          if_render_with_grad=False)
    with torch.no_grad():
        col = res["color_fine"].detach().numpy()
        print(f"[info] view {NOVEL_VIEW}: opacity {res['weights_sum'].mean():.3f}, colour range {col.min():.3f}..{col.max():.3f}")
        gold.update(novel_view=np.int64(NOVEL_VIEW), novel_c2w=c2w.astype(np.float32), novel_near_far=near_far, novel_sel=sel,
                    novel_color=col, novel_depth=res["depth"].detach().numpy(), novel_weights_sum=res["weights_sum"].detach().numpy())
    np.savez_compressed(os.path.join(GOLD, "views_mini.npz"), **gold)
    print("golden vectors written to", os.path.join(GOLD, "views_mini.npz"))
    print("ALL PINNED" if ok else "SOME CHECKS FAILED")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
