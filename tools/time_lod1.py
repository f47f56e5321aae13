"""export_mesh with num_lods 1 against 2 at the bench configuration (32 views of 256^2, 96^3 lod 0, 192^3 lod 1,
R = 256), seeded synthetic weights.  Prints the card and its power limit, the whole-call times (CUDA events, median of
REPS after one warm-up) and the per-stage times of the lod-1 glue.

    python tools/time_lod1.py [REPS]
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from o2345 import synthetic as S  # noqa: E402
from o2345.pipeline import build_networks, synthetic_sample  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b)


def main(reps=3):
    dev = torch.device("cuda:0")
    sample = synthetic_sample(dev, n_views=bench.N_VIEWS, H=bench.H, W=bench.W)
    states = {**S.all_states(0), **S.lod1_states(0)}
    res = {"card": card(), "config": {"views": bench.N_VIEWS, "hw": bench.H, "vol_dim": bench.VOL, "mesh_resolution": bench.MESH_RES}}
    for lods in (1, 2):
        tr = build_networks(dev, vol_dim=bench.VOL, states=states, perturb=0.0, num_lods=lods)
        tr(sample, mode="export_mesh", resolution=bench.MESH_RES)
        ms = [timed(lambda: tr(sample, mode="export_mesh", resolution=bench.MESH_RES))[1] for _ in range(reps)]
        res[f"export_mesh_ms_num_lods_{lods}"] = float(np.median(ms))
    # stages of the lod-1 glue (tr is the num_lods = 2 trainer)
    stages = {}
    for _ in range(reps):
        (imgs, fmaps, cond, sizeW, sizeH), t = timed(lambda: tr._conditional_features(sample))
        stages.setdefault("lod0_volume", []).append(t)
        origin = sample['partial_vol_origin']
        sdf0, t = timed(lambda: tr.sdf_network_lod0.get_sdf_volume(cond['dense_volume_scale0'], cond['valid_mask_volume_scale0'],
                                                                   cond['coords_scale0'], origin))
        stages.setdefault("sdf_volume", []).append(t)
        fm1, t = timed(lambda: tr.obtain_pyramid_feature_maps(imgs, lod=1))
        stages.setdefault("featurenet_lod1", []).append(t)
        (pc, pf), t = timed(lambda: tr.sdf_renderer_lod0.get_valid_sparse_coords_by_sdf(
            sdf0[0], cond['coords_scale0'][0], cond['valid_mask_volume_scale0'][0], cond['dense_volume_scale0'][0]))
        stages.setdefault("prune", []).append(t)
        pc[:, 1:] = pc[:, 1:] * 2
        cond1, t = timed(lambda: tr.sdf_network_lod1.get_conditional_volume(
            feature_maps=fm1[None], partial_vol_origin=origin, proj_mats=sample['affine_mats'], sizeH=sizeH, sizeW=sizeW,
            pre_coords=pc, pre_feats=pf))
        stages.setdefault("lod1_volume", []).append(t)
        _, t = timed(lambda: tr.validate_colored_mesh(
            tr.sdf_network_lod1, tr.sdf_renderer_lod1.extract_geometry, resolution=bench.MESH_RES,
            conditional_volume=cond1['dense_volume_scale1'], conditional_valid_mask_volume=cond1['valid_mask_volume_scale1'],
            feature_maps=fmaps, color_maps=imgs, w2cs=sample['w2cs'][0], intrinsics=sample['intrinsics'][0],
            rendering_network=tr.rendering_network_lod1, lod=1, threshold=0, query_c2w=sample['query_c2w'],
            scale_mat=sample['scale_mat'], trans_mat=sample['trans_mat'], img_wh=[sizeW, sizeH]))
        stages.setdefault("mesh_lod1", []).append(t)
    res["lod1_stages_ms"] = {k: float(np.median(v)) for k, v in stages.items()}
    res["survivors"] = int(pc.shape[0])
    res["lod1_rows"] = int(tr.sdf_network_lod1._last["count"].item())
    res["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    print(json.dumps(res, indent=1))
    return res


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 3)
