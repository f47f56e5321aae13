"""One reconstruction step at the bench configuration, for ncu.

    ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/launches.csv \
        python tools/profile_step.py --chunks 8
    ncu --set full --clock-control none --import-source on -k regex:render_blend -c 1 -o gpurun_out/blend \
        python tools/profile_step.py --chunks 1
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=8, help="number of 8192-ray chunks to render (8 = full image)")
    ap.add_argument("--mesh", action="store_true", help="also run export_mesh at R=256")
    args = ap.parse_args()
    from o2345 import synthetic as S
    from o2345.pipeline import build_networks
    dev = torch.device("cuda:0")
    tr = build_networks(dev, vol_dim=bench.VOL, states=S.all_states(0), perturb=0.0)
    from o2345.pipeline import synthetic_sample
    sample = synthetic_sample(dev, n_views=bench.N_VIEWS, H=bench.H, W=bench.W)
    imgs, fmaps, cond, sizeW, sizeH = tr._conditional_features(sample)
    vol, occ = cond['dense_volume_scale0'], cond['valid_mask_volume_scale0']
    near, far = sample['query_near_far'][0, :1], sample['query_near_far'][0, 1:]
    ro = sample['rays']['rays_o'][0].reshape(-1, 3)
    rd = sample['rays']['rays_v'][0].reshape(-1, 3)
    for a, b in list(zip(ro.split(bench.CHUNK), rd.split(bench.CHUNK)))[:args.chunks]:
        tr.sdf_renderer_lod0.render(a, b, near, far, tr.sdf_network_lod0, tr.rendering_network_lod0,
                                    perturb_overwrite=0, background_rgb=1.0, alpha_inter_ratio=1.0, lod=0,
                                    conditional_volume=vol, conditional_valid_mask_volume=occ, feature_maps=fmaps,
                                    color_maps=imgs, w2cs=sample['w2cs'][0], intrinsics=sample['intrinsics'][0],
                                    img_wh=[sizeW, sizeH], query_c2w=sample['query_c2w'])
    if args.mesh:
        tr(sample, mode="export_mesh", resolution=256)
    torch.cuda.synchronize()
    print("done")


if __name__ == "__main__":
    main()
