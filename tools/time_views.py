"""Any-camera rendering on the bench scene (96^3 volume, 32 source views of 256^2, num_lods = 1):
GenericTrainer.render_cameras (rays of all cameras in 65536-ray launch groups) against a per-camera loop of
SparseNeuSRenderer.render (bench.CHUNK = 65536-ray calls, as bench.py measures the query view), alternating the two in one
process.

    python tools/time_views.py [--rounds 2]

Workloads: the 8 stage-1 cameras at 256^2, and 36-frame orbits (pipeline.render_turntable's cameras) at 256^2 and 128^2.
The loop side generates and renders the same rays with each camera's query_c2w and scalar near / far; both sides get
the feature maps and the volume built beforehand, so what is timed is ray generation and the ray march (render_cameras
also sums the normals).  Prints one JSON line per (workload, round) and the
card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200")):
    sys.path.insert(0, p)
import numpy as np
import torch

import bench
from o2345 import synthetic as S
from o2345.pipeline import build_networks, synthetic_sample


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_views.py measures on the GPU"
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card()}), flush=True)
    tr = build_networks(dev, vol_dim=bench.VOL, states=S.all_states(0), perturb=0.0)
    sample = synthetic_sample(dev, n_views=bench.N_VIEWS, H=bench.H, W=bench.W)
    feats = tr._conditional_features(sample)
    tr._conditional_features = lambda s: feats           # volume built once: the ray march is what is timed
    imgs, fmaps, cond, sizeW, sizeH = feats
    meta = S.pose_json(60.0)
    cams = S.scene_cameras(meta, n_src=bench.N_VIEWS, img_wh=(bench.W, bench.H))
    poses = np.array(list(meta["c2ws"].values()))
    workloads = {"stage1_8_256": (poses[:8], 256), "orbit36_256": (S.orbit_cameras(meta, 36), 256),
                 "orbit36_128": (S.orbit_cameras(meta, 36), 128)}
    r = tr.sdf_renderer_lod0
    kw = dict(perturb_overwrite=0, lod=0, conditional_volume=cond['dense_volume_scale0'],
              conditional_valid_mask_volume=cond['valid_mask_volume_scale0'], feature_maps=fmaps, color_maps=imgs,
              w2cs=sample['w2cs'][0], intrinsics=sample['intrinsics'][0], img_wh=[sizeW, sizeH])

    for name, (c2w_b, hw) in workloads.items():
        K = np.array(meta["intrinsics"], np.float64)
        K[:2] *= hw / 256.0
        c2w, intr, nf = S.normalise_cameras(cams, c2w_b, K)
        n_rays = len(c2w) * hw * hw

        def batched():
            return tr.render_cameras(sample, c2w, intr, nf, img_wh=(hw, hw))

        def loop():
            for k, c, f in zip(intr, c2w, nf):
                ro, rd = (torch.from_numpy(x).to(dev) for x in S.query_rays(k, c, hw, hw))
                qc2w, near, far = torch.from_numpy(c)[None].to(dev), torch.tensor(f[:1], device=dev), torch.tensor(f[1:], device=dev)
                for a, b in zip(ro.split(bench.CHUNK), rd.split(bench.CHUNK)):
                    r.render(a, b, near, far, tr.sdf_network_lod0, tr.rendering_network_lod0, query_c2w=qc2w, **kw)

        batched(), loop()                                   # warm-up: every shape of the timed window
        for rnd in range(args.rounds):
            tb = timed(batched)
            tl = timed(loop)
            print(json.dumps({"workload": name, "round": rnd, "cameras": len(c2w), "rays": n_rays,
                              "render_cameras": {"s": tb, "M_rays_per_s": n_rays / tb / 1e6, "ms_per_frame": tb / len(c2w) * 1e3},
                              "render_loop": {"s": tl, "M_rays_per_s": n_rays / tl / 1e6, "ms_per_frame": tl / len(c2w) * 1e3}}),
                  flush=True)
    print(json.dumps({"card": card(), "peak_alloc_gb": torch.cuda.max_memory_allocated() / 1e9}), flush=True)


if __name__ == "__main__":
    main()
