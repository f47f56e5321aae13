"""Input-view projection (csrc/project.cu through o2345/mesh_texture.py): milliseconds of the bake with and without the
photo projected, on
  field     the bench scene's R = 256 marching-cubes mesh (bench.py's 96^3 volume, synthetic weights) through
            export_mesh_step(target_faces = 10 %, texture_size = 2048), with the query image as the photo at 256^2 (a
            1024^2 depth buffer) and upsampled to 2048^2 (a 4096^2 buffer); the projection covers the vertex colours and
            the texture, one depth buffer for both;
  example   the reference's example mesh (backpack_ours.obj) simplified to 10 % (6 996 faces) at N = 2048, colours
            transferred from the full mesh (transfer_fn), a seeded 256^2 photo from a rig camera.

    python tools/time_projection.py [--reps 5]

Each time is a host clock around a call that ends in a device synchronisation; with and without projection are timed
alternately, and the minimum of each over --reps calls after a warm-up call is printed, one JSON line per workload, with
the card's name, power limit and clocks read in the same run."""
import argparse
import gzip
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import numpy as np
import torch

from o2345 import mesh_io
from o2345 import mesh_raster as MR
from o2345 import mesh_texture as MT
from o2345.mesh_simplify import simplify
from time_raster import card
from time_simplify import bench_scene


def ms_pair(a, b, reps):
    """Minimum milliseconds of a and of b, timed alternately (a warm-up call of each first)."""
    out = ([], [])
    for _ in range(reps + 1):
        for k, fn in enumerate((a, b)):
            torch.cuda.synchronize()
            t = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            out[k].append(1e3 * (time.perf_counter() - t))
    return min(out[0][1:]), min(out[1][1:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_projection.py measures on the GPU"
    print(json.dumps({"card": card()}), flush=True)
    N = 2048
    tr, sample = bench_scene()
    full = tr.export_mesh_step(sample, resolution=256)
    target = len(full["triangles"]) // 10
    q = (sample["query_image"][0].permute(1, 2, 0).clamp(0, 1) * 255).round().to(torch.uint8).cpu().numpy()
    row = {"workload": "field_mc256_10pct", "faces": int(target), "N": N}
    for side in (256, 2048):
        photo = np.repeat(np.repeat(q, side // q.shape[0], 0), side // q.shape[1], 1)
        view = {"photo": photo, "alpha": None}
        plain, t = ms_pair(lambda: tr.export_mesh_step(sample, resolution=256, target_faces=target, texture_size=N),
                           lambda: tr.export_mesh_step(sample, resolution=256, target_faces=target, texture_size=N,
                                                       project_view=view), args.reps)
        seen = tr.export_mesh_step(sample, resolution=256, target_faces=target, texture_size=N, project_view=view)
        row.update({f"export_mesh_step_{side}_ms": plain, f"projected_{side}_ms": t, f"projection_{side}_ms": t - plain,
                    f"vertices_seen_{side}": float((seen["project_weight"] > 0).mean())})
    print(json.dumps(row), flush=True)

    tmp = tempfile.mkdtemp()
    try:
        obj = os.path.join(tmp, "backpack_ours.obj")
        with gzip.open(os.path.join(ROOT, "tests", "golden", "render_eval", "backpack_ours.obj.gz"), "rb") as s, \
                open(obj, "wb") as d:
            shutil.copyfileobj(s, d)
        v, f, c = mesh_io.read_obj(obj)
        v = v.astype(np.float32)
        sv, sf, _, _ = simplify(v, f, None, len(f) // 10)
        ctr = (sv.max(0) + sv.min(0)) / 2
        scale = np.abs(sv - ctr).max() * 2
        sv, v = ((sv - ctr) / scale).astype(np.float32), ((v - ctr) / scale).astype(np.float32)
        cfn = MT.transfer_fn(v, f, c, texture_size=N)
        c2w, K = MR.rig_cameras(1.5, 256)
        w2c, intr = MR.camera_arrays(c2w[2:3], K)
        rng = np.random.default_rng(0)
        view = {"photo": rng.integers(0, 256, (256, 256, 3), dtype=np.uint8), "alpha": None, "w2c": w2c[0],
                "intr": (intr[0, 0], intr[0, 1], intr[0, 2] - 0.5, intr[0, 3] - 0.5)}
        base, proj = ms_pair(lambda: MT.bake(sv, sf, N, cfn), lambda: MT.bake(sv, sf, N, cfn, view=view), args.reps)
        print(json.dumps({"workload": "transfer_example_10pct", "faces": int(len(sf)), "N": N, "bake_ms": base,
                          "bake_projected_ms": proj, "projection_ms": proj - base}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps({"card": card(), "peak_alloc_gb": torch.cuda.max_memory_allocated() / 1e9}), flush=True)


if __name__ == "__main__":
    main()
