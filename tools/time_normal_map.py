"""Normal-map baking (csrc/texture.cu through o2345/mesh_texture.py): milliseconds of the bake with and without a normal
map on
  transfer  the reference's example mesh (backpack_ours.obj) simplified to 10 % (6 996 faces) at N = 2048, colours and
            normals transferred from the full 69 960-face mesh (transfer_fn, normal_transfer_fn);
  field     the bench scene's R = 256 marching-cubes mesh (bench.py's 96^3 volume, synthetic weights) through
            export_mesh_step(target_faces = 10 %, texture_size = 2048), coloured by blend_points and, with normal_map, the
            SDF gradient at the texel points.

    python tools/time_normal_map.py [--reps 3]

Each time is a host clock around a call that ends in a device synchronisation (the bake downloads its textures); the
minimum over --reps calls after a warm-up call is printed, one JSON line per workload, with the card's name, power limit
and clocks read in the same run."""
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
from o2345 import mesh_texture as MT
from o2345.mesh_simplify import simplify
from time_raster import card
from time_simplify import bench_scene


def ms(fn, reps):
    out = []
    for _ in range(reps + 1):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(1e3 * (time.perf_counter() - t))
    return min(out[1:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_normal_map.py measures on the GPU"
    print(json.dumps({"card": card()}), flush=True)
    tmp = tempfile.mkdtemp()
    try:
        obj = os.path.join(tmp, "backpack_ours.obj")
        with gzip.open(os.path.join(ROOT, "tests", "golden", "render_eval", "backpack_ours.obj.gz"), "rb") as s, \
                open(obj, "wb") as d:
            shutil.copyfileobj(s, d)
        v, f, c = mesh_io.read_obj(obj)
        v = v.astype(np.float32)
        sv, sf, _, _ = simplify(v, f, None, len(f) // 10)
        N = 2048
        cfn = MT.transfer_fn(v, f, c, texture_size=N)
        colour = ms(lambda: MT.bake(sv, sf, N, cfn), args.reps)
        both = ms(lambda: MT.bake(sv, sf, N, cfn, normal_fn=MT.normal_transfer_fn(v, f, texture_size=N)), args.reps)
        print(json.dumps({"workload": "transfer_example_10pct", "faces": int(len(sf)), "N": N, "bake_colour_ms": colour,
                          "bake_colour_and_normal_ms": both, "normal_ms": both - colour}), flush=True)

        tr, sample = bench_scene()
        full = tr.export_mesh_step(sample, resolution=256)
        target = len(full["triangles"]) // 10
        plain = ms(lambda: tr.export_mesh_step(sample, resolution=256, target_faces=target, texture_size=N), args.reps)
        mapped = ms(lambda: tr.export_mesh_step(sample, resolution=256, target_faces=target, texture_size=N, normal_map=True),
                    args.reps)
        print(json.dumps({"workload": "field_mc256_10pct", "faces": int(target), "N": N, "export_mesh_step_ms": plain,
                          "export_mesh_step_normal_map_ms": mapped, "normal_ms": mapped - plain}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps({"card": card(), "peak_alloc_gb": torch.cuda.max_memory_allocated() / 1e9}), flush=True)


if __name__ == "__main__":
    main()
