"""Ambient occlusion (csrc/ao.cu through ops.ambient_occlusion): median milliseconds after warm-up, by CUDA events, of
  build   the call with one query point: the input check, the LBVH build and one warp of rays;
  full    the call at every vertex of the mesh with its vertex normals (mesh_texture.vertex_ao's work), so
  ao      full - build is the AO pass;
on
  example   the reference's example mesh (backpack_ours.obj, 69 960 faces);
  analytic  an R = 256 marching-cubes mesh of a ball, a distant small ball and a bubble inside the first (time_clean.py).

    python tools/time_ao.py [--reps 11]

One JSON line per workload, with the rays per second of the AO pass, and the card's name, power limit and clocks read
in the same run."""
import argparse
import gzip
import json
import os
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import numpy as np
import torch

from o2345 import mesh_io, mesh_texture as MT, ops
from time_clean import analytic
from time_raster import card


def median_ms(fn, reps):
    fn()                                           # warm-up
    t = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        t.append(a.elapsed_time(b))
    return float(np.median(t))


def row(name, v, f, reps):
    vt = torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda()
    ft = torch.from_numpy(np.ascontiguousarray(f, np.int32)).cuda()
    nrm = ops.vertex_normals(vt, ft)
    build = median_ms(lambda: ops.ambient_occlusion(vt, ft, vt[:1], nrm[:1]), reps)
    full = median_ms(lambda: ops.ambient_occlusion(vt, ft, vt, nrm), reps)
    ao = ops.ambient_occlusion(vt, ft, vt, nrm)
    rays = len(v) * MT.AO_RAYS
    out = {"workload": name, "faces": int(len(f)), "vertices": int(len(v)), "build_ms": build, "full_ms": full,
           "ao_ms": full - build, "gigarays_per_s": rays / ((full - build) * 1e-3) / 1e9, "ao_mean": float(ao.mean())}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=11)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_ao.py measures on the GPU"
    print(json.dumps({"card": card()}), flush=True)
    tmp = tempfile.mkdtemp()
    try:
        obj = os.path.join(tmp, "backpack_ours.obj")
        with gzip.open(os.path.join(ROOT, "tests", "golden", "render_eval", "backpack_ours.obj.gz"), "rb") as s, \
                open(obj, "wb") as d:
            shutil.copyfileobj(s, d)
        v, f, _ = mesh_io.read_obj(obj)
        v, f, _ = mesh_io.merge_vertices(v.astype(np.float32), f)
        row("example", v, f, args.reps)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    v, f = analytic(256)
    row("analytic_mc256", v, f, args.reps)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
