"""Mesh cleaning (csrc/clean.cu through ops.clean_mesh): median milliseconds of one call after warm-up, on
  example   the reference's example mesh (backpack_ours.obj, 69 960 faces, one component);
  field     the bench scene's R = 256 marching-cubes mesh (bench.py's 96^3 volume, synthetic weights), welded, with the
            time of export_mesh_step on the same scene beside it, so the cleaning's share of the export is printed;
  analytic  an R = 640 marching-cubes mesh (about 1 M faces) of a ball, a distant ball of a tenth its radius and a bubble
            inside the first.

    python tools/time_clean.py [--reps 11] [--min_component 0.05]

Each time is a host clock around a call that ends in a device synchronisation.  One JSON line per workload, with the
component counts, and the card's name, power limit and clocks read in the same run."""
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

from o2345 import mesh_io, ops
from time_raster import card
from time_simplify import bench_scene


def median_ms(fn, reps):
    fn()                                           # warm-up
    t = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(t))


def row(name, v, f, F, reps, **extra):
    vt = torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda()
    ft = torch.from_numpy(np.ascontiguousarray(f, np.int32)).cuda()
    _, _, st = ops.clean_mesh(vt, ft, F)
    ms = median_ms(lambda: ops.clean_mesh(vt, ft, F), reps)
    out = {"workload": name, "faces": int(len(f)), "vertices": int(len(v)), "min_component": F, "clean_ms": ms,
           **{k: st[k] for k in ("components", "dropped", "dropped_faces", "enclosed")}, **extra}
    print(json.dumps(out), flush=True)
    return ms


def analytic(R):
    x = torch.linspace(-1, 1, R, device="cuda", dtype=torch.float64)
    X, Y, Z = torch.meshgrid(x, x, x, indexing="ij")
    d = lambda c, r: torch.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r
    u = torch.minimum(torch.maximum(d((-0.3, 0, 0), 0.5), -d((-0.25, 0.05, 0), 0.2)), d((0.6, 0.55, 0.5), 0.05)).float()
    del X, Y, Z
    verts, tris, _ = ops.marching_cubes(u)
    return (verts.cpu().numpy() * (2.0 / (R - 1)) - 1.0).astype(np.float32), tris.cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--min_component", type=float, default=0.05)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_clean.py measures on the GPU"
    F = args.min_component
    print(json.dumps({"card": card()}), flush=True)

    tmp = tempfile.mkdtemp()
    try:
        obj = os.path.join(tmp, "backpack_ours.obj")
        with gzip.open(os.path.join(ROOT, "tests", "golden", "render_eval", "backpack_ours.obj.gz"), "rb") as s, \
                open(obj, "wb") as d:
            shutil.copyfileobj(s, d)
        v, f, _ = mesh_io.read_obj(obj)
        v, f, _ = mesh_io.merge_vertices(v.astype(np.float32), f)
        row("example", v, f, F, args.reps)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)

    tr, sample = bench_scene()
    export = median_ms(lambda: tr.export_mesh_step(sample, resolution=256), max(3, args.reps // 3))
    full = tr.export_mesh_step(sample, resolution=256)
    ms = row("field_mc256", full["vertices"], full["triangles"], F, args.reps, export_mesh_step_ms=export)
    print(json.dumps({"workload": "field_mc256", "clean_share_of_export": ms / export}), flush=True)

    v, f = analytic(640)
    row("analytic_mc640", v, f, F, args.reps)
    print(json.dumps({"card": card(), "peak_alloc_gb": torch.cuda.max_memory_allocated() / 1e9}), flush=True)


if __name__ == "__main__":
    main()
