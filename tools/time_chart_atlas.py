"""Chart atlas (ops.chart_atlas, --atlas charts) against the per-face atlas (ops.texture_atlas): milliseconds per call,
cut rounds and chart count on
  example   the reference's example mesh (backpack_ours.obj) at 10 % (6 996 faces) and in full (69 960 faces);
  bench     the bench scene's R = 256 marching-cubes mesh (bench.py's volume, synthetic weights), in full.
at N = 1024 and 2048.  The per-face atlas refuses where its boxes do not fit (printed as null).

    python tools/time_chart_atlas.py [--reps 3]

Each call ends in a device synchronisation; the minimum over --reps calls after a warm-up call is printed, one JSON line
per workload, with the card's name, power limit and clocks."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np
import torch

from o2345 import ops
from o2345._lib import O2345Error
from time_raster import card
from time_simplify import bench_scene


def best(fn, reps):
    out = fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(1e3 * (time.perf_counter() - t))
    return min(ts), out


def meshes():
    from test_simplify_host import GOLD, example_mesh
    v, f, _ = example_mesh()
    g = np.load(os.path.join(GOLD, "simplify", "backpack_ours_6996.npz"))
    yield "example 10%", v[g["vertex_index"]], g["faces"]
    yield "example full", v, f
    tr, sample = bench_scene()
    out = tr.export_mesh_step(sample, resolution=256)
    yield "bench R=256", out["vertices"].astype(np.float32), out["triangles"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    gpu = card()
    for name, v, f in meshes():
        vt = torch.from_numpy(np.ascontiguousarray(v, np.float32)).to(dev)
        ft = torch.from_numpy(np.ascontiguousarray(f, np.int32)).to(dev)
        for N in (1024, 2048):
            ms_c, at = best(lambda: ops.chart_atlas(vt, ft, N), args.reps)
            try:
                ms_f, af = best(lambda: ops.texture_atlas(vt, ft, N), args.reps)
                faces = {"ms": round(ms_f, 2), "rho": round(af["rho"], 2)}
            except O2345Error:
                faces = None
            print(json.dumps({"mesh": name, "faces": len(f), "N": N, "charts_ms": round(ms_c, 2), "rounds": at["rounds"],
                              "charts": at["charts"], "charts_rho": round(at["rho"], 2), "per_face_atlas": faces,
                              "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
