"""Isotropic remeshing (csrc/remesh.cu through ops.remesh_mesh / ops.closest_points): median milliseconds after
warm-up, by CUDA events, of
  lbvh      ops.closest_points with one query point: the input check and the LBVH build over the mesh;
  iter1     the remesh with one iteration (split, collapse and flip rounds, relaxation, projection);
  total     the remesh with the default iterations (mesh_remesh.REMESH_ITERATIONS), with the rounds it ran;
on
  example   the reference's example mesh (backpack_ours.obj, welded, 69 960 faces) to 20 %, 5 % and 1 % of its faces;
  analytic  an R = 256 marching-cubes mesh (time_clean.py) to 20 % of its faces.
The phases of one iteration are not timed apart: each synchronises once per round inside one call.

    python tools/time_remesh.py [--reps 5]

One JSON line per workload, and the card's name, power limit and clocks read in the same run."""
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

from o2345 import mesh_io, mesh_remesh, ops
from time_ao import median_ms
from time_clean import analytic
from time_raster import card


def row(name, v, f, frac, reps):
    vt = torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda()
    ft = torch.from_numpy(np.ascontiguousarray(f, np.int32)).cuda()
    N = int(round(len(f) * frac))
    L, _ = mesh_remesh.target_length(v, f, N)
    lbvh = median_ms(lambda: ops.closest_points(vt, ft, vt[:1]), reps)
    it1 = median_ms(lambda: ops.remesh_mesh(vt, ft, L, 1), reps)
    total = median_ms(lambda: ops.remesh_mesh(vt, ft, L, mesh_remesh.REMESH_ITERATIONS), reps)
    ov, of, rounds = ops.remesh_mesh(vt, ft, L, mesh_remesh.REMESH_ITERATIONS)
    print(json.dumps({"workload": name, "faces_in": int(len(f)), "target": N, "faces_out": int(of.shape[0]),
                      "lbvh_ms": lbvh, "iter1_ms": it1, "total_ms": total, "rounds": list(rounds)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_remesh.py measures on the GPU"
    print(json.dumps({"card": card()}), flush=True)
    tmp = tempfile.mkdtemp()
    try:
        obj = os.path.join(tmp, "backpack_ours.obj")
        with gzip.open(os.path.join(ROOT, "tests", "golden", "render_eval", "backpack_ours.obj.gz"), "rb") as s, \
                open(obj, "wb") as d:
            shutil.copyfileobj(s, d)
        v, f, _ = mesh_io.read_obj(obj)
        v, f, _ = mesh_io.merge_vertices(v.astype(np.float32), f)
        for frac in (0.2, 0.05, 0.01):
            row(f"example_{frac}", v, f, frac, args.reps)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    v, f = analytic(256)
    row("analytic_mc256_0.2", v, f, 0.2, args.reps)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
