"""Mesh simplification (csrc/simplify.cu through o2345/mesh_simplify.py): milliseconds per call and rounds on
  example     the reference's example mesh (backpack_ours.obj, 69 960 faces) at 50 %, 10 % and 1 % of its faces;
  bench_mc256 the marching-cubes mesh of the bench scene at R = 256 (bench.py's 96^3 volume, synthetic weights) at 10 %
              and 2 %;
  bench_mc512 the same scene meshed at R = 512, at 2 %;
and, for scale, GenericTrainer.export_mesh_step of the bench scene at R = 256 without simplification.

    python tools/time_simplify.py [--rounds 2] [--reps 3]

A call is timed on the host around mesh_simplify.simplify (numpy in, numpy out: upload, the kernels with their one
host synchronisation per round, download), which ends in a device synchronisation; the minimum and the median over
--reps calls after one warm-up call per workload are printed.  The rounds alternate the order of the workloads.  Prints
one JSON line per (round, workload, target) and the card's name, power limit and clocks."""
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
from o2345.mesh_simplify import simplify
from time_raster import card


def bench_scene():
    import bench
    from o2345 import synthetic as S
    from o2345.pipeline import build_networks, synthetic_sample
    dev = torch.device("cuda:0")
    tr = build_networks(dev, vol_dim=bench.VOL, states=S.all_states(0), perturb=0.0)
    tr.base_exp_dir = None
    return tr, synthetic_sample(dev, n_views=bench.N_VIEWS, H=bench.H, W=bench.W)


def wall(fn, reps):
    ts, out = [], None
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(1e3 * (time.perf_counter() - t))
    return float(np.min(ts)), float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_simplify.py measures on the GPU"
    print(json.dumps({"card": card()}), flush=True)
    tmp = tempfile.mkdtemp()
    try:
        obj = os.path.join(tmp, "backpack_ours.obj")
        with gzip.open(os.path.join(ROOT, "tests", "golden", "render_eval", "backpack_ours.obj.gz"), "rb") as s, \
                open(obj, "wb") as d:
            shutil.copyfileobj(s, d)
        v, f, _ = mesh_io.read_obj(obj)
        meshes = {"example": (v.astype(np.float32), f)}
        tr, sample = bench_scene()
        for R in (256, 512):
            m = tr.export_mesh_step(sample, resolution=R)
            meshes[f"bench_mc{R}"] = (m["vertices"], m["triangles"])
        t_min, t_med, _ = wall(lambda: tr.export_mesh_step(sample, resolution=256), args.reps + 1)
        print(json.dumps({"export_mesh_step_r256_ms_min": t_min, "export_mesh_step_r256_ms_median": t_med,
                          "faces": int(len(meshes["bench_mc256"][1]))}), flush=True)
        work = [("example", 50), ("example", 10), ("example", 1), ("bench_mc256", 10), ("bench_mc256", 2), ("bench_mc512", 2)]
        for name, pct in work:                      # warm-up of every workload
            vv, ff = meshes[name]
            simplify(vv, ff, None, len(ff) * pct // 100)
        for rnd in range(args.rounds):
            for name, pct in (work if rnd % 2 == 0 else work[::-1]):
                vv, ff = meshes[name]
                target = len(ff) * pct // 100
                t_min, t_med, out = wall(lambda: simplify(vv, ff, None, target), args.reps)
                print(json.dumps({"round": rnd, "workload": name, "percent": pct, "faces_in": int(len(ff)),
                                  "vertices_in": int(len(vv)), "faces_out": int(len(out[1])), "vertices_out": int(len(out[0])),
                                  "rounds": out[3], "ms_min": t_min, "ms_median": t_med}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps({"card": card(), "peak_alloc_gb": torch.cuda.max_memory_allocated() / 1e9}), flush=True)


if __name__ == "__main__":
    main()
