"""Mesh scoring (csrc/metrics.cu): surface sampling and both exact nearest-neighbour passes of the F-Score / Chamfer
protocol, at N = 10^4, 10^5 and 10^6 samples per surface, on two workloads:
  pair        the reference's example pair (backpack_ours.obj, 70 k triangles, against backpack_gt.glb, 3.8 k triangles);
  bench_mc256 the marching-cubes mesh of the bench scene at R = 256 (bench.py's 96^3 volume, synthetic weights) against
              itself rotated by 3 degrees about the vertical axis.
Beside the grid search, for N <= 10^5: a chunked torch.cdist(...).min(1) on the same device (its matrix-product
distances are not exact; the share of equal indices is printed).

    python tools/time_metrics.py [--rounds 2] [--reps 5]

Times are CUDA events over --reps back-to-back calls after a warm-up of every shape; each ops.surface_sample call
includes its one host synchronisation.  The rounds alternate the workloads and sizes.  Prints one JSON line per
(round, workload, N) and the card's name, power limit and clocks."""
import argparse
import gzip
import json
import math
import os
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import numpy as np
import torch

from o2345 import mesh_metrics as MM
from o2345 import ops
from time_raster import bench_mesh, card

SIZES = (10_000, 100_000, 1_000_000)


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps, out


def cdist_min(q, r):
    chunk = max(1, (1 << 28) // r.shape[0])          # at most 2^28 distances (1 GiB) per block
    d, i = zip(*[torch.cdist(q[a:a + chunk], r).min(1) for a in range(0, q.shape[0], chunk)])
    return torch.cat(d), torch.cat(i)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_metrics.py measures on the GPU"
    print(json.dumps({"card": card()}), flush=True)
    tmp = tempfile.mkdtemp()
    try:
        gold = os.path.join(ROOT, "tests", "golden", "render_eval")
        obj = os.path.join(tmp, "backpack_ours.obj")
        with gzip.open(os.path.join(gold, "backpack_ours.obj.gz"), "rb") as s, open(obj, "wb") as d:
            shutil.copyfileobj(s, d)
        ply = os.path.join(tmp, "mc256.ply")
        bench_mesh(ply)
        mc = MM.load_flat(ply)
        c, s = math.cos(math.radians(3)), math.sin(math.radians(3))
        rot = {**mc, "verts": (mc["verts"].astype(np.float64) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T).astype(np.float32)}
        work = {"pair": (MM.load_flat(obj), MM.load_flat(os.path.join(gold, "backpack_gt.glb"))), "bench_mc256": (rot, mc)}
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        meshes = {k: tuple((dev(f["verts"]), dev(f["faces"])) for f in v) for k, v in work.items()}

        def run(name, n, rnd, reps):
            (vp, fp), (vg, fg) = meshes[name]
            t_sp, (p, _) = timed(lambda: ops.surface_sample(vp, fp, n, 0), reps)
            t_sg, (g, _) = timed(lambda: ops.surface_sample(vg, fg, n, 1), reps)
            t_pg, (d_pg, i_pg) = timed(lambda: ops.nearest(p, g), reps)
            t_gp, _ = timed(lambda: ops.nearest(g, p), reps)
            rec = {"round": rnd, "workload": name, "faces": [int(fp.shape[0]), int(fg.shape[0])], "n": n,
                   "ms_sample_pred": t_sp, "ms_sample_gt": t_sg, "ms_nn_pred_to_gt": t_pg, "ms_nn_gt_to_pred": t_gp,
                   "ms_total": t_sp + t_sg + t_pg + t_gp, "M_queries_per_s": 2 * n / (t_pg + t_gp) / 1e3}
            if n <= 100_000:
                t_cd, (d_cd, i_cd) = timed(lambda: cdist_min(p, g), max(1, reps // 2 if n == 100_000 else reps))
                rec.update(ms_cdist_pred_to_gt=t_cd, cdist_same_index=float((i_cd.int() == i_pg).float().mean()),
                           cdist_max_abs_d2=float((d_cd.square() - d_pg).abs().max()))
            return rec

        for name in work:                            # warm-up of every shape
            for n in SIZES:
                run(name, n, -1, 1)
        for rnd in range(args.rounds):
            for name in (list(work) if rnd % 2 == 0 else list(work)[::-1]):
                for n in SIZES:
                    print(json.dumps(run(name, n, rnd, args.reps)), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps({"card": card(), "peak_alloc_gb": torch.cuda.max_memory_allocated() / 1e9}), flush=True)


if __name__ == "__main__":
    main()
