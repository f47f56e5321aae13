"""Mesh rasterizer (csrc/raster.cu) on the 24-view evaluation rig at 512^2, camera distance 1.3: the reference's example
pair (tests/golden/render_eval: backpack_gt.glb, 3.8 k textured triangles; backpack_ours.obj, 70 k triangles with vertex
colours) and the marching-cubes mesh of the bench scene at R = 256 (bench.py's 96^3 volume, synthetic weights).

    python tools/time_raster.py [--rounds 2] [--reps 20] [--splits 16,64,256,1000000000]

Every (mesh, split) pair is timed with CUDA events over --reps back-to-back renders (one ops.raster call each: memsets,
four kernels, output allocation from torch's cache), the pairs alternating within each round.  split is the bounding-box
pixel count above which a warp instead of one thread walks a triangle (o2345_debug_raster_split); 10^9 = never.
Prints one JSON line per (round, mesh, split) and the card's name, power limit and clocks."""
import argparse
import gzip
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "one-2-3-45_b200")):
    sys.path.insert(0, p)
import numpy as np
import torch

from o2345 import _lib as L
from o2345 import mesh_io, ops
from o2345 import mesh_raster as MR


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def bench_mesh(path):
    import bench
    from o2345 import synthetic as S
    from o2345.pipeline import build_networks, synthetic_sample
    dev = torch.device("cuda:0")
    tr = build_networks(dev, vol_dim=bench.VOL, states=S.all_states(0), perturb=0.0)
    tr.base_exp_dir = None
    m = tr.export_mesh_step(synthetic_sample(dev, n_views=bench.N_VIEWS, H=bench.H, W=bench.W), resolution=256)
    mesh_io.write_ply(path, m["vertices"], m["triangles"], m["colors"])
    del tr
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--splits", type=str, default="16,64,256,1000000000")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_raster.py measures on the GPU"
    print(json.dumps({"card": card()}), flush=True)
    tmp = tempfile.mkdtemp()
    try:
        gold = os.path.join(ROOT, "tests", "golden", "render_eval")
        obj = os.path.join(tmp, "backpack_ours.obj")
        with gzip.open(os.path.join(gold, "backpack_ours.obj.gz"), "rb") as s, open(obj, "wb") as d:
            shutil.copyfileobj(s, d)
        ply = os.path.join(tmp, "mc256.ply")
        bench_mesh(ply)
        paths = {"backpack_gt": os.path.join(gold, "backpack_gt.glb"), "backpack_ours": obj, "bench_mc256": ply}
        w2c, intr = MR.camera_arrays(*MR.rig_cameras(1.3, 512))
        cuda = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
        w2c, intr = cuda(w2c), cuda(intr)
        meshes = {}
        for name, p in paths.items():
            flat = MR.flatten(MR.normalize_scene(MR.load_scene(p)))
            meshes[name] = {k: cuda(v) for k, v in flat.items()}
        splits = [int(s) for s in args.splits.split(",")]

        def run(m):
            return ops.raster(m["verts"], m["faces"], w2c, intr, 512, 512, colors=m["colors"], uvs=m["uvs"],
                              face_tex=m["face_tex"], texels=m["texels"], tex_info=m["tex_info"])

        lib = L.load()
        ref = {}
        for name, m in meshes.items():               # warm-up, and the reference bits of every split
            for s in splits:
                lib.o2345_debug_raster_split(s)
                out = run(m)
                tri = out["tri"].cpu()
                ref.setdefault(name, tri)
                assert torch.equal(tri, ref[name]), (name, s)
        for rnd in range(args.rounds):
            for name, m in meshes.items():
                nf = int(m["faces"].shape[0])
                for s in splits:
                    lib.o2345_debug_raster_split(s)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.reps):
                        run(m)
                    e1.record()
                    e1.synchronize()
                    ms = e0.elapsed_time(e1) / args.reps
                    print(json.dumps({"round": rnd, "mesh": name, "triangles": nf, "vertices": int(m["verts"].shape[0]),
                                      "split": s, "ms_per_rig": ms, "M_triangle_views_per_s": 24 * nf / ms / 1e3,
                                      "coverage": float((ref[name] >= 0).float().mean())}), flush=True)
        lib.o2345_debug_raster_split(0)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps({"card": card(), "peak_alloc_gb": torch.cuda.max_memory_allocated() / 1e9}), flush=True)


if __name__ == "__main__":
    main()
