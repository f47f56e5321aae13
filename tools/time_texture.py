"""Texture baking (csrc/texture.cu through o2345/mesh_texture.py): milliseconds per stage on
  example   the reference's example mesh (backpack_ours.obj) simplified to 10 % (6 996 faces), colours transferred from the
            full mesh, at N = 1024, 2048 and 4096;
  bench     the bench scene's R = 256 marching-cubes mesh (bench.py's 96^3 volume, synthetic weights) simplified to 10 %
            and 2 %, at N = 2048, coloured by the reconstruction (export_mesh_step(texture_size=N): blend_points) and by
            transfer from the full mesh.

    python tools/time_texture.py [--reps 3]

Stages, each ended by a device synchronisation: atlas (ops.texture_atlas, with its host reads), texel points
(ops.texel_points, reading T), colour (the colour function on the T points: blend_points in 2^20-point chunks, or surface
sampling + nearest + transfer), fill (ops.texture_fill) and total (mesh_texture.bake: upload, the four stages, the
download and quantisation).  The minimum over --reps calls after a warm-up call is printed, one JSON line per workload,
with the card's name, power limit and clocks; also export_mesh_step at R = 256 with the target and without a texture."""
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
from o2345 import mesh_texture as MT
from o2345.mesh_simplify import simplify
from time_raster import card
from time_simplify import bench_scene


def staged(vertices, faces, N, colour_fn, out=None):
    """The stages of mesh_texture.bake, each timed -> dict of ms and T; out (a list) receives bake's (uv, texture)."""
    dev = torch.device("cuda:0")
    t = {}
    torch.cuda.synchronize()
    t0 = s = time.perf_counter()

    def lap(name):
        nonlocal s
        torch.cuda.synchronize()
        e = time.perf_counter()
        t[name] = 1e3 * (e - s)
        s = e
    vt = torch.from_numpy(np.ascontiguousarray(vertices, np.float32)).to(dev)
    ft = torch.from_numpy(np.ascontiguousarray(faces, np.int32)).to(dev)
    lap("upload")
    at = ops.texture_atlas(vt, ft, N)
    lap("atlas")
    idx, pts, _ = ops.texel_points(vt, ft, at["uv"], at["owner"], N)
    lap("texel_points")
    rgb = colour_fn(pts).float().contiguous()
    lap("colour")
    tex = ops.texture_fill(idx, rgb, at["owner"], N)
    lap("fill")
    result = at["uv"].cpu().numpy(), MT.quantise(tex)
    lap("download")
    if out is not None:
        out.append(result)
    t["total"] = 1e3 * (time.perf_counter() - t0)
    t["texels"], t["j"] = int(len(idx)), at["j"]
    return t


def best(runs):
    return {k: (min(r[k] for r in runs) if isinstance(runs[0][k], float) else runs[0][k]) for k in runs[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_texture.py measures on the GPU"
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
        for N in (1024, 2048, 4096):
            fn = MT.transfer_fn(v, f, c, texture_size=N)
            runs = [staged(sv, sf, N, fn) for _ in range(args.reps + 1)][1:]
            print(json.dumps({"workload": "example_10pct", "faces": int(len(sf)), "N": N, "colour": "transfer", **best(runs)}),
                  flush=True)

        tr, sample = bench_scene()
        full = tr.export_mesh_step(sample, resolution=256)
        fv, ff, fc = full["vertices"].astype(np.float32), full["triangles"], full["colors"]
        N = 2048
        for pct in (10, 2):
            target = len(ff) * pct // 100
            sv, sf, _, _ = simplify(fv, ff, None, target)
            fn = MT.transfer_fn(fv, ff, fc, texture_size=N)
            runs = [staged(sv, sf, N, fn) for _ in range(args.reps + 1)][1:]
            print(json.dumps({"workload": f"bench_mc256_{pct}pct", "faces": int(len(sf)), "N": N, "colour": "transfer",
                              **best(runs)}), flush=True)
            # the field path: export_mesh_step's own bake, its stages timed through the same colour function
            runs, real = [], MT.bake
            def timed_bake(vv, fff, n, colour_fn, device=None):
                got = []
                runs.append(staged(vv, fff, n, colour_fn, got))
                return got[0]
            MT.bake = timed_bake
            try:
                walls = []
                for _ in range(args.reps + 1):
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    tr.export_mesh_step(sample, resolution=256, target_faces=target, texture_size=N)
                    torch.cuda.synchronize()
                    walls.append(1e3 * (time.perf_counter() - t))
            finally:
                MT.bake = real
            plain = []
            for _ in range(args.reps + 1):
                torch.cuda.synchronize()
                t = time.perf_counter()
                tr.export_mesh_step(sample, resolution=256, target_faces=target)
                torch.cuda.synchronize()
                plain.append(1e3 * (time.perf_counter() - t))
            print(json.dumps({"workload": f"bench_mc256_{pct}pct", "faces": int(len(sf)), "N": N, "colour": "blend_points",
                              **best(runs[1:]), "export_mesh_step_ms": min(walls[1:]),
                              "export_mesh_step_no_texture_ms": min(plain[1:])}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps({"card": card(), "peak_alloc_gb": torch.cuda.max_memory_allocated() / 1e9}), flush=True)


if __name__ == "__main__":
    main()
