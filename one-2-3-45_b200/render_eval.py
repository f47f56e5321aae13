"""Renders meshes from the 24 views of the reference's evaluation rig on the GPU (o2345/mesh_raster.py, csrc/raster.cu).

Mirrors the reference's render/single_render_eval.py and render/launch_render_eval.py:

    python one-2-3-45_b200/render_eval.py --object_path mesh.glb --output_dir D [--camera_dist 1.5] [--resolution 512]
                                          [--shading unlit|lambert]
        -> D/0.png ... D/23.png (RGBA), D/depth.npy [24,H,W], D/normal.npy [24,H,W,3]
    python one-2-3-45_b200/render_eval.py --DATA_DIR dir [--camera_dist 1.3] [--resolution 512]
        -> output/<name>/render_<resolution>/ for every mesh in dir (the launcher passes --camera_dist 1.3)

Inputs: .obj, .glb and .ply (.ply is an extension: the reference script refuses it); .fbx is refused.  --resolution is
honoured (the reference script always renders 512^2).  --engine is accepted and ignored."""
from __future__ import annotations

import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

FORMATS = (".obj", ".glb", ".ply")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--object_path", type=str, help="mesh to render (.obj, .glb or .ply)")
    src.add_argument("--DATA_DIR", type=str, help="render every mesh of this folder into output/<name>/render_<res>/")
    ap.add_argument("--output_dir", type=str, default="./views")
    ap.add_argument("--engine", type=str, default=None, help="accepted for the reference's command line; ignored")
    ap.add_argument("--camera_dist", type=float, default=None,
                    help="camera distance (default 1.5 with --object_path, 1.3 with --DATA_DIR, as the reference)")
    ap.add_argument("--resolution", type=int, default=512)
    ap.add_argument("--shading", choices=("unlit", "lambert"), default="unlit")
    ap.add_argument("--out_root", type=str, default="output", help="--DATA_DIR: root of the output folders")
    args = ap.parse_args(argv)
    if args.resolution < 1 or args.resolution > 16384:
        ap.error("--resolution must be in [1, 16384]")
    if args.camera_dist is None:
        args.camera_dist = 1.3 if args.DATA_DIR else 1.5
    if args.camera_dist <= 0:
        ap.error("--camera_dist must be > 0")
    if args.object_path and os.path.splitext(args.object_path)[1].lower() not in FORMATS:
        ap.error(f"{args.object_path}: unsupported mesh format (only {', '.join(FORMATS)}; .fbx is not supported)")
    return args


def jobs(args):
    """(mesh path, output dir) pairs the command renders."""
    if args.object_path:
        return [(args.object_path, args.output_dir)]
    out = []
    for name in sorted(os.listdir(args.DATA_DIR)):
        if os.path.splitext(name)[1].lower() in FORMATS:
            out.append((os.path.join(args.DATA_DIR, name),
                        os.path.join(args.out_root, name.split(".")[0], f"render_{args.resolution}")))
    return out


def main(argv=None):
    args = parse_args(argv)
    if args.engine is not None:
        print(f"render_eval: --engine {args.engine} ignored (the GPU rasterizer renders every view)", file=sys.stderr)
    import time

    import torch
    from o2345 import mesh_raster
    for path, out_dir in jobs(args):
        t0 = time.time()
        out = mesh_raster.render_rig(path, args.camera_dist, args.resolution, args.shading)
        torch.cuda.synchronize()
        mesh_raster.write_views(out, out_dir)
        print(f"rendered {path} -> {out_dir} in {time.time() - t0:.2f} s")


if __name__ == "__main__":
    main()
