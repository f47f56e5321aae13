"""Scores generated meshes against their ground truth on the GPU (o2345/mesh_metrics.py, csrc/metrics.cu):

    python one-2-3-45_b200/eval_mesh.py --pred a.obj [b.ply ...] --gt a_gt.glb [b_gt.glb ...] \\
        [--n_points 100000] [--threshold 0.05 ...] [--seed 0] [--clip_ckpt zero123-xl.ckpt] \\
        [--resolution 512] [--camera_dist 1.3] [--out scores.json]

Pairs are taken in order (the i-th --pred against the i-th --gt).  Prints one line per pair and the mean over the pairs:
F-Score, precision and recall at every threshold and the Chamfer distance, in the rig frame of render_eval.py (largest
extent 0.8), plus the CLIP similarity of the 24 rig views when --clip_ckpt gives a Zero123 checkpoint to take the CLIP
image tower from.  --out writes the scores and the protocol's parameters as JSON.  Inputs: .obj, .glb and .ply."""
from __future__ import annotations

import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

FORMATS = (".obj", ".glb", ".ply")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--pred", nargs="+", required=True, help="generated meshes (.obj, .glb or .ply)")
    ap.add_argument("--gt", nargs="+", required=True, help="ground-truth meshes, one per --pred, in the same order")
    ap.add_argument("--n_points", type=int, default=100_000, help="surface samples per mesh")
    ap.add_argument("--threshold", type=float, nargs="+", default=[0.05],
                    help="F-Score distance thresholds in the rig frame (0.05 is this project's choice)")
    ap.add_argument("--seed", type=int, default=0, help="sampling seed (predicted mesh: seed, ground truth: seed + 1)")
    ap.add_argument("--clip_ckpt", type=str, default=None, help="Zero123 checkpoint with the CLIP image tower (CLIP similarity)")
    ap.add_argument("--resolution", type=int, default=512, help="CLIP: rig render resolution")
    ap.add_argument("--camera_dist", type=float, default=1.3, help="CLIP: rig camera distance")
    ap.add_argument("--out", type=str, default=None, help="JSON file for the scores and the protocol")
    args = ap.parse_args(argv)
    if len(args.pred) != len(args.gt):
        ap.error(f"{len(args.pred)} --pred meshes but {len(args.gt)} --gt meshes: they are taken in pairs")
    for p in args.pred + args.gt:
        if os.path.splitext(p)[1].lower() not in FORMATS:
            ap.error(f"{p}: unsupported mesh format (only {', '.join(FORMATS)})")
    if args.n_points < 1:
        ap.error("--n_points must be >= 1")
    if any(not t > 0 for t in args.threshold):
        ap.error("--threshold values must be > 0")
    if args.resolution < 1 or args.resolution > 16384:
        ap.error("--resolution must be in [1, 16384]")
    if not args.camera_dist > 0:
        ap.error("--camera_dist must be > 0")
    if not 0 <= args.seed < 2 ** 64:
        ap.error("--seed must be in [0, 2^64)")
    return args


def line(name, s, thresholds):
    parts = [f"F@{t:g}={s['fscore'][t]['fscore']:.6f} P={s['fscore'][t]['precision']:.6f} R={s['fscore'][t]['recall']:.6f}"
             for t in thresholds]
    parts.append(f"chamfer={s['chamfer']:.6f}")
    if "clip" in s:
        parts.append(f"clip={s['clip']['mean']:.6f}")
    return f"{name}: " + " ".join(parts)


def mean_scores(scores, thresholds):
    n = len(scores)
    out = {"fscore": {t: {k: sum(s["fscore"][t][k] for s in scores) / n for k in ("precision", "recall", "fscore")}
                      for t in thresholds},
           "chamfer": sum(s["chamfer"] for s in scores) / n}
    if scores and all("clip" in s for s in scores):
        out["clip"] = {"mean": sum(s["clip"]["mean"] for s in scores) / n}
    return out


def main(argv=None):
    args = parse_args(argv)
    from o2345 import mesh_metrics as MM
    embedder = None
    if args.clip_ckpt:
        from o2345.zero123 import load_clip_image_embedder
        embedder = load_clip_image_embedder(args.clip_ckpt, device="cuda")
    scores = []
    for pred, gt in zip(args.pred, args.gt):
        s = MM.score(pred, gt, args.n_points, tuple(args.threshold), args.seed, embedder, args.resolution, args.camera_dist)
        scores.append(s)
        print(line(f"{pred} vs {gt}", s, args.threshold), flush=True)
    mean = mean_scores(scores, args.threshold)
    print(line(f"mean over {len(scores)} pairs", mean, args.threshold))
    if args.out:
        key = lambda d: {f"{t:g}": v for t, v in d.items()}
        doc = {"protocol": {"frame": "mesh_raster.flatten(normalize_scene(load_scene(path))): largest extent 0.8, centred, "
                                     "OBJ / glTF Y-up -> Z-up, no alignment",
                            "n_points": args.n_points, "thresholds": args.threshold, "seed": args.seed,
                            "seed_gt": (args.seed + 1) % 2 ** 64, "distance": "exact nearest surface sample, fp32",
                            "chamfer": "(mean d(pred, gt) + mean d(gt, pred)) / 2, not squared",
                            "clip": None if embedder is None else {
                                "checkpoint": args.clip_ckpt, "views": 24, "resolution": args.resolution,
                                "camera_dist": args.camera_dist, "shading": "unlit", "background": "white",
                                "preprocessing": "Zero123 (bicubic, align_corners)"}},
               "pairs": [{**s, "fscore": key(s["fscore"])} for s in scores],
               "mean": {**mean, "fscore": key(mean["fscore"])}}
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)
    return scores


if __name__ == "__main__":
    main()
