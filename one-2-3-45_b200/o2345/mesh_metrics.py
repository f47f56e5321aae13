"""Scores a generated mesh against its ground truth: F-Score and Chamfer distance from surface samples (csrc/metrics.cu),
and the CLIP similarity of the 24 evaluation-rig views.  One-2-3-45 reports F-Score and CLIP similarity; the reference
ships only the renderer of that evaluation (render/), no metric code, so the protocol below is this project's definition
(DESIGN.md section 2, parity unpinned; oracle/metrics_oracle.py restates it in numpy):

  frame        both meshes through mesh_raster.flatten(normalize_scene(load_scene(path))): the frame the rig renders in
               (largest extent 0.8, centred, OBJ / glTF turned from Y-up to Z-up).  No ICP or other alignment.
  samples      n_points (default 100 000) area-uniform samples per surface; the predicted mesh from `seed`, the ground
               truth from seed + 1.
  F-Score      precision = share of predicted samples whose nearest GT sample is closer than tau, recall the other way
               (compared as squares in fp32: d2 < fp32(tau^2)); F = 2PR / (P + R), 0 when P + R = 0.  The default
               tau = 0.05 in the rig frame is a choice: the paper's threshold is not in the reference.
  Chamfer      (mean_p d(p, GT) + mean_g d(g, Pred)) / 2, Euclidean (not squared), summed in fp64.
  CLIP         both meshes rendered unlit from the 24 rig views (camera_dist 1.3 as the reference's launcher), composited
               over white (rgb * alpha + 1 - alpha), mapped to [-1, 1] and embedded with FrozenCLIPImageEmbedder, whose
               preprocessing is Zero123's (bicubic resize with align_corners to 224^2), not OpenAI's PIL pipeline;
               cosine similarity of view i with view i, and the mean over the 24 views.
"""
from __future__ import annotations

import numpy as np

from . import mesh_raster as MR

DEFAULT_N_POINTS = 100_000
DEFAULT_THRESHOLDS = (0.05,)
CLIP_RESOLUTION, CLIP_CAMERA_DIST = 512, 1.3


def load_flat(path, y_up=None):
    """A mesh file in the rig frame: mesh_raster.flatten's arrays."""
    return MR.flatten(MR.normalize_scene(MR.load_scene(path, y_up=y_up)))


def sample(flat, n, seed=0, device="cuda"):
    """n area-uniform samples of flatten()'s mesh -> pts [n,3] fp32 and face_id [n] int32, device tensors."""
    import torch
    from . import ops
    dev = torch.device(device)
    with torch.cuda.device(dev):
        return ops.surface_sample(torch.from_numpy(np.ascontiguousarray(flat["verts"])).to(dev),
                                  torch.from_numpy(np.ascontiguousarray(flat["faces"])).to(dev), n, seed)


def fscore_chamfer(flat_pred, flat_gt, n_points=DEFAULT_N_POINTS, thresholds=DEFAULT_THRESHOLDS, seed=0, device="cuda"):
    """-> {"fscore": {tau: {precision, recall, fscore, n_precise, n_recalled}}, "chamfer": float}, as
    oracle.metrics_oracle.fscore_chamfer computes it from the same samples."""
    import torch
    from . import ops
    p, _ = sample(flat_pred, n_points, seed, device)
    g, _ = sample(flat_gt, n_points, (seed + 1) % 2 ** 64, device)
    with torch.cuda.device(p.device):
        d2p, _ = ops.nearest(p, g)
        d2g, _ = ops.nearest(g, p)
        t2 = [float(np.float32(t * t)) for t in thresholds]
        counts = torch.stack([torch.stack([(d2p < v).sum(), (d2g < v).sum()]) for v in t2]).tolist()
        chamfer = 0.5 * (float(torch.sqrt(d2p.double()).mean()) + float(torch.sqrt(d2g.double()).mean()))
    out = {}
    for tau, (npr, nre) in zip(thresholds, counts):
        P, R = npr / n_points, nre / n_points
        out[tau] = {"precision": P, "recall": R, "fscore": 2 * P * R / (P + R) if P + R > 0 else 0.0,
                    "n_precise": npr, "n_recalled": nre}
    return {"fscore": out, "chamfer": chamfer}


def white_views(path, resolution=CLIP_RESOLUTION, camera_dist=CLIP_CAMERA_DIST, device="cuda"):
    """The 24 unlit rig views of a mesh composited over white, [24,3,H,W] in [-1, 1] (the embedder's input range)."""
    out = MR.render_rig(path, camera_dist, resolution, shading="unlit", device=device)
    a = out["alpha"][..., None]
    rgb = out["color"].clamp(0, 1) * a + (1 - a)
    return (rgb * 2 - 1).permute(0, 3, 1, 2).contiguous()


def clip_similarity(path_pred, path_gt, embedder, resolution=CLIP_RESOLUTION, camera_dist=CLIP_CAMERA_DIST, device="cuda"):
    """-> {"per_view": [24 cosines], "mean": float}: CLIP image embeddings of view i of both meshes, compared view by view."""
    import torch
    with torch.no_grad():
        e = [embedder(white_views(p, resolution, camera_dist, device)).double() for p in (path_pred, path_gt)]
        cos = torch.nn.functional.cosine_similarity(e[0], e[1], dim=1)
    per_view = cos.tolist()
    return {"per_view": per_view, "mean": float(np.mean(per_view))}


def score(pred_path, gt_path, n_points=DEFAULT_N_POINTS, thresholds=DEFAULT_THRESHOLDS, seed=0, embedder=None,
          resolution=CLIP_RESOLUTION, camera_dist=CLIP_CAMERA_DIST, device="cuda"):
    """The protocol on one pair of mesh files; "clip" only with an embedder."""
    out = {"pred": pred_path, "gt": gt_path,
           **fscore_chamfer(load_flat(pred_path), load_flat(gt_path), n_points, thresholds, seed, device)}
    if embedder is not None:
        out["clip"] = clip_similarity(pred_path, gt_path, embedder, resolution, camera_dist, device)
    return out
