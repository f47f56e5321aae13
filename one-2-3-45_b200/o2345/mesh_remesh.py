"""Isotropic remeshing on host arrays (run.py / simplify_mesh.py --remesh, GenericTrainer.validate_colored_mesh): the mesh goes
to the GPU, ops.remesh_mesh splits, collapses, flips, relaxes and projects it back onto itself (csrc/remesh.cu) to about
target_faces faces of near-equilateral triangles, and the new vertices come back.  Every output vertex lies on the input
surface; colours are taken by the caller at the new positions."""
from __future__ import annotations

import math

import numpy as np
import torch

from . import ops

REMESH_ITERATIONS = 5


def target_length(vertices, triangles, target_faces):
    """-> (L fp32, A): L = sqrt(4 A / (sqrt(3) N)) rounded once to fp32, the edge length of N equilateral triangles of the
    input's total area A (fp64, summed in ascending face order); +inf for N = 0."""
    v = np.asarray(vertices, np.float32).astype(np.float64).reshape(-1, 3)
    f = np.asarray(triangles, np.int64).reshape(-1, 3)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    e1, e2 = b - a, c - a
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    area = 0.5 * np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    A = float(np.cumsum(area)[-1]) if len(area) else 0.0
    if target_faces <= 0:
        return np.float32(np.inf), A
    return np.float32(math.sqrt(4.0 * A / (math.sqrt(3.0) * float(target_faces)))), A


def remesh(vertices, triangles, extra, target_faces, device=None, iterations=REMESH_ITERATIONS):
    """vertices [n,3], triangles [m,3] (numpy), extra: ignored except that it must be None (colours are the caller's:
    the vertices are new) -> (vertices fp32 [n',3], triangles int32 [m',3], stats dict(L, area, rounds, iterations)).
    A mesh without faces or area comes back with its faces that have three distinct corners and the vertices they
    reference, unmoved."""
    if target_faces < 0:
        raise ValueError(f"target_faces must be >= 0, got {target_faces}")
    if extra is not None:
        raise ValueError("remesh creates vertices: take colours at the returned positions instead")
    v = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)
    f = np.ascontiguousarray(triangles, np.int32).reshape(-1, 3)
    if len(f) and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError("a face index is outside [0, nv)")
    if not np.isfinite(v).all():
        raise ValueError("a vertex coordinate is not finite")
    L, A = target_length(v, f, target_faces)
    stats = {"L": float(L), "area": A, "rounds": (0, 0, 0), "iterations": iterations}
    if len(f) == 0 or not A > 0:
        # as the remesh itself leaves them: faces with three distinct corners, only the vertices they reference
        f = f[(f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])]
        used = np.zeros(len(v), bool)
        used[f.reshape(-1)] = True
        return v[used], (np.cumsum(used) - 1)[f].astype(np.int32).reshape(-1, 3), stats
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    with torch.cuda.device(dev):
        vt = torch.from_numpy(v).to(dev)
        ft = torch.from_numpy(f).to(dev)
        ov, of, rounds = ops.remesh_mesh(vt, ft, L, iterations)
        out_v, out_f = ov.cpu().numpy(), of.cpu().numpy()
    stats["rounds"] = rounds
    return out_v, out_f, stats


def describe(vertices, triangles, stats):
    """The line the command lines print."""
    s, c, fl = stats["rounds"]
    return (f"remesh: {len(triangles)} faces, {len(vertices)} vertices, L = {stats['L']:.6g}, "
            f"{stats['iterations']} iterations, rounds: {s} split, {c} collapse, {fl} flip")


def surface_colors(src_vertices, src_triangles, src_colors, points, device=None):
    """Colours uint8 [n,k] of the source mesh at points [n,3]: each point's exact closest point on the source (ops.
    closest_points) and the closest face's vertex colours interpolated there (ops.transfer_colors), rounded half-even, so
    a point on a source vertex takes its colour exactly."""
    c = np.asarray(src_colors)
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    with torch.cuda.device(dev):
        sv = torch.from_numpy(np.ascontiguousarray(src_vertices, np.float32)).to(dev)
        sf = torch.from_numpy(np.ascontiguousarray(src_triangles, np.int32).reshape(-1, 3)).to(dev)
        p = torch.from_numpy(np.ascontiguousarray(points, np.float32).reshape(-1, 3)).to(dev)
        _, face = ops.closest_points(sv, sf, p)
        idx = torch.arange(p.shape[0], dtype=torch.int32, device=dev)
        cols = []
        for k in range(0, c.shape[1], 3):
            part = np.zeros((len(c), 3), np.float32)
            part[:, :min(3, c.shape[1] - k)] = c[:, k:k + 3]
            rgb = ops.transfer_colors(sv, sf, torch.from_numpy(part).to(dev), p, idx, face)
            cols.append(torch.round(rgb[:, :min(3, c.shape[1] - k)]).clamp(0, 255).cpu().numpy())
    return np.concatenate(cols, 1).astype(c.dtype)
