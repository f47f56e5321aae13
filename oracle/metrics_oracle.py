"""numpy restatement of the mesh-scoring kernels (csrc/metrics.cu) and of the F-Score / Chamfer protocol
(o2345/mesh_metrics.py, DESIGN.md section 2).  The reference has no metric code, so nothing here is pinned against it:
this file is the definition the GPU path is tested against, operation for operation.

  surface_weights   twice the face areas, fp64 from the fp32 vertices: e1 = B - A, e2 = C - A, c = e1 x e2,
                    sqrt((cx*cx + cy*cy) + cz*cz); 0 for an index outside [0, nv) or a non-finite value
  surface_cdf       np.cumsum inside chunks of 1024 faces, np.cumsum over the chunk totals, each chunk's offset added
  surface_sample    three splitmix64 uniforms per sample, first face whose CDF exceeds u0 * total, barycentric point
  nearest           chunked brute force, d2 = (dx*dx + dy*dy) + dz*dz in fp32, ties to the lower reference index
  fscore_chamfer    precision / recall / F per threshold (d2 < fp32(tau^2)), chamfer = (mean d(P, G) + mean d(G, P)) / 2
"""
from __future__ import annotations

import numpy as np

CHUNK = 1024
GOLDEN = np.uint64(0x9E3779B97F4A7C15)


def splitmix64(seed, c):
    """Output c (uint64 array) of splitmix64 seeded with `seed`."""
    z = np.uint64(seed) + (np.asarray(c, np.uint64) + np.uint64(1)) * GOLDEN
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def uniforms(seed, c):
    return (splitmix64(seed, c) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def surface_weights(verts, faces):
    verts, faces = np.asarray(verts, np.float32), np.asarray(faces, np.int64).reshape(-1, 3)
    ok = ((faces >= 0) & (faces < len(verts))).all(1)
    f = np.where(ok[:, None], faces, 0)
    A, B, C = (verts[f[:, k]].astype(np.float64) for k in range(3))
    e1, e2 = B - A, C - A
    cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    with np.errstate(invalid="ignore", over="ignore"):
        w = np.sqrt((cx * cx + cy * cy) + cz * cz)
    return np.where(ok & np.isfinite(w), w, 0.0)


def surface_cdf(w):
    """-> (cdf [nf], total) with the kernel's chunked summation order."""
    nf = len(w)
    nchunks = -(-nf // CHUNK)
    loc = np.cumsum(np.concatenate([w, np.zeros(nchunks * CHUNK - nf)]).reshape(nchunks, CHUNK), axis=1)
    T = np.cumsum(loc[:, -1])
    off = np.concatenate([[0.0], T[:-1]])
    return (loc + off[:, None]).reshape(-1)[:nf], float(T[-1])


def surface_sample(verts, faces, n, seed=0):
    """-> pts float32 [n,3], face_id int32 [n], bit-identical to ops.surface_sample."""
    verts, faces = np.asarray(verts, np.float32), np.asarray(faces, np.int64).reshape(-1, 3)
    cdf, total = surface_cdf(surface_weights(verts, faces))
    if not total > 0:
        raise ValueError("the faces have no area")
    i = np.arange(n, dtype=np.uint64) * np.uint64(3)
    u0, u1, u2 = (uniforms(seed, i + np.uint64(k)) for k in range(3))
    f = np.searchsorted(cdf, u0 * total, side="right")
    f = np.where(f == len(cdf), np.searchsorted(cdf, total, side="left"), f)
    s = np.sqrt(u1)
    wa, wb, wc = 1.0 - s, s * (1.0 - u2), s * u2
    A, B, C = (verts[faces[f, k]].astype(np.float64) for k in range(3))
    p = (wa[:, None] * A + wb[:, None] * B) + wc[:, None] * C
    return p.astype(np.float32), f.astype(np.int32)


def nearest(query, ref, chunk=256):
    """Brute force -> dist2 float32 [nq], index int32 [nq] (the first minimum: ties to the lower index)."""
    q, r = np.asarray(query, np.float32).reshape(-1, 3), np.asarray(ref, np.float32).reshape(-1, 3)
    d2, idx = np.empty(len(q), np.float32), np.empty(len(q), np.int32)
    for a in range(0, len(q), chunk):
        qa = q[a:a + chunk]
        dx, dy, dz = (qa[:, None, k] - r[None, :, k] for k in range(3))
        d = (dx * dx + dy * dy) + dz * dz
        j = d.argmin(1)
        idx[a:a + chunk], d2[a:a + chunk] = j, d[np.arange(len(qa)), j]
    return d2, idx


def fscore_chamfer(d2_pred, d2_gt, thresholds=(0.05,)):
    """d2_pred: squared distance of every predicted sample to the GT samples, d2_gt the other way ->
    {"fscore": {tau: {precision, recall, fscore, n_precise, n_recalled}}, "chamfer": float}."""
    d2_pred, d2_gt = np.asarray(d2_pred, np.float32), np.asarray(d2_gt, np.float32)
    out = {}
    for tau in thresholds:
        t2 = np.float32(tau * tau)
        npr, nre = int((d2_pred < t2).sum()), int((d2_gt < t2).sum())
        P, R = npr / len(d2_pred), nre / len(d2_gt)
        out[tau] = {"precision": P, "recall": R, "fscore": 2 * P * R / (P + R) if P + R > 0 else 0.0,
                    "n_precise": npr, "n_recalled": nre}
    chamfer = 0.5 * (np.sqrt(d2_pred.astype(np.float64)).mean() + np.sqrt(d2_gt.astype(np.float64)).mean())
    return {"fscore": out, "chamfer": float(chamfer)}


def score(flat_pred, flat_gt, n_points, thresholds=(0.05,), seed=0):
    """The whole protocol on mesh_raster.flatten() arrays: predicted samples from `seed`, GT samples from seed + 1."""
    p, _ = surface_sample(flat_pred["verts"], flat_pred["faces"], n_points, seed)
    g, _ = surface_sample(flat_gt["verts"], flat_gt["faces"], n_points, (seed + 1) % 2 ** 64)
    return fscore_chamfer(nearest(p, g)[0], nearest(g, p)[0], thresholds)
