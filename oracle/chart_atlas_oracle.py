"""numpy restatement of o2345_chart_atlas (csrc/texture.cu, --atlas charts), bit for bit.

The reference has no texture baking, so every rule is this project's own (include/o2345.h, DESIGN §2):

  labels   n = (P1 - P0) x (P2 - P0) in fp64; axis a = argmax |n_a| (the lower axis on ties), label 2a + (n_a < 0); a zero
           or non-finite n gives label 6 (a chart of its own, projected along z);
  project  (u, v) = (p[(a+1) % 3], p[(a+2) % 3]) in fp32, u negated when n_a < 0;
  charts   connected components of faces sharing an edge with exactly two (face, edge) uses on two faces and the same key
           (round 0: the label, 6 + f for label 6); the edge -> face pairs come from sorted edge keys here (the device
           walks its vertex -> face lists); a chart's id is its least face;
  overlap  the separating-axis test of tri_overlap, touching does not count;
  cut      a chart with an overlap ranks its m faces by (x0 + x1) + x2 along its longer extent (u on ties), ties by face
           index; the first m // 2 go to side 0; the next key is 2 id + side; repeat until no chart overlaps;
  extent   per chart min / max of its corners; e = max - min in fp64 rounded up to fp32;
  packing  texture_oracle's boxes, shelves and ladder over the charts in id order, S = sum of e_u e_v;
  uv       (x + 2 + (p - min) rho) / N in fp64, rounded to fp32;
  owner    candidates: the chart's faces whose uv box (uv * N in fp32) grown by 2 holds the texel centre, inside the
           chart's box; key (fp32 squared distance, f), least wins; the distance is 0 inside or on the triangle.
"""
from __future__ import annotations

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from . import texture_oracle as T

PAD = T.PAD
OWN = 6


def labels(verts, faces):
    """-> (label [F] int32, puv [F,3,2] fp32 projected corners)."""
    v = np.asarray(verts, np.float32)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    p = v[f].astype(np.float64)
    e1, e2 = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    a = np.argmax(np.abs(n), 1)
    na = n[np.arange(len(f)), a]
    ok = (np.abs(na) > 0) & np.isfinite(n).all(1)
    a = np.where(ok, a, 2)
    neg = ok & (na < 0)
    lab = np.where(ok, 2 * a + neg, OWN).astype(np.int32)
    q = v[f]                                             # [F,3,3] fp32
    r = np.arange(len(f))[:, None]
    u = q[r, np.arange(3)[None], ((a + 1) % 3)[:, None]]
    w = q[r, np.arange(3)[None], ((a + 2) % 3)[:, None]]
    u = np.where(neg[:, None], -u, u)
    return lab, np.stack([u, w], -1).astype(np.float32)


def edge_pairs(faces, nv):
    """-> (f, g) int64 arrays: the faces of every edge with exactly two uses that belong to two faces."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    a = f.reshape(-1)
    b = f[:, [1, 2, 0]].reshape(-1)
    slot_face = np.repeat(np.arange(len(f)), 3)
    keep = a != b
    key = np.minimum(a, b)[keep] * nv + np.maximum(a, b)[keep]
    sf = slot_face[keep]
    o = np.argsort(key, kind="stable")
    key, sf = key[o], sf[o]
    start = np.r_[True, key[1:] != key[:-1]]
    idx = np.nonzero(start)[0]
    size = np.diff(np.r_[idx, len(key)])
    two = idx[size == 2]
    fa, fb = sf[two], sf[two + 1]
    ok = fa != fb
    return fa[ok], fb[ok]


def components(nf, fa, fb, key):
    """-> chart id [F] (the least face of each component of the pairs with equal keys)."""
    m = key[fa] == key[fb]
    g = coo_matrix((np.ones(int(m.sum())), (fa[m], fb[m])), shape=(nf, nf))
    _, comp = connected_components(g, directed=False)
    least = np.full(comp.max() + 1, nf, np.int64)
    np.minimum.at(least, comp, np.arange(nf))
    return least[comp]


def orient(ax, ay, bx, by, px, py):
    ax, ay, bx, by, px, py = (np.asarray(x, np.float64) for x in (ax, ay, bx, by, px, py))
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax)


def tri_overlap(P, Q):
    """P, Q [n,3,2] fp32 -> [n] bool: the projected triangles share an interior point (separating axes, touching does not
    count; a triangle of orient 0 has no interior)."""
    P, Q = np.asarray(P, np.float32), np.asarray(Q, np.float32)
    out = np.ones(len(P), bool)
    for A, B in ((P, Q), (Q, P)):
        out &= orient(A[:, 0, 0], A[:, 0, 1], A[:, 1, 0], A[:, 1, 1], A[:, 2, 0], A[:, 2, 1]) != 0
        for k in range(3):
            k1, k2 = (k + 1) % 3, (k + 2) % 3
            ax, ay, bx, by = A[:, k, 0], A[:, k, 1], A[:, k1, 0], A[:, k1, 1]
            s = orient(ax, ay, bx, by, A[:, k2, 0], A[:, k2, 1])
            o = np.stack([orient(ax, ay, bx, by, B[:, j, 0], B[:, j, 1]) for j in range(3)], 1)
            out &= ~((o.max(1) <= np.minimum(0.0, s)) | (o.min(1) >= np.maximum(0.0, s)))
    return out


def overlapping_charts(puv, chart):
    """-> sorted array of chart ids in which two faces overlap (a sweep over u inside each chart: the pairs whose uv
    boxes overlap with positive area, then tri_overlap)."""
    lo, hi = puv.min(1), puv.max(1)                      # [F,2]
    o = np.lexsort((lo[:, 0], chart))                    # by chart, then u min
    c, l0 = chart[o], lo[o, 0]
    n = len(o)
    upto = np.empty(n, np.int64)                         # faces i + 1 .. upto[i] - 1 of i's run start left of i's u max
    bounds = np.searchsorted(c, np.unique(c))
    for a, b in zip(bounds.tolist(), np.r_[bounds[1:], n].tolist()):
        upto[a:b] = a + np.searchsorted(l0[a:b], hi[o[a:b], 0], side="left")
    i = np.arange(n)
    cnt = np.maximum(upto - (i + 1), 0)
    total = int(cnt.sum())
    first = np.repeat(i, cnt)
    second = (np.arange(total) - np.repeat(np.cumsum(cnt) - cnt, cnt)) + np.repeat(i + 1, cnt)
    bad = set()
    step = 1 << 22
    for s in range(0, total, step):
        fi, fj = o[first[s:s + step]], o[second[s:s + step]]
        box = (hi[fj, 0] > lo[fi, 0]) & (lo[fj, 0] < hi[fi, 0]) & (hi[fj, 1] > lo[fi, 1]) & (lo[fj, 1] < hi[fi, 1])
        fi, fj = fi[box], fj[box]
        hit = tri_overlap(puv[fi], puv[fj])
        bad.update(np.unique(chart[fi[hit]]).tolist())
    return np.array(sorted(bad), np.int64)


def extents(puv, chart):
    """-> (ids [C] ascending, lo [C,2] fp32, e [C,2] fp32 rounded up)."""
    ids, inv = np.unique(chart, return_inverse=True)
    lo = np.full((len(ids), 2), np.inf, np.float32)
    hi = np.full((len(ids), 2), -np.inf, np.float32)
    np.minimum.at(lo, inv, puv.min(1))
    np.maximum.at(hi, inv, puv.max(1))
    d = hi.astype(np.float64) - lo.astype(np.float64)
    e = d.astype(np.float32)
    up = e.astype(np.float64) < d
    e[up] = np.nextafter(e[up], np.float32(np.inf))
    return ids, lo, e


def cut(puv, chart, bad, ids, e):
    """-> the next round's key [F]."""
    side = np.zeros(len(chart), np.int64)
    pos = {int(c): i for i, c in enumerate(ids)}
    for cid in bad.tolist():
        fs = np.nonzero(chart == cid)[0]
        eu, ev = e[pos[cid]]
        ax = 0 if eu >= ev else 1
        q = puv[fs, :, ax].astype(np.float64)
        c = (q[:, 0] + q[:, 1]) + q[:, 2]
        order = np.lexsort((fs, c))
        s = np.zeros(len(fs), np.int64)
        s[order[len(fs) // 2:]] = 1
        side[fs] = s
    return 2 * chart + side


def tri_dist2(q, a, b, c):
    """Squared distance [n] fp64 of points q [n,2] to triangles a, b, c [n,2] (fp64), 0 inside or on the triangle."""
    w0 = orient(b[:, 0], b[:, 1], c[:, 0], c[:, 1], q[:, 0], q[:, 1])
    w1 = orient(c[:, 0], c[:, 1], a[:, 0], a[:, 1], q[:, 0], q[:, 1])
    w2 = orient(a[:, 0], a[:, 1], b[:, 0], b[:, 1], q[:, 0], q[:, 1])
    ar = orient(a[:, 0], a[:, 1], b[:, 0], b[:, 1], c[:, 0], c[:, 1])
    inside = (ar != 0) & (((w0 >= 0) & (w1 >= 0) & (w2 >= 0)) | ((w0 <= 0) & (w1 <= 0) & (w2 <= 0)))
    z = np.zeros((len(q), 1))
    la, lb, lc = T.closest_point(*(np.concatenate([x, z], 1) for x in (q, a, b, c)))
    x = (la * a[:, 0] + lb * b[:, 0]) + lc * c[:, 0]
    y = (la * a[:, 1] + lb * b[:, 1]) + lc * c[:, 1]
    dx, dy = q[:, 0] - x, q[:, 1] - y
    return np.where(inside, 0.0, dx * dx + dy * dy)


def owner_map(uv, boxes, N):
    """-> owner [N*N] int32 of the faces' uv [F,3,2] inside their chart boxes [F,4]."""
    t = (np.asarray(uv, np.float32) * np.float32(N)).astype(np.float64)   # [F,3,2]
    bx, by, bw, bh = (boxes[:, k].astype(np.int64) for k in range(4))
    x0 = np.maximum(bx, np.ceil(t[:, :, 0].min(1) - (PAD + 0.5)).astype(np.int64))
    x1 = np.minimum(bx + bw - 1, np.floor(t[:, :, 0].max(1) + (PAD - 0.5)).astype(np.int64))
    y0 = np.maximum(by, np.ceil(t[:, :, 1].min(1) - (PAD + 0.5)).astype(np.int64))
    y1 = np.minimum(by + bh - 1, np.floor(t[:, :, 1].max(1) + (PAD - 0.5)).astype(np.int64))
    w, h = np.maximum(x1 - x0 + 1, 0), np.maximum(y1 - y0 + 1, 0)
    w, h = np.where(h > 0, w, 0), np.where(w > 0, h, 0)
    keys = np.full(N * N, np.iinfo(np.uint64).max, np.uint64)
    faces = np.arange(len(t))
    step = 1 << 14
    for s in range(0, len(t), step):
        fs = faces[s:s + step]
        cnt = w[fs] * h[fs]
        f = np.repeat(fs, cnt)
        i = np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        tx, ty = x0[f] + i % w[f], y0[f] + i // w[f]
        q = np.stack([tx + 0.5, ty + 0.5], 1).astype(np.float64)
        d = tri_dist2(q, t[f, 0], t[f, 1], t[f, 2]).astype(np.float32)
        key = (d.view(np.uint32).astype(np.uint64) << np.uint64(32)) | f.astype(np.uint64)
        np.minimum.at(keys, ty * N + tx, key)
    return np.where(keys == np.iinfo(np.uint64).max, -1, (keys & np.uint64(0xffffffff)).astype(np.int64)).astype(np.int32)


def atlas(verts, faces, N):
    """-> dict(j, rho, rounds, charts, label [F], chart [F], boxes [F,4], uv [F,3,2], owner [N*N]).  Raises ValueError
    where the C call returns O2345_EINVAL."""
    if not T.valid_size(N):
        raise ValueError("N must be a power of two in [64, 8192]")
    v = np.asarray(verts, np.float32)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(f) == 0 or f.min() < 0 or f.max() >= len(v):
        raise ValueError("a face index is outside [0, nv)")
    if not np.isfinite(v).all():
        raise ValueError("a vertex coordinate is not finite")
    nf = len(f)
    lab, puv = labels(v, f)
    fa, fb = edge_pairs(f, len(v))
    key = np.where(lab < OWN, lab, OWN + np.arange(nf)).astype(np.int64)
    rounds = 0
    while True:
        chart = components(nf, fa, fb, key)
        ids, lo, e = extents(puv, chart)
        bad = overlapping_charts(puv, chart)
        if len(bad) == 0:
            break
        rounds += 1
        key = cut(puv, chart, bad, ids, e)
    S = T.lh_sum(e[:, 0], e[:, 1])
    if not S > 0:
        raise ValueError("the charts have no area")
    r0 = T.rho0(N, S)
    packs = {}

    def fits_at(j):
        rho = T.rung(r0, j)
        w, hg = T.box_sides(e[:, 0], rho, N), T.box_sides(e[:, 1], rho, N)
        ok, x, y = T.pack(w, hg, N)
        packs[j] = (x, y, w, hg)
        return ok

    j = T.search(fits_at)
    if j is None:
        raise ValueError(f"{N}^2 texels cannot hold {len(ids)} charts")
    rho = T.rung(r0, j)
    x, y, w, hg = packs[j]
    cbox = np.stack([x, y, w, hg], 1).astype(np.int32)
    pos = np.searchsorted(ids, chart)
    boxes = cbox[pos]
    X = (boxes[:, 0] + PAD).astype(np.float64)[:, None]
    Y = (boxes[:, 1] + PAD).astype(np.float64)[:, None]
    m = lo[pos].astype(np.float64)
    u = (X + (puv[:, :, 0].astype(np.float64) - m[:, None, 0]) * rho) / N
    vv = (Y + (puv[:, :, 1].astype(np.float64) - m[:, None, 1]) * rho) / N
    uv = np.stack([u, vv], -1).astype(np.float32)
    owner = owner_map(uv, boxes, N)
    return {"j": j, "rho": rho, "rounds": rounds, "charts": len(ids), "label": lab, "chart": chart.astype(np.int32),
            "boxes": boxes, "uv": uv, "owner": owner, "puv": puv, "extent": e}
