"""numpy restatement of the mesh simplifier (csrc/simplify.cu, ops.simplify_mesh).  The reference has no simplifier, so
nothing here is pinned against it: this file is the definition the GPU path is tested against, operation for operation.

Parallel half-edge collapse driven by Garland-Heckbert quadrics.  A removed vertex u is merged into a neighbour v that
keeps its position, so every output vertex is an input vertex.  The work runs in rounds on the mesh as it stood at the
start of the round:

  input       faces with a repeated index are dropped; an index outside [0, nv) or a non-finite coordinate is refused
  quadrics    once: n = (B - A) x (C - A) in fp64 from the fp32 vertices, |n| = sqrt((nx*nx + ny*ny) + nz*nz),
              p = (nx/|n|, ny/|n|, nz/|n|, d), d = -((px*Ax + py*Ay) + pz*Az), w = |n| * 0.5, Q_f[ij] = w * (p_i * p_j)
              for the 10 entries (i <= j, row-major); 0 when |n| = 0.  Q_u = sum of its faces' Q_f in ascending face order
  locks       u is locked when an edge at u does not have exactly two faces, or its faces do not form one closed fan
  legal u->v  u unlocked, v a neighbour; the two faces of uv have third vertices o1 != o2 and N(u) & N(v) = {o1, o2};
              val(o1) >= 4, val(o2) >= 4, val(u) + val(v) - 4 >= 3; every face of u without v keeps n' . n > 0 (fp64,
              (n'x*nx + n'y*ny) + n'z*nz) when u is replaced by v
  cost        Q = Q_u + Q_v, r_i = ((Q_i0*x + Q_i1*y) + Q_i2*z) + Q_i3, c = ((r0*x + r1*y) + r2*z) + r3 at v = (x, y, z),
              rounded to fp32, anything not > 0 becomes +0; u proposes its legal neighbour with the least (c, v) under
              the key (bits(c) << 32) | u
  selection   every proposal's key is min-reduced onto the closed 1-rings of u and v; it is accepted when it holds the
              minimum on all of them; if more than k = ceil((F - target) / 2) are accepted only the k least keys are kept
  apply       u -> v in every face of u, the two faces of uv are deleted, Q_v += Q_u; faces keep their input order

Output: (vertex_index [nv'] int32, faces [nf', 3] int32 renumbered into it, rounds).
"""
from __future__ import annotations

import numpy as np

PAIRS = ((0, 0), (0, 1), (0, 2), (0, 3), (1, 1), (1, 2), (1, 3), (2, 2), (2, 3), (3, 3))
SYM = np.array([[0, 1, 2, 3], [1, 4, 5, 6], [2, 5, 7, 8], [3, 6, 8, 9]])    # Q entry of (row, column)
NO_CLAIM = np.uint64(2 ** 64 - 1)


def cross(P0, P1, P2):
    """(P1 - P0) x (P2 - P0) of fp64 arrays [..., 3], as metrics.cu's face weights compute it."""
    e1, e2 = P1 - P0, P2 - P0
    return np.stack([e1[..., 1] * e2[..., 2] - e1[..., 2] * e2[..., 1],
                     e1[..., 2] * e2[..., 0] - e1[..., 0] * e2[..., 2],
                     e1[..., 0] * e2[..., 1] - e1[..., 1] * e2[..., 0]], -1)


def face_quadrics(V, F):
    """V fp64 [nv,3], F [m,3] -> Q_f [m,10]."""
    A = V[F[:, 0]]
    n = cross(A, V[F[:, 1]], V[F[:, 2]])
    ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    ok = ln > 0
    s = np.where(ok, ln, 1.0)
    p = [n[:, 0] / s, n[:, 1] / s, n[:, 2] / s]
    p.append(-((p[0] * A[:, 0] + p[1] * A[:, 1]) + p[2] * A[:, 2]))
    w = ln * 0.5
    Q = np.stack([w * (p[i] * p[j]) for i, j in PAIRS], 1)
    return np.where(ok[:, None], Q, 0.0)


def incidence(F, nv):
    """-> (inc [nv, D] face indices ascending, -1 padded; slot [nv, D] corner of the vertex in that face; deg [nv])."""
    vert = F.reshape(-1)
    order = np.argsort(vert, kind="stable")             # corners are in face order: stable keeps faces ascending
    deg = np.bincount(vert, minlength=nv)
    start = np.concatenate([[0], np.cumsum(deg)[:-1]])
    rank = np.arange(len(vert)) - start[vert[order]]
    D = max(int(deg.max()) if len(deg) else 0, 1)
    inc, slot = np.full((nv, D), -1, np.int64), np.zeros((nv, D), np.int64)
    inc[vert[order], rank] = order // 3
    slot[vert[order], rank] = order % 3
    return inc, slot, deg


def vertex_quadrics(V, F):
    """Q_u [nv,10]: the sum of the vertex's face quadrics, face by face in ascending face order."""
    Qf = face_quadrics(V, F)
    inc, _, _ = incidence(F, len(V))
    Q = np.zeros((len(V), 10))
    for k in range(inc.shape[1]):
        has = inc[:, k] >= 0
        Q[has] = Q[has] + Qf[inc[has, k]]
    return Q


def _edge_key(a, b, nv):
    return np.minimum(a, b).astype(np.int64) * nv + np.maximum(a, b)


def locks_and_valence(F, nv, inc, slot, deg):
    """-> (locked [nv] bool, valence [nv], sorted undirected edge keys, their opposite vertices [E,2] or -1)."""
    a, b, o = F.reshape(-1), F[:, [1, 2, 0]].reshape(-1), F[:, [2, 0, 1]].reshape(-1)
    key = _edge_key(a, b, nv)
    order = np.argsort(key, kind="stable")
    ukey, first, cnt = np.unique(key[order], return_index=True, return_counts=True)
    lo, hi = ukey // nv, ukey % nv
    val = np.bincount(lo, minlength=nv) + np.bincount(hi, minlength=nv)
    locked = deg == 0
    bad = cnt != 2
    locked[lo[bad]] = True
    locked[hi[bad]] = True
    opp = np.full((len(ukey), 2), -1, np.int64)
    opp[~bad, 0] = o[order][first[~bad]]
    opp[~bad, 1] = o[order][first[~bad] + 1]
    # one closed fan: walk from the vertex's first face across its edges (each has exactly two faces here) and count
    # the faces met before the walk returns
    cand = np.nonzero(~locked)[0]
    fc = inc[cand]
    valid = fc >= 0
    A = np.where(valid, F[np.maximum(fc, 0), (slot[cand] + 1) % 3], -1)
    B = np.where(valid, F[np.maximum(fc, 0), (slot[cand] + 2) % 3], -1)
    ar = np.arange(len(cand))
    x, prev = B[:, 0].copy(), np.zeros(len(cand), np.int64)
    seen, done = np.ones(len(cand), np.int64), np.zeros(len(cand), bool)
    for _ in range(inc.shape[1]):
        hit = (A == x[:, None]) | (B == x[:, None])
        hit[ar, prev] = False
        j = hit.argmax(1)
        step = ~done & (j != 0)
        seen += step
        x = np.where(step, np.where(A[ar, j] == x, B[ar, j], A[ar, j]), x)
        prev = np.where(step, j, prev)
        done |= j == 0
    locked[cand[seen != deg[cand]]] = True
    return locked, val, ukey, opp


def neighbours(ukey, nv):
    """Distinct neighbours of every vertex, ascending, -1 padded [nv, Dn]."""
    lo, hi = ukey // nv, ukey % nv
    src, dst = np.concatenate([lo, hi]), np.concatenate([hi, lo])
    order = np.lexsort((dst, src))
    src, dst = src[order], dst[order]
    cnt = np.bincount(src, minlength=nv)
    start = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    nb = np.full((nv, max(int(cnt.max()) if nv else 0, 1)), -1, np.int64)
    nb[src, np.arange(len(src)) - start[src]] = dst
    return nb


def collapse_cost(Q, V, u, v):
    """fp32 cost of u -> v (arrays of vertex ids), negative or zero results as +0."""
    q = Q[u] + Q[v]
    x = [V[v, 0], V[v, 1], V[v, 2]]
    r = [((q[:, SYM[i, 0]] * x[0] + q[:, SYM[i, 1]] * x[1]) + q[:, SYM[i, 2]] * x[2]) + q[:, SYM[i, 3]] for i in range(4)]
    c = (((r[0] * x[0] + r[1] * x[1]) + r[2] * x[2]) + r[3]).astype(np.float32)
    return np.where(c > 0, c, np.float32(0))


def proposals(F, V, Q, locked, val, ukey, opp, nb, inc, random_cost=False, chunk=16384):
    """-> (u, v, key) of every unlocked vertex that has a legal collapse."""
    nv = len(V)
    u = np.repeat(np.arange(nv), (nb >= 0).sum(1))
    v = nb[nb >= 0]
    keep = ~locked[u]
    u, v = u[keep], v[keep]
    e = np.searchsorted(ukey, _edge_key(u, v, nv))
    o1, o2 = opp[e, 0], opp[e, 1]
    ok = (o1 != o2) & (val[o1] >= 4) & (val[o2] >= 4) & (val[u] + val[v] - 4 >= 3)
    # link condition: no neighbour of u other than v, o1, o2 is a neighbour of v
    x = nb[u]
    other = (x >= 0) & (x != v[:, None]) & (x != o1[:, None]) & (x != o2[:, None])
    kx = _edge_key(np.maximum(x, 0), v[:, None], nv)
    pos = np.minimum(np.searchsorted(ukey, kx), len(ukey) - 1)
    ok &= ~(other & (ukey[pos] == kx)).any(1)
    # no face of u without v flips or collapses
    for a in range(0, len(u), chunk):
        s = slice(a, a + chunk)
        fc = inc[u[s]]
        tri = F[np.maximum(fc, 0)]                                   # [n, D, 3]
        skip = (fc < 0) | (tri == v[s, None, None]).any(2)
        P = V[tri]                                                   # [n, D, 3, 3]
        n0 = cross(P[:, :, 0], P[:, :, 1], P[:, :, 2])
        P2 = np.where((tri == u[s, None, None])[..., None], V[v[s]][:, None, None, :], P)
        n1 = cross(P2[:, :, 0], P2[:, :, 1], P2[:, :, 2])
        dot = (n1[..., 0] * n0[..., 0] + n1[..., 1] * n0[..., 1]) + n1[..., 2] * n0[..., 2]
        ok[s] &= (skip | (dot > 0)).all(1)
    u, v = u[ok], v[ok]
    if random_cost:      # the control: a uniform in [0, 1) hashed from the edge instead of the quadric error
        from .metrics_oracle import uniforms
        c = uniforms(0, u.astype(np.uint64) * np.uint64(nv) + v.astype(np.uint64)).astype(np.float32)
    else:
        c = collapse_cost(Q, V, u, v)
    cb = c.view(np.uint32).astype(np.uint64)
    order = np.lexsort((v, cb, u))
    u, v, cb = u[order], v[order], cb[order]
    first = np.ones(len(u), bool)
    first[1:] = u[1:] != u[:-1]
    u, v, cb = u[first], v[first], cb[first]
    return u, v, (cb << np.uint64(32)) | u.astype(np.uint64)


def select(u, v, key, nb, nv):
    """Accepted proposals: those whose key is the least on every vertex of the closed 1-rings of u and v."""
    ring = np.concatenate([u[:, None], nb[u], v[:, None], nb[v]], 1)
    has = ring >= 0
    claim = np.full(nv, NO_CLAIM, np.uint64)
    np.minimum.at(claim, ring[has], np.broadcast_to(key[:, None], ring.shape)[has])
    return (~has | (claim[np.maximum(ring, 0)] == key[:, None])).all(1)


def prepare(verts, faces):
    """Checks the input and drops faces with a repeated index -> (V fp64 [nv,3], F int64 [m,3])."""
    V = np.asarray(verts, np.float32).reshape(-1, 3)
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(F) and (F.min() < 0 or F.max() >= len(V)):
        raise ValueError("a face index is outside [0, nv)")
    if not np.isfinite(V).all():
        raise ValueError("a vertex coordinate is not finite")
    rep = (F[:, 0] == F[:, 1]) | (F[:, 1] == F[:, 2]) | (F[:, 0] == F[:, 2])
    return V.astype(np.float64), F[~rep]


def simplify(verts, faces, target_faces, random_cost=False, trace=None):
    """-> (vertex_index int32 [nv'], faces int32 [nf',3], rounds).  random_cost=True replaces every cost by a hash of the
    edge (a control that keeps every rule but lets no geometry choose the collapses; with every cost 0 instead, the least
    index absorbs its neighbours about one collapse per round).  trace: a list that receives (u, v, cost fp32) of the collapses
    applied in each round."""
    if target_faces < 0:
        raise ValueError("target_faces must be >= 0")
    V, F = prepare(verts, faces)
    nv = len(V)
    Q = vertex_quadrics(V, F)
    rounds = 0
    while len(F) > target_faces:
        inc, slot, deg = incidence(F, nv)
        locked, val, ukey, opp = locks_and_valence(F, nv, inc, slot, deg)
        nb = neighbours(ukey, nv)
        u, v, key = proposals(F, V, Q, locked, val, ukey, opp, nb, inc, random_cost)
        if len(u) == 0:
            break
        acc = select(u, v, key, nb, nv)
        u, v, key = u[acc], v[acc], key[acc]
        k = (len(F) - target_faces + 1) // 2
        if len(u) > k:
            keep = np.argsort(key)[:k]
            u, v, key = u[keep], v[keep], key[keep]
        if trace is not None:
            trace.append((u, v, (key >> np.uint64(32)).astype(np.uint32).view(np.float32)))
        to = np.arange(nv)
        to[u] = v
        F = to[F]
        F = F[(F[:, 0] != F[:, 1]) & (F[:, 1] != F[:, 2]) & (F[:, 0] != F[:, 2])]
        Q[v] = Q[v] + Q[u]
        rounds += 1
    used = np.zeros(nv, bool)
    used[F.reshape(-1)] = True
    vertex_index = np.nonzero(used)[0]
    remap = np.cumsum(used) - 1
    return vertex_index.astype(np.int32), remap[F].astype(np.int32).reshape(-1, 3), rounds
