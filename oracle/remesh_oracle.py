"""numpy restatement of isotropic remeshing and closest points on a mesh (csrc/remesh.cu, ops.remesh_mesh,
ops.closest_points).  The reference has no remesher, so nothing here is pinned against it: this file is the definition the
GPU path is tested against, operation for operation.  The rules are written out in include/o2345.h (o2345_remesh,
o2345_closest_points); the remesh is Botsch & Kobbelt (2004): split long edges, collapse short ones, flip towards valence
6, relax tangentially, project back onto the input.

Closest point: closest_points() evaluates only the faces whose centroid lies within (d + r)(1 + 1e-9) + M 2^-40 of the
point (d the distance to the nearest centroid, r the largest centroid-corner distance, M the largest |coordinate|): the
face a search over all faces picks is within d of the point (up to rounding), so its centroid is within d + r, and
brute=True (every face) gives the same answer; the tests check both.
"""
from __future__ import annotations

import numpy as np

from . import simplify_oracle as S
from .normal_map_oracle import vertex_normals
from .texture_oracle import closest_point

ITERATIONS = 5
MAX_SPLIT_ROUNDS = 64
MAX_GAIN = 1 << 30


def target_length(verts, faces, target_faces):
    """L = sqrt(4 A / (sqrt(3) N)) rounded once to fp32, A the area summed in fp64 in ascending face order (sequentially);
    +inf for N = 0."""
    V = np.asarray(verts, np.float32).astype(np.float64).reshape(-1, 3)
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    n = S.cross(V[F[:, 0]], V[F[:, 1]], V[F[:, 2]])
    area = 0.5 * np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    A = float(np.cumsum(area)[-1]) if len(area) else 0.0
    if target_faces <= 0:
        return np.float32(np.inf), A
    return np.float32(np.sqrt(4.0 * A / (np.sqrt(3.0) * float(target_faces)))), A


# ----------------------------------------------------------------------------- closest point
def _candidates_eval(V, F, P, pi, fi):
    """(d2 fp64, q fp64 [n,3]) of points P[pi] against faces fi."""
    A, B, C = V[F[fi, 0]], V[F[fi, 1]], V[F[fi, 2]]
    p = P[pi]
    la, lb, lc = closest_point(p, A, B, C)
    q = (la[:, None] * A + lb[:, None] * B) + lc[:, None] * C
    d = q - p
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2], q


def _pick(n, pi, fi, d2, q):
    order = np.lexsort((fi, d2, pi))
    first = np.ones(len(order), bool)
    first[1:] = pi[order][1:] != pi[order][:-1]
    sel = order[first]
    face = np.full(n, -1, np.int64)
    out = np.full((n, 3), np.nan)
    face[pi[sel]] = fi[sel]
    out[pi[sel]] = q[sel]
    return out, face


def closest_points(verts, faces, points, brute=False, chunk=1 << 22):
    """-> (points fp32 [n,3], face int64 [n]): per point the least (squared distance, face index) over all faces of the
    7-region closest point; NaN / -1 for a non-finite point or no faces."""
    V = np.asarray(verts, np.float32).astype(np.float64).reshape(-1, 3)
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    P32 = np.asarray(points, np.float32).reshape(-1, 3)
    n = len(P32)
    ok = np.isfinite(P32).all(1)
    out, face = np.full((n, 3), np.nan), np.full(n, -1, np.int64)
    if len(F) == 0 or not ok.any():
        return out.astype(np.float32), face
    idx = np.nonzero(ok)[0]
    P = P32[idx].astype(np.float64)
    if brute:
        per = max(1, chunk // len(F))
        res_o, res_f = [], []
        for a in range(0, len(P), per):
            m = min(per, len(P) - a)
            pi = np.repeat(np.arange(m), len(F))
            fi = np.tile(np.arange(len(F)), m)
            d2, q = _candidates_eval(V, F, P[a:a + m], pi, fi)
            o, f = _pick(m, pi, fi, d2, q)
            res_o.append(o), res_f.append(f)
        o, f = np.concatenate(res_o), np.concatenate(res_f)
    else:
        from scipy.spatial import cKDTree
        cen = (V[F[:, 0]] + V[F[:, 1]] + V[F[:, 2]]) / 3.0
        r = max(float(np.sqrt(((V[F[:, k]] - cen) ** 2).sum(1)).max()) for k in range(3))
        M = float(np.abs(V).max()) if len(V) else 0.0
        tree = cKDTree(cen)
        dU, _ = tree.query(P)
        rad = (dU + r) * (1 + 1e-9) + M * 2.0 ** -40 + 1e-300
        lists = tree.query_ball_point(P, rad)
        cnt = np.array([len(x) for x in lists])
        pi = np.repeat(np.arange(len(P)), cnt)
        fi = np.concatenate([np.asarray(x, np.int64) for x in lists]) if len(pi) else np.zeros(0, np.int64)
        d2, q = _candidates_eval(V, F, P, pi, fi)
        o, f = _pick(len(P), pi, fi, d2, q)
    out[idx], face[idx] = o, f
    return out.astype(np.float32), face


# ----------------------------------------------------------------------------- remesh
def _len2(V, a, b):
    d = V[b].astype(np.float64) - V[a].astype(np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _half_edges(F, nv):
    """-> a, b, c [3F] (corner k, k + 1, k + 2 of each face), edge id per half-edge (its least half-edge), face count per
    half-edge, and the other half-edge of every two-face edge's canonical half-edge (-1 elsewhere)."""
    a, b, c = F.reshape(-1), F[:, [1, 2, 0]].reshape(-1), F[:, [2, 0, 1]].reshape(-1)
    key = np.minimum(a, b) * nv + np.maximum(a, b)
    order = np.argsort(key, kind="stable")
    _, first, inv, cnt = np.unique(key[order], return_index=True, return_inverse=True, return_counts=True)
    eid = np.empty(len(a), np.int64)
    eid[order] = order[first][inv]
    ecnt = np.empty(len(a), np.int64)
    ecnt[order] = cnt[inv]
    other = np.full(len(a), -1, np.int64)
    two = cnt == 2
    other[order[first[two]]] = order[first[two] + 1]
    return a, b, c, eid, ecnt, other


def _split_round(V, F, hi2):
    nv = len(V)
    a, b, _, eid, ecnt, other = _half_edges(F, nv)
    l2 = _len2(V, a, b)
    long = (l2 > hi2) & (ecnt <= 2)
    key = (l2.astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | eid.astype(np.uint64)
    kk = np.where(long, key, np.uint64(0)).reshape(-1, 3)
    fmax = kk.max(1)
    fk = np.where(fmax > 0, kk.argmax(1), -1)
    h = 3 * np.arange(len(F)) + np.maximum(fk, 0)
    canon = (fk >= 0) & (eid[h] == h)
    oface = np.where(other[h] >= 0, other[h] // 3, -1)
    split_h = np.zeros(len(a), bool)
    pick = canon & ((oface < 0) | (fmax[np.maximum(oface, 0)] == fmax))
    split_h[h[pick]] = True
    rows = np.nonzero(split_h)[0]
    if len(rows) == 0:
        return V, F, False
    hidx = np.full(len(a), -1, np.int64)
    hidx[rows] = np.arange(len(rows))
    e = (fmax & np.uint64(0xffffffff)).astype(np.int64)
    fflag = (fk >= 0) & split_h[e]
    mid = (V[a[rows]] + V[b[rows]]) * np.float32(0.5)
    V = np.concatenate([V, mid.astype(np.float32)])
    fr = np.nonzero(fflag)[0]
    k = fk[fr]
    m = nv + hidx[e[fr]]
    G = F[fr].copy()
    G[np.arange(len(fr)), k] = m
    F = F.copy()
    F[fr, (k + 1) % 3] = m
    return V, np.concatenate([F, G]), True


def _topology(F, nv):
    inc, slot, deg = S.incidence(F, nv)
    locked, val, ukey, opp = S.locks_and_valence(F, nv, inc, slot, deg)
    return inc, locked, val, ukey, opp


def _legal(F, V64, locked, val, ukey, opp, nb, inc, u, v, chunk=16384):
    """The simplifier's legal u -> v (u unlocked)."""
    nv = len(V64)
    e = np.searchsorted(ukey, S._edge_key(u, v, nv))
    o1, o2 = opp[e, 0], opp[e, 1]
    ok = (o1 != o2) & (val[o1] >= 4) & (val[o2] >= 4) & (val[u] + val[v] - 4 >= 3)
    x = nb[u]
    oth = (x >= 0) & (x != v[:, None]) & (x != o1[:, None]) & (x != o2[:, None])
    kx = S._edge_key(np.maximum(x, 0), v[:, None], nv)
    pos = np.minimum(np.searchsorted(ukey, kx), len(ukey) - 1)
    ok &= ~(oth & (ukey[pos] == kx)).any(1)
    for s0 in range(0, len(u), chunk):
        s = slice(s0, s0 + chunk)
        fc = inc[u[s]]
        tri = F[np.maximum(fc, 0)]
        skip = (fc < 0) | (tri == v[s, None, None]).any(2)
        P = V64[tri]
        n0 = S.cross(P[:, :, 0], P[:, :, 1], P[:, :, 2])
        P2 = np.where((tri == u[s, None, None])[..., None], V64[v[s]][:, None, None, :], P)
        n1 = S.cross(P2[:, :, 0], P2[:, :, 1], P2[:, :, 2])
        dot = (n1[..., 0] * n0[..., 0] + n1[..., 1] * n0[..., 1]) + n1[..., 2] * n0[..., 2]
        ok[s] &= (skip | (dot > 0)).all(1)
    return ok


def _collapse_round(V, F, lo2, hi2):
    nv = len(V)
    inc, locked, val, ukey, opp = _topology(F, nv)
    nb = S.neighbours(ukey, nv)
    u = np.repeat(np.arange(nv), (nb >= 0).sum(1))
    v = nb[nb >= 0]
    keep = ~locked[u]
    u, v = u[keep], v[keep]
    l2 = _len2(V, u, v)
    sh = l2 < lo2
    u, v, l2 = u[sh], v[sh], l2[sh]
    if len(u) == 0:
        return F, False
    V64 = V.astype(np.float64)
    ok = _legal(F, V64, locked, val, ukey, opp, nb, inc, u, v)
    X = nb[u]
    lx = _len2(V, v[:, None], np.maximum(X, 0))
    ok &= (~((X >= 0) & (X != v[:, None]) & (lx > hi2))).all(1)
    u, v, l2 = u[ok], v[ok], l2[ok]
    if len(u) == 0:
        return F, False
    cb = l2.astype(np.float32).view(np.uint32).astype(np.uint64)
    order = np.lexsort((v, cb, u))
    u, v, cb = u[order], v[order], cb[order]
    first = np.ones(len(u), bool)
    first[1:] = u[1:] != u[:-1]
    u, v, cb = u[first], v[first], cb[first]
    key = (cb << np.uint64(32)) | u.astype(np.uint64)
    acc = S.select(u, v, key, nb, nv)
    u, v = u[acc], v[acc]
    if len(u) == 0:
        return F, False
    to = np.arange(nv)
    to[u] = v
    F = to[F]
    return F[(F[:, 0] != F[:, 1]) & (F[:, 1] != F[:, 2]) & (F[:, 0] != F[:, 2])], True


def _dev(val, locked):
    e = val - np.where(locked, 4, 6)
    return e * e


def _flip_round(V, F):
    nv = len(V)
    _, locked, val, ukey, _ = _topology(F, nv)
    a, b, c, eid, ecnt, other = _half_edges(F, nv)
    h = np.arange(len(a))
    cand = (eid == h) & (ecnt == 2)
    oh = np.maximum(other, 0)
    cand &= (a[oh] == b) & (b[oh] == a)
    d = c[oh]
    cand &= (d != c) & (val[a] > 3) & (val[b] > 3)
    kcd = S._edge_key(c, d, nv)
    pos = np.minimum(np.searchsorted(ukey, kcd), len(ukey) - 1)
    cand &= ukey[pos] != kcd
    la, lb, lc, ld = locked[a], locked[b], locked[c], locked[d]
    before = _dev(val[a], la) + _dev(val[b], lb) + _dev(val[c], lc) + _dev(val[d], ld)
    after = _dev(val[a] - 1, la) + _dev(val[b] - 1, lb) + _dev(val[c] + 1, lc) + _dev(val[d] + 1, ld)
    gain = before - after
    cand &= gain > 0
    i = np.nonzero(cand)[0]
    if len(i) == 0:
        return F, False
    V64 = V.astype(np.float64)
    A, B, C, D = V64[a[i]], V64[b[i]], V64[c[i]], V64[d[i]]
    n0, n1, m0, m1 = S.cross(A, B, C), S.cross(B, A, D), S.cross(A, D, C), S.cross(D, B, C)
    dt = lambda x, y: (x[:, 0] * y[:, 0] + x[:, 1] * y[:, 1]) + x[:, 2] * y[:, 2]
    ok = (dt(m0, n0) > 0) & (dt(m0, n1) > 0) & (dt(m1, n0) > 0) & (dt(m1, n1) > 0)
    i = i[ok]
    if len(i) == 0:
        return F, False
    key = (np.uint64(MAX_GAIN) - gain[i].astype(np.uint64)) << np.uint64(32) | i.astype(np.uint64)
    quad = np.stack([a[i], b[i], c[i], d[i]], 1)
    claim = np.full(nv, S.NO_CLAIM, np.uint64)
    np.minimum.at(claim, quad.reshape(-1), np.repeat(key, 4))
    acc = (claim[quad] == key[:, None]).all(1)
    i, quad = i[acc], quad[acc]
    if len(i) == 0:
        return F, False
    F = F.copy()
    f, o = i // 3, oh[i] // 3
    F[f] = quad[:, [0, 3, 2]]
    F[o] = quad[:, [3, 1, 2]]
    return F, True


def _relax(V, F):
    nv = len(V)
    _, locked, _, ukey, _ = _topology(F, nv)
    nb = S.neighbours(ukey, nv)
    V64 = V.astype(np.float64)
    s = np.zeros((nv, 3))
    for k in range(nb.shape[1]):
        has = nb[:, k] >= 0
        s[has] = s[has] + V64[nb[has, k]]
    cnt = (nb >= 0).sum(1)
    move = ~locked
    c = s[move] / cnt[move, None].astype(np.float64)
    n = vertex_normals(V, F).astype(np.float64)[move]
    p = V64[move]
    e = c - p
    t = (e[:, 0] * n[:, 0] + e[:, 1] * n[:, 1]) + e[:, 2] * n[:, 2]
    out = V.copy()
    out[move] = (p + (e - n * t[:, None])).astype(np.float32)
    return out, locked


def prepare(verts, faces):
    V = np.asarray(verts, np.float32).reshape(-1, 3)
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(F) and (F.min() < 0 or F.max() >= len(V)):
        raise ValueError("a face index is outside [0, nv)")
    if not np.isfinite(V).all():
        raise ValueError("a vertex coordinate is not finite")
    return V, F


def remesh(verts, faces, L, iterations=ITERATIONS, relax=True, flip=True, project=True):
    """-> (verts fp32 [nv',3], faces int32 [nf',3], (split rounds, collapse rounds, flip rounds)) for target edge length L
    (fp32).  relax / flip / project=False switch a step off (controls for the tests; the library always runs them)."""
    V, Fin = prepare(verts, faces)
    L = np.float32(L)
    if not (L >= np.float32(2.0 ** -60)):
        raise ValueError("target length must be >= 2^-60")
    ref_V, ref_F = V.copy(), Fin.copy()
    rep = (Fin[:, 0] == Fin[:, 1]) | (Fin[:, 1] == Fin[:, 2]) | (Fin[:, 0] == Fin[:, 2])
    F = Fin[~rep]
    Ld = np.float64(L)
    hi, lo = Ld * (4.0 / 3.0), Ld * 0.8
    hi2, lo2 = hi * hi, lo * lo
    rounds = [0, 0, 0]
    for _ in range(iterations):
        if len(F) == 0:
            break
        for _ in range(MAX_SPLIT_ROUNDS):
            V, F, did = _split_round(V, F, hi2)
            if not did:
                break
            rounds[0] += 1
        while len(F):
            F, did = _collapse_round(V, F, lo2, hi2)
            if not did:
                break
            rounds[1] += 1
        while flip and len(F):
            F, did = _flip_round(V, F)
            if not did:
                break
            rounds[2] += 1
        if len(F) == 0:
            break
        if relax:
            V, locked = _relax(V, F)
        else:
            locked = _topology(F, len(V))[1]
        if project:
            idx = np.nonzero(~locked)[0]
            if len(idx):
                q, _ = closest_points(ref_V, ref_F, V[idx])
                V = V.copy()
                V[idx] = q
    used = np.zeros(len(V), bool)
    used[F.reshape(-1)] = True
    remap = np.cumsum(used) - 1
    return V[used], remap[F].astype(np.int32).reshape(-1, 3), tuple(rounds)
