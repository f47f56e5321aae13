"""numpy restatement of csrc/texture.cu (texture baking), bit for bit.

The reference has no texture baking (its convert_mesh_format writes vertex colours), so every rule here is this
project's own definition (DESIGN §2, parity unpinned):

  charts      per face, base = the longest of (v0v1, v1v2, v2v0) by fp32 squared length ((dx*dx + dy*dy) + dz*dz), the first
              on ties; a, b = the base's vertices, c the third; L = |b - a|, d = (c - a).(b - a) / L,
              h = |(b - a) x (c - a)| / L in fp64 from the fp32 vertices, rounded once to fp32 (0 for L = 0), d clamped to
              [0, L];
  scale       S = sum of L * h (fp64; sequential inside chunks of 1024 faces, then over the chunk totals),
              rho0 = sqrt(0.5 N^2 / S), rho_j = rho0 * j / 64;
  boxes       w = ceil(L rho) + 2P, hgt = ceil(h rho) + 2P, P = 2 (N + 1 when ceil(.) > N: it cannot fit);
  packing     sort by hgt descending then face index; next-fit shelves (a new shelf below the current one's tallest box
              when a box would cross x = N); fits when every box lies inside N x N;
  search      j = 1 must fit; then lo = 1, hi = 257, binary search keeping the largest j that fits;
  uv          a at (x + P, y + P), b at (x + P + L rho, y + P), c at (x + P + d rho, y + P + h rho), / N (fp64, rounded
              to fp32), row k of a face for its corner k;
  ownership   every texel of a box is owned by the box's face;
  points      the closest point of the chart's triangle (uv * N in fp32) to the texel centre (i + 0.5, j + 0.5), by the
              7-region test in fp64, then (la A + lb B) + lc C in fp32 with the weights rounded to fp32;
  fill        push-pull on fp32 rgb + weight (owned texels weigh 1): pull = weight sums and weight-normalised 2 x 2 means,
              push = every texel of weight 0 takes its parent's colour, coarse to fine;
  transfer    the closest point of the source face behind each point's nearest sample (nearest indices are an input)
              and the face's vertex colours interpolated with the same rounding.
"""
from __future__ import annotations

import numpy as np

PAD = 2
CHUNK = 1024
RUNGS, RUNG_DEN = 256, 64
MIN_N, MAX_N = 64, 8192


def valid_size(N):
    return isinstance(N, (int, np.integer)) and MIN_N <= N <= MAX_N and N & (N - 1) == 0


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def base_corner(verts, faces):
    """-> [F] index k0 of the corner that starts the longest edge (fp32 squared lengths, first on ties)."""
    v = np.asarray(verts, np.float32)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    l2 = []
    for k in range(3):
        e = v[f[:, (k + 1) % 3]] - v[f[:, k]]
        l2.append((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2])
    l2 = np.stack(l2, 1)
    k0 = np.zeros(len(f), np.int64)
    best = l2[:, 0].copy()
    for k in (1, 2):
        better = l2[:, k] > best
        k0[better], best[better] = k, l2[better, k]
    return k0


def charts(verts, faces):
    """-> (L, d, h) fp32 [F] and the base corner k0 [F]."""
    v = np.asarray(verts, np.float32)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    k0 = base_corner(v, f)
    r = np.arange(len(f))
    a = v[f[r, k0]].astype(np.float64)
    b = v[f[r, (k0 + 1) % 3]].astype(np.float64)
    c = v[f[r, (k0 + 2) % 3]].astype(np.float64)
    e1, e2 = b - a, c - a
    L = np.sqrt(_dot(e1, e1))
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    pos = L > 0
    safe = np.where(pos, L, 1.0)
    d = np.where(pos, _dot(e2, e1) / safe, 0.0)
    h = np.where(pos, np.sqrt(_dot(n, n)) / safe, 0.0)
    Lf, df, hf = L.astype(np.float32), d.astype(np.float32), h.astype(np.float32)
    df = np.minimum(np.maximum(df, np.float32(0)), Lf)
    return Lf, df, hf, k0


def lh_sum(L, h):
    p = np.asarray(L, np.float32).astype(np.float64) * np.asarray(h, np.float32).astype(np.float64)
    total = 0.0
    for a in range(0, len(p), CHUNK):
        run = 0.0
        for x in p[a:a + CHUNK]:
            run = run + float(x)
        total = total + run
    return total


def rho0(N, S):
    return float(np.sqrt(0.5 * (float(N) * float(N)) / S))


def rung(r0, j):
    return r0 * float(j) / float(RUNG_DEN)


def box_sides(e, rho, N):
    s = np.ceil(np.asarray(e, np.float32).astype(np.float64) * rho)
    return np.where(s > N, N + 1, np.minimum(s, N).astype(np.int64) + 2 * PAD)


def pack(w, hgt, N):
    """Next-fit shelf packing -> (fits, x [F], y [F]); x / y only meaningful when it fits."""
    w, hgt = np.asarray(w, np.int64), np.asarray(hgt, np.int64)
    x, y = np.zeros(len(w), np.int64), np.zeros(len(w), np.int64)
    if (w > N).any() or (hgt > N).any():
        return False, x, y
    order = np.argsort(-hgt, kind="stable")
    cx = cy = sh = 0
    for f in order.tolist():
        wf, hf = int(w[f]), int(hgt[f])
        if cx > 0 and cx + wf > N:
            cy, cx, sh = cy + sh, 0, 0
        if cx + wf > N or cy + hf > N:
            return False, x, y
        x[f], y[f] = cx, cy
        cx, sh = cx + wf, max(sh, hf)
    return True, x, y


def search(fits_at):
    """The ladder search over j in [1, 256] given fits_at(j) -> bool; None when j = 1 does not fit."""
    if not fits_at(1):
        return None
    lo, hi = 1, RUNGS + 1
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if fits_at(mid):
            lo = mid
        else:
            hi = mid
    return lo


def atlas(verts, faces, N):
    """-> dict(j, rho, boxes [F,4] int32 (x, y, w, hgt), uv [F,3,2] fp32, owner [N*N] int32, k0 [F]).
    Raises ValueError where the C call returns O2345_EINVAL."""
    if not valid_size(N):
        raise ValueError("N must be a power of two in [64, 8192]")
    v = np.asarray(verts, np.float32)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(f) == 0 or f.min() < 0 or f.max() >= len(v):
        raise ValueError("a face index is outside [0, nv)")
    if not np.isfinite(v).all():
        raise ValueError("a vertex coordinate is not finite")
    L, d, h, k0 = charts(v, f)
    S = lh_sum(L, h)
    if not S > 0:
        raise ValueError("the faces have no area")
    r0 = rho0(N, S)
    packs = {}

    def fits_at(j):
        rho = rung(r0, j)
        w, hg = box_sides(L, rho, N), box_sides(h, rho, N)
        ok, x, y = pack(w, hg, N)
        packs[j] = (x, y, w, hg)
        return ok

    j = search(fits_at)
    if j is None:
        raise ValueError(f"{N}^2 texels cannot hold {len(f)} charts")
    rho = rung(r0, j)
    x, y, w, hg = packs[j]
    boxes = np.stack([x, y, w, hg], 1).astype(np.int32)
    X, Y = (x + PAD).astype(np.float64), (y + PAD).astype(np.float64)
    px = np.stack([X, X + L.astype(np.float64) * rho, X + d.astype(np.float64) * rho], 1)
    py = np.stack([Y, Y, Y + h.astype(np.float64) * rho], 1)
    uv = np.zeros((len(f), 3, 2), np.float32)
    r = np.arange(len(f))
    for jj in range(3):
        k = (k0 + jj) % 3
        uv[r, k, 0] = (px[:, jj] / N).astype(np.float32)
        uv[r, k, 1] = (py[:, jj] / N).astype(np.float32)
    owner = np.full((N, N), -1, np.int32)
    for i, (bx, by, bw, bh) in enumerate(boxes.tolist()):
        owner[by:by + bh, bx:bx + bw] = i
    return {"j": j, "rho": rho, "boxes": boxes, "uv": uv, "owner": owner.reshape(-1), "k0": k0}


def closest_point(p, a, b, c):
    """Barycentrics (la, lb, lc) fp64 [n] of the point of triangle abc closest to p (all [n,3] fp64): corner a, corner b,
    edge ab, corner c, edge ac, edge bc, interior, the first region that applies; zero denominators take corner a / 0."""
    p, a, b, c = (np.asarray(x, np.float64) for x in (p, a, b, c))
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = _dot(ab, ap), _dot(ac, ap)
    bp = p - b
    d3, d4 = _dot(ab, bp), _dot(ac, bp)
    vc = d1 * d4 - d3 * d2
    cp = p - c
    d5, d6 = _dot(ab, cp), _dot(ac, cp)
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    e43, e56 = d4 - d3, d5 - d6
    t_ab, t_ac, t_bc = d1 - d3, d2 - d6, e43 + e56
    den = (va + vb) + vc
    with np.errstate(divide="ignore", invalid="ignore"):
        v_ab = np.where(t_ab > 0, d1 / np.where(t_ab > 0, t_ab, 1.0), 0.0)
        w_ac = np.where(t_ac > 0, d2 / np.where(t_ac > 0, t_ac, 1.0), 0.0)
        w_bc = np.where(t_bc > 0, e43 / np.where(t_bc > 0, t_bc, 1.0), 0.0)
        v_in = vb / np.where(den > 0, den, 1.0)
        w_in = vc / np.where(den > 0, den, 1.0)
    conds = [(d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0), (d6 >= 0) & (d5 <= d6),
             (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & (e43 >= 0) & (e56 >= 0), ~(den > 0)]
    one, zero = np.ones_like(d1), np.zeros_like(d1)
    la = np.select(conds, [one, zero, 1.0 - v_ab, zero, 1.0 - w_ac, zero, one], (1.0 - v_in) - w_in)
    lb = np.select(conds, [zero, one, v_ab, zero, zero, 1.0 - w_bc, zero], v_in)
    lc = np.select(conds, [zero, zero, zero, one, w_ac, w_bc, zero], w_in)
    return la, lb, lc


def region(p, a, b, c):
    """Index of the region closest_point takes (0 a, 1 b, 2 ab, 3 c, 4 ac, 5 bc, 6 interior) -- for the tests."""
    la, lb, lc = closest_point(p, a, b, c)
    out = np.full(len(la), 6)
    out[(lc == 0) & (la > 0) & (lb > 0)] = 2
    out[(lb == 0) & (la > 0) & (lc > 0)] = 4
    out[(la == 0) & (lb > 0) & (lc > 0)] = 5
    out[la == 1] = 0
    out[lb == 1] = 1
    out[lc == 1] = 3
    return out


def blend3(la, lb, lc, A, B, C):
    la, lb, lc = (np.asarray(x, np.float64).astype(np.float32)[:, None] for x in (la, lb, lc))
    A, B, C = (np.asarray(x, np.float32) for x in (A, B, C))
    return (la * A + lb * B) + lc * C


def texel_points(verts, faces, uv, owner, N):
    """-> (texel_index [T] int32 ascending, points [T,3] fp32, texel_face [T] int32)."""
    v = np.asarray(verts, np.float32)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    owner = np.asarray(owner).reshape(-1)
    t = np.nonzero(owner >= 0)[0]
    tf = owner[t].astype(np.int64)
    k0 = base_corner(v, f)[tf]
    ka, kb, kc = k0, (k0 + 1) % 3, (k0 + 2) % 3
    uvN = np.asarray(uv, np.float32).reshape(-1, 3, 2)[tf] * np.float32(N)
    r = np.arange(len(t))

    def corner(k):
        q = uvN[r, k].astype(np.float64)
        return np.stack([q[:, 0], q[:, 1], np.zeros(len(q))], 1)

    q = np.stack([(t % N).astype(np.float64) + 0.5, (t // N).astype(np.float64) + 0.5, np.zeros(len(t))], 1)
    la, lb, lc = closest_point(q, corner(ka), corner(kb), corner(kc))
    pts = blend3(la, lb, lc, v[f[tf, ka]], v[f[tf, kb]], v[f[tf, kc]])
    return t.astype(np.int32), pts, tf.astype(np.int32)


def fill(texel_index, rgb, owner, N):
    """-> texture [N,N,3] fp32: rgb at the owned texels, push-pull everywhere else."""
    owner = np.asarray(owner).reshape(N, N)
    tex = np.zeros((N * N, 3), np.float32)
    tex[np.asarray(texel_index, np.int64)] = np.asarray(rgb, np.float32)
    tex = tex.reshape(N, N, 3)
    level = np.concatenate([tex, (owner >= 0).astype(np.float32)[..., None]], -1)
    pyramid = []
    while level.shape[0] > 1:
        ch = [level[0::2, 0::2], level[0::2, 1::2], level[1::2, 0::2], level[1::2, 1::2]]
        sw = ((ch[0][..., 3] + ch[1][..., 3]) + ch[2][..., 3]) + ch[3][..., 3]
        num = ((ch[0][..., 3:] * ch[0][..., :3] + ch[1][..., 3:] * ch[1][..., :3]) + ch[2][..., 3:] * ch[2][..., :3]) \
            + ch[3][..., 3:] * ch[3][..., :3]
        with np.errstate(divide="ignore", invalid="ignore"):
            mean = np.where(sw[..., None] > 0, num / np.where(sw > 0, sw, np.float32(1))[..., None], np.float32(0))
        level = np.concatenate([mean.astype(np.float32), sw[..., None]], -1)
        pyramid.append(level)
    for l in range(len(pyramid) - 2, -1, -1):
        lv, par = pyramid[l], pyramid[l + 1]
        up = np.repeat(np.repeat(par[..., :3], 2, 0), 2, 1)
        empty = lv[..., 3] == 0
        lv[..., :3][empty] = up[empty]
    up = np.repeat(np.repeat(pyramid[0][..., :3], 2, 0), 2, 1)
    empty = owner < 0
    tex[empty] = up[empty]
    return tex


def transfer(src_v, src_f, src_c, points, nn_index, sample_face):
    """-> rgb [n,3] fp32: the colours of src (fp32 [nv,3]) at the closest point of each point's nearest sample's face."""
    v = np.asarray(src_v, np.float32)
    f = np.asarray(src_f, np.int64).reshape(-1, 3)
    col = np.asarray(src_c, np.float32)
    face = np.asarray(sample_face, np.int64)[np.asarray(nn_index, np.int64)]
    c = f[face]
    la, lb, lc = closest_point(np.asarray(points, np.float32).astype(np.float64), v[c[:, 0]], v[c[:, 1]], v[c[:, 2]])
    return blend3(la, lb, lc, col[c[:, 0]], col[c[:, 1]], col[c[:, 2]])
