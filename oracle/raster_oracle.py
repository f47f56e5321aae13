"""numpy restatement of the mesh rasterizer (csrc/raster.cu, include/o2345.h `o2345_raster`), rule for rule.

Every float operation is a float32 numpy operation in the kernel's order: numpy rounds each one to nearest and never
contracts a multiply and an add into an FMA, so the projection, the snapped fixed-point coordinates, the depth keys and
hence the winning triangle ids come out bit-identical to the kernel's.  The kernel's rules:
  * camera space c_r = ((M[r,0] x + M[r,1] y) + M[r,2] z) + M[r,3]; pixel x = (fx c_x / c_z + cx) * 256 rounded to the
    nearest integer, ties to even (8 subpixel bits); a vertex with c_z <= near or |x|, |y| >= 2^29 (fixed) is invalid;
  * a triangle with an invalid vertex, an index outside [0, nv) or zero area is dropped; a clockwise one has its slots 1
    and 2 swapped; pixel (i, j) is sampled at fixed (256 i + 128, 256 j + 128); int64 edge functions with the top-left
    rule (an edge owns the samples on it iff dy < 0, or dy == 0 and dx > 0);
  * b_k = w_k / area, 1/z = (b0 / z0 + b1 / z1) + b2 / z2, z = 1 / (1/z); the key (bits of z) << 32 | id is minimised;
  * resolve: p_k = b_k / z_k / (1/z) interpolates colour and uv; the texture is sampled bilinearly (texel centres at
    (i + 0.5) / w); the normal is the unit world face normal turned toward the camera centre -R^T t.
This module does not import the package: it is the independent statement the GPU tests compare against."""
from __future__ import annotations

import numpy as np

F = np.float32
SUB = 256
MAX_FIXED = F(536870912.0)
INVALID = np.iinfo(np.int32).min
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
SHADE_UNLIT, SHADE_LAMBERT = 0, 1


def project(verts, w2c, intr, near):
    """One view: fixed-point (X, Y) int64 [nv] (INVALID where the vertex is dropped) and camera z float32 [nv]."""
    p = np.asarray(verts, F)
    M = np.asarray(w2c, F).reshape(3, 4)
    K = np.asarray(intr, F).reshape(4)
    c = [((M[r, 0] * p[:, 0] + M[r, 1] * p[:, 1]) + M[r, 2] * p[:, 2]) + M[r, 3] for r in range(3)]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        sx = ((K[0] * c[0]) / c[2] + K[2]) * F(SUB)
        sy = ((K[1] * c[1]) / c[2] + K[3]) * F(SUB)
        ok = (c[2] > F(near)) & (np.abs(sx) < MAX_FIXED) & (np.abs(sy) < MAX_FIXED)
    X = np.where(ok, np.rint(np.where(ok, sx, 0)).astype(np.int64), INVALID)
    Y = np.where(ok, np.rint(np.where(ok, sy, 0)).astype(np.int64), INVALID)
    return X, Y, c[2].astype(F)


def setup(faces, X, Y, zc):
    """Triangle setup of one view -> dict of per-triangle slot arrays (x, y [nf,3] int64, r [nf,3], idx [nf,3], area) and
    the mask of kept triangles."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    nv = len(X)
    inb = ((f >= 0) & (f < nv)).all(1)
    fi = np.where(inb[:, None], f, 0)
    x, y = X[fi], Y[fi]
    with np.errstate(divide="ignore"):
        r = F(1.0) / zc[fi]
    ok = inb & (x != INVALID).all(1)
    area = (x[:, 1] - x[:, 0]) * (y[:, 2] - y[:, 0]) - (y[:, 1] - y[:, 0]) * (x[:, 2] - x[:, 0])
    ok &= area != 0
    sw = area < 0
    for a in (x, y, r, fi):
        a[sw, 1], a[sw, 2] = a[sw, 2].copy(), a[sw, 1].copy()
    return {"x": x, "y": y, "r": r, "idx": fi, "area": np.abs(area)}, ok


def _edge(xa, ya, xb, yb, sx, sy):
    return (xb - xa) * (sy - ya) - (yb - ya) * (sx - xa)


def _owns(w, xa, ya, xb, yb):
    dy, dx = yb - ya, xb - xa
    return (w > 0) | ((w == 0) & ((dy < 0) | ((dy == 0) & (dx > 0))))


def weights(T, t, px, py):
    """Edge functions w [n,3] of triangles t at pixels (px, py) and whether each pixel centre is covered."""
    x, y = T["x"][t], T["y"][t]
    sx, sy = px.astype(np.int64) * SUB + SUB // 2, py.astype(np.int64) * SUB + SUB // 2
    w, cov = [], np.ones(len(t), bool)
    for k, (a, b) in enumerate(((1, 2), (2, 0), (0, 1))):
        wk = _edge(x[:, a], y[:, a], x[:, b], y[:, b], sx, sy)
        cov &= _owns(wk, x[:, a], y[:, a], x[:, b], y[:, b])
        w.append(wk)
    return np.stack(w, 1), cov


def _to_f32(i64):
    assert np.all(np.abs(i64) < 2 ** 53), "edge function beyond 2^53: float64 would not hold it exactly"
    return i64.astype(np.float64).astype(F)   # exact to float64, then one rounding to float32 (= __ll2float_rn)


def depth(T, t, w):
    """Screen barycentrics b [n,3], 1/z and z (float32) in the kernel's order."""
    fa = _to_f32(T["area"][t])
    b = _to_f32(w) / fa[:, None]
    r = T["r"][t]
    iz = (b[:, 0] * r[:, 0] + b[:, 1] * r[:, 1]) + b[:, 2] * r[:, 2]
    return b, iz, F(1.0) / iz


def _span(a, b, n):
    lo = np.maximum((a - SUB // 2 + SUB - 1) >> 8, 0)
    hi = np.minimum((b - SUB // 2) >> 8, n - 1)
    return lo, hi


def fragments(T, ok, W, H):
    """Every covered (triangle, pixel) pair of one view -> (t, px, py, key)."""
    tk = np.nonzero(ok)[0]
    x0, x1 = _span(T["x"][tk].min(1), T["x"][tk].max(1), W)
    y0, y1 = _span(T["y"][tk].min(1), T["y"][tk].max(1), H)
    nx, ny = np.maximum(x1 - x0 + 1, 0), np.maximum(y1 - y0 + 1, 0)
    cnt = nx * ny
    tot = int(cnt.sum())
    start = np.repeat(np.cumsum(cnt) - cnt, cnt)
    rep = np.repeat(np.arange(len(tk)), cnt)
    k = np.arange(tot, dtype=np.int64) - start
    t = tk[rep]
    px, py = x0[rep] + k % nx[rep], y0[rep] + k // nx[rep]
    w, cov = weights(T, t, px, py)
    t, px, py, w = t[cov], px[cov], py[cov], w[cov]
    _, _, z = depth(T, t, w)
    key = (z.view(np.uint32).astype(np.uint64) << np.uint64(32)) | t.astype(np.uint64)
    return t, px, py, key


def coverage(verts, faces, w2c, intr, W, H, near=0.1):
    """How many triangles cover each pixel centre -> int [V,H,W] (tests of the fill rule)."""
    w2c = np.asarray(w2c, F).reshape(-1, 3, 4)
    out = np.zeros((len(w2c), H, W), np.int64)
    for v in range(len(w2c)):
        X, Y, zc = project(verts, w2c[v], np.asarray(intr, F).reshape(-1, 4)[v], near)
        T, ok = setup(faces, X, Y, zc)
        _, px, py, _ = fragments(T, ok, W, H)
        np.add.at(out[v], (py, px), 1)
    return out


def _wrap(i, n, mode):
    if mode == 1:
        return np.clip(i, 0, n - 1)
    if mode == 2:
        m = np.mod(i, 2 * n)
        return np.where(m < n, m, 2 * n - 1 - m)
    return np.mod(i, n)


def _lerp(a, b, t):
    return a * (F(1.0) - t) + b * t


def sample_texture(texels, info, u, v):
    base, w, h, ws, wt = (int(q) for q in info)
    fx = np.clip(u * F(w) - F(0.5), F(-16777216.0), F(16777216.0))
    fy = np.clip(v * F(h) - F(0.5), F(-16777216.0), F(16777216.0))
    flx, fly = np.floor(fx), np.floor(fy)
    ax, ay = fx - flx, fy - fly
    ix, iy = flx.astype(np.int64), fly.astype(np.int64)
    xa, xb, ya, yb = _wrap(ix, w, ws), _wrap(ix + 1, w, ws), _wrap(iy, h, wt), _wrap(iy + 1, h, wt)
    tex = np.asarray(texels, np.uint8).reshape(-1, 4)
    g = lambda yy, xx: tex[base + yy * w + xx, :3].astype(F) / F(255.0)
    top = _lerp(g(ya, xa), g(ya, xb), ax[:, None])
    bot = _lerp(g(yb, xa), g(yb, xb), ax[:, None])
    return _lerp(top, bot, ay[:, None])


def render(verts, faces, w2c, intr, W, H, near=0.1, shading=SHADE_UNLIT, colors=None, uvs=None, face_tex=None, texels=None,
           tex_info=None):
    """Same inputs and outputs as o2345.ops.raster, as numpy arrays."""
    verts = np.asarray(verts, F).reshape(-1, 3)
    w2c = np.asarray(w2c, F).reshape(-1, 3, 4)
    intr = np.asarray(intr, F).reshape(-1, 4)
    V = len(w2c)
    out = {"color": np.zeros((V, H, W, 3), F), "alpha": np.zeros((V, H, W), F), "depth": np.zeros((V, H, W), F),
           "normal": np.zeros((V, H, W, 3), F), "tri": np.full((V, H, W), -1, np.int32)}
    for v in range(V):
        X, Y, zc = project(verts, w2c[v], intr[v], near)
        T, ok = setup(faces, X, Y, zc)
        t, px, py, key = fragments(T, ok, W, H)
        kb = np.full(H * W, EMPTY, np.uint64)
        np.minimum.at(kb, py * W + px, key)
        pix = np.nonzero(kb != EMPTY)[0]
        kk = kb[pix]
        t = (kk & np.uint64(0xFFFFFFFF)).astype(np.int64)
        py, px = pix // W, pix % W
        w, _ = weights(T, t, px, py)
        b, iz, _ = depth(T, t, w)
        p = (b * T["r"][t]) / iz[:, None]
        idx = T["idx"][t]
        interp = lambda a: (p[:, 0] * a[idx[:, 0]] + p[:, 1] * a[idx[:, 1]]) + p[:, 2] * a[idx[:, 2]]
        if colors is not None:
            col = np.stack([interp(np.asarray(colors, F).reshape(-1, 3)[:, c]) for c in range(3)], 1)
        else:
            col = np.ones((len(t), 3), F)
        if face_tex is not None:
            ft = np.asarray(face_tex, np.int64)[t]
            info = np.asarray(tex_info, np.int64).reshape(-1, 5)
            uv = np.asarray(uvs, F).reshape(-1, 2)
            u, vv = interp(uv[:, 0]), interp(uv[:, 1])
            for ti in range(len(info)):
                sel = ft == ti
                if sel.any():
                    col[sel] = col[sel] * sample_texture(texels, info[ti], u[sel], vv[sel])
        P = [verts[idx[:, k]] for k in range(3)]
        e1, e2 = P[1] - P[0], P[2] - P[0]
        n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                      e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
        ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
        M = w2c[v]
        face = np.zeros(len(t), F)
        for c in range(3):
            cc = -((M[0, c] * M[0, 3] + M[1, c] * M[1, 3]) + M[2, c] * M[2, 3])
            face = face + n[:, c] * (cc - P[0][:, c])
        s = np.where(face < 0, F(-1.0), F(1.0))
        with np.errstate(divide="ignore", invalid="ignore"):
            nrm = np.where(ln[:, None] > 0, (s[:, None] * n) / ln[:, None], F(0.0)).astype(F)
        if shading == SHADE_LAMBERT:
            col = col * (F(0.4) + F(0.6) * np.maximum(nrm[:, 2], F(0.0)))[:, None]
        out["color"][v].reshape(-1, 3)[pix] = col
        out["normal"][v].reshape(-1, 3)[pix] = nrm
        out["alpha"][v].reshape(-1)[pix] = 1.0
        out["depth"][v].reshape(-1)[pix] = (kk >> np.uint64(32)).astype(np.uint32).view(F)
        out["tri"][v].reshape(-1)[pix] = t
    return out
