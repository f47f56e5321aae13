"""numpy restatement of ambient occlusion (csrc/ao.cu, include/o2345.h `o2345_ambient_occlusion`), rule for rule.

The direction table, the tangent frame, the padded box test and the watertight ray-triangle test are numpy float32 /
float64 operations in the kernel's order (numpy rounds each one to nearest and never contracts a multiply and an add into
an FMA), and every ray is tested against every face whose padded box is within reach, so the result is bit-identical to
the kernel's LBVH search.  This module does not import the package: it is the independent statement the GPU tests
compare against."""
from __future__ import annotations

import numpy as np

F, D = np.float32, np.float64
RAYS = 256                  # directions per point (mesh_texture.AO_RAYS)
T_MIN, T_MAX = 1e-3, 0.1    # segment ends as fractions of the box diagonal (mesh_texture.AO_T_MIN, AO_T_MAX)
PAD_SCALE = F(2.0 ** -13)   # face boxes grow by this times the diagonal (csrc/ao.cu kPadScale)
CHUNK = 4096                # faces per vectorised block (memory only: the result does not depend on it)


def directions(k=RAYS):
    """The golden-angle spiral on the unit disk lifted to the hemisphere (Malley): d = (r cos phi, r sin phi,
    sqrt(1 - r^2)), r = sqrt((i + 1/2) / k), phi = i pi (3 - sqrt 5), in fp64, rounded once -> float32 [k,3]."""
    i = np.arange(k, dtype=D)
    r2 = (i + 0.5) / k
    r, phi = np.sqrt(r2), i * (np.pi * (3.0 - np.sqrt(5.0)))
    return np.stack([r * np.cos(phi), r * np.sin(phi), np.sqrt(1.0 - r2)], 1).astype(F)


def diagonal(verts):
    """The diagonal of the box of the vertices, sqrt((dx dx + dy dy) + dz dz) in fp64 (0 without vertices)."""
    v = np.asarray(verts, F).reshape(-1, 3)
    if len(v) == 0:
        return D(0.0)
    e = v.max(0).astype(D) - v.min(0).astype(D)
    return np.sqrt((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2])


def distances(verts):
    """(t_min, t_max) float32: T_MIN and T_MAX times the diagonal in fp64, each rounded once."""
    d = diagonal(verts)
    return F(D(T_MIN) * d), F(D(T_MAX) * d)


def frame(normal):
    """(ok, T, B, u) of one normal: Duff et al. 2017 in float32 (ok False for a zero or non-finite length)."""
    nx, ny, nz = (F(c) for c in normal)
    with np.errstate(all="ignore"):
        ln = np.sqrt((nx * nx + ny * ny) + nz * nz)
        if not (ln > 0 and ln <= np.finfo(F).max):
            return False, None, None, None
        ux, uy, uz = nx / ln, ny / ln, nz / ln
        s = np.copysign(F(1), uz)
        a = F(-1) / (s + uz)
        b = (ux * uy) * a
        T = np.array([F(1) + ((s * ux) * ux) * a, s * b, -(s * ux)], F)
        B = np.array([b, s + (uy * uy) * a, -uy], F)
    return True, T, B, np.array([ux, uy, uz], F)


def rays(T, B, u, dirs):
    """w [k,3] = (d.x T + d.y B) + d.z u per component, float32."""
    d = np.asarray(dirs, F).reshape(-1, 3)
    return (d[:, :1] * T[None] + d[:, 1:2] * B[None]) + d[:, 2:3] * u[None]


def face_boxes(verts, faces, pad):
    """Corners [m,3,3] float32 and the padded boxes lo, hi [m,3] (min - pad, max + pad, rounded)."""
    c = np.asarray(verts, F).reshape(-1, 3)[np.asarray(faces, np.int64).reshape(-1, 3)]
    return c, c.min(1) - F(pad), c.max(1) + F(pad)


def any_hit(p, w, corners, lo, hi, t_min, t_max):
    """bool [k]: ray k (origin p [3], direction w [k,3], float32) hits one of the faces (corners [m,3,3], padded boxes lo, hi
    [m,3]) on [t_min, t_max]: the box test and the watertight test of the header."""
    p, w = np.asarray(p, F), np.asarray(w, F)
    t_min, t_max = F(t_min), F(t_max)
    k = len(w)
    hit = np.zeros(k, bool)
    with np.errstate(all="ignore"):
        inv = F(1) / w
        fin = np.isfinite(inv)
        kz = np.where(np.abs(w[:, 1]) > np.abs(w[:, 0]), 1, 0)
        kz = np.where(np.abs(w[:, 2]) > np.abs(w[np.arange(k), kz]), 2, kz)
        kx, ky = (kz + 1) % 3, (kz + 2) % 3
        neg = w[np.arange(k), kz] < 0
        kx, ky = np.where(neg, ky, kx), np.where(neg, kx, ky)
        wz = w[np.arange(k), kz]
        Sx, Sy, Sz = w[np.arange(k), kx] / wz, w[np.arange(k), ky] / wz, F(1) / wz
        for a in range(0, len(corners), CHUNK):
            c, l, h = corners[a:a + CHUNK], lo[a:a + CHUNK], hi[a:a + CHUNK]
            # box test on [0, t_max]
            tn = np.zeros((k, len(c)), F)
            tf = np.full((k, len(c)), t_max, F)
            ok = np.ones((k, len(c)), bool)
            for ax in range(3):
                t1 = (l[None, :, ax] - p[ax]) * inv[:, None, ax]
                t2 = (h[None, :, ax] - p[ax]) * inv[:, None, ax]
                f = fin[:, None, ax]
                tn = np.where(f, np.maximum(tn, np.minimum(t1, t2)), tn)
                tf = np.where(f, np.minimum(tf, np.maximum(t1, t2)), tf)
                inside = ((l[:, ax] <= p[ax]) & (p[ax] <= h[:, ax]))[None, :]
                ok &= f | inside
            ok &= tn <= tf
            # watertight test
            P = c - p[None, None, :]                                     # [m,3,3]
            z = [P[:, j, :][:, kz].T for j in range(3)]                  # [k,m]
            x = [P[:, j, :][:, kx].T - Sx[:, None] * z[j] for j in range(3)]
            y = [P[:, j, :][:, ky].T - Sy[:, None] * z[j] for j in range(3)]
            U = x[2] * y[1] - y[2] * x[1]
            V = x[0] * y[2] - y[0] * x[2]
            W = x[1] * y[0] - y[1] * x[0]
            zero = (U == 0) | (V == 0) | (W == 0)
            if zero.any():
                e64 = lambda a1, b1, a2, b2: (a1.astype(D) * b1.astype(D) - a2.astype(D) * b2.astype(D)).astype(F)
                U = np.where(zero, e64(x[2], y[1], y[2], x[1]), U)
                V = np.where(zero, e64(x[0], y[2], y[0], x[2]), V)
                W = np.where(zero, e64(x[1], y[0], y[1], x[0]), W)
            mixed = ((U < 0) | (V < 0) | (W < 0)) & ((U > 0) | (V > 0) | (W > 0))
            det = (U + V) + W
            T = (U * (Sz[:, None] * z[0]) + V * (Sz[:, None] * z[1])) + W * (Sz[:, None] * z[2])
            T = np.where(det < 0, -T, T)
            det = np.where(det < 0, -det, det)
            got = ok & ~mixed & (det != 0) & (t_min * det <= T) & (T <= t_max * det)
            hit |= got.any(1)
    return hit


def ambient_occlusion(verts, faces, points, normals, dirs=None, t_min=None, t_max=None):
    """AO float32 [n] of points [n,3] with normals [n,3] against the mesh verts [nv,3], faces [nf,3]: the share of the
    directions (default: directions()) whose segment [t_min, t_max] (default: distances(verts)) hits no face.  A face
    is only tested when its padded box lies within 1.01 |w| t_max of the point: farther, the box test cannot pass, whose
    rounded slab parameters are within a few units in the last place of the exact ones."""
    v = np.asarray(verts, F).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    pts, nrm = np.asarray(points, F).reshape(-1, 3), np.asarray(normals, F).reshape(-1, 3)
    dirs = directions() if dirs is None else np.asarray(dirs, F).reshape(-1, 3)
    dt = distances(v)
    t_min = dt[0] if t_min is None else F(t_min)
    t_max = dt[1] if t_max is None else F(t_max)
    pad = F(F(diagonal(v)) * PAD_SCALE)
    corners, lo, hi = face_boxes(v, f, pad)
    out = np.ones(len(pts), F)
    for i, (p, n) in enumerate(zip(pts, nrm)):
        ok, T, B, u = frame(n)
        if not ok or not np.isfinite(p).all() or len(f) == 0:
            continue
        w = rays(T, B, u, dirs)
        reach = 1.01 * float(t_max) * float(np.sqrt((w.astype(D) ** 2).sum(1)).max())
        gap = np.maximum(np.maximum(lo.astype(D) - p, p - hi.astype(D)), 0.0)
        near = np.sqrt((gap * gap).sum(1)) <= reach
        misses = (~any_hit(p, w, corners[near], lo[near], hi[near], t_min, t_max)).sum()
        out[i] = F(misses) / F(len(dirs))
    return out
