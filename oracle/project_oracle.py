"""numpy restatement of the input-view projection (csrc/project.cu, include/o2345.h `o2345_project_view` and
`o2345_face_normals`), rule for rule.

Every float operation of the projection is a float32 numpy operation in the kernel's order (numpy rounds each one to
nearest and never contracts a multiply and an add into an FMA), so the weights and colours come out bit-identical to the
kernel's; the face normals are fp64 and rounded once, as the kernel's.  The depth buffer is an input: the rasterizer that
makes it is pinned to oracle/raster_oracle.py.
This module does not import the package: it is the independent statement the GPU tests compare against."""
from __future__ import annotations

import numpy as np

F = np.float32
COS_LO, COS_HI, TAU_PIX = F(0.3), F(0.7), F(2.0)
FLT_MAX = np.finfo(np.float32).max


def face_normals(verts, faces, face_index):
    """Unit normals [n,3] fp32 of faces face_index: (B - A) x (C - A) in fp64 / its length, rounded once; (0, 0, 0) for
    an index out of range or a face without area."""
    v = np.asarray(verts, np.float32).astype(np.float64).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    fi = np.asarray(face_index, np.int64)
    ok = (fi >= 0) & (fi < len(f))
    c = f[np.where(ok, fi, 0)]
    ok &= ((c >= 0) & (c < len(v))).all(1)
    c = np.where(ok[:, None], c, 0)
    a, b, d = v[c[:, 0]], v[c[:, 1]], v[c[:, 2]]
    e1, e2 = b - a, d - a
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
        ok &= (ln > 0) & (ln < np.inf)
        out = n / np.where(ok, ln, 1.0)[:, None]
    return np.where(ok[:, None], out, 0.0).astype(np.float32)


def bilinear(img, x, y):
    """Bilinear sample [n, C] of uint8 img [H, W, C] at (x, y) inside [0, W-1] x [0, H-1], in byte units: taps nw, ne, sw,
    se summed in that order; a tap past the last column or row has weight 0 and reads the last one."""
    img = np.asarray(img)
    H, W = img.shape[:2]
    img = img.reshape(H, W, -1).astype(F)
    x0, y0 = np.floor(x), np.floor(y)
    x1, y1 = x0 + F(1), y0 + F(1)
    wnw, wne = ((x1 - x) * (y1 - y))[:, None], ((x - x0) * (y1 - y))[:, None]
    wsw, wse = ((x1 - x) * (y - y0))[:, None], ((x - x0) * (y - y0))[:, None]
    ix, iy = x0.astype(np.int64), y0.astype(np.int64)
    jx, jy = np.minimum(ix + 1, W - 1), np.minimum(iy + 1, H - 1)
    acc = img[iy, ix] * wnw
    acc = acc + img[iy, jx] * wne
    acc = acc + img[jy, ix] * wsw
    return acc + img[jy, jx] * wse


def project_view(points, normals, base, w2c, intr, photo, alpha, depth, near=0.1):
    """-> (colours [T,3], weight [T]) fp32 of o2345_project_view; depth [s H, s W] (its scale s = width / W)."""
    p = np.asarray(points, F).reshape(-1, 3)
    nrm = np.asarray(normals, F).reshape(-1, 3)
    b = np.asarray(base, F).reshape(-1, 3)
    M = np.asarray(w2c, F).reshape(-1, 4)[:3]
    fx, fy, cx, cy = (F(v) for v in intr)
    photo = np.asarray(photo, np.uint8)
    H, W = photo.shape[:2]
    depth = np.asarray(depth, F)
    s = depth.shape[1] // W
    assert depth.shape == (s * H, s * W) and s >= 1
    w = np.zeros(len(p), F)
    x = np.zeros(len(p), F)
    y = np.zeros(len(p), F)
    with np.errstate(all="ignore"):
        q = [((M[r, 0] * p[:, 0] + M[r, 1] * p[:, 1]) + M[r, 2] * p[:, 2]) + M[r, 3] for r in range(3)]
        xs = (fx * q[0]) / q[2] + cx
        ys = (fy * q[1]) / q[2] + cy
        nl = np.sqrt((nrm[:, 0] * nrm[:, 0] + nrm[:, 1] * nrm[:, 1]) + nrm[:, 2] * nrm[:, 2])
        m = (q[2] > F(near)) & (q[2] <= FLT_MAX)
        x[m], y[m] = xs[m], ys[m]
        m &= (xs >= 0) & (xs <= F(W - 1)) & (ys >= 0) & (ys <= F(H - 1)) & (nl > 0) & (nl <= FLT_MAX)
        c = [-((M[0, k] * M[0, 3] + M[1, k] * M[1, 3]) + M[2, k] * M[2, 3]) for k in range(3)]
        d = [c[k] - p[:, k] for k in range(3)]
        dl = np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
        cs = ((nrm[:, 0] / nl) * (d[0] / dl) + (nrm[:, 1] / nl) * (d[1] / dl)) + (nrm[:, 2] / nl) * (d[2] / dl)
        t = (cs - COS_LO) / (COS_HI - COS_LO)
        wa = np.where(t > 0, np.where(t < 1, t, F(1)), F(0)).astype(F)
        m &= wa > 0
        i = np.nonzero(m)[0]
        j = np.minimum(np.floor(F(s) * (x[i] + F(0.5))).astype(np.int64), s * W - 1)
        k = np.minimum(np.floor(F(s) * (y[i] + F(0.5))).astype(np.int64), s * H - 1)
        D = depth[k, j]
        tau = ((TAU_PIX * q[2][i]) / (F(s) * fx)) / np.maximum(cs[i], COS_LO)
        seen = (D <= 0) | ((q[2][i] - D) <= tau)
        i = i[seen]
        a = F(1) if alpha is None else np.minimum(bilinear(alpha, x[i], y[i])[:, 0] / F(255), F(1))
        w[i] = wa[i] * a
    out = b.copy()
    i = np.nonzero(w > 0)[0]
    photo_rgb = bilinear(photo, x[i], y[i]) / F(255)
    out[i] = b[i] + w[i, None] * (photo_rgb - b[i])
    return out.astype(F), w
