"""numpy restatement of the normal-map rules (csrc/texture.cu o2345_tangent_normals / o2345_normal_quantise /
o2345_vertex_normals, and the normal-map branch of csrc/raster.cu's resolve), bit for bit.

The reference has no texture or normal-map baking, so every rule here is this project's own definition (DESIGN §2,
parity unpinned):

  frames      per face, in fp64 from the fp32 corners P0, P1, P2 and uv rows (glTF: v down the image): e1 = P1 - P0,
              e2 = P2 - P0, (du1, dv1) = uv1 - uv0, (du2, dv2) = uv2 - uv0, det = du1 dv2 - du2 dv1,
              dp/du = (dv2 e1 - dv1 e2) / det, dp/dv = (du1 e2 - du2 e1) / det, T = dp/du / |dp/du|,
              B = -dp/dv / |dp/dv| (+Y up the image), N = e1 x e2 / |e1 x e2|;
  tangent     a world normal n in its texel's face frame: (n.T, n.B, n.N) / |n| rounded to fp32; (0, 0, 1) for det = 0
              (or not finite), a face without area, or n zero or not finite;
  quantise    v / |v| in fp32 ((0, 0, 1) when |v| is zero or not finite), each component round_half_even((c + 1) * 127.5);
  vertex n.   per vertex, the sum of its faces' (B - A) x (C - A) in ascending face order in fp64, divided by its length,
              rounded once to fp32 ((0, 0, 0) for a zero sum);
  raster      a face with a valid face_ntex, given normals and tangents: N, T = the perspective-correct interpolated
              normal and tangent xyz normalised in fp32, w = -1 where the interpolated tangent w < 0 else 1,
              B = (N x T) * w, t = 2 * bilinear sample - 1, n = normalize((t.x T + t.y B) + t.z N) times the sign that
              turns the face's normal in its own corner order toward the camera (the resolve works on slots 1 and 2
              swapped for a screen-clockwise triangle, whose normal is the opposite); a zero or non-finite length
              keeps the face normal.  n replaces the normal
              output and the Lambert term's normal; everything else is raster_oracle.render.
This module does not import the package: it is the independent statement the GPU tests compare against."""
from __future__ import annotations

import numpy as np

from . import raster_oracle as R
from .texture_oracle import _dot

F = np.float32


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _unit(a):
    """a / |a| (fp64 [n,3]) and whether |a| is a positive finite number."""
    with np.errstate(invalid="ignore", over="ignore"):
        ln = np.sqrt(_dot(a, a))
        ok = (ln > 0) & (ln < np.inf)
        return a / np.where(ok, ln, 1.0)[:, None], ok


def frames(verts, faces, uv):
    """-> T, B, N fp64 [F,3] and ok [F] (False for a degenerate face) of the tangent-frame rule."""
    v = np.asarray(verts, np.float32)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    q = np.asarray(uv, np.float32).reshape(-1, 3, 2).astype(np.float64)
    P0, P1, P2 = (v[f[:, k]].astype(np.float64) for k in range(3))
    e1, e2 = P1 - P0, P2 - P0
    du1, dv1 = q[:, 1, 0] - q[:, 0, 0], q[:, 1, 1] - q[:, 0, 1]
    du2, dv2 = q[:, 2, 0] - q[:, 0, 0], q[:, 2, 1] - q[:, 0, 1]
    det = du1 * dv2 - du2 * dv1
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        good = np.abs(det) > 0
        d = np.where(good, det, 1.0)[:, None]
        dpdu = (dv2[:, None] * e1 - dv1[:, None] * e2) / d
        dpdv = -(du1[:, None] * e2 - du2[:, None] * e1) / d
    T, okT = _unit(dpdu)
    B, okB = _unit(dpdv)
    N, okN = _unit(_cross(e1, e2))
    return T, B, N, good & okT & okB & okN


def tangent_normals(verts, faces, uv, texel_face, normals):
    """-> [n,3] fp32: normals [n,3] (fp32) in the frames of faces texel_face [n]."""
    T, B, N, ok = frames(verts, faces, uv)
    tf = np.asarray(texel_face, np.int64)
    w = np.asarray(normals, np.float32).reshape(-1, 3).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        ln = np.sqrt(_dot(w, w))
        good = ok[tf] & (ln > 0) & (ln < np.inf)
        s = np.where(good, ln, 1.0)
        t = np.stack([_dot(w, T[tf]) / s, _dot(w, B[tf]) / s, _dot(w, N[tf]) / s], 1).astype(np.float32)
    return np.where(good[:, None], t, np.array([0, 0, 1], np.float32))


def quantise_normals(texture):
    """-> uint8 [..., 3] of a fp32 texture [..., 3] of tangent-space vectors."""
    t = np.asarray(texture, np.float32)
    shape = t.shape
    t = t.reshape(-1, 3)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        ln = np.sqrt((t[:, 0] * t[:, 0] + t[:, 1] * t[:, 1]) + t[:, 2] * t[:, 2])
        ok = (ln > 0) & (ln < np.inf)
        c = np.where(ok[:, None], t / np.where(ok, ln, np.float32(1))[:, None], np.array([0, 0, 1], np.float32))
    code = np.rint((c.astype(np.float32) + np.float32(1)) * np.float32(127.5))
    return np.clip(code, 0, 255).astype(np.uint8).reshape(shape)


def vertex_normals(verts, faces):
    """-> [nv,3] fp32 unit vertex normals."""
    v = np.asarray(verts, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    fn = _cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    corner_v = f.reshape(-1)
    corner_f = np.repeat(np.arange(len(f)), 3)
    order = np.lexsort((corner_f, corner_v))            # by vertex, then face ascending
    cv, cf = corner_v[order], corner_f[order]
    start = np.searchsorted(cv, np.arange(len(v)))
    rank = np.arange(len(cv)) - start[cv]
    s = np.zeros((len(v), 3))
    for k in range(int(rank.max()) + 1 if len(rank) else 0):
        sel = rank == k
        s[cv[sel]] = s[cv[sel]] + fn[cf[sel]]
    n, ok = _unit(s)
    return np.where(ok[:, None], n, 0.0).astype(np.float32)


def _normalize32(v):
    """v / |v| in fp32 per row and whether |v| is a positive finite number."""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        ln = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
        ok = (ln > 0) & (ln < np.inf)
        return v / np.where(ok, ln, F(1.0))[:, None], ok


def render(verts, faces, w2c, intr, W, H, near=0.1, shading=R.SHADE_UNLIT, colors=None, uvs=None, face_tex=None,
           texels=None, tex_info=None, normals=None, tangents=None, face_ntex=None):
    """Same inputs and outputs as o2345.ops.raster (with the normal-map fields), as numpy arrays."""
    out = R.render(verts, faces, w2c, intr, W, H, near, R.SHADE_UNLIT, colors, uvs, face_tex, texels, tex_info)
    verts = np.asarray(verts, F).reshape(-1, 3)
    w2c = np.asarray(w2c, F).reshape(-1, 3, 4)
    intr = np.asarray(intr, F).reshape(-1, 4)
    mapped = face_ntex is not None and normals is not None and tangents is not None
    for v in range(len(w2c) if mapped else 0):
        X, Y, zc = R.project(verts, w2c[v], intr[v], near)
        T, _ = R.setup(faces, X, Y, zc)
        pix = np.nonzero(out["tri"][v].reshape(-1) >= 0)[0]
        t = out["tri"][v].reshape(-1)[pix].astype(np.int64)
        w, _ = R.weights(T, t, pix % W, pix // W)
        b, iz, _ = R.depth(T, t, w)
        p = (b * T["r"][t]) / iz[:, None]
        idx = T["idx"][t]
        interp = lambda a: (p[:, 0] * a[idx[:, 0]] + p[:, 1] * a[idx[:, 1]]) + p[:, 2] * a[idx[:, 2]]
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
        s = np.where(idx[:, 1] == np.asarray(faces, np.int64).reshape(-1, 3)[t, 1], s, -s)   # the face's own winding
        info = np.asarray(tex_info, np.int64).reshape(-1, 5)
        uv = np.asarray(uvs, F).reshape(-1, 2)
        u, vv = interp(uv[:, 0]), interp(uv[:, 1])
        fn = np.asarray(face_ntex, np.int64)[t]
        nv_, tg = np.asarray(normals, F).reshape(-1, 3), np.asarray(tangents, F).reshape(-1, 4)
        Nn, okN = _normalize32(np.stack([interp(nv_[:, c]) for c in range(3)], 1))
        Tt, okT = _normalize32(np.stack([interp(tg[:, c]) for c in range(3)], 1))
        sw = np.where(interp(tg[:, 3]) < 0, F(-1.0), F(1.0))
        B = np.stack([(Nn[:, 1] * Tt[:, 2] - Nn[:, 2] * Tt[:, 1]) * sw, (Nn[:, 2] * Tt[:, 0] - Nn[:, 0] * Tt[:, 2]) * sw,
                      (Nn[:, 0] * Tt[:, 1] - Nn[:, 1] * Tt[:, 0]) * sw], 1)
        tt = np.zeros((len(t), 3), F)
        for ti in range(len(info)):
            sel = fn == ti
            if sel.any():
                tt[sel] = F(2.0) * R.sample_texture(texels, info[ti], u[sel], vv[sel]) - F(1.0)
        m, okm = _normalize32((tt[:, 0:1] * Tt + tt[:, 1:2] * B) + tt[:, 2:3] * Nn)
        use = (fn >= 0) & (fn < len(info)) & (ln > 0) & okN & okT & okm
        nrm = out["normal"][v].reshape(-1, 3)
        nrm[pix[use]] = (s[use, None] * m[use]).astype(F)
    if shading == R.SHADE_LAMBERT:
        out["color"] = (out["color"] * (F(0.4) + F(0.6) * np.maximum(out["normal"][..., 2], F(0.0)))[..., None]).astype(F)
    return out
