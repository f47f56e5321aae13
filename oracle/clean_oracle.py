"""numpy restatement of mesh cleaning (csrc/clean.cu, include/o2345.h `o2345_clean_mesh`), rule for rule.

Components follow shared vertex indices and are numbered by their least face; areas and winding numbers are fp64 numpy
operations in the kernel's order (numpy rounds each one to nearest and never contracts a multiply and an add into an FMA)
and summed in the kernel's fixed order, so every output comes out bit-identical to the kernel's.
This module does not import the package: it is the independent statement the GPU tests compare against."""
from __future__ import annotations

import numpy as np

D = np.float64
CHUNK = 1024                                   # terms per sequential chunk of an ordered sum (kSumChunk)
ATAN_C = [D(1.0) / D(2 * k + 1) for k in range(12)]
PI, HALF_PI = D(3.141592653589793), D(1.5707963267948966)


def vertex_roots(nv, faces):
    """Each vertex's root: the least vertex index of its set, the sets joined along face edges (hooking and pointer
    jumping until no face has two roots)."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    p = np.arange(nv, dtype=np.int64)
    while True:
        r = p[f]
        m = r.min(axis=1)
        if (r == m[:, None]).all():
            return p
        for k in range(3):
            np.minimum.at(p, r[:, k], m)       # the root of each corner hooks under the face's least root
        while True:
            q = p[p]
            if (q == p).all():
                break
            p = q


def components(nv, faces):
    """-> (label [nf]: each face's component, heads [nc]: each component's least face, ascending)."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    root = vertex_roots(nv, f)[f[:, 0]]
    least = np.full(nv, len(f), np.int64)
    np.minimum.at(least, root, np.arange(len(f)))
    head = least[root]
    heads = np.unique(head)
    return np.searchsorted(heads, head), heads


def face_areas(verts, faces):
    """0.5 sqrt(n . n), n = (B - A) x (C - A) in fp64 from the fp32 positions."""
    v = np.asarray(verts, np.float32).astype(D).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    e1, e2 = b - a, c - a
    n = cross(e1, e2)
    return D(0.5) * np.sqrt(dot(n, n))


def dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def cross(u, v):
    return np.stack([u[..., 1] * v[..., 2] - u[..., 2] * v[..., 1], u[..., 2] * v[..., 0] - u[..., 0] * v[..., 2],
                     u[..., 0] * v[..., 1] - u[..., 1] * v[..., 0]], axis=-1)


def ordered_sum(x):
    """Sequential inside chunks of CHUNK consecutive terms, then sequential over the chunk totals, each from +0.0."""
    x = np.asarray(x, D)
    if len(x) == 0:
        return D(0.0)
    pad = np.zeros(-len(x) % CHUNK, D)
    chunks = np.concatenate([x, pad]).reshape(-1, CHUNK)
    tot = np.add.accumulate(np.concatenate([np.zeros((len(chunks), 1), D), chunks], axis=1), axis=1)[:, -1]
    return np.add.accumulate(np.concatenate([np.zeros(1, D), tot]))[-1]


def atan2(y, x):
    """The kernel's atan2 (0 for y = x = 0): t = min / max of |x|, |y|, halved twice by t / (1 + sqrt(1 + t^2)), the
    Taylor series to u^23 in Horner form, times 4, then the octant."""
    y, x = np.asarray(y, D), np.asarray(x, D)
    ax, ay = np.abs(x), np.abs(y)
    zero = (ax == 0) & (ay == 0)
    swap = ay > ax
    with np.errstate(divide="ignore", invalid="ignore"):
        u = np.where(swap, ax / np.where(swap, ay, 1.0), ay / np.where(swap | zero, 1.0, ax))
    u = np.where(zero, 0.0, u)
    for _ in range(2):
        u = u / (D(1.0) + np.sqrt(D(1.0) + u * u))
    u2 = u * u
    p = np.full_like(u, ATAN_C[11])
    for k in range(10, -1, -1):
        p = ATAN_C[k] - u2 * p
    r = D(4.0) * (u * p)
    r = np.where(swap, HALF_PI - r, r)
    r = np.where(x < 0, PI - r, r)
    r = np.where(y < 0, -r, r)
    return np.where(zero, 0.0, r)


def solid_angles(tri, p):
    """2 atan2(a . (b x c), ((|a||b|)|c| + (a . b)|c| + (a . c)|b|) + (b . c)|a|) of triangles tri [m,3,3] fp64 at p."""
    a, b, c = tri[:, 0] - p, tri[:, 1] - p, tri[:, 2] - p
    la, lb, lc = np.sqrt(dot(a, a)), np.sqrt(dot(b, b)), np.sqrt(dot(c, c))
    det = dot(a, cross(b, c))
    den = ((la * lb) * lc + dot(a, b) * lc) + dot(a, c) * lb
    den = den + dot(b, c) * la
    return D(2.0) * atan2(det, den)


def winding_number(verts, faces, point):
    """(ordered sum of the solid angles of faces, in their order, at point) / (4 pi)."""
    v = np.asarray(verts, np.float32).astype(D).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    return ordered_sum(solid_angles(v[f], np.asarray(point, D))) / (D(4.0) * PI)


def centroid(verts, face):
    v = np.asarray(verts, np.float32).astype(D).reshape(-1, 3)
    a, b, c = v[np.asarray(face, np.int64)]
    return ((a + b) + c) / D(3.0)


def clean_mesh(verts, faces, min_component):
    """-> dict(label, area, winding, keep, largest, enclosed, vertex_index, faces) of o2345_clean_mesh."""
    v = np.asarray(verts, np.float32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    F = D(min_component)
    assert 0.0 < F <= 1.0
    label, heads = components(len(v), f)
    nc = len(heads)
    fa = face_areas(v, f)
    order = np.argsort(label, kind="stable")                                 # by component, ascending faces inside
    off = np.concatenate([[0], np.cumsum(np.bincount(label, minlength=nc))])
    area = np.array([ordered_sum(fa[order[off[c]:off[c + 1]]]) for c in range(nc)], D)
    largest = int(np.argmax(area)) if nc else -1                              # the first of equal areas
    lfaces = f[order[off[largest]:off[largest + 1]]] if nc else f[:0]
    winding = np.zeros(nc, D)
    for c in range(nc):
        if c != largest:
            winding[c] = winding_number(v, lfaces, centroid(v, f[heads[c]]))
    enclosed = (np.abs(winding) >= 0.5) & (np.arange(nc) != largest)
    keep = (np.arange(nc) == largest) | (~enclosed & (area >= F * area[largest] if nc else False))
    fkeep = keep[label] if nc else np.zeros(0, bool)
    used = np.zeros(len(v), bool)
    used[f[fkeep].reshape(-1)] = True
    vertex_index = np.flatnonzero(used)
    remap = np.cumsum(used) - 1
    return {"label": label.astype(np.int32), "area": area, "winding": winding, "keep": keep.astype(np.uint8),
            "largest": largest, "enclosed": int(enclosed.sum()), "vertex_index": vertex_index.astype(np.int32),
            "faces": remap[f[fkeep]].astype(np.int32).reshape(-1, 3)}
