"""Mesh tail of the reconstruction path (SURVEY.md row B15) without trimesh (not installed here).

Restates, on plain numpy arrays:
  * `merge_vertices`        what `trimesh.Trimesh(vertices, faces, vertex_colors=...)` does with its default `process=True`
                            before reference reconstruction/models/trainer_generic.py:1374-1380 exports mesh.ply: vertices
                            that coincide after rounding to 8 decimals are merged (first occurrence kept, with its colour),
                            faces are re-indexed, vertices no face references are dropped.  trimesh's source is not under
                            /root/reference: PARITY UNPINNED (only the vertex ORDER could differ; geometry cannot).
  * `write_ply`             binary little-endian PLY with per-vertex RGBA, the layout trimesh emits.
  * `to_viewer_frame` + `write_obj` / `write_glb`
                            reference utils/utils.py:31-45 `convert_mesh_format`: rotate +90 degrees about x, 180 degrees
                            about z, negate x, reverse the face winding -- altogether (x, y, z) -> (x, z, y) with flipped
                            faces -- then `.obj` with `v x y z r g b` lines (trimesh's include_color=True) or a binary glTF.
  * `write_textured_glb` / `write_textured_obj`
                            a mesh with per-corner uv and a colour texture (o2345/mesh_texture.py; not in the reference):
                            glTF with an embedded PNG as baseColorTexture, or OBJ + MTL (map_Kd) + PNG; optionally a
                            tangent-space normal map in the frame of `tangent_frames` (normalTexture, or `norm` in the MTL).
"""
from __future__ import annotations

import json
import struct

import numpy as np


def merge_vertices(vertices, triangles, colors=None, digits=8, candidates=None):
    """candidates (optional): indices of the only vertices that can coincide with another one (marching cubes: those on a
    lattice point).  With fewer than two of them, or no coinciding pair among them, the arrays are returned untouched; the
    sort over all vertices is only paid when something really merges."""
    v = np.asarray(vertices)
    f = np.asarray(triangles)
    if len(v) == 0 or len(f) == 0:
        return v, f, colors
    if candidates is not None:
        cand = np.asarray(candidates, np.int64)
        if cand.size < 2:
            return v, f, colors
        ck = np.round(np.asarray(v[cand], np.float64) * 10.0 ** digits).astype(np.int64)
        if len(np.unique(ck, axis=0)) == len(ck):
            return v, f, colors
    v = np.asarray(v, np.float64)
    f = np.asarray(f, np.int64).reshape(-1, 3)
    key = np.round(v * 10.0 ** digits).astype(np.int64)
    _, first, inverse = np.unique(key, axis=0, return_index=True, return_inverse=True)
    inverse = np.asarray(inverse).reshape(-1)
    # keep the FIRST occurrence of every position, in order of first occurrence
    order = np.argsort(first, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    keep = first[order]
    remap = rank[inverse]
    f2 = remap[f]
    used = np.zeros(len(keep), bool)
    used[f2.reshape(-1)] = True
    if not used.all():
        compact = np.cumsum(used) - 1
        f2 = compact[f2]
        keep = keep[used]
    return v[keep], f2, (None if colors is None else np.asarray(colors)[keep])


def write_ply(path, vertices, triangles, colors):
    """Binary little-endian PLY with per-vertex RGBA."""
    v = np.asarray(vertices, np.float32)
    f = np.asarray(triangles, np.int32)
    c = np.asarray(colors, np.uint8)
    if c.shape[1] == 3:
        c = np.concatenate([c, np.full((len(c), 1), 255, np.uint8)], 1)
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
              "property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\n"
              "element face %d\nproperty list uchar int vertex_indices\nend_header\n") % (len(v), len(f))
    vrec = np.empty(len(v), dtype=[("p", "<f4", 3), ("c", "u1", 4)])
    vrec["p"], vrec["c"] = v, c
    frec = np.empty(len(f), dtype=[("n", "u1"), ("i", "<i4", 3)])
    frec["n"], frec["i"] = 3, f
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vrec.tobytes())
        fh.write(frec.tobytes())


def read_ply(path):
    """Reads back a file written by write_ply -> (vertices float32 [n,3], triangles int32 [m,3], colors uint8 [n,4])."""
    with open(path, "rb") as fh:
        raw = fh.read()
    end = raw.index(b"end_header\n") + len(b"end_header\n")
    head = raw[:end].decode("ascii")
    nv = int(head.split("element vertex ")[1].split("\n")[0])
    nf = int(head.split("element face ")[1].split("\n")[0])
    vrec = np.frombuffer(raw, dtype=[("p", "<f4", 3), ("c", "u1", 4)], count=nv, offset=end)
    frec = np.frombuffer(raw, dtype=[("n", "u1"), ("i", "<i4", 3)], count=nf, offset=end + nv * 16)
    return vrec["p"].copy(), frec["i"].copy(), vrec["c"].copy()


def to_viewer_frame(vertices, triangles, uv=None):
    """convert_mesh_format's transform chain (reference utils/utils.py:35-41), applied exactly in its order.  With uv
    [m,3,2] (one row per face corner) the rows of each face are reversed with its corners and returned third."""
    v = np.asarray(vertices, np.float64)
    rx = np.array([[1, 0, 0], [0, 0, -1], [0, 1, 0]], np.float64)        # rotation_matrix(pi / 2, [1, 0, 0])
    rz = np.array([[-1, 0, 0], [0, -1, 0], [0, 0, 1]], np.float64)       # rotation_matrix(pi, [0, 0, 1])
    v = v @ rx.T
    v = v @ rz.T
    v[:, 0] = -v[:, 0]
    if uv is not None:
        return v, np.fliplr(np.asarray(triangles)).copy(), np.asarray(uv)[:, ::-1].copy()
    return v, np.fliplr(np.asarray(triangles)).copy()


def write_obj(path, vertices, triangles, colors):
    v = np.asarray(vertices, np.float64)
    c = np.asarray(colors, np.float64)[:, :3] / 255.0
    f = np.asarray(triangles, np.int64) + 1
    with open(path, "w") as fh:
        fh.write("# o2345-b200\n")
        for p, q in zip(v, c):
            fh.write("v %.8f %.8f %.8f %.8f %.8f %.8f\n" % (p[0], p[1], p[2], q[0], q[1], q[2]))
        for t in f:
            fh.write("f %d %d %d\n" % (t[0], t[1], t[2]))


def write_glb(path, vertices, triangles, colors):
    """Binary glTF 2.0: one mesh, POSITION float32, COLOR_0 normalised uint8 RGBA, uint32 indices."""
    v = np.ascontiguousarray(vertices, np.float32)
    c = np.asarray(colors, np.uint8)
    if c.shape[1] == 3:
        c = np.concatenate([c, np.full((len(c), 1), 255, np.uint8)], 1)
    c = np.ascontiguousarray(c)
    idx = np.ascontiguousarray(np.asarray(triangles, np.uint32).reshape(-1))
    blobs = [v.tobytes(), c.tobytes(), idx.tobytes()]
    offs, total = [], 0
    for b in blobs:
        offs.append(total)
        total += (len(b) + 3) // 4 * 4
    bin_chunk = bytearray(total)
    for o, b in zip(offs, blobs):
        bin_chunk[o:o + len(b)] = b
    doc = {
        "asset": {"version": "2.0", "generator": "o2345-b200"},
        "scene": 0, "scenes": [{"nodes": [0]}], "nodes": [{"mesh": 0}],
        "meshes": [{"primitives": [{"attributes": {"POSITION": 0, "COLOR_0": 1}, "indices": 2, "mode": 4}]}],
        "buffers": [{"byteLength": total}],
        "bufferViews": [{"buffer": 0, "byteOffset": offs[0], "byteLength": len(blobs[0]), "target": 34962},
                        {"buffer": 0, "byteOffset": offs[1], "byteLength": len(blobs[1]), "target": 34962},
                        {"buffer": 0, "byteOffset": offs[2], "byteLength": len(blobs[2]), "target": 34963}],
        "accessors": [{"bufferView": 0, "componentType": 5126, "count": int(len(v)), "type": "VEC3",
                       "min": v.min(0).tolist() if len(v) else [0, 0, 0], "max": v.max(0).tolist() if len(v) else [0, 0, 0]},
                      {"bufferView": 1, "componentType": 5121, "normalized": True, "count": int(len(c)), "type": "VEC4"},
                      {"bufferView": 2, "componentType": 5125, "count": int(len(idx)), "type": "SCALAR"}],
    }
    js = json.dumps(doc, separators=(",", ":")).encode("utf-8")
    js += b" " * ((4 - len(js) % 4) % 4)
    with open(path, "wb") as fh:
        fh.write(struct.pack("<III", 0x46546C67, 2, 12 + 8 + len(js) + 8 + len(bin_chunk)))
        fh.write(struct.pack("<II", len(js), 0x4E4F534A))
        fh.write(js)
        fh.write(struct.pack("<II", len(bin_chunk), 0x004E4942))
        fh.write(bytes(bin_chunk))


def _png_bytes(texture):
    import io
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(texture, np.uint8)).save(buf, format="PNG")
    return buf.getvalue()


def tangent_frames(vertices, triangles, uv):
    """The tangent frame of every face (include/o2345.h, the rule the normal-map baker codes with): in fp64 from the fp32
    corners and uv rows (glTF: v down the image), T = dp/du, B = -dp/dv (+Y up the image), N = e1 x e2 (the winding as
    given), each normalised -> T, B, N float64 [m,3].  A degenerate face gets N = (0, 0, 1) where e1 x e2 = 0 and
    T = (1, 0, 0), B = N x T where its uv have no area."""
    v = np.asarray(vertices, np.float32).astype(np.float64)
    f = np.asarray(triangles, np.int64).reshape(-1, 3)
    q = np.asarray(uv, np.float32).reshape(-1, 3, 2).astype(np.float64)
    e1, e2 = v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]
    d1, d2 = q[:, 1] - q[:, 0], q[:, 2] - q[:, 0]
    det = d1[:, 0] * d2[:, 1] - d2[:, 0] * d1[:, 1]

    def unit(a, fallback):
        ln = np.linalg.norm(a, axis=1, keepdims=True)
        ok = (ln > 0) & np.isfinite(ln)
        return np.where(ok, a / np.where(ok, ln, 1.0), fallback)
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.where(det != 0, 1.0 / np.where(det != 0, det, 1.0), 0.0)[:, None]
    N = unit(np.cross(e1, e2), np.array([0.0, 0.0, 1.0]))
    T = unit((d2[:, 1:2] * e1 - d1[:, 1:2] * e2) * s, np.array([1.0, 0.0, 0.0]))
    B = unit(-(d1[:, 0:1] * e2 - d2[:, 0:1] * e1) * s, np.cross(N, T))
    return T, B, N


def write_textured_glb(path, vertices, triangles, uv, texture, normal_texture=None, occlusion_texture=None):
    """Binary glTF 2.0 of a textured mesh: vertices [n,3], triangles [m,3], uv [m,3,2] (row k for corner k, glTF's
    convention), texture uint8 [N,N,3].  Vertices are split per corner (3m of them: POSITION float32, TEXCOORD_0 float32,
    uint32 indices 0 .. 3m-1) and the material is unlit-friendly PBR: the texture as an embedded PNG baseColorTexture
    (CLAMP_TO_EDGE, LINEAR), metallic 0, roughness 1.  No COLOR_0.  With normal_texture uint8 [N,N,3] (tangent space, in
    the frame of tangent_frames) the corners also get NORMAL (the face normal of the written winding) and TANGENT (T, w)
    with w = sign((N x T) . B) in this frame, and the material a normalTexture (a second PNG).  With occlusion_texture
    uint8 [N,N] (ambient occlusion, 255 = open) the material gains an occlusionTexture in TEXCOORD_0: a grey PNG, whose
    R channel glTF reads."""
    f = np.asarray(triangles, np.int64).reshape(-1, 3)
    v = np.ascontiguousarray(np.asarray(vertices, np.float32)[f.reshape(-1)])
    t = np.ascontiguousarray(np.asarray(uv, np.float32).reshape(-1, 2))
    if len(t) != len(v):
        raise ValueError(f"uv has {len(t) // 3} faces, triangles {len(f)}")
    idx = np.arange(len(v), dtype=np.uint32)
    blobs = [v.tobytes(), t.tobytes(), idx.tobytes(), _png_bytes(texture)]
    if normal_texture is not None:
        T, B, N = tangent_frames(vertices, f, uv)
        w = np.where(np.einsum("ij,ij->i", np.cross(N, T), B) < 0, -1.0, 1.0)
        nrm = np.ascontiguousarray(np.repeat(N, 3, 0).astype(np.float32))
        tan = np.ascontiguousarray(np.repeat(np.concatenate([T, w[:, None]], 1), 3, 0).astype(np.float32))
        blobs += [_png_bytes(normal_texture), nrm.tobytes(), tan.tobytes()]
    if occlusion_texture is not None:
        blobs.append(_png_bytes(occlusion_texture))
    offs, total = [], 0
    for b in blobs:
        offs.append(total)
        total += (len(b) + 3) // 4 * 4
    bin_chunk = bytearray(total)
    for o, b in zip(offs, blobs):
        bin_chunk[o:o + len(b)] = b
    doc = {
        "asset": {"version": "2.0", "generator": "o2345-b200"},
        "scene": 0, "scenes": [{"nodes": [0]}], "nodes": [{"mesh": 0}],
        "meshes": [{"primitives": [{"attributes": {"POSITION": 0, "TEXCOORD_0": 1}, "indices": 2, "material": 0, "mode": 4}]}],
        "materials": [{"pbrMetallicRoughness": {"baseColorTexture": {"index": 0}, "metallicFactor": 0.0, "roughnessFactor": 1.0}}],
        "textures": [{"sampler": 0, "source": 0}],
        "samplers": [{"magFilter": 9729, "minFilter": 9729, "wrapS": 33071, "wrapT": 33071}],
        "images": [{"bufferView": 3, "mimeType": "image/png"}],
        "buffers": [{"byteLength": total}],
        "bufferViews": [{"buffer": 0, "byteOffset": offs[0], "byteLength": len(blobs[0]), "target": 34962},
                        {"buffer": 0, "byteOffset": offs[1], "byteLength": len(blobs[1]), "target": 34962},
                        {"buffer": 0, "byteOffset": offs[2], "byteLength": len(blobs[2]), "target": 34963},
                        {"buffer": 0, "byteOffset": offs[3], "byteLength": len(blobs[3])}],
        "accessors": [{"bufferView": 0, "componentType": 5126, "count": int(len(v)), "type": "VEC3",
                       "min": v.min(0).tolist() if len(v) else [0, 0, 0], "max": v.max(0).tolist() if len(v) else [0, 0, 0]},
                      {"bufferView": 1, "componentType": 5126, "count": int(len(t)), "type": "VEC2"},
                      {"bufferView": 2, "componentType": 5125, "count": int(len(idx)), "type": "SCALAR"}],
    }
    if normal_texture is not None:
        doc["meshes"][0]["primitives"][0]["attributes"].update(NORMAL=3, TANGENT=4)
        doc["materials"][0]["normalTexture"] = {"index": 1}
        doc["textures"].append({"sampler": 0, "source": 1})
        doc["images"].append({"bufferView": 4, "mimeType": "image/png"})
        doc["bufferViews"] += [{"buffer": 0, "byteOffset": offs[4], "byteLength": len(blobs[4])},
                               {"buffer": 0, "byteOffset": offs[5], "byteLength": len(blobs[5]), "target": 34962},
                               {"buffer": 0, "byteOffset": offs[6], "byteLength": len(blobs[6]), "target": 34962}]
        doc["accessors"] += [{"bufferView": 5, "componentType": 5126, "count": int(len(v)), "type": "VEC3"},
                             {"bufferView": 6, "componentType": 5126, "count": int(len(v)), "type": "VEC4"}]
    if occlusion_texture is not None:
        doc["materials"][0]["occlusionTexture"] = {"index": len(doc["textures"])}
        doc["textures"].append({"sampler": 0, "source": len(doc["images"])})
        doc["images"].append({"bufferView": len(blobs) - 1, "mimeType": "image/png"})
        doc["bufferViews"].append({"buffer": 0, "byteOffset": offs[-1], "byteLength": len(blobs[-1])})
    js = json.dumps(doc, separators=(",", ":")).encode("utf-8")
    js += b" " * ((4 - len(js) % 4) % 4)
    with open(path, "wb") as fh:
        fh.write(struct.pack("<III", 0x46546C67, 2, 12 + 8 + len(js) + 8 + len(bin_chunk)))
        fh.write(struct.pack("<II", len(js), 0x4E4F534A))
        fh.write(js)
        fh.write(struct.pack("<II", len(bin_chunk), 0x004E4942))
        fh.write(bytes(bin_chunk))


def write_textured_obj(path, vertices, triangles, uv, texture, normal_texture=None, occlusion_texture=None):
    """Wavefront OBJ of a textured mesh beside its material: `v x y z`, then one `vt u (1 - v)` per face corner (OBJ's v
    points up the image), then `f a/t b/t c/t`; <stem>.mtl (`map_Kd <stem>_albedo.png`) and the PNG next to it.  With
    normal_texture uint8 [N,N,3] (tangent space, the frame of tangent_frames) also one `vn` per face (its normal),
    `f a/t/n ...`, <stem>_normal.png and `norm <stem>_normal.png` in the MTL.  With occlusion_texture uint8 [N,N]
    also <stem>_occlusion.png and `map_ao <stem>_occlusion.png` in the MTL: map_ao is not part of the MTL standard, but
    several importers read it as the ambient occlusion map."""
    import os
    stem = os.path.splitext(os.path.basename(path))[0]
    folder = os.path.dirname(os.path.abspath(path))
    v = np.asarray(vertices, np.float64)
    f = np.asarray(triangles, np.int64).reshape(-1, 3)
    t = np.asarray(uv, np.float64).reshape(-1, 2)
    with open(os.path.join(folder, stem + "_albedo.png"), "wb") as fh:
        fh.write(_png_bytes(texture))
    mtl = "# o2345-b200\nnewmtl albedo\nKa 1 1 1\nKd 1 1 1\nKs 0 0 0\nillum 1\nmap_Kd %s_albedo.png\n" % stem
    if normal_texture is not None:
        with open(os.path.join(folder, stem + "_normal.png"), "wb") as fh:
            fh.write(_png_bytes(normal_texture))
        mtl += "norm %s_normal.png\n" % stem
    if occlusion_texture is not None:
        with open(os.path.join(folder, stem + "_occlusion.png"), "wb") as fh:
            fh.write(_png_bytes(occlusion_texture))
        mtl += "map_ao %s_occlusion.png\n" % stem
    with open(os.path.join(folder, stem + ".mtl"), "w") as fh:
        fh.write(mtl)
    with open(path, "w") as fh:
        fh.write("# o2345-b200\nmtllib %s.mtl\n" % stem)
        for p in v:
            fh.write("v %.8f %.8f %.8f\n" % (p[0], p[1], p[2]))
        for q in t:
            fh.write("vt %.8f %.8f\n" % (q[0], 1.0 - q[1]))
        if normal_texture is not None:
            for n in tangent_frames(v, f, uv)[2]:
                fh.write("vn %.8f %.8f %.8f\n" % (n[0], n[1], n[2]))
        fh.write("usemtl albedo\n")
        for i, q in enumerate(f + 1):
            if normal_texture is None:
                fh.write("f %d/%d %d/%d %d/%d\n" % (q[0], 3 * i + 1, q[1], 3 * i + 2, q[2], 3 * i + 3))
            else:
                fh.write("f %d/%d/%d %d/%d/%d %d/%d/%d\n" % (q[0], 3 * i + 1, i + 1, q[1], 3 * i + 2, i + 1, q[2], 3 * i + 3, i + 1))


def write_textured(path, vertices, triangles, uv, texture, normal_texture=None, occlusion_texture=None):
    """write_textured_glb or write_textured_obj by the extension of path."""
    if path.lower().endswith(".glb"):
        return write_textured_glb(path, vertices, triangles, uv, texture, normal_texture, occlusion_texture)
    if path.lower().endswith(".obj"):
        return write_textured_obj(path, vertices, triangles, uv, texture, normal_texture, occlusion_texture)
    raise ValueError(f"{path}: a textured mesh is written as .glb or .obj")


def convert_mesh_format(exp_dir, output_format=".obj"):
    """reference utils/utils.py:31-45: <exp_dir>/mesh.ply -> <exp_dir>/mesh.obj | mesh.glb in the viewer frame."""
    import os
    v, f, c = read_ply(os.path.join(exp_dir, "mesh.ply"))
    v2, f2 = to_viewer_frame(v, f)
    out = os.path.join(exp_dir, f"mesh{output_format}")
    if output_format == ".obj":
        write_obj(out, v2, f2, c)
    else:
        write_glb(out, v2, f2, c)
    return out


# ----------------------------------------------------------------------------- readers of the evaluation renderer
# (o2345/mesh_raster.py).  Each returns the file's own axes; the Blender import conventions live in mesh_raster.

def read_obj(path):
    """Wavefront OBJ: `v x y z [r g b]` vertices (trimesh's and write_obj's vertex colours) and `f` polygons (`a`, `a/b`,
    `a/b/c`, `a//c`, negative indices), fan-triangulated.  -> (vertices float64 [n,3], triangles int64 [m,3], colors float64
    [n,3] in [0, 1] or None when no vertex carries a colour).  Texture coordinates and materials are ignored."""
    verts, cols, faces = [], [], []
    with open(path, "r", errors="replace") as fh:
        for line in fh:
            if line.startswith("v "):
                q = line.split()
                verts.append([float(x) for x in q[1:4]])
                cols.append([float(x) for x in q[4:7]] if len(q) >= 7 else None)
            elif line.startswith("f "):
                idx = []
                for tok in line.split()[1:]:
                    i = int(tok.split("/")[0])
                    idx.append(i - 1 if i > 0 else len(verts) + i)
                faces.extend([idx[0], idx[k], idx[k + 1]] for k in range(1, len(idx) - 1))
    v = np.asarray(verts, np.float64).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(f) and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError(f"{path}: a face refers to a vertex that does not exist")
    has = [c is not None for c in cols]
    c = None
    if any(has):
        c = np.ones((len(v), 3), np.float64)
        for i, ci in enumerate(cols):
            if ci is not None:
                c[i] = ci
    return v, f, c


_GLTF_TYPES = {5120: np.int8, 5121: np.uint8, 5122: np.int16, 5123: np.uint16, 5125: np.uint32, 5126: np.float32}
_GLTF_WIDTH = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4, "MAT4": 16}


def _glb_accessor(doc, binary, i):
    a = doc["accessors"][i]
    if "sparse" in a or "bufferView" not in a:
        raise ValueError("glTF: sparse accessors and accessors without a bufferView are not supported")
    bv = doc["bufferViews"][a["bufferView"]]
    if bv.get("buffer", 0) != 0:
        raise ValueError("glTF: only the GLB's own binary chunk is supported as a buffer")
    dt = np.dtype(_GLTF_TYPES[a["componentType"]]).newbyteorder("<")
    width, count = _GLTF_WIDTH[a["type"]], a["count"]
    start = bv.get("byteOffset", 0) + a.get("byteOffset", 0)
    stride = bv.get("byteStride") or width * dt.itemsize
    rows = np.ndarray((count, width), dt, buffer=binary, offset=start, strides=(stride, dt.itemsize))
    out = rows.astype(np.float64) if dt.kind == "f" else rows.astype(np.int64)
    if a.get("normalized"):
        info = np.iinfo(dt)
        out = np.maximum(out / info.max, -1.0)
    return out


def _gltf_node_matrix(n):
    if "matrix" in n:
        return np.asarray(n["matrix"], np.float64).reshape(4, 4).T     # column-major
    x, y, z, w = n.get("rotation", [0.0, 0.0, 0.0, 1.0])
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], np.float64)
    M = np.eye(4)
    M[:3, :3] = R * np.asarray(n.get("scale", [1.0, 1.0, 1.0]), np.float64)[None, :]
    M[:3, 3] = n.get("translation", [0.0, 0.0, 0.0])
    return M


_GLTF_WRAP = {10497: 0, 33071: 1, 33648: 2}     # REPEAT, CLAMP_TO_EDGE, MIRRORED_REPEAT -> O2345_WRAP_*


def read_glb(path):
    """Binary glTF 2.0 -> dict:
      roots     [4x4] world matrix of every root node of the default scene that has a mesh below it;
      meshes    one entry per node with a mesh: verts [n,3], faces [m,3] (every indexed or non-indexed triangle primitive of
                the mesh, joined), colors [n,3] (COLOR_0 times the material's baseColorFactor, white without either), uvs
                [n,2] (TEXCOORD_0, or None), face_tex [m] (texture of the material's baseColorTexture, -1 without), normals
                [n,3] (NORMAL, zeros for a primitive without, or None), tangents [n,4] (TANGENT alike), face_ntex [m]
                (texture of the material's normalTexture where the primitive has TEXCOORD_0, NORMAL and TANGENT, -1
                without), face_otex [m] (texture of the material's occlusionTexture where the primitive has TEXCOORD_0, -1
                without; glTF reads its R channel), root (index into roots), local_to_root [4x4] (product of the node
                matrices below the root's own);
      textures  [(RGBA uint8 [h,w,4], wrap s, wrap t)] decoded with PIL.
    All in glTF's own (Y-up) axes.  Primitives that are not triangle lists, alpha modes, metallic-roughness textures,
    the occlusion strength, the normal map's scale and texture transforms are ignored; a texture is sampled at TEXCOORD_0."""
    import io
    raw = open(path, "rb").read()
    magic, version, _ = struct.unpack_from("<III", raw, 0)
    if magic != 0x46546C67 or version != 2:
        raise ValueError(f"{path}: not a binary glTF 2.0 file")
    jlen, jtype = struct.unpack_from("<II", raw, 12)
    if jtype != 0x4E4F534A:
        raise ValueError(f"{path}: the first GLB chunk is not JSON")
    doc = json.loads(raw[20:20 + jlen].decode("utf-8"))
    binary = b""
    off = 20 + jlen
    if off + 8 <= len(raw):
        blen, btype = struct.unpack_from("<II", raw, off)
        if btype == 0x004E4942:
            binary = raw[off + 8:off + 8 + blen]

    textures, tex_of_image = [], {}

    def texture(ti):
        t = doc["textures"][ti]
        src = t.get("source")
        if src is None:
            return -1
        samp = doc.get("samplers", [{}])[t["sampler"]] if "sampler" in t else {}
        key = (src, samp.get("wrapS", 10497), samp.get("wrapT", 10497))
        if key not in tex_of_image:
            from PIL import Image
            img = doc["images"][src]
            if "bufferView" not in img:
                raise ValueError(f"{path}: image {src} is not embedded in the GLB")
            bv = doc["bufferViews"][img["bufferView"]]
            data = binary[bv.get("byteOffset", 0):bv.get("byteOffset", 0) + bv["byteLength"]]
            rgba = np.asarray(Image.open(io.BytesIO(data)).convert("RGBA"), np.uint8)
            tex_of_image[key] = len(textures)
            textures.append((rgba, _GLTF_WRAP.get(key[1], 0), _GLTF_WRAP.get(key[2], 0)))
        return tex_of_image[key]

    def mesh(mi):
        vs, fs, cs, us, ts, ns, gs, nts, ots, n = [], [], [], [], [], [], [], [], [], 0
        for prim in doc["meshes"][mi]["primitives"]:
            if prim.get("mode", 4) != 4:
                continue
            att = prim["attributes"]
            v = _glb_accessor(doc, binary, att["POSITION"])
            f = (_glb_accessor(doc, binary, prim["indices"]).reshape(-1, 3) if "indices" in prim
                 else np.arange(len(v) - len(v) % 3, dtype=np.int64).reshape(-1, 3))
            mat = doc["materials"][prim["material"]] if "material" in prim else {}
            pbr = mat.get("pbrMetallicRoughness", {})
            c = np.ones((len(v), 3))
            if "COLOR_0" in att:
                c = _glb_accessor(doc, binary, att["COLOR_0"])[:, :3].astype(np.float64)
            c = c * np.asarray(pbr.get("baseColorFactor", [1.0, 1.0, 1.0, 1.0])[:3], np.float64)
            tex = texture(pbr["baseColorTexture"]["index"]) if "baseColorTexture" in pbr and "TEXCOORD_0" in att else -1
            mapped = "normalTexture" in mat and all(k in att for k in ("TEXCOORD_0", "NORMAL", "TANGENT"))
            nts.append(np.full(len(f), texture(mat["normalTexture"]["index"]) if mapped else -1, np.int64))
            occluded = "occlusionTexture" in mat and "TEXCOORD_0" in att
            ots.append(np.full(len(f), texture(mat["occlusionTexture"]["index"]) if occluded else -1, np.int64))
            ns.append(_glb_accessor(doc, binary, att["NORMAL"])[:, :3] if "NORMAL" in att else np.zeros((len(v), 3)))
            gs.append(_glb_accessor(doc, binary, att["TANGENT"])[:, :4] if "TANGENT" in att else np.zeros((len(v), 4)))
            vs.append(v[:, :3])
            fs.append(f + n)
            cs.append(c)
            us.append(_glb_accessor(doc, binary, att["TEXCOORD_0"]) if "TEXCOORD_0" in att else np.zeros((len(v), 2)))
            ts.append(np.full(len(f), tex, np.int64))
            n += len(v)
        if not vs:
            return None
        has = lambda key: any(key in p["attributes"] for p in doc["meshes"][mi]["primitives"])
        return {"verts": np.concatenate(vs), "faces": np.concatenate(fs), "colors": np.concatenate(cs),
                "uvs": np.concatenate(us) if has("TEXCOORD_0") else None, "face_tex": np.concatenate(ts),
                "normals": np.concatenate(ns) if has("NORMAL") else None,
                "tangents": np.concatenate(gs) if has("TANGENT") else None, "face_ntex": np.concatenate(nts),
                "face_otex": np.concatenate(ots)}

    roots, meshes = [], []

    def walk(ni, root, rel):
        node = doc["nodes"][ni]
        if "mesh" in node:
            m = mesh(node["mesh"])
            if m is not None:
                m.update(root=root, local_to_root=rel)
                meshes.append(m)
        for ch in node.get("children", []):
            walk(ch, root, rel @ _gltf_node_matrix(doc["nodes"][ch]))

    if "scenes" in doc:
        top = doc["scenes"][doc.get("scene", 0)].get("nodes", [])
    else:   # no scene: every node that is nobody's child
        kids = {c for n in doc.get("nodes", []) for c in n.get("children", [])}
        top = [i for i in range(len(doc.get("nodes", []))) if i not in kids]
    for ni in top:
        before = len(meshes)
        walk(ni, len(roots), np.eye(4))
        if len(meshes) > before:
            roots.append(_gltf_node_matrix(doc["nodes"][ni]))
    return {"roots": roots, "meshes": meshes, "textures": textures}
