"""CPU: the evaluation rig of the mesh renderer (o2345/mesh_raster.py) -- cameras, normalize_scene, the loaders and
their axis conventions --, the fill and depth rules of the numpy rasterizer oracle (oracle/raster_oracle.py), the
render_eval.py command line and the argument checks of o2345_raster."""
import ctypes as C
import json
import math
import os
import struct
import sys

import numpy as np
import pytest

from o2345 import mesh_io
from o2345 import mesh_raster as MR
from oracle import raster_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ----------------------------------------------------------------------------- rig
@pytest.mark.parametrize("r", [1.3, 1.5])
def test_rig_cameras(r):
    c2w, K = MR.rig_cameras(r, 512)
    assert c2w.shape == (24, 4, 4) and K[0, 0] == K[1, 1] == 560.0 and K[0, 2] == K[1, 2] == 256.0
    centres = c2w[:, :3, 3]
    np.testing.assert_allclose(np.linalg.norm(centres, axis=1), r, rtol=1e-12)
    np.testing.assert_allclose(np.degrees(np.arccos(centres[:, 2] / r)), [60.0] * 12 + [90.0] * 12, atol=1e-9)
    for R, c in zip(c2w[:, :3, :3], centres):
        np.testing.assert_allclose(R.T @ R, np.eye(3), atol=1e-12)
        assert np.linalg.det(R) > 0
        np.testing.assert_allclose(np.cross(R[:, 2], -c), 0, atol=1e-12)    # the optical axis passes through the origin
        assert R[:, 2] @ -c > 0
        assert -R[2, 1] >= -1e-12                                            # image up (-y) has a non-negative world z
        assert abs(R[2, 0]) < 1e-12                                          # no roll: image x stays horizontal
    _, K2 = MR.rig_cameras(r, 128)
    assert K2[0, 0] == 140.0 and K2[0, 2] == 64.0


# ----------------------------------------------------------------------------- hand-built glTF
def write_glb(path, doc, binary):
    binary = binary + b"\0" * ((4 - len(binary) % 4) % 4)
    doc = dict(doc, asset={"version": "2.0"}, buffers=[{"byteLength": len(binary)}])
    js = json.dumps(doc).encode()
    js += b" " * ((4 - len(js) % 4) % 4)
    with open(path, "wb") as fh:
        fh.write(struct.pack("<III", 0x46546C67, 2, 28 + len(js) + len(binary)))
        fh.write(struct.pack("<II", len(js), 0x4E4F534A) + js)
        fh.write(struct.pack("<II", len(binary), 0x004E4942) + binary)


def glb_blobs(*arrays):
    """bufferViews / accessors for the arrays (float32 VEC2/VEC3, uint16 or uint32 SCALAR) packed into one buffer."""
    binary, views, accs = b"", [], []
    types = {np.dtype(np.float32): 5126, np.dtype(np.uint16): 5123, np.dtype(np.uint32): 5125, np.dtype(np.uint8): 5121}
    for a in arrays:
        binary += b"\0" * ((4 - len(binary) % 4) % 4)
        views.append({"buffer": 0, "byteOffset": len(binary), "byteLength": a.nbytes})
        width = 1 if a.ndim == 1 else a.shape[1]
        accs.append({"bufferView": len(views) - 1, "componentType": types[a.dtype], "count": len(a),
                     "type": {1: "SCALAR", 2: "VEC2", 3: "VEC3", 4: "VEC4"}[width]})
        binary += a.tobytes()
    return binary, views, accs


TETRA = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
TETRA_F = np.array([0, 2, 1, 0, 1, 3, 0, 3, 2, 1, 2, 3], np.uint16)


def test_normalize_two_nodes_with_a_rotated_child(tmp_path):
    binary, views, accs = glb_blobs(TETRA, TETRA_F)
    h = math.sqrt(0.5)
    doc = {"scene": 0, "scenes": [{"nodes": [0]}],
           "nodes": [{"translation": [1, 0, 0], "children": [1]},
                     {"rotation": [0, h, 0, h], "translation": [2, 0, 0], "mesh": 0}],   # 90 deg about glTF +y
           "meshes": [{"primitives": [{"attributes": {"POSITION": 0}, "indices": 1}]}], "bufferViews": views, "accessors": accs}
    p = str(tmp_path / "two.glb")
    write_glb(p, doc, binary)
    sc = MR.load_scene(p)
    # Blender frame: local AABB of C v is x [0,1], y [-1,0], z [0,1]; the child turns it 90 deg about z and moves it by
    # (2,0,0), the root by (1,0,0): x [3,4], y [0,1], z [0,1].  Rotated by 45 deg instead the corner box would differ.
    lo, hi = MR.scene_bbox(sc)
    np.testing.assert_allclose(lo, [3, 0, 0], atol=1e-12)
    np.testing.assert_allclose(hi, [4, 1, 1], atol=1e-12)

    doc["nodes"][1]["rotation"] = [0, math.sin(math.pi / 8), 0, math.cos(math.pi / 8)]   # 45 deg: corner box != vertex box
    write_glb(p, doc, binary)
    sc = MR.load_scene(p)
    lo, hi = MR.scene_bbox(sc)
    r2 = math.sqrt(2.0)
    # corners (x, y) of [0,1] x [-1,0] turned 45 deg about z: x' = (x - y) / sqrt2 in [0, sqrt2], y' = (x + y) / sqrt2
    np.testing.assert_allclose(lo, [3, -1 / r2, 0], atol=1e-12)
    np.testing.assert_allclose(hi, [3 + r2, 1 / r2, 1], atol=1e-12)
    MR.normalize_scene(sc)
    s = 0.8 / r2
    root = sc["roots"][0]
    np.testing.assert_allclose(root[:3, :3], s * np.eye(3), atol=1e-12)               # scaled about the root's origin
    # before centring: x in [1 + 2s, 1 + (2 + sqrt2) s], y in [-s/sqrt2, s/sqrt2], z in [0, s]
    np.testing.assert_allclose(root[:3, 3], [1 - (1 + (2 + r2 / 2) * s), 0, -s / 2], atol=1e-12)
    lo, hi = MR.scene_bbox(sc)
    np.testing.assert_allclose(lo, [-0.4, -0.4, -s / 2], atol=1e-12)
    np.testing.assert_allclose(hi, [0.4, 0.4, s / 2], atol=1e-12)
    # the vertices themselves span less than the corner box in x: the box, not the vertices, is normalised
    v = MR.flatten(sc)["verts"]
    assert v[:, 0].max() - v[:, 0].min() < 0.8 - 0.1


def test_normalize_single_obj_is_the_plain_aabb(tmp_path):
    rng = np.random.default_rng(0)
    v = rng.uniform([-1, 2, 5], [3, 2.5, 6], size=(50, 3))
    f = rng.integers(0, 50, size=(30, 3))
    p = str(tmp_path / "m.obj")
    mesh_io.write_obj(p, v, f, np.full((50, 3), 128))
    w = MR.flatten(MR.normalize_scene(MR.load_scene(p)))["verts"].astype(np.float64)
    ref = v @ MR.Y_UP_TO_Z_UP.T
    ref = (ref - (ref.min(0) + ref.max(0)) / 2) * (0.8 / (ref.max(0) - ref.min(0)).max())
    np.testing.assert_allclose(w, ref, atol=1e-6)
    np.testing.assert_allclose((w.max(0) - w.min(0)).max(), 0.8, atol=1e-6)


# ----------------------------------------------------------------------------- loaders
@pytest.mark.parametrize("ext", [".ply", ".obj", ".glb"])
def test_loaders_round_trip_mesh_io(tmp_path, ext):
    rng = np.random.default_rng(1)
    v = rng.normal(size=(40, 3)).astype(np.float32)
    f = rng.integers(0, 40, size=(60, 3))
    c = rng.integers(0, 256, size=(40, 3)).astype(np.uint8)
    p = str(tmp_path / f"m{ext}")
    {".ply": mesh_io.write_ply, ".obj": mesh_io.write_obj, ".glb": mesh_io.write_glb}[ext](p, v, f, c)
    flat = MR.flatten(MR.load_scene(p))
    expect = v.astype(np.float64) if ext == ".ply" else v.astype(np.float64) @ MR.Y_UP_TO_Z_UP.T
    np.testing.assert_allclose(flat["verts"], expect, atol=1e-6)
    assert np.array_equal(flat["faces"], f)
    np.testing.assert_allclose(flat["colors"], c / 255.0, atol=1e-6)


def test_textured_glb_with_matrix_and_trs_nodes(tmp_path):
    quad = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float32)
    uv = np.array([[0, 1], [1, 1], [1, 0], [0, 0]], np.float32)
    idx = np.array([0, 1, 2, 0, 2, 3], np.uint32)
    binary, views, accs = glb_blobs(quad, uv, idx)
    from io import BytesIO

    from PIL import Image
    tex = np.arange(2 * 3 * 4, dtype=np.uint8).reshape(2, 3, 4) * 10
    buf = BytesIO()
    Image.fromarray(tex, "RGBA").save(buf, "PNG")
    png = buf.getvalue()
    binary += b"\0" * ((4 - len(binary) % 4) % 4)
    views.append({"buffer": 0, "byteOffset": len(binary), "byteLength": len(png)})
    binary += png
    M = np.array([[2, 0, 0, 5], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float64)     # scale x by 2, move x by 5
    doc = {"scene": 0, "scenes": [{"nodes": [0]}],
           "nodes": [{"matrix": M.T.reshape(-1).tolist(), "children": [1]},
                     {"translation": [0, 0, -3], "scale": [1, 3, 1], "mesh": 0}],
           "meshes": [{"primitives": [{"attributes": {"POSITION": 0, "TEXCOORD_0": 1}, "indices": 2, "material": 0}]}],
           "materials": [{"pbrMetallicRoughness": {"baseColorTexture": {"index": 0}, "baseColorFactor": [0.5, 1, 1, 1]}}],
           "textures": [{"source": 0, "sampler": 0}], "samplers": [{"wrapS": 33071, "wrapT": 33648}],
           "images": [{"bufferView": 3, "mimeType": "image/png"}], "bufferViews": views, "accessors": accs}
    p = str(tmp_path / "tex.glb")
    write_glb(p, doc, binary)
    flat = MR.flatten(MR.load_scene(p))
    world_gltf = np.stack([2 * quad[:, 0] + 5, 3 * quad[:, 1], quad[:, 2] - 3], 1)
    np.testing.assert_allclose(flat["verts"], world_gltf @ MR.Y_UP_TO_Z_UP.T, atol=1e-6)
    np.testing.assert_allclose(flat["uvs"], uv)
    np.testing.assert_allclose(flat["colors"], np.tile([0.5, 1, 1], (4, 1)))
    assert flat["face_tex"].tolist() == [0, 0]
    assert flat["tex_info"].tolist() == [[0, 3, 2, 1, 2]]
    assert np.array_equal(flat["texels"].reshape(2, 3, 4), tex)


def test_example_meshes_load():
    sc = MR.normalize_scene(MR.load_scene(os.path.join(ROOT, "tests", "golden", "render_eval", "backpack_gt.glb")))
    assert len(sc["meshes"]) == 53 and len(sc["textures"]) == 1
    lo, hi = MR.scene_bbox(sc)
    np.testing.assert_allclose((hi - lo).max(), 0.8, atol=1e-9)
    np.testing.assert_allclose(lo + hi, 0, atol=1e-9)


def test_fbx_and_unknown_formats_are_refused(tmp_path):
    for ext in (".fbx", ".stl"):
        p = tmp_path / f"m{ext}"
        p.write_bytes(b"")
        with pytest.raises(ValueError):
            MR.load_scene(str(p))


# ----------------------------------------------------------------------------- oracle rules
PLANE_W2C = np.array([[[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]]], np.float32)   # z = 1: pixel coordinates = (x, y)
PLANE_K = np.array([[1, 1, 0, 0]], np.float32)


def plane(xy):
    return np.concatenate([np.asarray(xy, np.float32), np.ones((len(xy), 1), np.float32)], 1)


def test_shared_edge_through_pixel_centres_covers_each_once():
    v = plane([[0.5, 0.5], [6.5, 0.5], [0.5, 6.5], [6.5, 6.5]])
    for faces in ([[0, 1, 2], [1, 3, 2]], [[0, 2, 1], [1, 2, 3]]):       # either winding
        cov = RO.coverage(v, faces, PLANE_W2C, PLANE_K, 8, 8)[0]
        expect = np.zeros((8, 8), np.int64)
        expect[:6, :6] = 1                                                # top and left edges owned, right and bottom not
        assert np.array_equal(cov, expect)


def test_fan_centre_on_a_pixel_centre_is_covered_once():
    ring = [[3.5 + 3 * math.cos(a), 3.5 + 3 * math.sin(a)] for a in np.linspace(0, 2 * math.pi, 9)[:-1]]
    v = plane([[3.5, 3.5]] + ring)
    faces = [[0, 1 + k, 1 + (k + 1) % 8] for k in range(8)]
    cov = RO.coverage(v, faces, PLANE_W2C, PLANE_K, 8, 8)[0]
    assert cov[3, 3] == 1 and cov.max() == 1


def test_closed_convex_mesh_is_covered_exactly_twice():
    from scipy.spatial import ConvexHull
    rng = np.random.default_rng(3)
    p = rng.normal(size=(60, 3))
    p = p / np.linalg.norm(p, axis=1, keepdims=True) + [0, 0, 4]
    faces = ConvexHull(p).simplices
    cov = RO.coverage(p.astype(np.float32), faces, PLANE_W2C, np.array([[40, 40, 16, 16]], np.float32), 32, 32)[0]
    assert set(np.unique(cov)) == {0, 2} and (cov == 2).sum() > 100


def test_coplanar_duplicates_go_to_the_lower_id_and_nearer_wins():
    tri = plane([[0.2, 0.3], [7.1, 0.9], [1.0, 6.8]])
    v = np.concatenate([tri, tri * 0.5])     # the second copy at half the depth: same pixels, nearer
    out = RO.render(v, [[0, 1, 2], [0, 1, 2]], PLANE_W2C, PLANE_K, 8, 8)
    assert set(np.unique(out["tri"])) == {-1, 0}
    out = RO.render(v, [[0, 1, 2], [0, 1, 2], [3, 4, 5]], PLANE_W2C, PLANE_K, 8, 8)
    assert set(np.unique(out["tri"])) == {-1, 2} and np.allclose(out["depth"][out["tri"] == 2], 0.5, rtol=2e-7, atol=0)


# ----------------------------------------------------------------------------- command line, ABI
def test_command_line():
    sys.path.insert(0, os.path.join(ROOT, "one-2-3-45_b200"))
    import render_eval as RE
    a = RE.parse_args(["--object_path", "x.glb", "--output_dir", "d", "--engine", "CYCLES"])
    assert a.camera_dist == 1.5 and a.resolution == 512 and a.shading == "unlit"
    assert RE.jobs(a) == [("x.glb", "d")]
    a = RE.parse_args(["--DATA_DIR", os.path.join(ROOT, "tests", "golden", "render_eval"), "--resolution", "128"])
    assert a.camera_dist == 1.3
    names = [os.path.basename(p) for p, _ in RE.jobs(a)]
    assert names == ["backpack_gt.glb"]                                   # the .obj.gz is not a mesh format
    assert RE.jobs(a)[0][1] == os.path.join("output", "backpack_gt", "render_128")
    for bad in (["--object_path", "x.fbx"], ["--object_path", "x.glb", "--resolution", "0"], []):
        with pytest.raises(SystemExit):
            RE.parse_args(bad)


def test_raster_refuses_bad_arguments_without_a_device():
    from o2345 import _lib
    lib = _lib.load()
    fake = 0x1000
    good = _lib.RasterMesh(verts=fake, faces=fake, nv=3, nf=1)
    need = lib.o2345_raster_scratch_bytes(3, 1, 1, 8, 8)
    assert need > 8 * 64 and lib.o2345_raster_scratch_bytes(-1, 1, 1, 8, 8) == -1
    f = C.c_void_p(fake)

    def call(mesh=good, V=1, W=8, H=8, near=0.1, shading=0, scratch=f, scratch_bytes=need):
        return lib.o2345_raster(C.byref(mesh) if mesh is not None else None, V, f, f, W, H, near, shading, scratch,
                                scratch_bytes, f, f, f, f, f, None)
    cases = [dict(mesh=None), dict(mesh=_lib.RasterMesh(verts=fake, nv=3, nf=1)), dict(mesh=_lib.RasterMesh(verts=fake, faces=fake, nv=0, nf=1)),
             dict(V=0), dict(W=0), dict(H=20000), dict(near=0.0), dict(shading=2), dict(scratch_bytes=need - 1),
             dict(mesh=_lib.RasterMesh(verts=fake, faces=fake, face_tex=fake, nv=3, nf=1)),
             dict(scratch=C.c_void_p(fake + 4))]
    for i, kw in enumerate(cases):
        assert call(**kw) == -1, (i, _lib.last_error())
        assert "o2345_raster" in _lib.last_error()
