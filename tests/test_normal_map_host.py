"""CPU tests of normal-map baking: the tangent-frame rule and its byte codes (oracle/normal_map_oracle.py), vertex
normals, the writers' NORMAL / TANGENT / normalTexture, the reader, the command lines and the ABI argument checks."""
import ctypes as C
import json
import struct

import numpy as np
import pytest

from oracle import normal_map_oracle as NO

S2 = np.float32(np.sqrt(np.float64(0.5)))


def _tri(uv):
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    return v, np.array([[0, 1, 2]]), np.asarray(uv, np.float32).reshape(1, 3, 2)


# P1 - P0 = +x goes right in the image, P2 - P0 = +y goes up (v falls): T = +x, B = +y, N = +z
UP = [[0.25, 0.75], [0.5, 0.75], [0.25, 0.5]]
MIRRORED = [[0.25, 0.5], [0.5, 0.5], [0.25, 0.75]]          # +y goes down the image: B = -y
ROTATED = [[0.5, 0.5], [0.5, 0.25], [0.25, 0.5]]            # +x goes up the image, +y goes left: T = -y, B = +x


@pytest.mark.parametrize("uv, T, B", [(UP, [1, 0, 0], [0, 1, 0]), (MIRRORED, [1, 0, 0], [0, -1, 0]),
                                      (ROTATED, [0, -1, 0], [1, 0, 0])])
def test_frame_of_each_chart_orientation(uv, T, B):
    v, f, q = _tri(uv)
    t, b, n, ok = NO.frames(v, f, q)
    assert ok.all()
    np.testing.assert_array_equal(t[0], T)
    np.testing.assert_array_equal(b[0], B)
    np.testing.assert_array_equal(n[0], [0, 0, 1])
    w = np.sign(np.dot(np.cross(n[0], t[0]), b[0]))
    assert w == (-1 if uv is MIRRORED else 1)


def test_face_normal_codes_to_128_128_255():
    for uv in (UP, MIRRORED, ROTATED):
        v, f, q = _tri(uv)
        t = NO.tangent_normals(v, f, q, [0, 0], np.array([[0, 0, 1], [0, 0, 7.5]], np.float32))
        np.testing.assert_array_equal(t, [[0, 0, 1], [0, 0, 1]])
        np.testing.assert_array_equal(NO.quantise_normals(t), [[128, 128, 255]] * 2)


def test_tilted_normals_have_hand_computed_codes():
    v, f, q = _tri(UP)
    n = np.array([[1, 0, 1], [0, 1, 0], [0, -1, 0], [-1, 0, 0], [1, 1, 1]], np.float32)
    t = NO.tangent_normals(v, f, q, np.zeros(5, np.int64), n)
    r3 = np.float32(1 / np.sqrt(np.float64(3)))
    np.testing.assert_array_equal(t, np.array([[S2, 0, S2], [0, 1, 0], [0, -1, 0], [-1, 0, 0], [r3, r3, r3]], np.float32))
    # (c + 1) * 127.5: sqrt(1/2) -> 217.66 -> 218, 0 -> 127.5 -> 128 (ties to even), -1 -> 0, 1 -> 255, 1/sqrt(3) -> 201.1
    np.testing.assert_array_equal(NO.quantise_normals(t), [[218, 128, 218], [128, 255, 128], [128, 0, 128],
                                                           [0, 128, 128], [201, 201, 201]])
    v, f, q = _tri(MIRRORED)                     # the same world normal codes with the opposite y in a mirrored chart
    np.testing.assert_array_equal(NO.quantise_normals(NO.tangent_normals(v, f, q, [0], n[1:2])), [[128, 0, 128]])


def test_zero_nonfinite_normals_and_degenerate_faces_code_as_the_face_normal():
    v, f, q = _tri(UP)
    bad = np.array([[0, 0, 0], [np.nan, 0, 1], [np.inf, 0, 0], [0, -np.inf, 1]], np.float32)
    np.testing.assert_array_equal(NO.tangent_normals(v, f, q, np.zeros(4, np.int64), bad), [[0, 0, 1]] * 4)
    flat_uv = np.array([[[0.1, 0.1], [0.2, 0.2], [0.3, 0.3]]], np.float32)        # det = 0
    np.testing.assert_array_equal(NO.tangent_normals(v, f, flat_uv, [0], [[1, 0, 0]]), [[0, 0, 1]])
    line = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0]], np.float32)                  # no area
    np.testing.assert_array_equal(NO.tangent_normals(line, f, q, [0], [[1, 0, 0]]), [[0, 0, 1]])
    empty = np.array([[0, 0, 0], [np.nan, 1, 0], [np.inf, 0, 0], [3, 4, 0]], np.float32)
    np.testing.assert_array_equal(NO.quantise_normals(empty), [[128, 128, 255]] * 3 + [[204, 230, 128]])


def test_vertex_normals_of_a_tetrahedron_and_a_cube():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    r3 = np.float32(1 / np.sqrt(np.float64(3)))
    np.testing.assert_array_equal(NO.vertex_normals(v, f), [[-r3, -r3, -r3], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    cube = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    cf = np.array([t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))])
    n = NO.vertex_normals(cube, cf)
    # every corner sees its three faces: twice the area-weighted outward normal of one face and once that of the others
    # or the same on each axis, depending on the split; the direction is outward in every octant
    assert (np.sign(n) == np.sign(cube)).all() and np.allclose(np.linalg.norm(n, axis=1), 1, atol=1e-7)
    lone = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 5]], np.float32)    # a vertex without faces
    np.testing.assert_array_equal(NO.vertex_normals(lone, [[0, 1, 2]])[3], [0, 0, 0])


# ----------------------------------------------------------------------------- writers and reader
def _quad():
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0.5], [0, 1, 0]], np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]])
    uv = np.array([[[0.1, 0.9], [0.4, 0.9], [0.4, 0.5]], [[0.5, 0.5], [0.9, 0.1], [0.5, 0.1]]], np.float32)
    rng = np.random.default_rng(1)
    return v, f, uv, rng.integers(0, 256, (64, 64, 3), dtype=np.uint8), rng.integers(0, 256, (64, 64, 3), dtype=np.uint8)


def _doc(path):
    raw = open(path, "rb").read()
    return json.loads(raw[20:20 + struct.unpack_from("<I", raw, 12)[0]])


@pytest.mark.parametrize("viewer", [False, True])
def test_glb_normal_map_round_trips_in_the_baked_frame(tmp_path, viewer):
    from o2345 import mesh_io
    v, f, uv, tex, ntex = _quad()
    if viewer:
        v, f, uv = mesh_io.to_viewer_frame(v, f, uv)
    p = str(tmp_path / "m.glb")
    mesh_io.write_textured_glb(p, v, f, uv, tex, normal_texture=ntex)
    doc = _doc(p)
    prim = doc["meshes"][0]["primitives"][0]
    assert doc["materials"][0]["normalTexture"] == {"index": 1} and len(doc["images"]) == 2
    assert {"NORMAL", "TANGENT"} <= set(prim["attributes"])
    g = mesh_io.read_glb(p)
    (m,) = g["meshes"]
    assert (m["face_ntex"] == 1).all() and (m["face_tex"] == 0).all()
    assert np.array_equal(g["textures"][1][0][..., :3], ntex)
    tan, nrm = m["tangents"], m["normals"]
    np.testing.assert_allclose(np.linalg.norm(tan[:, :3], axis=1), 1, atol=1e-6)
    np.testing.assert_allclose(np.linalg.norm(nrm, axis=1), 1, atol=1e-6)
    assert set(np.unique(tan[:, 3])) <= {-1.0, 1.0}
    # the frame a viewer decodes (T, (N x T) w) is (dp/du, -dp/dv) of the written uv, normalised
    T, B, N, ok = NO.frames(v, f, uv)
    assert ok.all()
    tc, nc = tan.reshape(-1, 3, 4), nrm.reshape(-1, 3, 3)
    for k in range(3):
        np.testing.assert_allclose(tc[:, k, :3], T, atol=1e-6)
        np.testing.assert_allclose(nc[:, k], N, atol=1e-6)
        np.testing.assert_allclose(np.cross(nc[:, k], tc[:, k, :3]) * tc[:, k, 3:], B, atol=1e-6)


def test_viewer_frame_flips_the_tangent_handedness(tmp_path):
    from o2345 import mesh_io
    v, f, uv, tex, ntex = _quad()
    w = []
    for args in ((v, f, uv), mesh_io.to_viewer_frame(v, f, uv)):
        p = str(tmp_path / "m.glb")
        mesh_io.write_textured_glb(p, *args, tex, normal_texture=ntex)
        w.append(mesh_io.read_glb(p)["meshes"][0]["tangents"][:, 3])
    np.testing.assert_array_equal(w[0], -w[1])


def test_glb_without_normal_map_is_unchanged(tmp_path):
    from o2345 import mesh_io
    v, f, uv, tex, _ = _quad()
    p = str(tmp_path / "m.glb")
    mesh_io.write_textured_glb(p, v, f, uv, tex)
    doc = _doc(p)
    assert "normalTexture" not in doc["materials"][0] and len(doc["images"]) == 1
    m = mesh_io.read_glb(p)["meshes"][0]
    assert m["normals"] is None and m["tangents"] is None and (m["face_ntex"] == -1).all()


def test_obj_normal_map_lines_and_files(tmp_path):
    from PIL import Image
    from o2345 import mesh_io
    v, f, uv, tex, ntex = _quad()
    p = str(tmp_path / "mesh.obj")
    mesh_io.write_textured_obj(p, v, f, uv, tex, normal_texture=ntex)
    lines = open(p).read().splitlines()
    vn = np.array([[float(x) for x in l.split()[1:]] for l in lines if l.startswith("vn ")])
    np.testing.assert_allclose(vn, NO.frames(v, f, uv)[2], atol=1e-8)
    assert [l for l in lines if l.startswith("f ")] == ["f 1/1/1 2/2/1 3/3/1", "f 1/4/2 3/5/2 4/6/2"]
    mtl = open(tmp_path / "mesh.mtl").read().splitlines()
    assert "norm mesh_normal.png" in mtl and "map_Kd mesh_albedo.png" in mtl
    assert np.array_equal(np.asarray(Image.open(tmp_path / "mesh_normal.png")), ntex)
    rv, rf, _ = mesh_io.read_obj(p)
    assert np.array_equal(rf, f)


def test_backpack_gt_flattens_as_without_normal_maps():
    import os
    from o2345 import mesh_raster as MR
    p = os.path.join(os.path.dirname(__file__), "golden", "render_eval", "backpack_gt.glb")
    scene = MR.load_scene(p)
    assert any(m["normals"] is not None for m in scene["meshes"])        # it has NORMAL and TANGENT, no normalTexture
    flat = MR.flatten(scene)
    assert flat["normals"] is None and flat["tangents"] is None and flat["face_ntex"] is None


def test_flatten_carries_normals_and_tangents_into_world_space(tmp_path):
    from o2345 import mesh_io, mesh_raster as MR
    v, f, uv, tex, ntex = _quad()
    p = str(tmp_path / "m.glb")
    mesh_io.write_textured_glb(p, v, f, uv, tex, normal_texture=ntex)
    sc = MR.load_scene(p)
    R = np.diag([2.0, -1.0, 1.0, 1.0])                    # a reflection with scale
    sc["roots"][0] = R @ sc["roots"][0]
    flat = MR.flatten(sc)
    g = mesh_io.read_glb(p)["meshes"][0]
    A = R[:3, :3] @ MR.Y_UP_TO_Z_UP
    np.testing.assert_allclose(flat["tangents"][:, :3], g["tangents"][:, :3] @ A.T, atol=1e-6)
    np.testing.assert_allclose(flat["tangents"][:, 3], -g["tangents"][:, 3])
    np.testing.assert_allclose(flat["normals"], g["normals"] @ np.linalg.inv(A), atol=1e-6)
    # world normals stay perpendicular to world tangents
    np.testing.assert_allclose(np.einsum("ij,ij->i", flat["normals"], flat["tangents"][:, :3]), 0, atol=1e-6)
    assert (flat["face_ntex"] == 1).all() and flat["tex_info"].shape == (2, 5)


def test_package_frame_matches_the_oracle():
    from o2345 import mesh_io
    rng = np.random.default_rng(3)
    v = rng.normal(size=(30, 3)).astype(np.float32)
    f = rng.integers(0, 30, (40, 3))
    f = f[(f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])]
    uv = rng.random((len(f), 3, 2)).astype(np.float32)
    T, B, N = mesh_io.tangent_frames(v, f, uv)
    t, b, n, ok = NO.frames(v, f, uv)
    assert ok.all()
    np.testing.assert_allclose(T, t, atol=1e-12)
    np.testing.assert_allclose(B, b, atol=1e-12)
    np.testing.assert_allclose(N, n, atol=1e-12)


# ----------------------------------------------------------------------------- command lines and the ABI
def test_run_py_normal_map_arguments():
    import run as run_cli
    a = run_cli.parse_args(["--texture_size", "1024", "--output_format", ".glb", "--normal_map"])
    assert a.normal_map and not run_cli.parse_args([]).normal_map
    assert run_cli._texture_kw(a) == {"texture_size": 1024, "normal_map": True}
    for bad in (["--normal_map"], ["--normal_map", "--output_format", ".glb"],
                ["--normal_map", "--texture_size", "1024", "--output_format", ".ply"]):
        with pytest.raises(SystemExit):
            run_cli.parse_args(bad)


def test_simplify_mesh_normal_map_arguments():
    import simplify_mesh as SM
    a = SM.parse_args(["--in", "a.ply", "--out", "b.obj", "--target_faces", "10", "--texture_size", "256", "--normal_map"])
    assert a.normal_map
    for bad in (["--out", "b.glb", "--normal_map"], ["--out", "b.ply", "--texture_size", "256", "--normal_map"]):
        with pytest.raises(SystemExit):
            SM.parse_args(["--in", "a.ply", "--target_faces", "10", *bad])


def test_normal_map_abi_checks_return_einval_without_touching_the_gpu():
    from o2345 import _lib
    lib = _lib.load()
    fake = C.c_void_p(0x1000)
    assert lib.o2345_vertex_normals_scratch_bytes(0, 1) == -1 and lib.o2345_vertex_normals_scratch_bytes(4, 0) == -1
    assert lib.o2345_vertex_normals_scratch_bytes(4, 4) > 0
    mesh = _lib.RasterMesh(verts=0x1000, faces=0x1000, face_ntex=0x1000, nv=3, nf=1)   # face_ntex without textures
    cases = [
        lambda: lib.o2345_tangent_normals(None, 3, fake, 1, fake, fake, fake, 10, fake, None),
        lambda: lib.o2345_tangent_normals(fake, 3, fake, 1, fake, fake, fake, 0, fake, None),
        lambda: lib.o2345_tangent_normals(fake, 0, fake, 1, fake, fake, fake, 10, fake, None),
        lambda: lib.o2345_normal_quantise(fake, 0, fake, None),
        lambda: lib.o2345_normal_quantise(None, 10, fake, None),
        lambda: lib.o2345_vertex_normals(fake, 3, fake, 1, fake, 8, fake, None),
        lambda: lib.o2345_vertex_normals(fake, 3, fake, 0, fake, 1 << 20, fake, None),
        lambda: lib.o2345_vertex_normals(fake, 3, fake, 1, C.c_void_p(0x1004), 1 << 20, fake, None),
        lambda: lib.o2345_raster(C.byref(mesh), 1, fake, fake, 8, 8, 0.1, 0, fake, 1 << 20, fake, fake, fake, fake, fake, None),
    ]
    for i, call in enumerate(cases):
        assert call() == -1, (i, _lib.last_error())
        assert len(_lib.last_error()) > 0
