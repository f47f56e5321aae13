"""CPU: texture baking's numpy oracle (oracle/texture_oracle.py) on hand-computed cases, invariants of its atlas of the
frozen 10 % example mesh, the textured GLB / OBJ writers, the command lines' argument checks and the C-ABI's argument
checks (no GPU needed)."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import texture_oracle as TO
from test_simplify_host import GOLD, example_mesh

P = TO.PAD


def one(v):
    return np.asarray(v, np.float32), np.array([[0, 1, 2]])


# ----------------------------------------------------------------------------- charts, boxes, uv, rho
def test_exact_triangle_has_the_hand_computed_atlas():
    # L = 2, d = 1, h = 1, S = 2; N = 64: rho0 = sqrt(0.5 * 4096 / 2) = 32, rho_j = j / 2, w = j + 4 <= 64 -> j = 60
    v, f = one([[0, 0, 0], [2, 0, 0], [1, 1, 0]])
    a = TO.atlas(v, f, 64)
    assert a["j"] == 60 and a["rho"] == 30.0
    assert a["boxes"].tolist() == [[0, 0, 64, 34]]
    assert np.array_equal(a["uv"][0] * 64, [[P, P], [P + 60, P], [P + 30, P + 30]])


def test_right_triangle_takes_the_hypotenuse_as_base():
    v, f = one([[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    L, d, h, k0 = TO.charts(v, f)
    assert k0.tolist() == [1]                                           # v1v2 is the longest edge
    np.testing.assert_allclose([L[0], d[0], h[0]], [2 ** 0.5, 2 ** -0.5, 2 ** -0.5], rtol=1e-7)
    a = TO.atlas(v, f, 64)
    rho = a["rho"]
    np.testing.assert_allclose(rho, 64 / 2 ** 0.5 * a["j"] / 64, rtol=1e-6)
    uv = a["uv"][0] * 64                                                # rows: corners 0, 1, 2 = c, a, b
    np.testing.assert_allclose(uv[1], [P, P])
    np.testing.assert_allclose(uv[2], [P + 2 ** 0.5 * rho, P], rtol=1e-6)
    np.testing.assert_allclose(uv[0], [P + 2 ** -0.5 * rho, P + 2 ** -0.5 * rho], rtol=1e-6)
    assert a["boxes"][0, 2] == np.ceil(np.float32(2 ** 0.5) * rho) + 2 * P


def test_equilateral_triangle_is_isometric():
    s = np.float32(3 ** 0.5 / 2)
    v, f = one([[0, 0, 0], [1, 0, 0], [0.5, s, 0]])
    a = TO.atlas(v, f, 128)
    uv = a["uv"][0].astype(np.float64) * 128
    for i, j in ((0, 1), (1, 2), (2, 0)):
        np.testing.assert_allclose(np.linalg.norm(uv[i] - uv[j]), a["rho"] * np.linalg.norm(v[i] - v[j]), rtol=1e-5)


def test_longest_edge_ties_go_to_the_first():
    v, f = one([[0, 0, 0], [2, 0, 0], [1, 3, 0]])                      # |v1v2|^2 = |v2v0|^2 = 10 > 4
    assert TO.base_corner(v, f).tolist() == [1]
    v, f = one([[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    v2 = v[[1, 2, 0]]                                                  # the same triangle rotated: ties by order
    assert TO.base_corner(v2, f).tolist() == [0]


def test_zero_area_and_collinear_faces_get_minimal_boxes():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 5], [2, 0, 0], [3, 0, 0], [4, 0, 0]], np.float32)
    f = np.array([[0, 1, 2], [3, 3, 3], [4, 5, 6]])
    L, d, h, _ = TO.charts(v, f)
    assert (L[1], d[1], h[1]) == (0, 0, 0) and h[2] == 0 and L[2] == 2 and d[2] == 1
    a = TO.atlas(v, f, 64)
    assert a["boxes"][1, 2:].tolist() == [2 * P, 2 * P] and a["boxes"][2, 3] == 2 * P
    assert np.all(a["uv"][1] * 64 == a["boxes"][1, :2] + P)             # all three corners at the box's inner corner


def test_shelf_positions():
    w = np.array([10, 30, 20, 40, 5, 64])
    hgt = np.array([5, 8, 8, 6, 9, 4])
    ok, x, y = TO.pack(w, hgt, 64)
    # order: 4 (9), 1 (8), 2 (8), 3 (6), 0 (5), 5 (4); shelf 0: 4, 1, 2 (x 0, 5, 35; 55 + 40 > 64), shelf 1 at y = 9: 3,
    # 0 (x 0, 40), shelf 2 at y = 15: 5 (64 wide)
    assert ok
    assert x.tolist() == [40, 5, 35, 0, 0, 0] and y.tolist() == [9, 0, 0, 9, 0, 15]
    assert not TO.pack(w, hgt, 32)[0] and not TO.pack([65], [4], 64)[0]
    assert not TO.pack([64] * 17, [4] * 17, 64)[0] and TO.pack([64] * 16, [4] * 16, 64)[0]


def test_ladder_search():
    assert TO.search(lambda j: j <= 173) == 173
    assert TO.search(lambda j: True) == 256
    assert TO.search(lambda j: j == 1) == 1
    assert TO.search(lambda j: False) is None


def test_infeasible_atlas_is_refused():
    # 200 tiny charts: at j = 1 every box is 5 x 5 and 64^2 texels hold 12 x 12 of them
    k = np.arange(200, dtype=np.float32)[:, None]
    v = np.concatenate([np.concatenate([k, 0 * k, 0 * k], 1), np.concatenate([k + 1e-3, 0 * k, 0 * k], 1),
                        np.concatenate([k, 1e-3 + 0 * k, 0 * k], 1)]).astype(np.float32)
    f = np.stack([np.arange(200), np.arange(200) + 200, np.arange(200) + 400], 1)
    with pytest.raises(ValueError, match="cannot hold 200 charts"):
        TO.atlas(v, f, 64)
    assert TO.atlas(v, f, 128)["j"] >= 1


def test_bad_input_is_refused():
    v, f = one([[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    for N in (32, 100, 16384):
        with pytest.raises(ValueError, match="power of two"):
            TO.atlas(v, f, N)
    with pytest.raises(ValueError, match="outside"):
        TO.atlas(v, np.array([[0, 1, 3]]), 64)
    with pytest.raises(ValueError, match="no area"):
        TO.atlas(np.zeros((3, 3), np.float32), f, 64)


# ----------------------------------------------------------------------------- closest points
def test_closest_point_regions():
    a, b, c = np.array([0.0, 0, 0]), np.array([4.0, 0, 0]), np.array([0.0, 4, 0])
    pts = {0: [-1, -1, 0], 1: [5, -1, 0], 2: [2, -1, 0], 3: [-1, 5, 0], 4: [-1, 2, 0], 5: [3, 3, 0], 6: [1, 1, 0]}
    p = np.array([pts[k] for k in range(7)], np.float64)
    A, B, Cc = (np.repeat(x[None], 7, 0) for x in (a, b, c))
    assert TO.region(p, A, B, Cc).tolist() == list(range(7))
    la, lb, lc = TO.closest_point(p, A, B, Cc)
    q = la[:, None] * A + lb[:, None] * B + lc[:, None] * Cc
    want = np.array([[0, 0, 0], [4, 0, 0], [2, 0, 0], [0, 4, 0], [0, 2, 0], [2, 2, 0], [1, 1, 0]], np.float64)
    np.testing.assert_allclose(q, want, atol=1e-12)
    assert np.all((la >= 0) & (lb >= 0) & (lc >= 0))
    # a degenerate triangle does not divide by zero
    z = np.zeros((1, 3))
    assert [x.tolist() for x in TO.closest_point(np.ones((1, 3)), z, z, z)] == [[1.0], [0.0], [0.0]]


def test_corner_texels_get_the_vertex_exactly():
    v, f = one([[0.1, 0.2, 0.3], [1.7, 0.25, -0.4], [0.6, 1.3, 0.9]])
    a = TO.atlas(v, f, 64)
    t, pts, tf = TO.texel_points(v, f, a["uv"], a["owner"], 64)
    assert (tf == 0).all() and len(t) == np.prod(a["boxes"][0, 2:])
    ix, iy = t % 64, t // 64
    bx, by = a["boxes"][0, :2]
    assert np.array_equal(pts[(ix == bx) & (iy == by)][0], v[f[0, a["k0"][0]]])   # the padding's corner is a


# ----------------------------------------------------------------------------- push-pull
def test_push_pull_2x2_and_4x4():
    # 2 x 2 is below the smallest texture; the rule is the same at any size
    owner = np.array([0, -1, -1, -1])
    tex = TO.fill([0], [[0.2, 0.4, 0.6]], owner, 2)
    assert np.array_equal(tex.reshape(4, 3), np.array([[0.2, 0.4, 0.6]] * 4, np.float32))
    owner = -np.ones(16, np.int64)
    owner[[0, 1, 15]] = 0
    rgb = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    tex = TO.fill([0, 1, 15], rgb, owner, 4).reshape(16, 3)
    assert np.array_equal(tex[[0, 1, 15]], rgb)                         # owned texels unchanged
    q0 = np.float32(0.5)                                                # top-left quadrant: mean of (1,0,0) and (0,1,0)
    for t in (4, 5):
        assert np.array_equal(tex[t], [q0, q0, 0])
    assert np.array_equal(tex[10], [0, 0, 1])                           # bottom-right quadrant: texel 15 only
    top = np.float32(1) / np.float32(3)                                 # empty quadrants: the 1 x 1 mean of all three
    for t in (2, 3, 6, 7, 8, 9, 12, 13):
        assert np.array_equal(tex[t], [top, top, top])


# ----------------------------------------------------------------------------- invariants on the example mesh
@pytest.fixture(scope="module")
def example6996():
    v, _, _ = example_mesh()
    g = np.load(os.path.join(GOLD, "simplify", "backpack_ours_6996.npz"))
    return v[g["vertex_index"]], g["faces"]


def test_oracle_atlas_of_the_example_mesh(example6996):
    v, f = example6996
    N = 1024
    a = TO.atlas(v, f, N)
    b = a["boxes"].astype(np.int64)
    assert (b[:, :2] >= 0).all() and (b[:, 0] + b[:, 2] <= N).all() and (b[:, 1] + b[:, 3] <= N).all()
    cover = np.zeros((N, N), np.int64)
    for x, y, w, h in b.tolist():
        cover[y:y + h, x:x + w] += 1
    assert cover.max() == 1                                              # boxes are disjoint
    assert (a["owner"] >= 0).sum() == cover.sum()
    uv = a["uv"].astype(np.float64) * N
    for i, j in ((0, 1), (1, 2), (2, 0)):
        l3 = np.linalg.norm(v[f[:, i]].astype(np.float64) - v[f[:, j]], axis=1)
        l2 = np.linalg.norm(uv[:, i] - uv[:, j], axis=1)
        # uv is fp32: each end is within half an ulp of 1.0 (N * 2^-24 texels), so 1e-5 relative holds from 16 texels on
        big = l3 * a["rho"] >= 16
        assert big.sum() > 100
        np.testing.assert_allclose(l2[big], a["rho"] * l3[big], rtol=1e-5)
        np.testing.assert_allclose(l2, a["rho"] * l3, rtol=1e-6, atol=4 * N * 2.0 ** -24)
    # every texel whose centre is inside a chart's triangle is owned by that face
    owner = a["owner"].reshape(N, N)
    for fi in range(0, len(f), 7):
        x, y, w, h = b[fi]
        gx, gy = np.meshgrid(np.arange(x, x + w) + 0.5, np.arange(y, y + h) + 0.5)
        p = uv[fi]
        s = [(p[(k + 1) % 3, 0] - p[k, 0]) * (gy - p[k, 1]) - (p[(k + 1) % 3, 1] - p[k, 1]) * (gx - p[k, 0]) for k in range(3)]
        inside = ((s[0] >= 0) & (s[1] >= 0) & (s[2] >= 0)) | ((s[0] <= 0) & (s[1] <= 0) & (s[2] <= 0))
        assert (owner[y:y + h, x:x + w][inside] == fi).all()
    assert 0.3 < (a["owner"] >= 0).mean() <= 1


# ----------------------------------------------------------------------------- writers
def _textured_quad():
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]], np.int64)
    uv = np.array([[[0.1, 0.1], [0.4, 0.1], [0.4, 0.4]], [[0.6, 0.6], [0.9, 0.6], [0.9, 0.9]]], np.float32)
    tex = np.random.default_rng(0).integers(0, 256, (64, 64, 3), dtype=np.uint8)
    return v, f, uv, tex


def test_textured_glb_round_trips(tmp_path):
    from o2345 import mesh_io
    v, f, uv, tex = _textured_quad()
    p = str(tmp_path / "m.glb")
    mesh_io.write_textured_glb(p, v, f, uv, tex)
    g = mesh_io.read_glb(p)
    (m,) = g["meshes"]
    assert len(m["faces"]) == 2 and np.array_equal(m["verts"], v[f.reshape(-1)])
    assert np.array_equal(m["uvs"].astype(np.float32), uv.reshape(-1, 2))
    assert np.array_equal(m["colors"], np.ones((6, 3))) and (m["face_tex"] == 0).all()   # no COLOR_0: white
    rgba, ws, wt = g["textures"][0]
    assert np.array_equal(rgba[..., :3], tex) and (ws, wt) == (1, 1)                      # CLAMP_TO_EDGE
    import json
    import struct
    raw = open(p, "rb").read()
    doc = json.loads(raw[20:20 + struct.unpack_from("<I", raw, 12)[0]])
    assert "COLOR_0" not in doc["meshes"][0]["primitives"][0]["attributes"]
    pbr = doc["materials"][0]["pbrMetallicRoughness"]
    assert pbr["metallicFactor"] == 0 and pbr["roughnessFactor"] == 1
    assert doc["samplers"][0]["magFilter"] == doc["samplers"][0]["minFilter"] == 9729


def test_textured_obj_has_flipped_vt_and_a_material(tmp_path):
    from PIL import Image
    from o2345 import mesh_io
    v, f, uv, tex = _textured_quad()
    p = str(tmp_path / "mesh.obj")
    mesh_io.write_textured_obj(p, v, f, uv, tex)
    lines = open(p).read().splitlines()
    assert "mtllib mesh.mtl" in lines and "usemtl albedo" in lines
    vt = np.array([[float(x) for x in l.split()[1:]] for l in lines if l.startswith("vt ")])
    np.testing.assert_allclose(vt[:, 0], uv.reshape(-1, 2)[:, 0], atol=1e-7)
    np.testing.assert_allclose(vt[:, 1], 1 - uv.reshape(-1, 2)[:, 1].astype(np.float64), atol=1e-7)
    fl = [l for l in lines if l.startswith("f ")]
    assert fl == ["f 1/1 2/2 3/3", "f 1/4 3/5 4/6"]
    assert "map_Kd mesh_albedo.png" in open(tmp_path / "mesh.mtl").read().splitlines()
    assert np.array_equal(np.asarray(Image.open(tmp_path / "mesh_albedo.png")), tex)
    rv, rf, rc = mesh_io.read_obj(p)                                    # read_obj still ignores vt and materials
    assert np.array_equal(rf, f) and rc is None


def test_viewer_frame_flip_keeps_each_uv_with_its_corner():
    from o2345 import mesh_io
    v, f, uv, _ = _textured_quad()
    v2, f2, uv2 = mesh_io.to_viewer_frame(v, f, uv)
    v3, f3 = mesh_io.to_viewer_frame(v, f)
    assert np.array_equal(v2, v3) and np.array_equal(f2, f3)
    for i in range(len(f)):
        for k in range(3):
            k2 = int(np.nonzero(f2[i] == f[i, k])[0][0])
            assert np.array_equal(uv2[i, k2], uv[i, k])


# ----------------------------------------------------------------------------- command lines and the ABI
def test_run_py_texture_arguments():
    import run as run_cli
    a = run_cli.parse_args(["--texture_size", "1024", "--output_format", ".glb"])
    assert a.texture_size == 1024
    assert run_cli.parse_args(["--texture_size", "64", "--output_format", ".obj"]).texture_size == 64
    assert run_cli.parse_args([]).texture_size is None
    for bad in (["--texture_size", "1024"], ["--texture_size", "1024", "--output_format", ".ply"],
                ["--texture_size", "1000", "--output_format", ".glb"], ["--texture_size", "32", "--output_format", ".glb"],
                ["--texture_size", "16384", "--output_format", ".obj"]):
        with pytest.raises(SystemExit):
            run_cli.parse_args(bad)


def test_simplify_mesh_texture_arguments():
    import simplify_mesh as SM
    a = SM.parse_args(["--in", "a.ply", "--out", "b.glb", "--target_faces", "10", "--texture_size", "256"])
    assert a.texture_size == 256
    assert SM.parse_args(["--in", "a.ply", "--out", "b.ply", "--target_faces", "10"]).texture_size is None
    for bad in (["--out", "b.ply", "--texture_size", "256"], ["--out", "b.glb", "--texture_size", "300"]):
        with pytest.raises(SystemExit):
            SM.parse_args(["--in", "a.ply", "--target_faces", "10", *bad])


def test_mesh_texture_size_check():
    from o2345.mesh_texture import check_size
    assert check_size(64) == 64 and check_size(8192) == 8192
    for bad in (0, 32, 96, 16384, 100.5):
        with pytest.raises(ValueError):
            check_size(bad)


def test_texture_abi_checks_return_einval_without_touching_the_gpu():
    from o2345 import _lib
    lib = _lib.load()
    fake = C.c_void_p(0x1000)
    assert lib.o2345_texture_atlas_scratch_bytes(0) == -1 and lib.o2345_texture_atlas_scratch_bytes(10) > 0
    assert lib.o2345_texel_points_scratch_bytes(100) == -1 and lib.o2345_texture_fill_scratch_bytes(32) == -1
    assert lib.o2345_texel_points_scratch_bytes(64) > 0 and lib.o2345_texture_fill_scratch_bytes(64) > 0
    j, rho = C.c_int32(0), C.c_double(0)
    cases = [
        lambda: lib.o2345_texture_atlas(fake, 3, fake, 1, 100, fake, 1 << 20, fake, fake, fake, C.byref(j), C.byref(rho), None),
        lambda: lib.o2345_texture_atlas(None, 3, fake, 1, 64, fake, 1 << 20, fake, fake, fake, None, None, None),
        lambda: lib.o2345_texture_atlas(fake, 3, fake, 1, 64, fake, 8, fake, fake, fake, None, None, None),
        lambda: lib.o2345_texel_points(fake, 3, fake, 1, fake, fake, 16384, fake, 1 << 30, fake, fake, fake, fake, None),
        lambda: lib.o2345_texture_fill(fake, fake, fake, fake, 64, fake, 0, fake, None),
        lambda: lib.o2345_transfer_colors(fake, 3, fake, 1, fake, fake, 0, fake, fake, 10, fake, None),
    ]
    for i, call in enumerate(cases):
        assert call() == -1, (i, _lib.last_error())
        assert len(_lib.last_error()) > 0
