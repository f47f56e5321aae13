"""CPU tests of ambient occlusion: the model of oracle/ao_oracle.py on the direction table, lone surfaces, closed meshes
with rays aimed exactly through shared edges and vertices, the analytic floor-and-wall scene (and its control), the
t_min / t_max boundaries, degenerate normals and empty inputs; the occlusion texture through the GLB and OBJ writers and
read_glb; the command lines and the ABI checks."""
import ctypes as C
import hashlib
import os
import re

import numpy as np
import pytest

from oracle import ao_oracle as AO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
UP = np.array([0.0, 0.0, 1.0], F32)


# ----------------------------------------------------------------------------- meshes
def quad(a, b, c, d):
    """Two triangles a b c, a c d (counter-clockwise seen from their normal's side)."""
    return [a, b, c, d], [[0, 1, 2], [0, 2, 3]]


def join(*parts):
    vs, fs, n = [], [], 0
    for v, f in parts:
        vs.append(np.asarray(v, F32).reshape(-1, 3))
        fs.append(np.asarray(f, np.int64).reshape(-1, 3) + n)
        n += len(vs[-1])
    return np.concatenate(vs), np.concatenate(fs).astype(np.int32)


def grid(n, x0, x1, y0, y1, z=0.0):
    """An n x n grid of quads on z, normals +z."""
    xs, ys = np.linspace(x0, x1, n + 1), np.linspace(y0, y1, n + 1)
    v = np.stack(np.meshgrid(xs, ys, indexing="ij"), -1).reshape(-1, 2)
    v = np.concatenate([v, np.full((len(v), 1), z)], 1)
    i = np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]
    a, b, c, d = i, i + (n + 1), i + (n + 2), i + 1
    f = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)])
    return v.astype(F32), f.astype(np.int32)


def floor_and_wall(x_wall=0.5, n=8):
    """A floor [x_wall - 2, x_wall] x [-1, 1] at z = 0 (normals +z) and a wall at x = x_wall, y in [-1, 1], z in [0, 1]
    (normal -x): box diagonal 3, so t_max = 0.3 and t_min = 0.003."""
    floor = grid(n, x_wall - 2.0, x_wall, -1.0, 1.0)
    wall = quad([x_wall, -1, 0], [x_wall, -1, 1], [x_wall, 1, 1], [x_wall, 1, 0])
    return join(floor, wall)


def octahedron(r=1.0):
    v = np.array([[r, 0, 0], [-r, 0, 0], [0, r, 0], [0, -r, 0], [0, 0, r], [0, 0, -r]], F32)
    f = [[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]]
    return v, np.array(f, np.int32)


def icosphere(level=2, r=1.0):
    t = (1 + 5 ** 0.5) / 2
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
         [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7],
         [9, 8, 1]]
    v = [np.array(p, float) / np.linalg.norm(p) for p in v]
    for _ in range(level):
        mid, nf = {}, []

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[k] = len(v) - 1
            return mid[k]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return (np.array(v) * r).astype(F32), np.array(f, np.int32)


def half_plane_discrepancy(dirs):
    """sup over a of | #{k: d_k.x >= a} / K - S(a) |, S(a) = (acos a - a sqrt(1 - a^2)) / pi the cosine-weighted share of
    the hemisphere with x >= a (the disk's area beyond the chord x = a, over pi).  The count steps at the table's x
    values and S is continuous and decreasing, so the supremum is taken at a step, on either side of it."""
    x = np.sort(dirs[:, 0].astype(np.float64))[::-1]
    K = len(x)
    S = (np.arccos(x) - x * np.sqrt(1 - x * x)) / np.pi
    j = np.arange(1, K + 1)
    return float(max(np.abs(j / K - S).max(), np.abs((j - 1) / K - S).max()))


def wall_ao(a):
    """The analytic AO of a point on the floor at distance a t_max from the wall (0 < a <= 1)."""
    return 1.0 - (np.arccos(a) - a * np.sqrt(1.0 - a * a)) / np.pi


# hand cases shared with the GPU tests: name -> (verts, faces, points, normals, dirs or None, t_min or None, t_max or None)
def hand_cases():
    cases = {}
    v, f = join(quad([-1, -1, 0], [1, -1, 0], [1, 1, 0], [-1, 1, 0]), quad([-1, -1, -1], [1, -1, -1], [1, 1, -1], [-1, 1, -1]))
    rng = np.random.default_rng(1)
    p = np.concatenate([rng.uniform(-0.5, 0.5, (16, 2)), np.zeros((16, 1))], 1).astype(F32)
    cases["lone_plane"] = (v, f, p, np.tile(UP, (16, 1)), None, None, None)
    v, f = icosphere(2)
    d = rng.standard_normal((24, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    cases["convex_outside"] = (v, f, (1.05 * d).astype(F32), d.astype(F32), None, None, None)
    v, f = octahedron()
    aim = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]] +
                   [[sx, sy, 0] for sx in (1, -1) for sy in (1, -1)] + [[sx, 0, sz] for sx in (1, -1) for sz in (1, -1)] +
                   [[0, sy, sz] for sy in (1, -1) for sz in (1, -1)], F32)
    cases["octahedron_aimed"] = (v, f, np.zeros((1, 3), F32), UP[None], aim, 1e-3, 4.0)
    pin = rng.uniform(-0.2, 0.2, (16, 3)).astype(F32)
    nin = rng.standard_normal((16, 3)).astype(F32)
    cases["octahedron_inside"] = (v, f, pin, nin, None, 1e-3, 4.0)
    v, f = icosphere(2)
    cases["icosphere_vertices_aimed"] = (v, f, np.zeros((1, 3), F32), UP[None], v.copy(), 1e-3, 4.0)
    v, f = floor_and_wall()
    ds = np.array([0.01, 0.03, 0.06, 0.1, 0.15, 0.2, 0.25, 0.29, 0.31, 0.4], F32)
    p = np.stack([0.5 - ds, np.linspace(-0.3, 0.3, len(ds)), np.zeros(len(ds))], 1).astype(F32)
    cases["floor_and_wall"] = (v, f, p, np.tile(UP, (len(ds), 1)), None, None, None)
    v, f = join(quad([-1, -1, 0.5], [1, -1, 0.5], [1, 1, 0.5], [-1, 1, 0.5]))
    cases["t_boundaries"] = (v, f, np.array([[0.25, 0.125, 0.0]], F32), UP[None], np.array([[0, 0, 1]], F32), None, None)
    v, f = octahedron()
    bad = np.array([[0, 0, 0], [np.nan, 0, 1], [np.inf, 0, 0], [1e-30, 0, 0], [0, 0, 1]], F32)
    pts = np.array([[0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0], [np.nan, 0, 0]], F32)
    cases["degenerate_normals"] = (v, f, pts, bad, None, 1e-3, 4.0)
    return cases


def run_case(case, **kw):
    v, f, p, n, dirs, t0, t1 = case
    return AO.ambient_occlusion(v, f, p, n, dirs=dirs, t_min=t0, t_max=t1)


# ----------------------------------------------------------------------------- the rule
def test_direction_table():
    from o2345 import mesh_texture as MT
    d = AO.directions()
    assert d.dtype == F32 and d.shape == (256, 3) and np.array_equal(d, MT.ao_directions())
    assert MT.AO_RAYS == AO.RAYS and MT.AO_T_MIN == AO.T_MIN and MT.AO_T_MAX == AO.T_MAX
    assert np.abs(np.linalg.norm(d.astype(np.float64), axis=1) - 1).max() < 2 ** -22     # unit to fp32
    assert (d[:, 2] > 0).all()
    # z_k = sqrt(1 - u_k), u_k = (k + 1/2) / K: the midpoint rule for the integral of sqrt(1 - u) over [0, 1] = 2/3.  By
    # Koksma-Hlawka the error is at most the variation of sqrt(1 - u) (1) times the star discrepancy of the midpoints
    # (1 / (2K)).
    assert abs(d[:, 2].astype(np.float64).mean() - 2 / 3) <= 1 / (2 * 256)


def test_distances_follow_the_box_diagonal():
    from o2345 import mesh_texture as MT
    v, _ = floor_and_wall()
    assert AO.diagonal(v) == 3.0
    assert AO.distances(v) == (F32(0.003), F32(0.3)) and MT.ao_distances(v) == AO.distances(v)
    assert MT.ao_distances(np.zeros((0, 3))) == (0.0, 0.0)


def test_lone_surfaces_are_open():
    cases = hand_cases()
    assert (run_case(cases["lone_plane"]) == 1).all()
    assert (run_case(cases["convex_outside"]) == 1).all()


def test_every_ray_from_inside_a_closed_mesh_hits():
    cases = hand_cases()
    assert (run_case(cases["octahedron_inside"]) == 0).all()
    assert (run_case(cases["octahedron_aimed"]) == 0).all()
    assert (run_case(cases["icosphere_vertices_aimed"]) == 0).all()


@pytest.mark.parametrize("name", ["octahedron", "icosphere"])
def test_rays_exactly_through_shared_edges_and_vertices_hit(name):
    """From the centre, rays exactly through every vertex (and, on the octahedron, every edge midpoint): each one hits,
    whatever the watertight test's edge functions decide between the faces that share the edge or vertex."""
    v, f = octahedron() if name == "octahedron" else icosphere(2)
    aim = hand_cases()["octahedron_aimed"][4] if name == "octahedron" else v
    pad = F32(F32(AO.diagonal(v)) * AO.PAD_SCALE)
    corners, lo, hi = AO.face_boxes(v, f, pad)
    assert AO.any_hit(np.zeros(3, F32), aim, corners, lo, hi, 1e-3, 4.0).all()
    # ... and face by face, each exact vertex ray is accepted by faces around that vertex only
    hits = np.stack([AO.any_hit(np.zeros(3, F32), v, corners[g:g + 1], lo[g:g + 1], hi[g:g + 1], 1e-3, 4.0)
                     for g in range(len(f))], 1)
    for i in range(len(v)):
        assert hits[i].any() and all(i in f[g] for g in np.flatnonzero(hits[i])), (i, np.flatnonzero(hits[i]))


def test_floor_and_wall_match_the_analytic_share_within_the_discrepancy():
    v, f, p, n, _, _, _ = hand_cases()["floor_and_wall"]
    got = run_case(hand_cases()["floor_and_wall"])
    t_max = AO.distances(v)[1]
    disc = half_plane_discrepancy(AO.directions())
    print(f"half-plane discrepancy of the 256-direction table: {disc:.5f}")
    assert disc < 0.02                       # under 5 of the 256 rays
    d = 0.5 - p[:, 0].astype(np.float64)
    for di, g in zip(d, got):
        want = wall_ao(di / float(t_max)) if di < t_max else 1.0
        assert abs(float(g) - want) <= disc + 1e-6, (di, g, want)
    # the control: the wall beyond t_max leaves the floor open
    assert (got[d > float(t_max)] == 1).all() and (got[d < 0.25] < 0.95).all()


def test_t_min_and_t_max_are_inclusive():
    """A plane at z = 0.5 above the point, the ray straight up: T = det / 2 exactly (a power of two), so the hit at
    t = 0.5 counts for t_max = 0.5 and t_min = 0.5 and not for either moved past it."""
    v, f, p, n, dirs, _, _ = hand_cases()["t_boundaries"]
    ao = lambda t0, t1: AO.ambient_occlusion(v, f, p, n, dirs=dirs, t_min=t0, t_max=t1)[0]
    lo, hi = F32(0.5 * (1 - 2 ** -20)), F32(0.5 * (1 + 2 ** -20))
    assert ao(0.001, 0.5) == 0 and ao(0.5, 0.5) == 0 and ao(0.001, 1.0) == 0
    assert ao(0.001, lo) == 1 and ao(hi, 1.0) == 1


def test_degenerate_and_non_finite_normals_and_points_give_one():
    # inside a closed octahedron every ray hits, but a zero, non-finite or underflowing normal or a NaN point gives 1
    got = run_case(hand_cases()["degenerate_normals"])
    np.testing.assert_array_equal(got, np.ones(5, F32))


def test_empty_inputs():
    v, f = octahedron()
    assert AO.ambient_occlusion(v, f, np.zeros((0, 3)), np.zeros((0, 3))).shape == (0,)
    got = AO.ambient_occlusion(v, f[:0], np.zeros((3, 3)), np.tile(UP, (3, 1)), t_min=0.0, t_max=1.0)
    np.testing.assert_array_equal(got, np.ones(3, F32))


# ----------------------------------------------------------------------------- writers and reader
def _textured(seed=0):
    rng = np.random.default_rng(seed)
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0.5]], F32)
    f = np.array([[0, 1, 2], [1, 3, 2]], np.int32)
    uv = rng.uniform(0, 1, (2, 3, 2)).astype(F32)
    tex = rng.integers(0, 256, (64, 64, 3), dtype=np.uint8)
    nrm = rng.integers(0, 256, (64, 64, 3), dtype=np.uint8)
    occ = rng.integers(0, 256, (64, 64), dtype=np.uint8)
    return v, f, uv, tex, nrm, occ


def _sha(paths):
    h = hashlib.sha256()
    for p in paths:
        h.update(open(p, "rb").read())
    return h.hexdigest()


# sha256 of the writers' files for _textured(0) before the occlusion texture existed
BYTES_BEFORE = {
    "glb": "93bd38255c1f1d9436d0da7b8d09ecf9ab803a17ef1f6ddb6484554ac1e89e92",
    "glb_normal": "30ed6479d053144eb4d89a94db9d798b9d7e3a24ac583fdcbaa0aa0d5aadf93e",
    "obj": "c6ce960400da6c5de491f4abf6b75d49144dff060e22885d347e1e7fddca3aa2",
    "obj_normal": "584d86d9c5c145f68de2b10832955c9f39d132a50b1386d737a74e1715a173b8",
}


def test_writers_without_occlusion_are_unchanged(tmp_path):
    from o2345 import mesh_io
    v, f, uv, tex, nrm, _ = _textured()
    for key, nt in (("", None), ("_normal", nrm)):
        p = str(tmp_path / f"m{key}.glb")
        mesh_io.write_textured_glb(p, v, f, uv, tex, nt)
        assert _sha([p]) == BYTES_BEFORE["glb" + key]
        p = str(tmp_path / f"m{key}.obj")
        mesh_io.write_textured_obj(p, v, f, uv, tex, nt)
        stem = p[:-4]
        files = [p, stem + ".mtl", stem + "_albedo.png"] + ([stem + "_normal.png"] if nt is not None else [])
        assert _sha(files) == BYTES_BEFORE["obj" + key]
        assert not os.path.exists(stem + "_occlusion.png")


@pytest.mark.parametrize("with_normal", [False, True])
def test_glb_round_trips_the_occlusion_texture(tmp_path, with_normal):
    from o2345 import mesh_io
    v, f, uv, tex, nrm, occ = _textured()
    p = str(tmp_path / "m.glb")
    mesh_io.write_textured(p, v, f, uv, tex, nrm if with_normal else None, occ)
    g = mesh_io.read_glb(p)
    m = g["meshes"][0]
    assert (m["face_otex"] == m["face_otex"][0]).all() and m["face_otex"][0] >= 0
    rgba = g["textures"][m["face_otex"][0]][0]
    np.testing.assert_array_equal(rgba[..., 0], occ)
    np.testing.assert_array_equal(g["textures"][m["face_tex"][0]][0][..., :3], tex)
    if with_normal:
        np.testing.assert_array_equal(g["textures"][m["face_ntex"][0]][0][..., :3], nrm)
    mesh_io.write_textured(p, v, f, uv, tex)
    assert (mesh_io.read_glb(p)["meshes"][0]["face_otex"] == -1).all()


def test_obj_writes_the_occlusion_png_and_map_ao(tmp_path):
    from PIL import Image
    from o2345 import mesh_io
    v, f, uv, tex, nrm, occ = _textured()
    p = str(tmp_path / "m.obj")
    mesh_io.write_textured(p, v, f, uv, tex, nrm, occ)
    mtl = open(str(tmp_path / "m.mtl")).read()
    assert "map_ao m_occlusion.png\n" in mtl and "norm m_normal.png\n" in mtl
    np.testing.assert_array_equal(np.asarray(Image.open(str(tmp_path / "m_occlusion.png"))), occ)


# ----------------------------------------------------------------------------- command lines and the ABI
def test_command_lines_refuse_ambient_occlusion_without_texture_size(capsys):
    import run
    import simplify_mesh
    with pytest.raises(SystemExit):
        run.parse_args(["--ambient_occlusion"])
    with pytest.raises(SystemExit):
        simplify_mesh.parse_args(["--in", "a.ply", "--out", "b.glb", "--target_faces", "10", "--ambient_occlusion"])
    assert "--ambient_occlusion needs --texture_size" in capsys.readouterr().err


def test_command_lines_take_ambient_occlusion():
    import run
    import simplify_mesh
    a = run.parse_args(["--ambient_occlusion", "--texture_size", "512", "--output_format", ".glb"])
    assert a.ambient_occlusion and run._texture_kw(a) == {"texture_size": 512, "ambient_occlusion": True}
    assert "ambient_occlusion" not in run._texture_kw(run.parse_args([]))
    b = simplify_mesh.parse_args(["--in", "a.ply", "--out", "b.glb", "--target_faces", "10", "--texture_size", "64",
                                  "--ambient_occlusion"])
    assert b.ambient_occlusion


def test_pipeline_refuses_ambient_occlusion_without_texture_size():
    from o2345.pipeline import _simplify_kw
    assert _simplify_kw(None, 256, ambient_occlusion=True) == {"texture_size": 256, "ambient_occlusion": True}
    assert "ambient_occlusion" not in _simplify_kw(None, 256)


def test_ao_entry_points_are_declared_and_bound():
    from o2345 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "o2345.h")).read(), flags=re.S)
    assert re.search(r"\bint o2345_ambient_occlusion\s*\(", src)
    assert re.search(r"\bint64_t o2345_ambient_occlusion_scratch_bytes\s*\(", src)
    for name in ("o2345_ambient_occlusion", "o2345_ambient_occlusion_scratch_bytes"):
        assert name in _lib.EXPORTED
    assert "0x1p-13f" in open(os.path.join(ROOT, "one-2-3-45_b200", "csrc", "ao.cu")).read() and AO.PAD_SCALE == 2.0 ** -13


def test_ao_abi_checks_return_einval_without_touching_the_gpu():
    from o2345 import _lib
    lib = _lib.load()
    fake = C.c_void_p(0x1000)                                   # never dereferenced: the checks fail first
    nb = lib.o2345_ambient_occlusion_scratch_bytes(10, 10)
    assert nb > 0 and lib.o2345_ambient_occlusion_scratch_bytes(-1, 10) == -1
    assert lib.o2345_ambient_occlusion_scratch_bytes(10, -1) == -1 and lib.o2345_ambient_occlusion_scratch_bytes(0, 0) > 0

    def call(nv=10, nf=10, n=4, k=256, t0=0.01, t1=1.0, scratch=fake, nbytes=nb, verts=fake, dirs=fake):
        return lib.o2345_ambient_occlusion(verts, nv, fake, nf, fake, fake, n, dirs, k, t0, t1, scratch, nbytes, fake, None)
    for case in (dict(nv=-1), dict(nf=-1), dict(n=-1), dict(k=0), dict(t0=-0.1), dict(t0=2.0), dict(t1=float("nan")),
                 dict(t1=float("inf")), dict(nbytes=nb - 1), dict(scratch=None), dict(scratch=C.c_void_p(0x1004)),
                 dict(verts=None), dict(dirs=None)):
        assert call(**case) == -1, case
        assert _lib.last_error().startswith("o2345_ambient_occlusion"), case
