"""CPU tests of mesh cleaning: the model of oracle/clean_oracle.py on hand cases (a small distant sphere, a bubble in
either orientation, a sphere in a torus's hole, a bowtie, a tie, zero-area faces, empty meshes, unreferenced vertices),
its partition against scipy's connected components and its enclosure decisions against a ray-parity count, the example
mesh left as it is, the command lines and the ABI checks."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle import clean_oracle as CO
from test_simplify_host import example_mesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ----------------------------------------------------------------------------- meshes
def icosphere(r=1.0, centre=(0.0, 0.0, 0.0), level=2, flip=False, grid=None):
    """A closed icosphere, outward faces (inward with flip); grid: positions rounded to multiples of 1 / grid first, so
    a translated copy has bit-identical edge vectors."""
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
    v = np.array(v) * r
    if grid:
        v = np.round(v * grid) / grid
    f = np.array(f, np.int32)
    return (v + np.asarray(centre)).astype(np.float32), (f[:, ::-1] if flip else f).copy()


def torus(R=1.0, r=0.3, n=32, m=16):
    i, j = np.meshgrid(np.arange(n), np.arange(m), indexing="ij")
    u, w = 2 * np.pi * i / n, 2 * np.pi * j / m
    v = np.stack([(R + r * np.cos(w)) * np.cos(u), (R + r * np.cos(w)) * np.sin(u), r * np.sin(w)], -1).reshape(-1, 3)
    idx = lambda a, b: (a % n) * m + (b % m)
    f = []
    for a in range(n):
        for b in range(m):
            f += [[idx(a, b), idx(a + 1, b), idx(a + 1, b + 1)], [idx(a, b), idx(a + 1, b + 1), idx(a, b + 1)]]
    return v.astype(np.float32), np.array(f, np.int32)


def tetra(centre, s=1.0):
    v = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], float) * s + centre
    return v.astype(np.float32), np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]], np.int32)


def join(*meshes):
    vs, fs, n = [], [], 0
    for v, f in meshes:
        vs.append(v), fs.append(f + n)
        n += len(v)
    return np.concatenate(vs).astype(np.float32), np.concatenate(fs).astype(np.int32)


def bowtie():
    """Two tetrahedra sharing one vertex (index 0 of both)."""
    (v1, f1), (v2, f2) = tetra((0, 0, 0)), tetra((0, 0, 0))
    v2 = -v2 + 2 * v1[0]                       # point reflection through v1[0]: v2[0] == v1[0]
    v = np.concatenate([v1, v2[1:]]).astype(np.float32)
    f2 = np.where(f2 == 0, 0, f2 + 3)
    return v, np.concatenate([f1, f2[:, ::-1]]).astype(np.int32)


def degenerate(centre, n=3):
    """n faces of zero area: collinear corners and a repeated corner."""
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [0, 1, 0]], float) * 0.1 + centre
    f = np.array([[0, 1, 2], [1, 2, 0], [3, 3, 0]][:n], np.int32)
    return v.astype(np.float32), f


HAND = {
    "far_small": lambda: join(icosphere(1.0), icosphere(0.1, (3, 0, 0))),
    "bubble_out": lambda: join(icosphere(1.0), icosphere(0.5, (0.1, 0, 0))),
    "bubble_in": lambda: join(icosphere(1.0), icosphere(0.5, (0.1, 0, 0), flip=True)),
    "bubble_both_in": lambda: join(icosphere(1.0, flip=True), icosphere(0.5, (0.1, 0, 0), flip=True)),
    "torus_hole": lambda: join(torus(), icosphere(0.1, level=1)),
    "bowtie": bowtie,
    "tie": lambda: join(icosphere(1.0, grid=1024), icosphere(1.0, (4, 0, 0), grid=1024)),
    "zero_area": lambda: join(icosphere(1.0), degenerate((3, 0, 0))),
    "zero_largest": lambda: join(degenerate((0, 0, 0)), degenerate((3, 0, 0), 2)),
    "unreferenced": lambda: (np.concatenate([icosphere(1.0)[0], np.full((3, 3), 5, np.float32)]), icosphere(1.0)[1]),
}


def run(name, F):
    v, f = HAND[name]()
    return v, f, CO.clean_mesh(v, f, F)


def kept_components(out):
    return list(np.flatnonzero(out["keep"]))


# ----------------------------------------------------------------------------- hand cases
@pytest.mark.parametrize("F, kept", [(0.02, [0]), (0.005, [0, 1])])
def test_small_distant_sphere_goes_by_area(F, kept):
    v, f, out = run("far_small", F)
    assert len(out["area"]) == 2 and out["largest"] == 0
    assert abs(out["area"][1] / out["area"][0] - 0.01) < 1e-6
    assert kept_components(out) == kept and out["enclosed"] == 0
    assert abs(out["winding"][1]) < 1e-3


@pytest.mark.parametrize("name", ["bubble_out", "bubble_in", "bubble_both_in"])
@pytest.mark.parametrize("F", [1e-6, 0.5, 1.0])
def test_bubble_is_dropped_at_every_F_in_either_orientation(name, F):
    v, f, out = run(name, F)
    assert out["largest"] == 0 and kept_components(out) == [0] and out["enclosed"] == 1
    assert abs(abs(out["winding"][1]) - 1.0) < 1e-9         # +1 or -1 with the outer sphere's orientation
    np.testing.assert_array_equal(out["faces"], f[:len(icosphere()[1])])
    np.testing.assert_array_equal(out["vertex_index"], np.arange(len(icosphere()[0])))


def test_sphere_in_the_hole_of_a_torus_is_kept():
    v, f, out = run("torus_hole", 0.005)
    tv = torus()[0]
    assert np.all(np.abs(v[-1]) < tv.max(0))                 # inside the torus's bounding box ...
    assert out["largest"] == 0 and abs(out["winding"][1]) < 1e-9   # ... but not enclosed
    assert kept_components(out) == [0, 1] and out["enclosed"] == 0


def test_bowtie_vertex_joins_its_two_fans():
    v, f, out = run("bowtie", 1.0)
    assert len(out["area"]) == 1 and list(out["label"]) == [0] * 8
    np.testing.assert_array_equal(out["faces"], f)


def test_equal_areas_tie_to_the_least_face_and_both_stay():
    v, f, out = run("tie", 1.0)
    assert out["area"][0] == out["area"][1] and out["largest"] == 0
    assert kept_components(out) == [0, 1]
    np.testing.assert_array_equal(out["faces"], f)


def test_zero_area_component_goes_for_every_F():
    for F in (1e-9, 1.0):
        v, f, out = run("zero_area", F)
        assert out["area"][1] == 0.0 and kept_components(out) == [0]


def test_zero_area_largest_keeps_every_component_that_is_not_enclosed():
    v, f, out = run("zero_largest", 1.0)
    assert list(out["area"]) == [0.0, 0.0] and out["largest"] == 0
    assert list(out["winding"]) == [0.0, 0.0] and kept_components(out) == [0, 1]


def test_unreferenced_vertices_are_dropped():
    v, f, out = run("unreferenced", 0.5)
    np.testing.assert_array_equal(out["vertex_index"], np.arange(len(v) - 3))
    np.testing.assert_array_equal(out["faces"], f)


def test_empty_mesh():
    out = CO.clean_mesh(np.zeros((4, 3), np.float32), np.zeros((0, 3), np.int32), 0.5)
    assert len(out["area"]) == 0 and out["largest"] == -1
    assert out["vertex_index"].shape == (0,) and out["faces"].shape == (0, 3)


def test_components_are_numbered_by_least_face():
    (va, fa), (vb, fb) = icosphere(0.2, (3, 0, 0), level=1), icosphere(1.0, level=1)
    v, f = join((va, fa), (vb, fb))
    f = np.concatenate([f[:5], f[len(fa):len(fa) + 3], f[5:len(fa)], f[len(fa) + 3:]])   # interleaved
    out = CO.clean_mesh(v, f, 0.5)
    assert list(out["label"][:10]) == [0] * 5 + [1] * 3 + [0] * 2
    assert out["largest"] == 1 and kept_components(out) == [1]
    np.testing.assert_array_equal(out["vertex_index"], np.arange(len(va), len(v)))


# ----------------------------------------------------------------------------- the model's pieces
def test_atan2_matches_numpy_to_a_few_ulp():
    rng = np.random.default_rng(0)
    y, x = rng.standard_normal(20000) * 10.0 ** rng.integers(-5, 5, 20000), rng.standard_normal(20000)
    y = np.concatenate([y, [0.0, 0.0, 1.0, -1.0, 1.0, 0.0]])
    x = np.concatenate([x, [0.0, -1.0, 0.0, 0.0, 1.0, 1.0]])
    a, want = CO.atan2(y, x), np.arctan2(y, x)
    assert np.all(np.abs(a - want) <= 4 * np.spacing(np.abs(want) + 1e-300))
    assert CO.atan2(0.0, 0.0) == 0.0 and CO.atan2(0.0, -1.0) == CO.PI


def test_ordered_sum_is_chunked_and_sequential():
    rng = np.random.default_rng(1)
    x = rng.random(3000) * 10.0 ** rng.integers(-8, 8, 3000)
    want, run_ = 0.0, 0.0
    for k in range(0, len(x), CO.CHUNK):
        s = 0.0
        for t in x[k:k + CO.CHUNK]:
            s += t
        run_ += s
    assert CO.ordered_sum(x) == run_ and CO.ordered_sum([]) == 0.0


def _random_meshes():
    rng = np.random.default_rng(2)
    for nv, nf in ((30, 12), (200, 90), (500, 400), (50, 1)):
        v = rng.standard_normal((nv, 3)).astype(np.float32)
        yield v, rng.integers(0, nv, (nf, 3)).astype(np.int32)
    yield HAND["bowtie"]()
    yield HAND["torus_hole"]()


def test_partition_equals_scipy_connected_components():
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    for v, f in _random_meshes():
        label, heads = CO.components(len(v), f)
        e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
        g = coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(len(v), len(v)))
        _, lab = connected_components(g, directed=False)
        comp = lab[f[:, 0]]
        # the same partition of the faces ...
        assert len(np.unique(comp)) == len(heads)
        for c in range(len(heads)):
            assert len(np.unique(comp[label == c])) == 1
        # ... numbered by least face
        assert np.all(np.diff(heads) > 0) and np.all(label[heads] == np.arange(len(heads)))
        assert all(label[:heads[c]].max(initial=-1) < c for c in range(len(heads)))


def _ray_parity(v, f, p, d):
    """Crossings of the ray p + t d (t > 0) with triangles v[f] (Moeller-Trumbore), mod 2."""
    a, b, c = v[f[:, 0]].astype(float), v[f[:, 1]].astype(float), v[f[:, 2]].astype(float)
    e1, e2 = b - a, c - a
    h = np.cross(d, e2)
    det = (e1 * h).sum(1)
    s = p - a
    u = (s * h).sum(1) / det
    q = np.cross(s, e1)
    w = (d * q).sum(1) / det
    t = (e2 * q).sum(1) / det
    return int(np.sum((u >= 0) & (w >= 0) & (u + w <= 1) & (t > 0))) % 2


@pytest.mark.parametrize("name", ["far_small", "bubble_out", "bubble_in", "bubble_both_in", "torus_hole", "tie"])
def test_enclosure_equals_a_ray_parity_count(name):
    v, f, out = run(name, 1e-6)
    L = out["largest"]
    lf = f[out["label"] == L]
    d = np.array([0.3141, 0.5926, 0.7419])
    for c in range(len(out["area"])):
        if c != L:
            p = CO.centroid(v, f[np.flatnonzero(out["label"] == c)[0]])
            assert (abs(out["winding"][c]) >= 0.5) == bool(_ray_parity(v, lf, p, d / np.linalg.norm(d))), c


@pytest.mark.parametrize("F", [1e-6, 0.05, 1.0])
def test_example_mesh_is_returned_unchanged(F):
    v, f, _ = example_mesh()
    out = CO.clean_mesh(v, f, F)
    assert len(out["area"]) == 1 and out["enclosed"] == 0
    np.testing.assert_array_equal(out["vertex_index"], np.arange(len(v)))
    np.testing.assert_array_equal(out["faces"], f)


# ----------------------------------------------------------------------------- command lines and the ABI
@pytest.mark.parametrize("bad", ["0", "-0.1", "1.5", "nan"])
def test_command_lines_refuse_min_component_outside_0_1(bad, capsys):
    import run
    import simplify_mesh
    with pytest.raises(SystemExit):
        run.parse_args(["--min_component", bad])
    with pytest.raises(SystemExit):
        simplify_mesh.parse_args(["--in", "a.ply", "--out", "b.ply", "--target_faces", "10", "--min_component", bad])
    assert "--min_component must lie in (0, 1]" in capsys.readouterr().err


def test_command_lines_take_min_component():
    import run
    import simplify_mesh
    a = run.parse_args(["--min_component", "0.05", "--img_path", "a.png", "b.png"])
    assert a.min_component == 0.05 and run._texture_kw(a) == {"min_component": 0.05}
    assert run.parse_args([]).min_component is None and "min_component" not in run._texture_kw(run.parse_args([]))
    b = simplify_mesh.parse_args(["--in", "a.ply", "--out", "b.ply", "--target_faces", "10", "--min_component", "1"])
    assert b.min_component == 1.0


def test_clean_entry_points_are_declared_and_bound():
    from o2345 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "o2345.h")).read(), flags=re.S)
    assert re.search(r"\bint o2345_clean_mesh\s*\(", src) and re.search(r"\bint64_t o2345_clean_mesh_scratch_bytes\s*\(", src)
    for name in ("o2345_clean_mesh", "o2345_clean_mesh_scratch_bytes"):
        assert name in _lib.EXPORTED
    assert CO.CHUNK == 1024


def test_clean_abi_checks_return_einval_without_touching_the_gpu():
    from o2345 import _lib
    lib = _lib.load()
    fake = C.c_void_p(0x1000)                                   # never dereferenced: the checks fail first
    counts = (C.c_int32 * 6)()
    nb = lib.o2345_clean_mesh_scratch_bytes(10, 10)
    assert nb > 0 and lib.o2345_clean_mesh_scratch_bytes(0, 10) == -1 and lib.o2345_clean_mesh_scratch_bytes(10, 0) == -1

    def call(nv=10, nf=10, F=0.5, scratch=fake, nbytes=nb, verts=fake):
        return lib.o2345_clean_mesh(verts, nv, fake, nf, F, scratch, nbytes, fake, fake, fake, fake, fake, fake, counts, None)
    for case in (dict(F=0.0), dict(F=-1.0), dict(F=1.5), dict(F=float("nan")), dict(nv=0), dict(nf=0),
                 dict(nbytes=nb - 1), dict(scratch=None), dict(verts=None), dict(scratch=C.c_void_p(0x1004))):
        assert call(**case) == -1, case
        assert _lib.last_error().startswith("o2345_clean_mesh"), case
