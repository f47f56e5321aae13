"""CPU: the mesh-simplification oracle (oracle/simplify_oracle.py) on hand-built cases with known answers and on the
reference's example mesh, the simplify_mesh.py / run.py command lines and the argument checks of o2345_simplify."""
import ctypes as C
import gzip
import os
import shutil
import sys

import numpy as np
import pytest

from oracle import metrics_oracle as MO
from oracle import simplify_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


# ----------------------------------------------------------------------------- meshes with known answers
def tetrahedron():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    return v, np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)


def grid(n):
    """Flat n x n patch in z = 0 split into 2 n^2 triangles."""
    g = np.arange(n + 1, dtype=np.float32) / np.float32(n)
    v = np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2)
    v = np.concatenate([v, np.zeros((len(v), 1), np.float32)], 1)
    i, j = (a.reshape(-1) for a in np.meshgrid(np.arange(n), np.arange(n), indexing="ij"))
    p = lambda a, b: a * (n + 1) + b
    f = np.concatenate([np.stack([p(i, j), p(i + 1, j), p(i + 1, j + 1)], 1), np.stack([p(i, j), p(i + 1, j + 1), p(i, j + 1)], 1)])
    return v, f.astype(np.int32)


def cube(n):
    """[-1, 1]^3 with every side an n x n grid of triangles, welded, outward winding."""
    from o2345.mesh_io import merge_vertices
    vs, fs, g = [], [], np.linspace(-1, 1, n + 1)
    for ax in range(3):
        for s in (-1.0, 1.0):
            a, b = [k for k in range(3) if k != ax]
            P = np.zeros((n + 1, n + 1, 3))
            P[..., ax] = s
            P[..., a], P[..., b] = np.meshgrid(g, g, indexing="ij")
            gv, gf = grid(n)
            flip = (s > 0) != ((ax % 2) == 0)
            fs.append((gf[:, ::-1] if flip else gf) + sum(len(x) for x in vs))
            vs.append(P.reshape(-1, 3))
    v, f, _ = merge_vertices(np.concatenate(vs), np.concatenate(fs))
    return v.astype(np.float32), f.astype(np.int32)


def sphere(n=600):
    """Convex hull of n Fibonacci points on the unit sphere: closed, genus 0."""
    from scipy.spatial import ConvexHull
    k = np.arange(n) + 0.5
    z, phi = 1 - 2 * k / n, np.pi * (1 + 5 ** 0.5) * k
    r = np.sqrt(1 - z * z)
    v = np.stack([r * np.cos(phi), r * np.sin(phi), z], 1).astype(np.float32)
    return v, ConvexHull(v).simplices.astype(np.int32)


def nonmanifold():
    """A grid with a fin: a third face on the interior edge (40, 41)."""
    v, f = grid(8)
    v = np.concatenate([v, [[0.5, 0.5, 1.0]]]).astype(np.float32)
    return v, np.concatenate([f, [[40, 41, len(v) - 1]]]).astype(np.int32)


def bowtie():
    """Two closed tetrahedra that share vertex 0."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0.3, 0.3, 1], [-1, 0, 0], [0, -1, 0], [-0.3, -0.3, -1]], np.float32)
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3], [0, 4, 5], [0, 6, 4], [0, 5, 6], [4, 6, 5]], np.int32)
    return v, f


def cases():
    """name -> (verts, faces, target): every hand-built case, also run bit for bit on the GPU."""
    tv, tf = tetrahedron()
    return {"tetrahedron": (tv, tf, 0), "grid": (*grid(8), 0), "cube": (*cube(4), 12), "sphere_300": (*sphere(), 300),
            "sphere_101": (*sphere(), 101), "sphere_40": (*sphere(), 40), "nonmanifold": (*nonmanifold(), 0),
            "bowtie": (*bowtie(), 0), "repeated": (tv, np.concatenate([tf, [[0, 0, 1], [2, 3, 3]]]).astype(np.int32), 0)}


def edges(f):
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    return np.unique(e, axis=0, return_counts=True)


def components(nv, f):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    e, _ = edges(f)
    return connected_components(coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(nv, nv)), directed=False)[0]


def check_closed(vertex_index, f, euler):
    """Every edge has two faces, one component, V - E + F = euler."""
    e, cnt = edges(f)
    assert (cnt == 2).all()
    assert components(len(vertex_index), f) == 1
    assert len(vertex_index) - len(e) + len(f) == euler
    assert (np.diff(vertex_index) > 0).all() and np.array_equal(np.unique(f), np.arange(len(vertex_index)))


# ----------------------------------------------------------------------------- the rules on hand-built cases
def test_tetrahedron_has_no_legal_collapse():
    v, f = tetrahedron()
    vi, out, rounds = SO.simplify(v, f, 0)
    assert vi.tolist() == [0, 1, 2, 3] and np.array_equal(out, f) and rounds == 0


def test_flat_patch_keeps_its_boundary_and_loses_its_interior_at_zero_cost():
    v, f = grid(8)
    trace = []
    vi, out, rounds = SO.simplify(v, f, 0, trace=trace)
    boundary = np.nonzero((v[:, 0] == 0) | (v[:, 0] == 1) | (v[:, 1] == 0) | (v[:, 1] == 1))[0]
    assert np.array_equal(vi, boundary) and len(out) == len(boundary) - 2     # a disc triangulated without interior points
    assert all((c == 0).all() for _, _, c in trace) and sum(len(u) for u, _, _ in trace) == 49
    assert (v[vi, 2] == 0).all()
    n = SO.cross(*(v[vi][out[:, k]].astype(np.float64) for k in range(3)))
    assert (n[:, 2] > 0).all() and (n[:, :2] == 0).all()                      # planar, winding kept, nothing flipped


# The cube with 4 x 4 grid sides reduces to its 8 corners; every collapse on the way costs 0 (no corner moves) and the
# 12 faces are frozen here.
CUBE_12 = [[3, 2, 0], [1, 3, 0], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [7, 6, 2], [3, 7, 2], [6, 4, 0], [2, 6, 0],
           [1, 5, 7], [1, 7, 3]]


def test_cube_reduces_to_its_corners_at_zero_cost():
    v, f = cube(4)
    trace = []
    vi, out, rounds = SO.simplify(v, f, 12, trace=trace)
    assert (np.abs(v[vi]) == 1).all(1).all() and len(vi) == 8
    assert all((c == 0).all() for _, _, c in trace)
    assert out.tolist() == CUBE_12
    check_closed(vi, out, 2)


def test_nonmanifold_edge_and_bowtie_vertex_are_locked():
    for (v, f), locked_ids in ((nonmanifold(), [40, 41]), (bowtie(), [0])):
        F = np.asarray(f, np.int64)
        inc, slot, deg = SO.incidence(F, len(v))
        locked, val, _, _ = SO.locks_and_valence(F, len(v), inc, slot, deg)
        interior = ~locked
        assert locked[locked_ids].all()
        vi, out, _ = SO.simplify(v, f, 0)
        assert set(locked_ids) <= set(vi.tolist())
    # bowtie: every other vertex of the two tetrahedra is a closed fan of valence 3
    assert interior[1:].all() and (val[1:] == 3).all() and val[0] == 6


def test_repeated_index_faces_are_dropped_and_bad_input_refused():
    v, f = tetrahedron()
    vi, out, _ = SO.simplify(v, np.concatenate([f, [[0, 0, 1], [2, 3, 3]]]), 0)
    assert np.array_equal(out, f) and len(vi) == 4
    with pytest.raises(ValueError, match="outside"):
        SO.simplify(v, [[0, 1, 4]], 0)
    with pytest.raises(ValueError, match="outside"):
        SO.simplify(v, [[0, -1, 2]], 0)
    bad = v.copy()
    bad[2, 1] = np.inf
    with pytest.raises(ValueError, match="finite"):
        SO.simplify(bad, f, 0)
    with pytest.raises(ValueError):
        SO.simplify(v, f, -1)


@pytest.mark.parametrize("target", [1000, 500, 301, 120, 40])
def test_face_count_stops_at_the_target(target):
    v, f = sphere()
    vi, out, rounds = SO.simplify(v, f, target)
    assert len(out) in (min(target, len(f)), target - 1) and (rounds == 0) == (target >= len(f))
    check_closed(vi, out, 2)


# ----------------------------------------------------------------------------- the reference's example mesh
def example_mesh():
    """backpack_ours.obj as simplify_mesh.py reads it (welded, fp32, the file's own coordinates); also its rig frame."""
    from o2345 import mesh_io
    from o2345 import mesh_metrics as MM
    import tempfile
    d = tempfile.mkdtemp()
    try:
        obj = os.path.join(d, "backpack_ours.obj")
        with gzip.open(os.path.join(GOLD, "render_eval", "backpack_ours.obj.gz"), "rb") as src, open(obj, "wb") as dst:
            shutil.copyfileobj(src, dst)
        v, f, _ = mesh_io.read_obj(obj)
        wv, wf, _ = mesh_io.merge_vertices(v.astype(np.float32), f)
        assert len(wv) == len(v)                      # already welded: indices of the file and of the mesh agree
        return wv.astype(np.float32), wf.astype(np.int32), MM.load_flat(obj)
    finally:
        shutil.rmtree(d, ignore_errors=True)


EXAMPLE_TARGET = 6996                                 # 10 % of 69 960
# oracle/metrics_oracle.py at N = 20 000, seed 0, in the rig frame (largest extent 0.8): the simplified mesh against the
# original, and the control against the original.  The control keeps every rule but replaces the quadric cost by a hash
# of the edge, so no geometry chooses the collapses.  (With every cost 0 the least index absorbs its neighbours about one
# collapse per round: 464 rounds for the 1 180-face sphere, far too many for this mesh.)
N_SCORE, TAUS = 20000, (0.01, 0.005)
SCORE_QEM = {"fscore": {0.01: 0.9851478658072376, 0.005: 0.6505186964374927}, "chamfer": 0.00432553267999027}
SCORE_CONTROL = {"fscore": {0.01: 0.9444347564849127, 0.005: 0.5129018665626981}, "chamfer": 0.005317682607564614}


@pytest.fixture(scope="module")
def example():
    return example_mesh()


def test_example_mesh_at_ten_percent(example):
    v, f, flat = example
    vi, out, rounds = SO.simplify(v, f, EXAMPLE_TARGET)
    gold = np.load(os.path.join(GOLD, "simplify", "backpack_ours_6996.npz"))
    assert np.array_equal(vi, gold["vertex_index"]) and np.array_equal(out, gold["faces"]) and rounds == int(gold["rounds"])
    assert len(out) == EXAMPLE_TARGET
    check_closed(vi, out, -2)
    cvi, cout, _ = SO.simplify(v, f, EXAMPLE_TARGET, random_cost=True)
    assert len(cout) == EXAMPLE_TARGET
    s = MO.score({"verts": flat["verts"][vi], "faces": out}, flat, N_SCORE, TAUS, seed=0)
    z = MO.score({"verts": flat["verts"][cvi], "faces": cout}, flat, N_SCORE, TAUS, seed=0)
    for t in TAUS:
        assert s["fscore"][t]["fscore"] == SCORE_QEM["fscore"][t] and z["fscore"][t]["fscore"] == SCORE_CONTROL["fscore"][t]
        assert s["fscore"][t]["fscore"] > z["fscore"][t]["fscore"]
    assert abs(s["chamfer"] - SCORE_QEM["chamfer"]) < 1e-12 and abs(z["chamfer"] - SCORE_CONTROL["chamfer"]) < 1e-12
    assert s["chamfer"] < z["chamfer"]


# ----------------------------------------------------------------------------- command lines, ABI
def test_command_lines():
    sys.path.insert(0, os.path.join(ROOT, "one-2-3-45_b200"))
    import run
    import simplify_mesh as SM
    a = SM.parse_args(["--in", "a.ply", "--out", "b.glb", "--target_faces", "100"])
    assert (a.inp, a.out, a.target_faces) == ("a.ply", "b.glb", 100)
    assert SM.parse_args(["--in", "a.OBJ", "--out", "b.obj", "--target_faces", "0"]).target_faces == 0
    for bad in (["--in", "a.glb", "--out", "b.ply", "--target_faces", "5"], ["--in", "a.ply", "--out", "b.stl", "--target_faces", "5"],
                ["--in", "a.ply", "--out", "b.ply", "--target_faces", "-1"], ["--in", "a.ply", "--out", "b.ply"],
                ["--in", "a.ply", "--target_faces", "5"], []):
        with pytest.raises(SystemExit):
            SM.parse_args(bad)
    assert run.parse_args([]).target_faces is None and run.parse_args(["--target_faces", "500"]).target_faces == 500
    with pytest.raises(SystemExit):
        run.parse_args(["--target_faces", "-2"])


def test_simplify_refuses_bad_arguments_without_a_device():
    from o2345 import _lib
    lib = _lib.load()
    p = C.c_void_p(0x1000)
    need = lib.o2345_simplify_scratch_bytes(100, 50)
    assert need > 80 * 100 + 3 * 12 * 50
    assert lib.o2345_simplify_scratch_bytes(0, 5) == -1 and lib.o2345_simplify_scratch_bytes(5, 0) == -1
    assert lib.o2345_simplify_scratch_bytes(5, 2 ** 31 // 3 + 1) == -1

    def call(verts=p, nv=100, faces=p, nf=50, target=10, scratch=p, nbytes=need, vi=p, out=p, counts=p):
        return lib.o2345_simplify(verts, nv, faces, nf, target, scratch, nbytes, vi, out, counts, None)
    cases = [dict(verts=None), dict(faces=None), dict(vi=None), dict(out=None), dict(counts=None), dict(nv=0), dict(nf=0),
             dict(nf=-4), dict(target=-1), dict(nbytes=need - 1), dict(scratch=None), dict(scratch=C.c_void_p(0x1008))]
    for i, kw in enumerate(cases):
        assert call(**kw) == -1, (i, _lib.last_error())
        assert "o2345_simplify" in _lib.last_error()
