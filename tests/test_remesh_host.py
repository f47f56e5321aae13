"""CPU tests of isotropic remeshing: the model of oracle/remesh_oracle.py on one hand case per step (split rounds on a
long strip, a fan of short edges, a quad flip that helps and one that would fold, relaxation of a lifted grid vertex),
closest points against the search over all faces on ties, a lat-long sphere to several targets (topology, distance to
the input, face count, quality against the input and against a control without relaxation and flips), a torus, an open
grid's boundary, a bowtie, empty / degenerate / zero-target inputs and refused inputs; the command lines and the ABI."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle import remesh_oracle as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


# ----------------------------------------------------------------------------- meshes
def uv_sphere(nlat=12, nlon=24):
    """A lat-long unit sphere: poles with fans of nlon thin triangles, the rest quads split on one diagonal."""
    v = [[0.0, 0.0, 1.0]]
    for i in range(1, nlat):
        th = np.pi * i / nlat
        for j in range(nlon):
            ph = 2 * np.pi * j / nlon
            v.append([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
    v.append([0.0, 0.0, -1.0])
    f = [[0, 1 + j, 1 + (j + 1) % nlon] for j in range(nlon)]
    for i in range(nlat - 2):
        for j in range(nlon):
            a, b = 1 + i * nlon + j, 1 + i * nlon + (j + 1) % nlon
            f += [[a, a + nlon, b + nlon], [a, b + nlon, b]]
    s = len(v) - 1
    base = 1 + (nlat - 2) * nlon
    f += [[base + j, s, base + (j + 1) % nlon] for j in range(nlon)]
    return np.asarray(v, F32), np.asarray(f, np.int32)


def torus(n=24, m=12, R0=1.0, r=0.35):
    u, w = np.meshgrid(np.arange(n), np.arange(m), indexing="ij")
    a, b = 2 * np.pi * u / n, 2 * np.pi * w / m
    v = np.stack([(R0 + r * np.cos(b)) * np.cos(a), (R0 + r * np.cos(b)) * np.sin(a), r * np.sin(b)], -1).reshape(-1, 3)
    idx = lambda i, j: (i % n) * m + (j % m)
    f = []
    for i in range(n):
        for j in range(m):
            f += [[idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)], [idx(i, j), idx(i + 1, j + 1), idx(i, j + 1)]]
    return v.astype(F32), np.asarray(f, np.int32)


def grid(n, size=1.0):
    xs = np.linspace(0.0, size, n + 1)
    v = np.stack(np.meshgrid(xs, xs, indexing="ij"), -1).reshape(-1, 2)
    v = np.concatenate([v, np.zeros((len(v), 1))], 1).astype(F32)
    i = np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]
    a, b, c, d = i, i + n + 1, i + n + 2, i + 1
    f = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)])
    return v, f.astype(np.int32)


def strip(length=8.0):
    """Two triangles spanning a 1 x length rectangle."""
    v = np.array([[0, 0, 0], [length, 0, 0], [length, 1, 0], [0, 1, 0]], F32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def edges(f):
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    return np.unique(e, axis=0)


def euler(v, f):
    used = np.unique(f)
    return len(used) - len(edges(f)) + len(f)


def components(f):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    e = edges(f)
    n = int(f.max()) + 1
    g = coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(n, n))
    _, lab = connected_components(g, directed=False)
    return len(np.unique(lab[np.unique(f)]))


def boundary_edges(f):
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    u, c = np.unique(e, axis=0, return_counts=True)
    return u[c == 1]


def quality(v, f):
    """-> (share of faces with min angle < 20 deg, share with q < 0.5, share of valence-6 vertices, min angle)."""
    v = v.astype(np.float64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    ar = 0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1)
    e2 = ((b - a) ** 2).sum(1) + ((c - b) ** 2).sum(1) + ((a - c) ** 2).sum(1)
    q = 4 * np.sqrt(3) * ar / np.maximum(e2, 1e-300)

    def ang(p, q_, r):
        x, y = q_ - p, r - p
        cs = (x * y).sum(1) / np.maximum(np.linalg.norm(x, axis=1) * np.linalg.norm(y, axis=1), 1e-300)
        return np.degrees(np.arccos(np.clip(cs, -1, 1)))
    mina = np.minimum(np.minimum(ang(a, b, c), ang(b, c, a)), ang(c, a, b))
    val = np.bincount(edges(f).ravel(), minlength=len(v))
    return float((mina < 20).mean()), float((q < 0.5).mean()), float((val[val > 0] == 6).mean()), float(mina.min())


def hand_cases():
    """name -> (verts, faces, L, iterations): the inputs the GPU test repeats."""
    sv, sf = uv_sphere()
    tv, tf = torus()
    gv, gf = grid(6)
    lifted = gv.copy()
    lifted[3 * 7 + 3, 2] = 0.2
    fan_v = [[0.0, 0.0, 0.0]] + [[0.05 * np.cos(t), 0.05 * np.sin(t), 0.0] for t in np.linspace(0, 2 * np.pi, 9)[:-1]]
    fan_v += [[np.cos(t), np.sin(t), 0.0] for t in np.linspace(0, 2 * np.pi, 9)[:-1]]
    fan_f = [[0, 1 + k, 1 + (k + 1) % 8] for k in range(8)]
    fan_f += [[1 + k, 9 + k, 1 + (k + 1) % 8] for k in range(8)] + [[1 + (k + 1) % 8, 9 + k, 9 + (k + 1) % 8] for k in range(8)]
    bow_v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [-1, 0, 0], [-1, -1, 0]], F32)
    bow_f = np.array([[0, 1, 2], [0, 3, 4]], np.int32)
    return {
        "strip": (*strip(), F32(1.0), 1),
        "fan": (np.asarray(fan_v, F32), np.asarray(fan_f, np.int32), F32(0.8), 1),
        "lifted_grid": (lifted, gf, F32(1 / 6), 2),
        "sphere_200": (sv, sf, R.target_length(sv, sf, 200)[0], 5),
        "sphere_2000": (sv, sf, R.target_length(sv, sf, 2000)[0], 5),
        "torus": (tv, tf, R.target_length(tv, tf, 300)[0], 5),
        "open_grid": (gv, gf, R.target_length(gv, gf, 150)[0], 5),
        "bowtie": (bow_v, bow_f, F32(0.3), 3),
    }


# ----------------------------------------------------------------------------- one step at a time
def test_a_long_strip_splits_over_several_rounds():
    v, f = strip()
    ov, of, rounds = R.remesh(v, f, F32(1.0), iterations=1, relax=False, flip=False, project=False)
    assert rounds[0] >= 3
    ln = np.linalg.norm(ov[edges(of)[:, 0]] - ov[edges(of)[:, 1]], axis=1)
    assert ln.max() <= 4 / 3 + 1e-6
    assert np.isclose(abs(np.cross(ov[of[:, 1]] - ov[of[:, 0]], ov[of[:, 2]] - ov[of[:, 0]])[:, 2]).sum() / 2, 8.0)
    assert euler(ov, of) == 1


def test_a_fan_of_short_edges_collapses():
    v, f, L, _ = hand_cases()["fan"]
    ov, of, rounds = R.remesh(v, f, L, iterations=1, relax=False, flip=False, project=False)
    assert rounds[0] == 0 and rounds[1] >= 1 and len(of) < len(f)
    assert (np.linalg.norm(ov, axis=1) < 0.1).sum() < 9          # the centre and its ring of 8 lost vertices
    assert len(boundary_edges(of)) == 8                 # the outer octagon is locked and kept


def test_flips_lower_the_valence_deviation_without_folding():
    v, f = uv_sphere()
    F = f.astype(np.int64)
    dev = lambda F: ((np.bincount(edges(F).ravel(), minlength=len(v)) - 6) ** 2).sum()
    f2, did = R._flip_round(v, F)
    assert did and dev(f2) < dev(F)
    V = v.astype(np.float64)
    n = np.cross(V[f2[:, 1]] - V[f2[:, 0]], V[f2[:, 2]] - V[f2[:, 0]])
    assert ((n * V[f2].mean(1)).sum(1) > 0).all()              # every face still faces outwards
    assert euler(v, f2) == 2
    # one flip the round takes: its quad a, b (the old edge), c, d (the new one); its endpoints have valence >= 4
    new = {tuple(x) for x in edges(f2)} - {tuple(x) for x in edges(F)}
    c, d = sorted(new)[0]
    quad = [x for x in F if c in x or d in x]
    a, b = [x for x in set(np.concatenate([q for q in quad if c in q and d not in q or d in q and c not in q]).tolist())
            if x not in (c, d) and sum((x in q) for q in quad) >= 2][:2]
    val = np.bincount(edges(F).ravel(), minlength=len(v))
    assert val[a] >= 4 and val[b] >= 4
    # a moved to the middle of triangle c d b: the quad is concave at a, so the flip to cd would fold, and the round
    # refuses it although its valence gain is unchanged
    V2 = v.copy()
    V2[a] = (v[c] + v[d] + v[b]) / F32(3)
    f3, _ = R._flip_round(V2, F)
    assert (min(c, d), max(c, d)) not in {tuple(x) for x in edges(f3)}


def test_relaxation_moves_a_vertex_towards_its_neighbours_within_the_plane():
    v, f, L, it = hand_cases()["lifted_grid"]
    out, locked = R._relax(v, f.astype(np.int64))
    i = 3 * 7 + 3
    assert not locked[i] and out[i, 2] == v[i, 2]             # the normal component stays: only the tangent moves
    g = v.copy()
    g[:, 2] = 0
    g[i, :2] += F32(0.06)
    out, _ = R._relax(g, f.astype(np.int64))
    assert (out[:, 2] == 0).all() and np.linalg.norm(out[i, :2] - [0.5, 0.5]) < np.linalg.norm(g[i, :2] - [0.5, 0.5])


# ----------------------------------------------------------------------------- closest point
def tie_case():
    """Two coplanar triangles sharing an edge, a duplicate of the second, and points on the shared edge, at shared
    vertices, in the duplicated face and above them."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]], F32)
    f = np.array([[0, 1, 2], [1, 3, 2], [1, 3, 2], [2, 1, 3]], np.int32)
    p = np.array([[0.5, 0.5, 0], [0.5, 0.5, 1], [1, 0, 0], [0, 1, 0.5], [0.75, 0.75, 0], [0.75, 0.75, -2],
                  [2, 2, 0], [-1, -1, 0], [0.25, 0.25, 0]], F32)
    return v, f, p


def test_closest_points_break_ties_by_the_least_face():
    v, f, p = tie_case()
    q, face = R.closest_points(v, f, p, brute=True)
    assert face.tolist() == [0, 0, 0, 0, 1, 1, 1, 0, 0]
    qa, fa = R.closest_points(v, f, p)
    np.testing.assert_array_equal(q.view(np.uint32), qa.view(np.uint32))
    np.testing.assert_array_equal(face, fa)


def test_closest_points_candidate_search_equals_the_full_search():
    v, f = uv_sphere(20, 40)
    p = np.random.default_rng(1).normal(size=(800, 3)).astype(F32) * F32(1.3)
    p = np.concatenate([p, v[:50], (v[f[:40, 0]] + v[f[:40, 1]]) * F32(0.5)])
    a, fa = R.closest_points(v, f, p)
    b, fb = R.closest_points(v, f, p, brute=True)
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))
    np.testing.assert_array_equal(fa, fb)
    assert (np.abs(np.linalg.norm(a, axis=1) - 1) < 0.02).all()


# ----------------------------------------------------------------------------- whole meshes
# frozen from the oracle's own runs of the sphere (min angle < 20 deg share, q < 0.5 share, valence-6 share)
SPHERE_BOUNDS = {200: (0.005, 0.005, 0.70), 1000: (0.005, 0.005, 0.70), 3000: (0.005, 0.005, 0.70)}


@pytest.mark.parametrize("N", sorted(SPHERE_BOUNDS))
def test_sphere_remesh_is_closed_close_and_better_than_input_and_control(N):
    v, f = uv_sphere()
    L, _ = R.target_length(v, f, N)
    ov, of, _ = R.remesh(v, f, L)
    assert euler(ov, of) == 2 and components(of) == 1 and len(boundary_edges(of)) == 0
    a, b, c = ov[of[:, 0]].astype(np.float64), ov[of[:, 1]].astype(np.float64), ov[of[:, 2]].astype(np.float64)
    assert (np.linalg.norm(np.cross(b - a, c - a), axis=1) > 0).all()
    q, _ = R.closest_points(v, f, ov)
    assert np.abs(q - ov).max() <= 4 * np.finfo(F32).eps                  # every vertex is on the input surface
    assert 0.7 * N <= len(of) <= 1.5 * N
    lo20, q05, val6 = SPHERE_BOUNDS[N]
    got = quality(ov, of)
    inp = quality(v, f)
    assert got[0] <= lo20 and got[1] <= q05 and got[2] >= val6
    assert got[0] < inp[0] and got[1] < inp[1] and got[3] > inp[3]   # (the input is valence 6 off the poles)
    cv, cf, _ = R.remesh(v, f, L, relax=False, flip=False)
    ctl = quality(cv, cf)
    assert not (ctl[0] <= lo20 and ctl[1] <= q05 and ctl[2] >= val6)


def test_torus_keeps_its_genus():
    v, f, L, it = hand_cases()["torus"]
    ov, of, _ = R.remesh(v, f, L, it)
    assert euler(ov, of) == 0 and components(of) == 1 and len(boundary_edges(of)) == 0


def test_open_grid_keeps_its_boundary_and_its_boundary_vertices():
    v, f, L, it = hand_cases()["open_grid"]
    ov, of, _ = R.remesh(v, f, L, it)
    be = boundary_edges(of)
    assert len(be) > 0 and euler(ov, of) == 1
    # every input boundary vertex is still there, bit for bit, and every output boundary vertex lies on the square
    bin_ = np.unique(boundary_edges(f))
    out = {tuple(x) for x in ov.view(np.uint32)[np.unique(be)]}
    assert all(tuple(x) in out for x in v.view(np.uint32)[bin_])
    pb = ov[np.unique(be)]
    assert (np.isclose(pb[:, 0], 0) | np.isclose(pb[:, 0], 1) | np.isclose(pb[:, 1], 0) | np.isclose(pb[:, 1], 1)).all()


def test_a_bowtie_vertex_stays_locked():
    v, f, L, it = hand_cases()["bowtie"]
    ov, of, _ = R.remesh(v, f, L, it)
    assert any((ov == v[0]).all(1))
    assert euler(ov, of) == len(np.unique(of)) - len(edges(of)) + len(of)


def test_empty_degenerate_and_zero_target_inputs():
    ov, of, r = R.remesh(np.zeros((0, 3), F32), np.zeros((0, 3), np.int32), F32(1.0))
    assert len(ov) == 0 and len(of) == 0
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0]], F32)        # collinear: no area
    ov, of, _ = R.remesh(v, np.array([[0, 1, 2], [0, 0, 1]], np.int32), F32(1.0))
    assert len(of) >= 1 and np.isfinite(ov).all() and (ov[:, 1:] == 0).all()
    sv, sf = uv_sphere()
    L, _ = R.target_length(sv, sf, 0)
    assert L == np.inf
    ov, of, _ = R.remesh(sv, sf, L)
    assert euler(ov, of) == 2 and len(of) < len(sf)


def test_bad_inputs_are_refused():
    v, f = strip()
    with pytest.raises(ValueError):
        R.remesh(v, np.array([[0, 1, 7]]), F32(1))
    bad = v.copy()
    bad[0, 0] = np.nan
    with pytest.raises(ValueError):
        R.remesh(bad, f, F32(1))
    with pytest.raises(ValueError):
        R.remesh(v, f, F32(0))


def test_target_length_matches_the_equilateral_formula():
    v, f = grid(4, 2.0)
    L, A = R.target_length(v, f, 100)
    assert np.isclose(A, 4.0) and L == F32(np.sqrt(4 * 4.0 / (np.sqrt(3) * 100)))
    from o2345 import mesh_remesh
    assert mesh_remesh.target_length(v, f, 100) == (L, A)
    assert mesh_remesh.REMESH_ITERATIONS == R.ITERATIONS == 5


# ----------------------------------------------------------------------------- command lines and the ABI
def test_simplify_mesh_takes_remesh():
    import simplify_mesh
    b = simplify_mesh.parse_args(["--in", "a.ply", "--out", "b.glb", "--target_faces", "10", "--remesh"])
    assert b.remesh and not simplify_mesh.parse_args(["--in", "a.ply", "--out", "b.glb", "--target_faces", "10"]).remesh


def test_run_py_takes_remesh_and_needs_target_faces(capsys):
    import run
    with pytest.raises(SystemExit):
        run.parse_args(["--remesh"])
    assert "--remesh needs --target_faces" in capsys.readouterr().err
    a = run.parse_args(["--remesh", "--target_faces", "5000"])
    assert a.remesh and run._texture_kw(a) == {"remesh": True}
    assert "remesh" not in run._texture_kw(run.parse_args(["--target_faces", "5000"]))


def test_pipeline_passes_remesh_only_with_target_faces():
    from o2345.pipeline import _simplify_kw
    assert _simplify_kw(100, remesh=True) == {"target_faces": 100, "remesh": True}
    assert "remesh" not in _simplify_kw(100)
    with pytest.raises(ValueError):
        _simplify_kw(None, remesh=True)


def test_remesh_wrapper_returns_degenerate_meshes_without_unreferenced_vertices():
    from o2345 import mesh_remesh
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [5, 5, 5]], F32)      # collinear, and one unreferenced vertex
    ov, of, st = mesh_remesh.remesh(v, np.array([[0, 1, 2], [0, 0, 1]], np.int32), None, 10)
    assert len(ov) == 3 and of.tolist() == [[0, 1, 2]] and st["rounds"] == (0, 0, 0)


def test_remesh_entry_points_are_declared_and_bound():
    from o2345 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "o2345.h")).read(), flags=re.S)
    for name in ("o2345_remesh", "o2345_closest_points"):
        assert re.search(r"\bint %s\s*\(" % name, src)
        assert re.search(r"\bint64_t %s_scratch_bytes\s*\(" % name, src)
        assert name in _lib.EXPORTED and name + "_scratch_bytes" in _lib.EXPORTED
    assert re.search(r"#define O2345_ENOSPC \(-4\)", src) and _lib.ENOSPC == -4
    assert re.search(r"#define O2345_ABI_VERSION 14\b", src) and _lib.ABI_VERSION == 14


def test_remesh_abi_checks_fail_without_touching_the_gpu():
    from o2345 import _lib
    lib = _lib.load()
    fake = C.c_void_p(0x1000)                                   # never dereferenced: the checks fail first
    assert lib.o2345_remesh_scratch_bytes(10, 10, 20, 20) > 0
    assert lib.o2345_remesh_scratch_bytes(10, 10, 5, 20) == -1 and lib.o2345_remesh_scratch_bytes(0, 10, 10, 10) == -1
    assert lib.o2345_closest_points_scratch_bytes(0, 0) > 0 and lib.o2345_closest_points_scratch_bytes(-1, 0) == -1
    counts = (C.c_int64 * 5)()
    assert lib.o2345_remesh(fake, 10, fake, 10, 1.0, 5, 5, 20, fake, 1 << 20, fake, fake, counts, None) == _lib.ENOSPC
    assert counts[0] == 10 and counts[1] == 10
    assert lib.o2345_remesh(fake, 10, fake, 10, 0.0, 5, 10, 10, fake, 1 << 20, fake, fake, counts, None) == -1
    assert lib.o2345_remesh(fake, 10, fake, 10, 1.0, -1, 10, 10, fake, 1 << 20, fake, fake, counts, None) == -1
    assert lib.o2345_closest_points(fake, 10, fake, 10, fake, 5, fake, 0, fake, fake, None) == -1
