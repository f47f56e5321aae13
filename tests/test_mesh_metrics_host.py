"""CPU: the mesh-scoring oracle (oracle/metrics_oracle.py) on hand-computed cases and on the reference's example pair,
the eval_mesh.py command line, and the argument checks of o2345_surface_sample / o2345_nearest."""
import ctypes as C
import gzip
import os
import shutil
import sys

import numpy as np
import pytest

from o2345 import mesh_metrics as MM
from oracle import metrics_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "render_eval")
TRI = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)


# ----------------------------------------------------------------------------- sampling
def test_samples_of_a_right_triangle_stay_inside_and_centre_on_the_centroid():
    n = 20000
    p, f = MO.surface_sample(TRI, [[0, 1, 2]], n, seed=3)
    assert p.dtype == np.float32 and (f == 0).all() and (p[:, 2] == 0).all()
    assert (p[:, :2] >= 0).all() and (p[:, 0].astype(np.float64) + p[:, 1] <= 1 + 1e-6).all()
    # x and y of a uniform point on this triangle have mean 1/3 and variance 1/18: 5 standard errors of the mean
    assert np.abs(p[:, :2].mean(0) - 1 / 3).max() < 5 * np.sqrt(1 / 18 / n)


def test_sample_counts_follow_the_areas():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0], [5, 0, 0], [8, 0, 0], [5, 2, 0]], np.float32)    # areas 1 and 3
    n = 40000
    _, f = MO.surface_sample(v, [[0, 1, 2], [3, 4, 5]], n, seed=0)
    # binomial(n, 1/4): standard deviation sqrt(n * 3/16) = 87; allow 5 of them
    assert abs(int((f == 0).sum()) - n / 4) < 5 * np.sqrt(n * 3 / 16)


def test_zero_area_and_bad_index_faces_get_no_samples():
    v = np.concatenate([TRI, [[2, 2, 2], [3, 3, 3]]]).astype(np.float32)
    faces = [[0, 0, 1], [3, 4, 9], [0, 1, 2], [-1, 1, 2], [3, 3, 4], [0, 1, 5], [2, 1, 0]]
    w = MO.surface_weights(v, faces)
    assert w.tolist() == [0, 0, 1, 0, 0, 0, 1]
    _, f = MO.surface_sample(v, faces, 5000, seed=1)
    assert set(np.unique(f)) == {2, 6}
    with pytest.raises(ValueError):
        MO.surface_sample(v, [[0, 0, 1], [0, 1, 7]], 10)


def test_chunked_cdf_and_seeds():
    w = np.random.default_rng(0).uniform(size=2500)
    cdf, total = MO.surface_cdf(w)
    np.testing.assert_allclose(cdf, np.cumsum(w), rtol=1e-13)
    assert total == cdf[-1] and (np.diff(cdf) >= 0).all()
    assert cdf[1023] == np.cumsum(w[:1024])[-1] and cdf[1024] == cdf[1023] + w[1024]
    a, _ = MO.surface_sample(TRI, [[0, 1, 2]], 100, seed=0)
    b, _ = MO.surface_sample(TRI, [[0, 1, 2]], 100, seed=1)
    assert np.array_equal(a, MO.surface_sample(TRI, [[0, 1, 2]], 100, seed=0)[0]) and not np.array_equal(a, b)
    u = MO.uniforms(2 ** 64 - 1, np.arange(10000, dtype=np.uint64))
    assert u.min() >= 0 and u.max() < 1 and abs(u.mean() - 0.5) < 0.02


# ----------------------------------------------------------------------------- distances and scores
def lattice(n, step):
    g = np.arange(n, dtype=np.float32) * np.float32(step)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)


def test_identical_clouds_score_one_and_zero():
    p = np.random.default_rng(0).uniform(size=(500, 3)).astype(np.float32)
    d2, idx = MO.nearest(p, p)
    assert (d2 == 0).all() and (idx == np.arange(500)).all()
    s = MO.fscore_chamfer(d2, d2, (0.01, 0.05))
    assert s["chamfer"] == 0 and all(v["fscore"] == 1 for v in s["fscore"].values())


@pytest.mark.parametrize("delta,step,fscore", [(0.03125, 0.125, 1.0), (0.0625, 0.25, 0.0)])
def test_shifted_lattice(delta, step, fscore):
    a = lattice(6, step)
    b = a + np.array([delta, 0, 0], np.float32)
    d_ab, i_ab = MO.nearest(a, b)
    d_ba, _ = MO.nearest(b, a)
    assert (i_ab == np.arange(len(a))).all()
    s = MO.fscore_chamfer(d_ab, d_ba, (0.05,))
    assert s["fscore"][0.05]["fscore"] == fscore and s["chamfer"] == delta


def test_f_is_zero_without_matches_and_ties_go_to_the_lower_index():
    s = MO.fscore_chamfer(np.ones(4, np.float32), np.ones(3, np.float32), (0.5,))
    assert s["fscore"][0.5] == {"precision": 0, "recall": 0, "fscore": 0.0, "n_precise": 0, "n_recalled": 0}
    ref = np.array([[-1, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0]], np.float32)
    d2, idx = MO.nearest(np.array([[0, 0, 0], [-1, 0, 0], [0.5, 0.5, 0]], np.float32), ref, chunk=2)
    assert idx.tolist() == [0, 0, 1] and d2.tolist() == [1, 0, 0.5]
    # the squares are compared in fp32: a distance equal to tau is not within tau
    t = np.float32(0.05 * 0.05)
    s = MO.fscore_chamfer(np.array([t], np.float32), np.array([np.nextafter(t, 0)], np.float32), (0.05,))
    assert s["fscore"][0.05]["n_precise"] == 0 and s["fscore"][0.05]["n_recalled"] == 1


# oracle/metrics_oracle.py on the reference's example pair (backpack_ours.obj against backpack_gt.glb, both in the rig
# frame), N = 20 000, seed 0, tau = 0.05: 18 021 of the predicted and 18 244 of the GT samples lie within tau, F = 0.90659,
# chamfer = 0.022769.  With the OBJ loaded without the Y-up -> Z-up change: F = 0.47481, chamfer = 0.056314.
PAIR_N, PAIR_TAU = 20000, 0.05
PAIR_MEASURED = {"n_precise": 18021, "n_recalled": 18244, "fscore": 0.9065907183234524, "chamfer": 0.02276941382568176}
PAIR_WRONG_AXIS = {"fscore": 0.4748118768096868, "chamfer": 0.056314087903429524}


@pytest.fixture(scope="module")
def pair(tmp_path_factory):
    obj = str(tmp_path_factory.mktemp("pair") / "backpack_ours.obj")
    with gzip.open(os.path.join(GOLD, "backpack_ours.obj.gz"), "rb") as src, open(obj, "wb") as dst:
        shutil.copyfileobj(src, dst)
    return {"gt": os.path.join(GOLD, "backpack_gt.glb"), "ours": obj}


def test_example_pair_through_the_oracle(pair):
    gt = MM.load_flat(pair["gt"])
    s = MO.score(MM.load_flat(pair["ours"]), gt, PAIR_N, (PAIR_TAU,), seed=0)
    f = s["fscore"][PAIR_TAU]
    assert f["n_precise"] == PAIR_MEASURED["n_precise"] and f["n_recalled"] == PAIR_MEASURED["n_recalled"]
    assert f["fscore"] == PAIR_MEASURED["fscore"] and abs(s["chamfer"] - PAIR_MEASURED["chamfer"]) < 1e-12
    # negative control: the wrong axis convention scores far lower
    w = MO.score(MM.load_flat(pair["ours"], y_up=False), gt, PAIR_N, (PAIR_TAU,), seed=0)
    assert w["fscore"][PAIR_TAU]["fscore"] == PAIR_WRONG_AXIS["fscore"]
    assert w["fscore"][PAIR_TAU]["fscore"] < f["fscore"] - 0.3 and w["chamfer"] > 2 * s["chamfer"]


# ----------------------------------------------------------------------------- command line, ABI
def test_command_line():
    sys.path.insert(0, os.path.join(ROOT, "one-2-3-45_b200"))
    import eval_mesh as EM
    a = EM.parse_args(["--pred", "a.obj", "--gt", "a.glb"])
    assert (a.n_points, a.threshold, a.seed, a.clip_ckpt, a.resolution, a.camera_dist, a.out) == \
        (100000, [0.05], 0, None, 512, 1.3, None)
    a = EM.parse_args(["--pred", "a.obj", "b.PLY", "--gt", "a.glb", "b.glb", "--threshold", "0.02", "0.05", "--n_points", "7"])
    assert a.pred == ["a.obj", "b.PLY"] and a.threshold == [0.02, 0.05] and a.n_points == 7
    for bad in (["--pred", "a.obj", "b.obj", "--gt", "a.glb"], ["--pred", "a.fbx", "--gt", "a.glb"],
                ["--pred", "a.obj", "--gt", "a.stl"], ["--pred", "a.obj", "--gt", "a.glb", "--n_points", "0"],
                ["--pred", "a.obj", "--gt", "a.glb", "--threshold", "-1"], ["--pred", "a.obj", "--gt", "a.glb", "--resolution", "0"],
                ["--pred", "a.obj", "--gt", "a.glb", "--camera_dist", "0"], ["--pred", "a.obj"], []):
        with pytest.raises(SystemExit):
            EM.parse_args(bad)
    s = {"fscore": {0.05: {"precision": 0.5, "recall": 1.0, "fscore": 2 / 3}}, "chamfer": 0.25}
    assert EM.line("x", s, [0.05]) == "x: F@0.05=0.666667 P=0.500000 R=1.000000 chamfer=0.250000"
    m = EM.mean_scores([s, {**s, "chamfer": 0.75}], [0.05])
    assert m["chamfer"] == 0.5 and m["fscore"][0.05]["fscore"] == 2 / 3 and "clip" not in m


def test_metrics_refuse_bad_arguments_without_a_device():
    from o2345 import _lib
    lib = _lib.load()
    f = C.c_void_p(0x1000)
    need_s = lib.o2345_surface_sample_scratch_bytes(10)
    need_n = lib.o2345_nn_scratch_bytes(100, 50)
    assert need_s == 8 * (10 + 1 + 1) and lib.o2345_surface_sample_scratch_bytes(0) == -1
    assert need_n > 16 * 100 and lib.o2345_nn_scratch_bytes(0, 5) == -1 and lib.o2345_nn_scratch_bytes(5, 0) == -1

    def sample(verts=f, nv=3, faces=f, nf=10, n=5, scratch=f, nbytes=need_s, pts=f, fid=f):
        return lib.o2345_surface_sample(verts, nv, faces, nf, n, 0, scratch, nbytes, pts, fid, None)

    def nearest(ref=f, nr=100, query=f, nq=50, scratch=f, nbytes=need_n, d2=f, idx=f):
        return lib.o2345_nearest(ref, nr, query, nq, scratch, nbytes, d2, idx, None)
    cases = [(sample, dict(verts=None)), (sample, dict(faces=None)), (sample, dict(pts=None)), (sample, dict(fid=None)),
             (sample, dict(nv=0)), (sample, dict(nf=0)), (sample, dict(n=0)), (sample, dict(n=-3)),
             (sample, dict(nbytes=need_s - 1)), (sample, dict(scratch=None)), (sample, dict(scratch=C.c_void_p(0x1004))),
             (nearest, dict(ref=None)), (nearest, dict(query=None)), (nearest, dict(d2=None)), (nearest, dict(idx=None)),
             (nearest, dict(nr=0)), (nearest, dict(nq=0)), (nearest, dict(nbytes=need_n - 1)), (nearest, dict(scratch=None)),
             (nearest, dict(scratch=C.c_void_p(0x1008)))]
    for i, (fn, kw) in enumerate(cases):
        assert fn(**kw) == -1, (i, _lib.last_error())
        assert ("o2345_surface_sample" if fn is sample else "o2345_nearest") in _lib.last_error()
