"""CPU: the multi-face chart atlas (oracle/chart_atlas_oracle.py, the rules of o2345_chart_atlas) on hand-built meshes
with known answers, its invariants checked by independent means on the frozen 10 % example mesh, and the --atlas
command-line flags."""
import os
import sys

import numpy as np
import pytest

from oracle import chart_atlas_oracle as CA
from test_simplify_host import GOLD, ROOT, example_mesh

PKG = os.path.join(ROOT, "one-2-3-45_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)


# ----------------------------------------------------------------------------- hand meshes
def grid(n=6, scale=0.25):
    x, y = np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing="xy")
    v = np.stack([x.ravel() * scale, y.ravel() * scale, np.zeros(x.size)], 1).astype(np.float32)
    f = []
    for j in range(n):
        for i in range(n):
            a = j * (n + 1) + i
            f += [[a, a + 1, a + n + 2], [a, a + n + 2, a + n + 1]]
    return v, np.array(f, np.int64)


def cube():
    v = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32)
    quads = [[0, 1, 3, 2], [4, 6, 7, 5], [0, 4, 5, 1], [2, 3, 7, 6], [0, 2, 6, 4], [1, 5, 7, 3]]
    f = []
    for a, b, c, d in quads:
        f += [[a, b, c], [a, c, d]]
    return v, np.array(f, np.int64)


def octahedron():
    v = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)
    f = [[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]]
    return v, np.array(f, np.int64)


def helicoid(turns=1.5, n=36):
    """A strip winding around z more than once, slowly rising: every face's normal is closest to +z, so the label alone
    makes one chart, and the projection overlaps itself."""
    t = np.linspace(0, 2 * np.pi * turns, int(n * turns) + 1)
    inner = np.stack([np.cos(t), np.sin(t), 0.02 * t], 1)
    outer = np.stack([2 * np.cos(t), 2 * np.sin(t), 0.02 * t], 1)
    v = np.concatenate([inner, outer]).astype(np.float32)
    m = len(t)
    f = []
    for i in range(m - 1):
        f += [[i, m + i, m + i + 1], [i, m + i + 1, i + 1]]
    return v, np.array(f, np.int64)


def fin():
    """Three faces on one edge (0, 1): non-manifold, so it cuts even between faces of one label."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0.5, 1, 0], [0.5, -1, 0], [0.5, 0.3, 0.01]], np.float32)
    return v, np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4]], np.int64)


def bowtie():
    """Two fans sharing only vertex 0: two charts."""
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [-1, 0, 0], [-1, -1, 0]], np.float32)
    return v, np.array([[0, 1, 2], [0, 3, 4]], np.int64)


def degenerate():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [2, 0, 0], [3, 0, 0]], np.float32)
    # a good pair, a face with a repeated index on the pair's edge and a zero-area line
    return v, np.array([[0, 1, 2], [1, 3, 2], [1, 2, 2], [1, 4, 5]], np.int64)


HAND = {"grid": (grid, 256), "cube": (cube, 128), "octahedron": (octahedron, 128), "helicoid": (helicoid, 512),
        "fin": (fin, 64), "bowtie": (bowtie, 64), "degenerate": (degenerate, 64)}


def hand_case(name):
    make, N = HAND[name]
    v, f = make()
    return v, f, N


# ----------------------------------------------------------------------------- rules on hand meshes
def test_flat_grid_is_one_chart_with_uv_its_xy_scaled():
    v, f, N = hand_case("grid")
    r = CA.atlas(v, f, N)
    assert r["charts"] == 1 and r["rounds"] == 0 and (r["chart"] == 0).all() and (r["label"] == 4).all()
    x, y, w, h = r["boxes"][0]
    want_u = (x + CA.PAD + (v[f][:, :, 0].astype(np.float64) - 0.0) * r["rho"]) / N
    want_v = (y + CA.PAD + v[f][:, :, 1].astype(np.float64) * r["rho"]) / N
    assert np.array_equal(r["uv"][..., 0], want_u.astype(np.float32))
    assert np.array_equal(r["uv"][..., 1], want_v.astype(np.float32))
    # every texel centre strictly inside the grid's square is covered
    own = r["owner"].reshape(N, N)
    assert (own[y + CA.PAD + 1:y + h - CA.PAD - 1, x + CA.PAD + 1:x + w - CA.PAD - 1] >= 0).all()


def test_cube_gives_six_charts_one_per_side():
    v, f, N = hand_case("cube")
    r = CA.atlas(v, f, N)
    assert r["charts"] == 6 and r["rounds"] == 0
    assert sorted(np.unique(r["label"]).tolist()) == [0, 1, 2, 3, 4, 5]
    for c in np.unique(r["chart"]):
        assert len(np.unique(r["label"][r["chart"] == c])) == 1 and (r["chart"] == c).sum() == 2


def test_octahedron_ties_go_to_the_lower_axis():
    v, f, N = hand_case("octahedron")
    lab, _ = CA.labels(v, f)
    # |n| components are all equal: axis x, the sign of n_x
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert np.array_equal(lab, np.where(n[:, 0] < 0, 1, 0))
    r = CA.atlas(v, f, N)
    # the four +x faces form a diamond around vertex 0 in the yz projection, the four -x faces one around vertex 1
    assert r["charts"] == 2 and r["rounds"] == 0 and sorted(np.unique(r["chart"]).tolist()) == [0, 1]


HELICOID_ROUNDS = 1


def test_helicoid_is_cut_until_it_does_not_overlap():
    v, f, N = hand_case("helicoid")
    lab, puv = CA.labels(v, f)
    assert (lab == 4).all()
    one = np.zeros(len(f), np.int64)
    assert len(CA.overlapping_charts(puv, one)) == 1             # uncut, it overlaps itself
    r = CA.atlas(v, f, N)
    assert r["rounds"] == HELICOID_ROUNDS and r["charts"] > 1
    assert len(CA.overlapping_charts(r["puv"], r["chart"].astype(np.int64))) == 0


def test_non_manifold_fin_bowtie_and_degenerate_faces():
    v, f, N = hand_case("fin")
    r = CA.atlas(v, f, N)
    assert r["charts"] == 3
    v, f, N = hand_case("bowtie")
    r = CA.atlas(v, f, N)
    assert r["charts"] == 2 and r["chart"].tolist() == [0, 1]
    v, f, N = hand_case("degenerate")
    r = CA.atlas(v, f, N)
    # edge (1, 2) has three uses (faces 0, 1 and the repeated-index face 2): faces 0 and 1 stay apart
    assert r["label"].tolist()[2:] == [CA.OWN, CA.OWN] and r["chart"].tolist() == [0, 1, 2, 3]


def test_bad_input_is_refused():
    v, f = cube()
    with pytest.raises(ValueError):
        CA.atlas(v, f, 100)
    with pytest.raises(ValueError):
        CA.atlas(v, np.array([[0, 1, 8]]), 64)
    bad = v.copy()
    bad[0, 0] = np.nan
    with pytest.raises(ValueError):
        CA.atlas(bad, f, 64)
    with pytest.raises(ValueError):          # no area: one zero-length face
        CA.atlas(np.zeros((3, 3), np.float32), np.array([[0, 1, 2]]), 64)


def test_separating_axis_test_ignores_touching():
    a = np.array([[[0, 0], [1, 0], [0, 1]]], np.float32)
    assert not CA.tri_overlap(a, a + np.float32([1, 0]))[0]               # share a corner
    assert not CA.tri_overlap(a, np.array([[[1, 0], [0, 1], [1, 1]]], np.float32))[0]   # share an edge
    assert CA.tri_overlap(a, a + np.float32([0.25, 0.25]))[0]
    assert CA.tri_overlap(a, a[:, ::-1])[0]                               # the same triangle, either winding


# ----------------------------------------------------------------------------- the example mesh
@pytest.fixture(scope="module")
def example():
    v0, _, _ = example_mesh()
    g = np.load(os.path.join(GOLD, "simplify", "backpack_ours_6996.npz"))
    v, f = v0[g["vertex_index"]], g["faces"].astype(np.int64)
    return v, f, CA.atlas(v, f, 1024)


# frozen from the oracle: 6 996 faces at N = 1024
EXAMPLE = {"charts": 207, "rounds": 8, "j": 76}


def test_example_mesh_frozen_numbers(example):
    v, f, r = example
    fa, fb = CA.edge_pairs(f, len(v))
    seams = int((r["chart"][fa] != r["chart"][fb]).sum())
    n = np.cross(v[f[:, 1]].astype(np.float64) - v[f[:, 0]], v[f[:, 2]].astype(np.float64) - v[f[:, 0]])
    area = 0.5 * np.linalg.norm(n, axis=1).sum()
    covered = r["rho"] ** 2 * area / 1024 ** 2
    print(f"charts {r['charts']}, rounds {r['rounds']}, seam edges {seams} of {len(fa)}, rho {r['rho']:.4f}, "
          f"surface share {covered:.4f}, owned share {(r['owner'] >= 0).mean():.4f}")
    assert {k: r[k] for k in EXAMPLE} == EXAMPLE
    assert seams == EXAMPLE_SEAMS
    assert r["rho"] == pytest.approx(EXAMPLE_RHO, rel=1e-12)
    assert covered == pytest.approx(EXAMPLE_SHARE, abs=5e-4)


EXAMPLE_SEAMS, EXAMPLE_RHO, EXAMPLE_SHARE = 1431, 579.5724726390532, 0.4595


def test_invariants_by_independent_means(example):
    v, f, r = example
    N, uv, boxes, chart = 1024, r["uv"], r["boxes"], r["chart"]
    # |n . axis| >= |n| / sqrt(3) for every labelled face
    n = np.cross(v[f[:, 1]].astype(np.float64) - v[f[:, 0]], v[f[:, 2]].astype(np.float64) - v[f[:, 0]])
    ok = r["label"] < CA.OWN
    ax = r["label"][ok] // 2
    assert (np.abs(n[ok, ax]) * np.sqrt(3) >= np.linalg.norm(n[ok], axis=1) * (1 - 1e-12)).all()
    # each chart is edge-connected, its faces all of one label (union-find over shared edges inside the chart)
    for c in np.unique(chart):
        fs = np.nonzero(chart == c)[0]
        assert len(np.unique(r["label"][fs])) == 1
        parent = {int(x): int(x) for x in fs}

        def find(x):
            while parent[x] != x:
                x = parent[x]
            return x
        edges = {}
        for x in fs:
            for k in range(3):
                e = tuple(sorted((f[x, k], f[x, (k + 1) % 3])))
                edges.setdefault(e, []).append(int(x))
        for fl in edges.values():
            for y in fl[1:]:
                parent[find(y)] = find(fl[0])
        assert len({find(int(x)) for x in fs}) == 1
    # boxes disjoint and inside N x N; every uv at least P inside its box
    cb = np.unique(boxes, axis=0)
    assert (cb[:, 0] >= 0).all() and (cb[:, 1] >= 0).all()
    assert (cb[:, 0] + cb[:, 2] <= N).all() and (cb[:, 1] + cb[:, 3] <= N).all()
    paint = np.zeros((N, N), np.int32)
    for x, y, w, h in cb.tolist():
        paint[y:y + h, x:x + w] += 1
    assert paint.max() == 1
    t = uv.astype(np.float64) * N
    assert (t[..., 0] >= boxes[:, None, 0] + CA.PAD).all() and (t[..., 0] <= boxes[:, None, 0] + boxes[:, None, 2] - CA.PAD).all()
    assert (t[..., 1] >= boxes[:, None, 1] + CA.PAD).all() and (t[..., 1] <= boxes[:, None, 1] + boxes[:, None, 3] - CA.PAD).all()
    # no texel centre lies strictly inside two faces of one chart (rasterised by barycentric signs)
    hits = np.zeros(N * N, np.int32)
    for x in range(len(f)):
        p = t[x]
        lo, hi = np.floor(p.min(0)).astype(int), np.ceil(p.max(0)).astype(int)
        xs, ys = np.meshgrid(np.arange(lo[0], hi[0] + 1) + 0.5, np.arange(lo[1], hi[1] + 1) + 0.5)
        xs, ys = xs.ravel(), ys.ravel()
        w = [(p[(k + 1) % 3, 0] - p[k, 0]) * (ys - p[k, 1]) - (p[(k + 1) % 3, 1] - p[k, 1]) * (xs - p[k, 0]) for k in range(3)]
        inside = ((w[0] > 0) & (w[1] > 0) & (w[2] > 0)) | ((w[0] < 0) & (w[1] < 0) & (w[2] < 0))
        hits[(ys[inside] - 0.5).astype(int) * N + (xs[inside] - 0.5).astype(int)] += 1
    assert hits.max() <= 1
    # a texel strictly inside a face is owned by it
    own = r["owner"]
    assert (own[hits == 1] >= 0).all()


# ----------------------------------------------------------------------------- command lines
def test_atlas_flags_need_texture_size():
    import run
    import simplify_mesh as SM
    assert run.parse_args(["--img_path", "a.png", "--texture_size", "512", "--output_format", ".glb",
                           "--atlas", "charts"]).atlas == "charts"
    assert run.parse_args(["--img_path", "a.png"]).atlas == "faces"
    with pytest.raises(SystemExit):
        run.parse_args(["--img_path", "a.png", "--atlas", "charts"])
    with pytest.raises(SystemExit):
        run.parse_args(["--img_path", "a.png", "--texture_size", "512", "--output_format", ".glb", "--atlas", "boxes"])
    base = ["--in", "a.ply", "--out", "b.glb", "--target_faces", "10"]
    assert SM.parse_args(base + ["--texture_size", "64", "--atlas", "charts"]).atlas == "charts"
    with pytest.raises(SystemExit):
        SM.parse_args(base + ["--atlas", "charts"])
    assert run._texture_kw(run.parse_args(["--img_path", "a.png"])) == {}
    kw = run._texture_kw(run.parse_args(["--img_path", "a.png", "--texture_size", "512", "--output_format", ".glb",
                                         "--atlas", "charts"]))
    assert kw == {"texture_size": 512, "atlas": "charts"}


def test_pipeline_keywords_and_bake_refuse_an_unknown_atlas():
    from o2345 import pipeline
    from o2345.mesh_texture import check_atlas
    assert pipeline._simplify_kw(None, 512) == {"texture_size": 512}
    assert pipeline._simplify_kw(None, 512, atlas="charts") == {"texture_size": 512, "atlas": "charts"}
    with pytest.raises(ValueError):
        pipeline._simplify_kw(None, None, atlas="charts")
    with pytest.raises(ValueError):
        check_atlas("boxes")
