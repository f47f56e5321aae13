"""GPU: mesh cleaning (csrc/clean.cu) bit-identical to oracle/clean_oracle.py on the hand cases, the example mesh and a
marching-cubes mesh of an analytic field, deterministic; the chart atlas on the shared union-find unchanged; the field
path through image_to_mesh, images_to_meshes (with and without the projection, the bake and simplification), run.py and
simplify_mesh.py."""
import os

import numpy as np
import pytest
import torch

from oracle import clean_oracle as CO
from test_clean_host import HAND, icosphere, join
from test_gpu_chart_atlas import check as check_charts
from test_gpu_project import STEPS, _photo, nets  # noqa: F401 (fixture)
from test_gpu_texture import _image, dev_t
from test_simplify_host import example_mesh

pytestmark = pytest.mark.gpu


def gpu_clean(v, f, F):
    from o2345 import ops
    return ops.clean_mesh(dev_t(v, np.float32).view(-1, 3), dev_t(f, np.int32).view(-1, 3), F)


def same(got, want):
    index, faces, st = got
    assert st["components"] == len(want["area"]) and st["largest"] == want["largest"]
    assert st["enclosed"] == want["enclosed"] and st["dropped"] == int((want["keep"] == 0).sum())
    assert np.array_equal(st["label"].cpu().numpy(), want["label"])
    for k in ("area", "winding"):
        assert np.array_equal(st[k].cpu().numpy().view(np.uint64), want[k].view(np.uint64)), k
    assert np.array_equal(st["keep"].cpu().numpy(), want["keep"])
    assert np.array_equal(index.cpu().numpy(), want["vertex_index"])
    assert np.array_equal(faces.cpu().numpy(), want["faces"])
    assert st["dropped_faces"] == len(st["label"]) - len(want["faces"])


def check(v, f, F):
    want = CO.clean_mesh(v, f, F)
    got = gpu_clean(v, f, F)
    same(got, want)
    again = gpu_clean(v, f, F)                      # two runs, the same bits
    assert torch.equal(got[0], again[0]) and torch.equal(got[1], again[1])
    for k in ("label", "area", "winding", "keep"):
        assert torch.equal(got[2][k], again[2][k]), k
    return want, got


# ----------------------------------------------------------------------------- kernels against the oracle
@pytest.mark.parametrize("name", sorted(HAND))
@pytest.mark.parametrize("F", [1e-6, 0.005, 0.02, 1.0])
def test_hand_cases_are_bit_identical_to_the_oracle(name, F):
    v, f = HAND[name]()
    check(v, f, F)


def test_many_small_components_and_an_empty_mesh():
    rng = np.random.default_rng(5)
    v = rng.standard_normal((3000, 3)).astype(np.float32)
    f = rng.integers(0, 3000, (600, 3)).astype(np.int32)         # a hundred and more components of a few faces
    want, _ = check(v, f, 0.3)
    assert len(want["area"]) > 100
    big = join(icosphere(1.0, level=4), *[icosphere(0.05, (1.5 + 0.2 * i, 0, 0), level=0) for i in range(40)])
    check(*big, 0.001)
    # a largest component of 320 000 faces: more chunks than one block's threads take in one round
    n = 400
    i, j = np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing="ij")
    pv = np.stack([i / n, j / n, np.zeros_like(i, float)], -1).reshape(-1, 3)
    a, b = (x.ravel() for x in np.meshgrid(np.arange(n), np.arange(n), indexing="ij"))
    at = lambda p, q: p * (n + 1) + q
    pf = np.concatenate([np.stack([at(a, b), at(a + 1, b), at(a + 1, b + 1)], 1), np.stack([at(a, b), at(a + 1, b + 1), at(a, b + 1)], 1)])
    tri = (np.array([[0.5, 0.5, 0.1], [0.6, 0.5, 0.1], [0.5, 0.6, 0.1]]), np.array([[0, 1, 2]]))
    want, _ = check(*join((pv.astype(np.float32), pf.astype(np.int32)), (tri[0].astype(np.float32), tri[1].astype(np.int32))), 1e-6)
    assert len(want["area"]) == 2 and want["keep"].all()
    index, faces, st = gpu_clean(v, f[:0], 0.5)
    assert index.numel() == 0 and faces.shape == (0, 3) and st["components"] == 0


def test_bad_input_is_refused():
    from o2345._lib import O2345Error
    v, f = HAND["bowtie"]()
    with pytest.raises(O2345Error):
        gpu_clean(v, np.array([[0, 1, 99]]), 0.5)
    bad = v.copy()
    bad[0, 0] = np.inf
    with pytest.raises(O2345Error):
        gpu_clean(bad, f, 0.5)
    with pytest.raises(O2345Error):
        gpu_clean(v, f, 0.0)


def test_example_mesh_is_returned_unchanged():
    from o2345.mesh_clean import clean
    v, f, _ = example_mesh()
    check(v, f, 0.05)
    c = np.arange(len(v) * 3, dtype=np.float32).reshape(-1, 3)
    for F in (1e-6, 1.0):
        v2, f2, c2, st = clean(v, f, c, F)
        assert st["components"] == 1 and st["dropped"] == 0
        assert np.array_equal(v2.view(np.uint32), v.view(np.uint32)) and np.array_equal(f2, f) and np.array_equal(c2, c)


def analytic_mesh(R=128):
    """A ball, a distant ball of a tenth its radius and a bubble inside the first, by ops.marching_cubes."""
    from o2345 import ops
    x = torch.linspace(-1, 1, R, device="cuda", dtype=torch.float64)
    X, Y, Z = torch.meshgrid(x, x, x, indexing="ij")
    d = lambda c, r: torch.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r
    ball, small, bubble = d((-0.3, 0, 0), 0.5), d((0.6, 0.55, 0.5), 0.05), d((-0.25, 0.05, 0), 0.2)
    u = torch.minimum(torch.maximum(ball, -bubble), small).float()
    verts, tris, _ = ops.marching_cubes(u)
    return (verts.cpu().numpy() * (2.0 / (R - 1)) - 1.0).astype(np.float32), tris.cpu().numpy()


def test_marching_cubes_mesh_keeps_only_the_ball():
    v, f = analytic_mesh()
    want, (index, faces, st) = check(v, f, 0.05)
    print(f"analytic: {len(f)} faces, areas {want['area']}, winding {want['winding']}")
    assert st["components"] == 3 and st["dropped"] == 2 and st["enclosed"] == 1
    assert abs(want["area"][want["largest"]] - 4 * np.pi * 0.25) < 0.02
    kept = want["label"] == want["largest"]
    assert len(faces) == kept.sum()


def test_chart_atlas_on_the_shared_union_find_is_unchanged():
    from test_chart_atlas_host import HAND as CHART_HAND, hand_case
    for name in sorted(CHART_HAND):
        check_charts(*hand_case(name), points=False)


# ----------------------------------------------------------------------------- the field path
R = 64
F = 0.05


def _ply(d):
    from o2345 import mesh_io
    return mesh_io.read_ply(os.path.join(d, "mesh.ply"))


def _cleaned(d):
    from o2345.mesh_clean import clean
    v, f, c = _ply(d)
    return clean(v, f, c, F)


def _same_mesh(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def test_image_to_mesh_cleans_the_welded_mesh(nets, tmp_path):
    from o2345.mesh_simplify import simplify
    from o2345.pipeline import image_to_mesh
    z, tr, dev = nets
    x = _image(3)
    kw = dict(polar_angle=60, resolution=R, **STEPS)
    runs = {"plain": {}, "clean": dict(min_component=F), "project": dict(min_component=F, project_view=_photo(3)),
            "bake": dict(min_component=F, target_faces=1500, texture_size=512)}
    out = {}
    for k, extra in runs.items():
        torch.cuda.manual_seed(11)
        out[k] = image_to_mesh(z, tr, x, exp_dir=str(tmp_path / k), **kw, **extra)
    want = _cleaned(tmp_path / "plain")
    print(f"field path: {len(out['plain']['triangles'])} faces, {want[3]}")
    assert want[3]["dropped"] > 0                         # the synthetic weights' mesh has fragments to drop
    assert out["clean"]["clean"] == want[3] and "clean" not in out["plain"]
    _same_mesh(_ply(tmp_path / "clean"), want[:3])
    # the projection ran on the cleaned mesh: same geometry, one weight per cleaned vertex
    pv, pf, _ = _ply(tmp_path / "project")
    _same_mesh((pv, pf), want[:2])
    w = out["project"]["project_weight"]
    assert w.shape == (len(want[0]),) and (w > 0).any()
    # simplified and baked: the cleaned mesh
    sv, sf, _, _ = simplify(want[0], want[1], None, 1500)
    _same_mesh((out["bake"]["vertices"].astype(np.float32), out["bake"]["triangles"]), (sv, sf))
    assert out["bake"]["uv"].shape == (len(sf), 3, 2) and out["bake"]["texture"].shape == (512, 512, 3)


def test_images_to_meshes_cleans_every_mesh(nets, tmp_path):
    from o2345.pipeline import images_to_meshes
    z, tr, dev = nets
    xs = [_image(3), _image(4)]
    for k, extra in (("plain", {}), ("clean", dict(min_component=F))):
        dirs = [str(tmp_path / k / str(i)) for i in range(2)]
        got = dict(images_to_meshes(z, tr, xs, [60, 60], seed=9, resolution=R, exp_dirs=dirs, **STEPS, **extra))
        assert ("clean" in got[0]) == (k == "clean")
    for i in range(2):
        want = _cleaned(tmp_path / "plain" / str(i))
        _same_mesh(_ply(tmp_path / "clean" / str(i)), want[:3])


def test_run_py_and_simplify_mesh_py_take_min_component(tmp_path, monkeypatch, capsys):
    from PIL import Image
    import run as run_cli
    import simplify_mesh
    from o2345 import mesh_io
    monkeypatch.chdir(tmp_path)
    img = str(tmp_path / "obj.png")
    Image.fromarray(_image(3)).save(img)
    run_cli.main(["--img_path", img, "--mesh_resolution", str(R), "--seed", "2", "--min_component", str(F)])
    assert "components, dropped" in capsys.readouterr().out
    ply = tmp_path / "exp" / "obj" / "mesh.ply"
    assert ply.exists()
    v, f, c = mesh_io.read_ply(str(ply))
    # a fragment far from the mesh is dropped again by simplify_mesh.py, which then simplifies the rest
    fv, ff = icosphere(0.01, (5, 5, 5), level=1)
    mesh_io.write_ply(str(tmp_path / "in.ply"), np.concatenate([v, fv]), np.concatenate([f, ff + len(v)]),
                      np.concatenate([c, np.full((len(fv), 4), 255, np.uint8)]))
    out = simplify_mesh.main(["--in", str(tmp_path / "in.ply"), "--out", str(tmp_path / "small.ply"),
                              "--target_faces", "500", "--min_component", str(F)])
    printed = capsys.readouterr().out
    assert "cleaned:" in printed and "dropped 1 " in printed
    assert len(out[1]) <= 500 and out[0].max(0)[0] < 4
