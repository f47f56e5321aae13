"""GPU: mesh simplification (csrc/simplify.cu through ops / mesh_simplify) bit-identical to the numpy oracle
(oracle/simplify_oracle.py) on the hand-built cases, the reference's example mesh and a clipped marching-cubes mesh;
determinism; the mesh tail (image_to_mesh, run.py) and the simplify_mesh.py command line."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import simplify_oracle as SO
from test_simplify_host import EXAMPLE_TARGET, GOLD, ROOT, cases, check_closed, edges, example_mesh

pytestmark = pytest.mark.gpu
PKG = os.path.join(ROOT, "one-2-3-45_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)


def gpu(verts, faces, target):
    from o2345 import ops
    vi, f, rounds = ops.simplify_mesh(torch.from_numpy(np.asarray(verts, np.float32)).cuda(),
                                      torch.from_numpy(np.asarray(faces, np.int32)).cuda(), target)
    return vi.cpu().numpy(), f.cpu().numpy(), rounds


def same(a, b):
    assert a[0].dtype == b[0].dtype == np.int32 and np.array_equal(a[0], b[0])
    assert a[1].dtype == b[1].dtype == np.int32 and a[1].shape == b[1].shape and np.array_equal(a[1], b[1])
    assert a[2] == b[2]


@pytest.mark.parametrize("name", sorted(cases()))
def test_hand_built_cases_are_bit_identical_to_the_oracle(name):
    v, f, target = cases()[name]
    same(gpu(v, f, target), SO.simplify(v, f, target))


def test_bad_input_is_refused():
    from o2345 import _lib
    v, f, _ = cases()["tetrahedron"]
    with pytest.raises(_lib.O2345Error, match="outside"):
        gpu(v, np.concatenate([f, [[0, 1, 4]]]), 0)
    bad = v.copy()
    bad[1, 0] = np.nan
    with pytest.raises(_lib.O2345Error, match="finite"):
        gpu(bad, f, 0)


@pytest.fixture(scope="module")
def example():
    return example_mesh()


@pytest.mark.parametrize("share", [50, 10, 1])
def test_example_mesh_is_bit_identical_to_the_oracle(example, share):
    v, f, _ = example
    target = len(f) * share // 100
    got = gpu(v, f, target)
    same(got, SO.simplify(v, f, target))
    assert len(got[1]) in (target, target - 1)
    check_closed(got[0], got[1], -2)
    if target == EXAMPLE_TARGET:
        gold = np.load(os.path.join(GOLD, "simplify", "backpack_ours_6996.npz"))
        assert np.array_equal(got[0], gold["vertex_index"]) and np.array_equal(got[1], gold["faces"])
    same(got, gpu(v, f, target))                                   # two runs, the same bits


def clipped_sphere(R=48):
    """Oracle marching cubes of a sphere that sticks out of the [-1, 1]^3 lattice: an open surface with a boundary."""
    from o2345.mesh_io import merge_vertices
    from oracle.recon_oracle import marching_cubes
    g = np.linspace(-1, 1, R)
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    u = 0.9 - np.sqrt((x - 0.35) ** 2 + (y + 0.05) ** 2 + z ** 2)
    v, f, _ = marching_cubes(u, 0.0)
    v, f, _ = merge_vertices(v, f)
    return v.astype(np.float32), f.astype(np.int32)


def test_clipped_marching_cubes_mesh_keeps_its_boundary():
    v, f = clipped_sphere()
    e, cnt = edges(f)
    boundary = np.unique(e[cnt == 1])
    assert len(boundary) > 50
    for target in (len(f) // 4, 200):
        got = gpu(v, f, target)
        same(got, SO.simplify(v, f, target))
        assert np.isin(boundary, got[0]).all()                  # boundary vertices are never removed
        e2, c2 = edges(got[1])
        assert set(c2.tolist()) <= {1, 2} and np.array_equal(np.sort(got[0][np.unique(e2[c2 == 1])]), boundary)


# ----------------------------------------------------------------------------- the mesh tail
STEPS = dict(ddim_steps=4, stage2_steps=2)
R = 64


def _image(seed=7):
    rng = np.random.default_rng(seed)
    im = np.full((256, 256, 3), 255, np.uint8)
    im[48:208, 56:200] = rng.integers(0, 255, (160, 144, 3), dtype=np.uint8)
    return im


def test_image_to_mesh_with_a_target_is_the_helper_on_the_full_mesh(tmp_path):
    from o2345 import synthetic as S
    from o2345.mesh_io import read_ply
    from o2345.mesh_simplify import simplify
    from o2345.pipeline import build_networks, image_to_mesh, images_to_meshes
    from o2345.zero123 import build_zero123
    dev = torch.device("cuda:0")
    z = build_zero123(dev, seed=0, clip=True).half()
    tr = build_networks(dev, vol_dim=96, states=S.all_states(0), perturb=0.0)
    x = _image()
    torch.cuda.manual_seed(5)
    full = image_to_mesh(z, tr, x, polar_angle=60, resolution=R, exp_dir=str(tmp_path / "full"), **STEPS)
    target = len(full["triangles"]) // 5
    torch.cuda.manual_seed(5)
    small = image_to_mesh(z, tr, x, polar_angle=60, resolution=R, exp_dir=str(tmp_path / "small"), target_faces=target, **STEPS)
    v, f, c, rounds = simplify(full["vertices"], full["triangles"], full["colors"], target)
    assert rounds > 0 and len(f) in (target, target - 1)
    for k, want in (("vertices", v), ("triangles", f), ("colors", c)):
        assert small[k].dtype == want.dtype and np.array_equal(small[k], want), k
    pv, pf, pc = read_ply(str(tmp_path / "small" / "mesh.ply"))
    assert np.array_equal(pv, v.astype(np.float32)) and np.array_equal(pf, f) and np.array_equal(pc[:, :3], c[:, :3])
    (_, many), = images_to_meshes(z, tr, [x], [60], seed=5, resolution=R, target_faces=target, **STEPS)
    assert len(many["triangles"]) in (target, target - 1)


def test_run_py_writes_the_simplified_mesh(tmp_path, monkeypatch):
    from PIL import Image
    import run as run_cli
    from o2345 import mesh_io
    from o2345.mesh_simplify import simplify
    monkeypatch.chdir(tmp_path)
    img = str(tmp_path / "obj.png")
    Image.fromarray(_image(3)).save(img)
    run_cli.main(["--img_path", img, "--mesh_resolution", "64", "--seed", "2"])
    v, f, c = mesh_io.read_ply(str(tmp_path / "exp" / "obj" / "mesh.ply"))
    target = len(f) // 3
    out = run_cli.main(["--img_path", img, "--mesh_resolution", "64", "--seed", "2", "--target_faces", str(target),
                        "--output_format", ".glb"])
    assert out.endswith("mesh.glb")
    sv, sf, sc, _ = simplify(v, f, c, target)
    ref = tmp_path / "ref"
    ref.mkdir()
    mesh_io.write_ply(str(ref / "mesh.ply"), sv, sf, sc)
    mesh_io.convert_mesh_format(str(ref), ".glb")
    assert (ref / "mesh.ply").read_bytes() == (tmp_path / "exp" / "obj" / "mesh.ply").read_bytes()
    assert (ref / "mesh.glb").read_bytes() == open(out, "rb").read()


def test_simplify_mesh_command_line_round_trips_the_example_obj(tmp_path, capsys):
    import gzip
    import shutil
    import simplify_mesh as SM
    from o2345 import mesh_io
    obj = str(tmp_path / "backpack_ours.obj")
    with gzip.open(os.path.join(GOLD, "render_eval", "backpack_ours.obj.gz"), "rb") as src, open(obj, "wb") as dst:
        shutil.copyfileobj(src, dst)
    out = str(tmp_path / "small.obj")
    SM.main(["--in", obj, "--out", out, "--target_faces", str(EXAMPLE_TARGET)])
    gold = np.load(os.path.join(GOLD, "simplify", "backpack_ours_6996.npz"))
    v0, _, c0 = mesh_io.read_obj(obj)
    v1, f1, c1 = mesh_io.read_obj(out)
    assert np.array_equal(f1, gold["faces"])
    np.testing.assert_allclose(v1, v0.astype(np.float32)[gold["vertex_index"]], rtol=0, atol=1e-8)
    assert c1 is not None
    lines = capsys.readouterr().out.splitlines()
    assert lines[0].endswith(f"{len(v0)} vertices, 69960 faces")
    assert lines[2] == f"simplified: {len(gold['vertex_index'])} vertices, {EXAMPLE_TARGET} faces in {int(gold['rounds'])} rounds"
    glb = str(tmp_path / "small.glb")
    SM.main(["--in", out, "--out", glb, "--target_faces", "1000"])
    g = mesh_io.read_glb(glb)
    assert len(g["meshes"][0]["faces"]) in (1000, 999)
