"""GPU tests of closest points and isotropic remeshing (csrc/remesh.cu): bit-identity to oracle/remesh_oracle.py on the
tie cases, random and on-surface points around the example mesh and a 10^6-face soup; the remesh on every host case,
on the welded example mesh and on a clipped marching-cubes mesh; determinism; the O2345_ENOSPC retry; fidelity to the
input against a control without projection; simplify_mesh.py --remesh end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import remesh_oracle as R
from test_remesh_host import F32, hand_cases, tie_case, uv_sphere
from test_simplify_host import example_mesh

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev_t(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def gpu_closest(v, f, p):
    from o2345 import ops
    q, face = ops.closest_points(dev_t(v, np.float32).view(-1, 3), dev_t(f, np.int32).view(-1, 3), dev_t(p, np.float32).view(-1, 3))
    return q.cpu().numpy(), face.cpu().numpy()


def gpu_remesh(v, f, L, it, **kw):
    from o2345 import ops
    ov, of, rounds = ops.remesh_mesh(dev_t(v, np.float32).view(-1, 3), dev_t(f, np.int32).view(-1, 3), L, it, **kw)
    return ov.cpu().numpy(), of.cpu().numpy(), rounds


def same_closest(v, f, p, brute=False):
    q, face = gpu_closest(v, f, p)
    rq, rf = R.closest_points(v, f, p, brute=brute)
    np.testing.assert_array_equal(q.view(np.uint32), rq.view(np.uint32))
    np.testing.assert_array_equal(face, rf)


def same_remesh(v, f, L, it):
    ov, of, rounds = gpu_remesh(v, f, L, it)
    rv, rf, rr = R.remesh(v, f, L, it)
    np.testing.assert_array_equal(ov.view(np.uint32), rv.view(np.uint32))
    np.testing.assert_array_equal(of, rf)
    assert rounds == rr
    return ov, of


def marching_cubes_mesh(R_=64):
    """A clipped sphere from the project's marching cubes: an open mesh with a boundary loop."""
    from o2345 import ops
    g = torch.linspace(-1, 1, R_, device="cuda")
    x, y, z = torch.meshgrid(g, g, g, indexing="ij")
    sdf = torch.sqrt(x * x + y * y + (z * 1.3) ** 2) - 0.7
    v, f, _ = ops.marching_cubes(sdf.contiguous(), 0.0)
    v, f = v.cpu().numpy().astype(np.float32), f.cpu().numpy().astype(np.int32)
    from o2345 import mesh_io
    v, f, _ = mesh_io.merge_vertices(v, f)
    keep = (v[f][:, :, 2] < R_ * 0.7).all(1)
    return v.astype(np.float32), f[keep].astype(np.int32)


def test_closest_points_ties_and_surfaces():
    v, f, p = tie_case()
    same_closest(v, f, p, brute=True)
    sv, sf = uv_sphere(20, 40)
    rng = np.random.default_rng(0)
    p = np.concatenate([rng.normal(size=(2000, 3)).astype(F32), sv, (sv[sf[:, 0]] + sv[sf[:, 1]]) * F32(0.5)])
    same_closest(sv, sf, p, brute=True)


def test_closest_points_around_the_example_mesh():
    v, f, _ = example_mesh()
    rng = np.random.default_rng(1)
    lo, hi = v.min(0), v.max(0)
    p = np.concatenate([rng.uniform(lo - 0.1 * (hi - lo), hi + 0.1 * (hi - lo), (20000, 3)).astype(F32), v[::7],
                        ((v[f[::5, 0]] + v[f[::5, 1]]) * F32(0.5))])
    same_closest(v, f, p)
    same_closest(v, f, p[:40], brute=True)


def test_closest_points_on_a_million_face_soup():
    rng = np.random.default_rng(2)
    c = rng.uniform(-1, 1, (1 << 20, 1, 3)).astype(F32)
    v = (c + rng.normal(scale=0.01, size=(1 << 20, 3, 3)).astype(F32)).reshape(-1, 3)
    f = np.arange(len(v), dtype=np.int32).reshape(-1, 3)
    p = rng.uniform(-1.1, 1.1, (20000, 3)).astype(F32)
    same_closest(v, f, p)


@pytest.mark.parametrize("name", sorted(hand_cases()))
def test_remesh_hand_cases_are_bit_identical_to_the_oracle(name):
    v, f, L, it = hand_cases()[name]
    same_remesh(v, f, L, it)


def test_remesh_is_deterministic_and_independent_of_the_capacities():
    v, f, L, it = hand_cases()["sphere_2000"]
    a = gpu_remesh(v, f, L, it)
    b = gpu_remesh(v, f, L, it)
    c = gpu_remesh(v, f, L, it, vertex_capacity=len(v), face_capacity=len(f))     # forced through O2345_ENOSPC
    for x in (b, c):
        np.testing.assert_array_equal(a[0].view(np.uint32), x[0].view(np.uint32))
        np.testing.assert_array_equal(a[1], x[1])


GOLD = os.path.join(ROOT, "tests", "golden", "remesh")


@pytest.mark.parametrize("N", [13992, 3498, 700])
def test_remesh_example_mesh_at_three_targets_is_bit_identical_to_the_oracle(N):
    """The oracle's own remesh of the welded example mesh at 20 %, 5 % and 1 % of its faces, with the default
    iterations (frozen in tests/golden/remesh: about 4 minutes of numpy for the three)."""
    from o2345 import mesh_remesh
    v, f, _ = example_mesh()
    g = np.load(os.path.join(GOLD, f"backpack_remesh_{N}.npz"))
    L, _ = R.target_length(v, f, N)
    assert L == g["L"] and mesh_remesh.REMESH_ITERATIONS == R.ITERATIONS
    ov, of, rounds = gpu_remesh(v, f, L, R.ITERATIONS)
    np.testing.assert_array_equal(ov.view(np.uint32), g["verts"].view(np.uint32))
    np.testing.assert_array_equal(of, g["faces"])
    assert rounds == tuple(g["rounds"].tolist())
    assert 0.8 * N <= len(of) <= 1.25 * N


def test_remesh_clipped_marching_cubes_mesh_is_bit_identical_to_the_oracle():
    v, f = marching_cubes_mesh()
    L, _ = R.target_length(v, f, len(f) // 3)
    same_remesh(v, f, L, 3)


def bumpy_sphere(nlat=40, nlon=80):
    v, f = uv_sphere(nlat, nlon)
    th = np.arccos(np.clip(v[:, 2], -1, 1))
    ph = np.arctan2(v[:, 1], v[:, 0])
    return (v * (1 + 0.15 * np.sin(5 * th) * np.sin(5 * ph))[:, None]).astype(F32), f


def chamfer(v1, f1, v2, f2, n=1 << 20):
    """Mean nearest-sample distance both ways between 2^20 area-uniform samples of each mesh (ops.surface_sample,
    ops.nearest)."""
    from o2345 import ops
    p, _ = ops.surface_sample(dev_t(v1, np.float32), dev_t(f1, np.int32), n, seed=1)
    q, _ = ops.surface_sample(dev_t(v2, np.float32), dev_t(f2, np.int32), n, seed=2)
    d1, _ = ops.nearest(p, q)
    d2, _ = ops.nearest(q, p)
    return float(d1.double().sqrt().mean() + d2.double().sqrt().mean())


# frozen from the oracle's runs (numpy samples of 10^6 points): 0.00595 with projection, 0.00639 without it
CHAMFER_BOUND = 0.0062


def test_remesh_chamfer_to_the_input_is_bounded_and_the_control_without_projection_fails():
    v, f = bumpy_sphere()
    L, _ = R.target_length(v, f, 6000)
    ov, of, _ = gpu_remesh(v, f, L, R.ITERATIONS)
    got = chamfer(v, f, ov, of)
    cv, cf, _ = R.remesh(v, f, L, R.ITERATIONS, project=False)
    ctl = chamfer(v, f, cv, cf)
    print(f"chamfer: remesh {got:.6f}, without projection {ctl:.6f}, bound {CHAMFER_BOUND}")
    assert got < CHAMFER_BOUND < ctl
    q, _ = gpu_closest(v, f, ov)
    assert np.abs(q - ov).max() <= 4 * np.finfo(F32).eps * np.abs(v).max()


def test_simplify_mesh_remesh_end_to_end(tmp_path):
    from o2345 import mesh_io, mesh_remesh
    from test_gpu_texture import _backpack_obj
    obj = _backpack_obj(str(tmp_path))
    out = str(tmp_path / "even.ply")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "one-2-3-45_b200", "simplify_mesh.py"), "--in", obj, "--out",
                        out, "--target_faces", "4000", "--remesh"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "remesh: " in r.stdout
    v, f, c = mesh_io.read_ply(out)
    assert 2000 <= len(f) <= 6000
    # the colours written are the input's at each vertex's exact closest point
    import simplify_mesh
    iv, if_, irgba = simplify_mesh.read_mesh(obj)
    iv, if_, irgba = mesh_io.merge_vertices(iv, if_, irgba)
    np.testing.assert_array_equal(c, mesh_remesh.surface_colors(iv, if_, irgba, v))
    # ... and exact where an output vertex is an input vertex: the locked boundary of an open grid with random colours
    from test_remesh_host import grid
    gv, gf = grid(12)
    gc = np.concatenate([np.random.default_rng(3).integers(0, 256, (len(gv), 3)), np.full((len(gv), 1), 255)], 1)
    src, dst = str(tmp_path / "grid.ply"), str(tmp_path / "grid_even.ply")
    mesh_io.write_ply(src, gv, gf, gc.astype(np.uint8))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "one-2-3-45_b200", "simplify_mesh.py"), "--in", src, "--out",
                        dst, "--target_faces", "150", "--remesh"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    v2, _, c2 = mesh_io.read_ply(dst)
    key = {tuple(x): i for i, x in enumerate(gv.view(np.uint32))}
    hits = [(j, key[tuple(x)]) for j, x in enumerate(np.asarray(v2, np.float32).view(np.uint32)) if tuple(x) in key]
    assert len(hits) >= 4 * 12
    j, i = np.array(hits).T
    np.testing.assert_array_equal(c2[j], gc[i].astype(np.uint8)[:, :c2.shape[1]])


# ----------------------------------------------------------------------------- the field path
from test_gpu_project import STEPS, _photo, nets  # noqa: E402,F401 (fixture)
from test_gpu_texture import _image  # noqa: E402

RES = 64


def test_image_to_mesh_remeshes_the_welded_mesh_in_the_normalised_frame(nets, monkeypatch):
    from o2345 import mesh_remesh
    from o2345.pipeline import image_to_mesh
    z, tr, dev = nets
    seen = {}
    real = mesh_remesh.remesh

    def spy(v, f, extra, n, *a, **k):
        out = real(v, f, extra, n, *a, **k)
        seen.update(v=np.asarray(v).copy(), f=np.asarray(f).copy(), out=out)
        return out
    monkeypatch.setattr(mesh_remesh, "remesh", spy)
    kw = dict(polar_angle=60, resolution=RES, **STEPS)
    torch.cuda.manual_seed(5)
    plain = image_to_mesh(z, tr, _image(3), **kw)
    torch.cuda.manual_seed(5)
    got = image_to_mesh(z, tr, _image(3), target_faces=1500, remesh=True, **kw)
    # the input of the remesh is the plain run's welded mesh, in the normalised frame
    np.testing.assert_array_equal(seen["f"], plain["triangles"])
    A = np.concatenate([seen["v"].astype(np.float64), np.ones((len(seen["v"]), 1))], 1)
    M, *_ = np.linalg.lstsq(A, plain["vertices"].astype(np.float64), rcond=None)
    np.testing.assert_allclose(A @ M, plain["vertices"], atol=1e-5)
    # its output, transformed by the same map, is the mesh; the remesh of that input gives it again, bit for bit
    ov, of, st = seen["out"]
    np.testing.assert_array_equal(got["triangles"], of)
    Bv = np.concatenate([ov.astype(np.float64), np.ones((len(ov), 1))], 1) @ M
    np.testing.assert_allclose(got["vertices"], Bv, atol=1e-5)
    again = real(seen["v"], seen["f"], None, 1500)
    np.testing.assert_array_equal(again[0].view(np.uint32), ov.view(np.uint32))
    assert got["remesh"]["rounds"] == st["rounds"] and 1000 <= len(of) <= 2250
    # colours: the trainer's colour() at the remeshed points, quantised as for the full mesh
    assert got["colors"].shape[0] == len(ov) and got["colors"].dtype == np.uint8


@pytest.mark.parametrize("atlas", ["faces", "charts"])
def test_image_to_mesh_remesh_composes_with_clean_bake_and_projection(nets, atlas):
    from o2345.pipeline import image_to_mesh
    z, tr, dev = nets
    torch.cuda.manual_seed(5)
    m = image_to_mesh(z, tr, _image(3), polar_angle=60, resolution=RES, target_faces=1500, remesh=True, min_component=0.05,
                      texture_size=512, normal_map=True, ambient_occlusion=True, atlas=atlas, project_view=_photo(3),
                      **STEPS)
    n = len(m["triangles"])
    assert m["uv"].shape == (n, 3, 2) and m["texture"].shape == (512, 512, 3)
    assert m["normal_texture"].shape == (512, 512, 3) and m["occlusion_texture"].shape == (512, 512)
    assert m["project_weight"].shape == (len(m["vertices"]),) and "clean" in m and "remesh" in m


def test_images_to_meshes_and_run_py_remesh(nets, tmp_path, monkeypatch):
    from PIL import Image
    import run as run_cli
    from o2345 import mesh_io
    from o2345.pipeline import images_to_meshes
    z, tr, dev = nets
    got = dict(images_to_meshes(z, tr, [_image(3), _image(4)], [60, 60], seed=9, resolution=RES, target_faces=1500,
                                remesh=True, **STEPS))
    assert sorted(got) == [0, 1] and all("remesh" in m for m in got.values())
    monkeypatch.chdir(tmp_path)
    img = str(tmp_path / "obj.png")
    Image.fromarray(_image(3)).save(img)
    out = run_cli.main(["--img_path", img, "--mesh_resolution", str(RES), "--seed", "2", "--target_faces", "1500",
                        "--remesh", "--output_format", ".glb"])
    g = mesh_io.read_glb(out)
    assert 700 <= len(g["meshes"][0]["faces"]) <= 2250
