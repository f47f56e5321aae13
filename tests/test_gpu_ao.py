"""GPU: ambient occlusion (csrc/ao.cu) through the C-ABI, bit-identical to oracle/ao_oracle.py on the host cases, the
example mesh's vertices, random points and normals around it, a mesh of coplanar and duplicated faces and a 10^6-face
soup, deterministic; the floor-and-wall bake against the analytic AO (and its flipped-normal control); the other outputs
unchanged by the option; the field path through image_to_mesh, images_to_meshes, run.py and simplify_mesh.py."""
import os

import numpy as np
import pytest
import torch

from oracle import ao_oracle as AO
from test_ao_host import F32, UP, floor_and_wall, grid, half_plane_discrepancy, hand_cases, join, wall_ao
from test_gpu_project import STEPS, nets  # noqa: F401 (fixture)
from test_gpu_texture import _backpack_obj, _image, dev_t
from test_simplify_host import example_mesh

pytestmark = pytest.mark.gpu


def gpu_ao(v, f, p, n, dirs=None, t_min=None, t_max=None):
    """o2345_ambient_occlusion through the C-ABI with the oracle's defaults -> AO float32 [n]."""
    from o2345 import _lib as L, ops
    v, f = np.asarray(v, F32).reshape(-1, 3), np.asarray(f, np.int32).reshape(-1, 3)
    dirs = AO.directions() if dirs is None else np.asarray(dirs, F32).reshape(-1, 3)
    dt = AO.distances(v)
    t_min, t_max = dt[0] if t_min is None else t_min, dt[1] if t_max is None else t_max
    vt, ft, pt, nt, dd = (dev_t(a, d) for a, d in ((v, F32), (f, np.int32), (p, F32), (n, F32), (dirs, F32)))
    nbytes = L.load().o2345_ambient_occlusion_scratch_bytes(len(v), len(f))
    scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device="cuda")
    out = torch.empty(len(np.asarray(p).reshape(-1, 3)), dtype=torch.float32, device="cuda")
    L.call("o2345_ambient_occlusion", ops._f(vt), len(v), ops._p(ft, torch.int32), len(f), ops._f(pt), ops._f(nt), out.numel(),
           ops._f(dd), len(dirs), float(t_min), float(t_max), ops._p(scratch), nbytes, ops._f(out), ops._stream())
    return out.cpu().numpy()


def check(v, f, p, n, dirs=None, t_min=None, t_max=None):
    want = AO.ambient_occlusion(v, f, p, n, dirs=dirs, t_min=t_min, t_max=t_max)
    got = gpu_ao(v, f, p, n, dirs, t_min, t_max)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.flatnonzero(got != want)[:10]
    assert np.array_equal(gpu_ao(v, f, p, n, dirs, t_min, t_max), got)          # two runs, the same bits
    return got


# ----------------------------------------------------------------------------- kernels against the oracle
@pytest.mark.parametrize("name", sorted(hand_cases()))
def test_hand_cases_are_bit_identical_to_the_oracle(name):
    check(*hand_cases()[name])


def test_empty_inputs():
    v, f, _, _, _, _, _ = hand_cases()["octahedron_inside"]
    assert gpu_ao(v, f, np.zeros((0, 3), F32), np.zeros((0, 3), F32)).shape == (0,)
    assert (check(v, f[:0], np.zeros((3, 3), F32), np.tile(UP, (3, 1)), t_min=0.0, t_max=1.0) == 1).all()


def test_bad_input_is_refused():
    from o2345 import _lib as L
    v, f, p, n, _, _, _ = hand_cases()["octahedron_inside"]
    with pytest.raises(L.O2345Error, match="face index"):
        gpu_ao(v, np.where(f == 5, 6, f), p, n)
    bad = v.copy()
    bad[2, 1] = np.inf
    with pytest.raises(L.O2345Error, match="not finite"):
        gpu_ao(bad, f, p, n, t_min=1e-3, t_max=4.0)


@pytest.fixture(scope="module")
def example():
    v, f, _ = example_mesh()
    return v, f


def test_example_mesh_vertices_are_bit_identical(example):
    from o2345 import mesh_texture as MT, ops
    v, f = example
    vt, ft = dev_t(v, F32).view(-1, 3), dev_t(f, np.int32).view(-1, 3)
    nrm = ops.vertex_normals(vt, ft)
    ao = ops.ambient_occlusion(vt, ft, vt, nrm)
    assert torch.equal(ao, MT.vertex_ao(vt, ft))
    ao, nrm = ao.cpu().numpy(), nrm.cpu().numpy()
    print(f"example: {len(f)} faces, vertex AO mean {ao.mean():.4f}, min {ao.min():.4f}, {np.mean(ao < 1):.3f} occluded")
    assert 0.3 < ao.mean() < 1 and ao.min() < 0.5
    sel = np.random.default_rng(0).choice(len(v), 256, replace=False)
    want = AO.ambient_occlusion(v, f, v[sel], nrm[sel])
    assert np.array_equal(ao[sel].view(np.uint32), want.view(np.uint32))
    assert np.array_equal(gpu_ao(v, f, v[sel], nrm[sel]), want)


def test_random_points_and_normals_around_the_example(example):
    v, f = example
    rng = np.random.default_rng(1)
    lo, hi = v.min(0), v.max(0)
    c, e = (lo + hi) / 2, (hi - lo) / 2
    p = (c + rng.uniform(-1.2, 1.2, (256, 3)) * e).astype(F32)
    n = rng.standard_normal((256, 3)).astype(F32)
    n[:12] = [[0, 0, 1], [0, 0, -1], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 0], [np.nan, 0, 0],
              [0, 0, -0.0], [1e-3, 0, 0], [3, 4, 0], [0, -2, 1e-7]]
    got = check(v, f, p, n)
    assert (got < 1).sum() > 50


def test_coplanar_and_duplicated_faces():
    """Every Morton code repeated: a 16 x 16 grid, four copies of it (two reversed) and a twin grid slightly above."""
    gv, gf = grid(16, -1, 1, -1, 1)
    v, f = join((gv, gf), (gv, gf), (gv, gf[:, ::-1]), (gv, gf[:, ::-1]), (gv + np.float32([0, 0, 0.01]), gf))
    rng = np.random.default_rng(2)
    p = np.concatenate([rng.uniform(-0.9, 0.9, (96, 2)), rng.uniform(-0.2, 0.2, (96, 1))], 1).astype(F32)
    n = rng.standard_normal((96, 3)).astype(F32)
    got = check(v, f, p, n, t_min=1e-3, t_max=0.5)
    assert 0 < got.mean() < 1


def test_a_million_face_soup():
    rng = np.random.default_rng(3)
    m = 1 << 20
    c = rng.uniform(-1, 1, (m, 1, 3))
    v = (c + rng.uniform(-0.004, 0.004, (m, 3, 3))).astype(F32).reshape(-1, 3)
    f = np.arange(3 * m, dtype=np.int32).reshape(-1, 3)
    p = rng.uniform(-0.8, 0.8, (16, 3)).astype(F32)
    n = rng.standard_normal((16, 3)).astype(F32)
    got = check(v, f, p, n)
    print(f"soup: {m} faces, AO {np.round(got, 3)}")
    assert 0.5 < got.mean() < 1


# ----------------------------------------------------------------------------- the bake
GRID = 96                     # floor quads per side: one chart of 2 GRID^2 faces


def _floor_bake(flip=False, N=256):
    """Bakes the floor-and-wall scene (floor GRID x GRID quads) into a chart atlas with the AO of its own vertices (normals
    flipped for the control) -> (mesh, uv, occlusion map, atlas dict, nearest-sample distance per owned texel)."""
    from o2345 import mesh_texture as MT, ops
    v, f = floor_and_wall(n=GRID)
    vt, ft = dev_t(v, F32).view(-1, 3), dev_t(f, np.int32).view(-1, 3)
    nrm = ops.vertex_normals(vt, ft)
    ao = ops.ambient_occlusion(vt, ft, vt, -nrm if flip else nrm)
    fn = MT._transfer(vt, ft, ao[:, None].expand(-1, 3).contiguous(), N, MT.TRANSFER_SEED)
    uv, tex, occ, at = MT.bake(v, f, N, lambda p: torch.zeros_like(p), atlas="charts", return_atlas=True,
                               ao_fn=lambda p: fn(p)[:, 0])
    samples, _ = ops.surface_sample(vt, ft, MT.TRANSFER_SAMPLES * N * N, MT.TRANSFER_SEED)
    d2, _ = ops.nearest(at["points"], samples)
    return (v, f), occ, at, np.sqrt(d2.cpu().numpy().astype(np.float64))


def _floor_errors(occ, at, s, v):
    t_max = float(AO.distances(v)[1])
    h = 2.0 / GRID
    idx, pts, face = (at[k].cpu().numpy() for k in ("texel_index", "points", "texel_face"))
    d = 0.5 - pts[:, 0].astype(np.float64)
    use = (face < 2 * GRID * GRID) & (np.abs(pts[:, 1]) < 0.6) & (d < 1.5) & (d >= 2 * h + s)
    a = np.minimum(d / t_max, 1.0)
    want = np.where(d < t_max, wall_ao(a), 1.0)
    got = occ.reshape(-1)[idx].astype(np.float64) / 255
    # vertex AO within the table's half-plane discrepancy of the analytic value; linear interpolation over a face of
    # diameter h sqrt 2 and the step s to the nearest sample's face move the analytic value by at most its largest slope
    # 2 / (pi t_max) times that distance; the 8-bit code adds 1/255
    bound = half_plane_discrepancy(AO.directions()) + 2 / (np.pi * t_max) * (h * np.sqrt(2) + s) + 1 / 255
    return use, np.abs(got - want), bound


def test_floor_and_wall_bake_is_within_the_analytic_bound():
    mesh, occ, at, s = _floor_bake()
    assert occ.shape == (256, 256) and occ.dtype == np.uint8
    use, err, bound = _floor_errors(occ, at, s, mesh[0])
    print(f"floor bake: {use.sum()} texels, worst error {err[use].max():.4f}, bound {bound[use].min():.4f} .. "
          f"{bound[use].max():.4f}, nearest sample up to {s[use].max():.4f}")
    assert use.sum() > 5000 and (err[use] <= bound[use]).all()
    # the control: normals flipped, the floor looks down at nothing and the wall's shadow is gone
    mesh, occ, at, s = _floor_bake(flip=True)
    use, err, bound = _floor_errors(occ, at, s, mesh[0])
    assert (err[use] > bound[use]).sum() > 500


def test_bake_outputs_are_unchanged_by_the_occlusion_map(example):
    from o2345 import mesh_texture as MT
    from o2345.mesh_simplify import simplify
    v, f = example
    sv, sf, _, _ = simplify(v, f, None, 3000)
    colour = MT.transfer_fn(v, f, np.full((len(v), 3), 200, np.uint8) - (np.arange(len(v)) % 50)[:, None].astype(np.uint8),
                            texture_size=512)
    nfn = MT.normal_transfer_fn(v, f, texture_size=512)
    plain = MT.bake(sv, sf, 512, colour, normal_fn=nfn)
    with_ao = MT.bake(sv, sf, 512, colour, normal_fn=nfn, ao_fn=MT.ao_transfer_fn(v, f, texture_size=512))
    assert len(with_ao) == 4 and with_ao[3].shape == (512, 512) and with_ao[3].min() < 128
    for a, b in zip(plain, with_ao):
        assert np.array_equal(a, b)


# ----------------------------------------------------------------------------- the field path
R = 64


def test_image_to_mesh_bakes_the_full_meshes_occlusion(nets, tmp_path, monkeypatch):
    import run as run_cli
    from o2345 import mesh_io, mesh_texture as MT
    from o2345.pipeline import image_to_mesh
    z, tr, dev = nets
    seen = {}
    real = MT.ao_transfer_fn

    def spy(src_v, src_f, *a, **k):
        seen["faces"] = len(src_f)
        return real(src_v, src_f, *a, **k)
    monkeypatch.setattr(MT, "ao_transfer_fn", spy)
    kw = dict(polar_angle=60, resolution=R, target_faces=1500, texture_size=512, normal_map=True, **STEPS)
    out = {}
    for k, extra in (("plain", {}), ("ao", dict(ambient_occlusion=True))):
        torch.cuda.manual_seed(11)
        out[k] = image_to_mesh(z, tr, _image(3), exp_dir=str(tmp_path / k), **kw, **extra)
    a, b = out["plain"], out["ao"]
    for key in ("vertices", "triangles", "colors", "uv", "texture", "normal_texture"):
        assert np.array_equal(a[key], b[key]), key
    assert open(tmp_path / "plain" / "mesh.ply", "rb").read() == open(tmp_path / "ao" / "mesh.ply", "rb").read()
    occ = b["occlusion_texture"]
    print(f"field path: AO of a {seen['faces']}-face mesh baked onto {len(b['triangles'])} faces, mean {occ.mean() / 255:.3f}")
    assert "occlusion_texture" not in a and occ.shape == (512, 512) and seen["faces"] > 1500
    glb = run_cli._write_format(str(tmp_path / "ao"), ".glb", b)
    g = mesh_io.read_glb(glb)
    m = g["meshes"][0]
    assert (m["face_otex"] == 2).all() and np.array_equal(g["textures"][2][0][..., 0], occ)


def test_images_to_meshes_bake_occlusion(nets, tmp_path):
    from o2345 import mesh_io
    from o2345.pipeline import images_to_meshes
    z, tr, dev = nets
    got = dict(images_to_meshes(z, tr, [_image(3), _image(4)], [60, 60], seed=9, resolution=R, target_faces=1500,
                                texture_size=512, ambient_occlusion=True, **STEPS))
    for i, mesh in got.items():
        p = str(tmp_path / f"m{i}.glb")
        mesh_io.write_textured(p, *mesh_io.to_viewer_frame(mesh["vertices"], mesh["triangles"], mesh["uv"]), mesh["texture"],
                               occlusion_texture=mesh["occlusion_texture"])
        assert (mesh_io.read_glb(p)["meshes"][0]["face_otex"] == 1).all()


def test_run_py_and_simplify_mesh_py_write_occlusion(tmp_path, monkeypatch):
    from PIL import Image
    import run as run_cli
    import simplify_mesh as SM
    from o2345 import mesh_io
    monkeypatch.chdir(tmp_path)
    img = str(tmp_path / "obj.png")
    Image.fromarray(_image(3)).save(img)
    out = run_cli.main(["--img_path", img, "--mesh_resolution", str(R), "--seed", "2", "--target_faces", "2000",
                        "--texture_size", "512", "--ambient_occlusion", "--output_format", ".glb"])
    g = mesh_io.read_glb(out)
    assert len(g["textures"]) == 2 and (g["meshes"][0]["face_otex"] == 1).all()
    obj = _backpack_obj(str(tmp_path))
    for ext in (".glb", ".obj"):
        res = SM.main(["--in", obj, "--out", str(tmp_path / f"small{ext}"), "--target_faces", "3000", "--texture_size", "512",
                       "--normal_map", "--ambient_occlusion"])
        assert res[-1].shape == (512, 512) and res[-1].min() < 128
    g = mesh_io.read_glb(str(tmp_path / "small.glb"))
    assert len(g["textures"]) == 3 and (g["meshes"][0]["face_otex"] == 2).all()
    assert "map_ao small_occlusion.png" in open(tmp_path / "small.mtl").read()
