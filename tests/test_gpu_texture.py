"""GPU: texture baking (csrc/texture.cu through ops / mesh_texture) bit-identical to the numpy oracle
(oracle/texture_oracle.py) on hand-built cases and the frozen 10 % example mesh; determinism; an analytic colour baked
onto a sphere and read back through the rasterizer; unchanged geometry of the textured GLB; real colours transferred
from the full example mesh; the field path (export_mesh_step, image_to_mesh, run.py) and simplify_mesh.py."""
import gzip
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from oracle import texture_oracle as TO
from test_simplify_host import GOLD, ROOT, example_mesh

pytestmark = pytest.mark.gpu
PKG = os.path.join(ROOT, "one-2-3-45_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)


def dev_t(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def gpu_atlas(v, f, N):
    from o2345 import ops
    vt, ft = dev_t(v, np.float32).view(-1, 3), dev_t(f, np.int32).view(-1, 3)
    at = ops.texture_atlas(vt, ft, N)
    return vt, ft, at


def same_atlas(at, want):
    assert at["j"] == want["j"] and at["rho"] == want["rho"]
    assert np.array_equal(at["boxes"].cpu().numpy(), want["boxes"])
    uv = at["uv"].cpu().numpy()
    assert uv.dtype == np.float32 and np.array_equal(uv.view(np.uint32), want["uv"].view(np.uint32))
    assert np.array_equal(at["owner"].cpu().numpy(), want["owner"])


def hand_cases():
    s = np.float32(3 ** 0.5 / 2)
    k = np.arange(100, dtype=np.float32)[:, None]
    z = 0 * k
    tiny = np.concatenate([np.concatenate([k, z, z], 1), np.concatenate([k + 0.01, z, z], 1), np.concatenate([k, z + 0.02, z], 1)])
    return {
        "exact": ([[0, 0, 0], [2, 0, 0], [1, 1, 0]], [[0, 1, 2]], 64),
        "right": ([[0, 0, 0], [1, 0, 0], [0, 1, 0]], [[0, 1, 2]], 64),
        "equilateral": ([[0, 0, 0], [1, 0, 0], [0.5, s, 0]], [[0, 1, 2]], 128),
        "tie": ([[0, 0, 0], [2, 0, 0], [1, 3, 0]], [[0, 1, 2]], 64),
        "degenerate": ([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 5], [2, 0, 0], [3, 0, 0], [4, 0, 0]],
                       [[0, 1, 2], [3, 3, 3], [4, 5, 6]], 64),
        "many_tiny": (tiny, np.stack([np.arange(100), np.arange(100) + 100, np.arange(100) + 200], 1), 128),
    }


@pytest.mark.parametrize("name", sorted(hand_cases()))
def test_hand_cases_are_bit_identical_to_the_oracle(name):
    from o2345 import ops
    v, f, N = hand_cases()[name]
    v, f = np.asarray(v, np.float32), np.asarray(f, np.int64)
    want = TO.atlas(v, f, N)
    vt, ft, at = gpu_atlas(v, f, N)
    same_atlas(at, want)
    idx, pts, face = ops.texel_points(vt, ft, at["uv"], at["owner"], N)
    wi, wp, wf = TO.texel_points(v, f, want["uv"], want["owner"], N)
    assert np.array_equal(idx.cpu().numpy(), wi) and np.array_equal(face.cpu().numpy(), wf)
    assert np.array_equal(pts.cpu().numpy().view(np.uint32), wp.view(np.uint32))


def test_infeasible_and_bad_input_are_refused():
    from o2345 import _lib
    k = np.arange(200, dtype=np.float32)[:, None]
    z = 0 * k
    v = np.concatenate([np.concatenate([k, z, z], 1), np.concatenate([k + 1e-3, z, z], 1), np.concatenate([k, z + 1e-3, z], 1)])
    f = np.stack([np.arange(200), np.arange(200) + 200, np.arange(200) + 400], 1)
    with pytest.raises(_lib.O2345Error, match="cannot hold 200 charts"):
        gpu_atlas(v, f, 64)
    with pytest.raises(_lib.O2345Error, match="outside"):
        gpu_atlas(v, np.array([[0, 1, 600]]), 64)
    bad = v.copy()
    bad[3, 1] = np.inf
    with pytest.raises(_lib.O2345Error, match="finite"):
        gpu_atlas(bad, f, 1024)


@pytest.fixture(scope="module")
def example6996():
    from o2345 import mesh_io
    v, _, _ = example_mesh()
    g = np.load(os.path.join(GOLD, "simplify", "backpack_ours_6996.npz"))
    return v, g["vertex_index"], g["faces"]


@pytest.mark.parametrize("N", [1024, 2048])
def test_example_mesh_atlas_points_and_fill_are_bit_identical(example6996, N):
    from o2345 import ops
    v0, vi, f = example6996
    v = v0[vi]
    want = TO.atlas(v, f, N)
    vt, ft, at = gpu_atlas(v, f, N)
    same_atlas(at, want)
    idx, pts, face = ops.texel_points(vt, ft, at["uv"], at["owner"], N)
    wi, wp, wf = TO.texel_points(v, f, want["uv"], want["owner"], N)
    assert np.array_equal(idx.cpu().numpy(), wi) and np.array_equal(face.cpu().numpy(), wf)
    assert np.array_equal(pts.cpu().numpy().view(np.uint32), wp.view(np.uint32))
    rgb = np.random.default_rng(N).random((len(wi), 3), dtype=np.float32)
    tex = ops.texture_fill(idx, dev_t(rgb, np.float32), at["owner"], N).cpu().numpy()
    assert np.array_equal(tex.view(np.uint32), TO.fill(wi, rgb, want["owner"], N).view(np.uint32))
    # two runs, the same bits
    _, _, at2 = gpu_atlas(v, f, N)
    assert all(torch.equal(at[k], at2[k]) for k in ("uv", "boxes", "owner"))
    idx2, pts2, _ = ops.texel_points(vt, ft, at2["uv"], at2["owner"], N)
    assert torch.equal(idx, idx2) and torch.equal(pts.view(torch.int32), pts2.view(torch.int32))


def _backpack_obj(tmp):
    obj = os.path.join(tmp, "backpack_ours.obj")
    with gzip.open(os.path.join(GOLD, "render_eval", "backpack_ours.obj.gz"), "rb") as src, open(obj, "wb") as dst:
        shutil.copyfileobj(src, dst)
    return obj


def test_transfer_kernel_is_bit_identical_to_the_oracle(example6996, tmp_path):
    from o2345 import mesh_io, ops
    from o2345.mesh_simplify import simplify
    v0, _, _ = example6996
    _, f0, c0 = mesh_io.read_obj(_backpack_obj(str(tmp_path)))
    N = 128                                                   # 128^2 texels hold a 500-face mesh's charts
    v, f, _, _ = simplify(v0, f0, None, 500)
    vt, ft, at = gpu_atlas(v, f, N)
    _, pts, _ = ops.texel_points(vt, ft, at["uv"], at["owner"], N)
    sv, sf, sc = dev_t(v0, np.float32), dev_t(f0, np.int32), dev_t(c0, np.float32)
    samples, sface = ops.surface_sample(sv, sf, 4 * N * N, 0)
    _, nn = ops.nearest(pts, samples)
    got = ops.transfer_colors(sv, sf, sc, pts, nn, sface).cpu().numpy()
    want = TO.transfer(v0, f0, c0.astype(np.float32), pts.cpu().numpy(), nn.cpu().numpy(), sface.cpu().numpy())
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.isfinite(got).all() and got.min() >= 0 and got.max() <= 1


# ----------------------------------------------------------------------------- rendering the baked texture
def _flat_textured(v, f, uv, tex):
    fi = np.asarray(f, np.int64).reshape(-1)
    return {"verts": np.ascontiguousarray(np.asarray(v, np.float32)[fi]), "faces": np.arange(len(fi), dtype=np.int32).reshape(-1, 3),
            "colors": None, "uvs": np.ascontiguousarray(np.asarray(uv, np.float32).reshape(-1, 2)),
            "face_tex": np.zeros(len(f), np.int32),
            "texels": np.concatenate([tex, np.full(tex.shape[:2] + (1,), 255, np.uint8)], -1).reshape(-1),
            "tex_info": np.array([[0, tex.shape[1], tex.shape[0], 1, 1]], np.int32)}


def _sphere(target=2000):
    from o2345.mesh_io import merge_vertices
    from o2345.mesh_simplify import simplify
    from oracle.recon_oracle import marching_cubes
    g = np.linspace(-1, 1, 64)
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    v, f, _ = marching_cubes(0.4 - np.sqrt(x ** 2 + y ** 2 + z ** 2), 0.0)
    v, f, _ = merge_vertices(v / 63 * 2 - 1, f)                # lattice indices -> [-1, 1]
    v, f, _, _ = simplify(v.astype(np.float32), f.astype(np.int32), None, target)
    return v.astype(np.float32), f


def test_analytic_colour_round_trips_through_the_rasterizer():
    from o2345 import mesh_raster as MR
    from o2345.mesh_texture import bake
    v, f = _sphere()
    N, omega = 512, 6.0
    uv, tex, at = bake(v, f, N, lambda p: 0.5 + 0.5 * torch.sin(omega * p), return_atlas=True)
    c2w, K = MR.rig_cameras(1.5, 256)
    lip, rho = 0.5 * omega, at["rho"]
    bound = lip * 2 ** 0.5 / rho + 1 / 255

    def worst(uv_used):
        out = MR.render(_flat_textured(v, f, uv_used, tex), c2w, K, 256, 256)
        col, alpha, depth = (out[k].cpu().numpy() for k in ("color", "alpha", "depth"))
        errs = []
        for i in range(len(c2w)):
            yy, xx = np.nonzero(alpha[i] > 0)
            zc = depth[i, yy, xx].astype(np.float64)
            pc = np.stack([(xx + 0.5 - K[0, 2]) / K[0, 0] * zc, (yy + 0.5 - K[1, 2]) / K[1, 1] * zc, zc, np.ones_like(zc)], 1)
            pw = (pc @ c2w[i].T)[:, :3]
            errs.append(np.abs(col[i, yy, xx] - (0.5 + 0.5 * np.sin(omega * pw))).max())
        return max(errs)
    good = worst(uv)
    flipped = uv.copy()
    flipped[..., 1] = 1 - flipped[..., 1]
    bad = worst(flipped)
    print(f"analytic round trip: rho {rho:.1f}, bound {bound:.4f}, worst {good:.4f}, v flipped {bad:.4f}")
    assert good <= bound + 2e-4          # 2e-4: the point recovered from fp32 depth
    assert bad > bound


def test_textured_glb_keeps_the_geometry(example6996, tmp_path):
    from o2345 import mesh_io
    from o2345 import mesh_raster as MR
    from o2345.mesh_texture import bake
    v0, vi, f = example6996
    v = v0[vi]
    uv, tex = bake(v, f, 1024, lambda p: torch.full_like(p, 0.5))
    a, b = str(tmp_path / "a.glb"), str(tmp_path / "b.glb")
    mesh_io.write_glb(a, v, f, np.full((len(v), 3), 128, np.uint8))
    mesh_io.write_textured_glb(b, v, f, uv, tex)
    ra, rb = MR.render_rig(a, resolution=256), MR.render_rig(b, resolution=256)
    assert torch.equal(ra["tri"], rb["tri"]) and torch.equal(ra["alpha"], rb["alpha"])
    assert (ra["tri"] >= 0).sum() > 1000


# measured on an H100 80GB HBM3 at 700 W (DESIGN §2): PSNR over pixels covered in both renders against the 69 960-face
# original, 24 rig views at 512^2, unlit: texture 45.14 dB, vertex colours 29.05 dB, a margin of 16.09 dB
PSNR_MARGIN, PSNR_SLACK = 16.09, 1.0


def test_transferred_texture_beats_vertex_colours(example6996, tmp_path):
    from o2345 import mesh_io
    from o2345 import mesh_raster as MR
    from o2345.mesh_texture import bake, transfer_fn
    v0, vi, f = example6996
    obj = _backpack_obj(str(tmp_path))
    _, f0, c0 = mesh_io.read_obj(obj)
    flat0 = MR.flatten(MR.normalize_scene(MR.load_scene(obj)))
    rig = flat0["verts"]                                          # the original in the rig frame (y-up converted, scaled)
    N = 2048
    uv, tex = bake(v0[vi], f, N, transfer_fn(v0, f0, c0, texture_size=N))
    c2w, K = MR.rig_cameras(1.5, 512)
    ref = MR.render(flat0, c2w, K, 512, 512)
    vc = {"verts": rig[vi], "faces": f.astype(np.int32), "colors": c0[vi].astype(np.float32), "uvs": None, "face_tex": None,
          "texels": None, "tex_info": None}
    r_vc = MR.render(vc, c2w, K, 512, 512)
    r_tx = MR.render(_flat_textured(rig[vi], f, uv, tex), c2w, K, 512, 512)

    def psnr(r):
        m = (ref["alpha"] > 0) & (r["alpha"] > 0)
        mse = float(((r["color"] - ref["color"]) ** 2)[m].mean())
        return 10 * np.log10(1.0 / mse)
    p_vc, p_tx = psnr(r_vc), psnr(r_tx)
    print(f"PSNR against the original: vertex colours {p_vc:.3f} dB, texture {p_tx:.3f} dB")
    assert p_tx - p_vc > PSNR_MARGIN - PSNR_SLACK


# ----------------------------------------------------------------------------- the field path
STEPS = dict(ddim_steps=4, stage2_steps=2)
R = 64


def _image(seed=7):
    rng = np.random.default_rng(seed)
    im = np.full((256, 256, 3), 255, np.uint8)
    im[48:208, 56:200] = rng.integers(0, 255, (160, 144, 3), dtype=np.uint8)
    return im


def test_export_mesh_bakes_the_reconstruction_colours(tmp_path, monkeypatch):
    from o2345 import mesh_texture as MT
    from o2345 import synthetic as S
    from o2345.pipeline import build_networks, image_to_mesh, images_to_meshes
    from o2345.zero123 import build_zero123
    dev = torch.device("cuda:0")
    z = build_zero123(dev, seed=0, clip=True).half()
    tr = build_networks(dev, vol_dim=96, states=S.all_states(0), perturb=0.0)
    x = _image()
    torch.cuda.manual_seed(5)
    plain = image_to_mesh(z, tr, x, polar_angle=60, resolution=R, exp_dir=str(tmp_path / "plain"), target_faces=2000, **STEPS)
    seen = {}
    real = MT.bake

    def spy(vertices, faces, n, colour_fn, device=None):
        uv, tex, at = real(vertices, faces, n, colour_fn, device, return_atlas=True)
        seen.update(at=at, colour_fn=colour_fn, vertices=vertices)
        return uv, tex
    monkeypatch.setattr(MT, "bake", spy)
    torch.cuda.manual_seed(5)
    out = image_to_mesh(z, tr, x, polar_angle=60, resolution=R, exp_dir=str(tmp_path / "tex"), target_faces=2000,
                        texture_size=256, **STEPS)
    for k in ("vertices", "triangles", "colors"):
        assert np.array_equal(out[k], plain[k]), k
    assert (tmp_path / "tex" / "mesh.ply").read_bytes() == (tmp_path / "plain" / "mesh.ply").read_bytes()
    tex, uv, at = out["texture"], out["uv"], seen["at"]
    assert tex.shape == (256, 256, 3) and tex.dtype == np.uint8 and uv.shape == (len(out["triangles"]), 3, 2)
    idx = at["texel_index"].cpu().numpy()
    again = MT.quantise(seen["colour_fn"](at["points"]))
    assert np.array_equal(tex.reshape(-1, 3)[idx], again)              # owned texels: quantised blend_points of their points
    # corner texels: the texel holding a chart's corner a gets the vertex's position, so the vertex's colour byte
    pts, faces = at["points"].cpu().numpy(), out["triangles"]
    k0 = TO.base_corner(seen["vertices"], faces)
    b = at["boxes"].cpu().numpy()
    corner = b[:, 1].astype(np.int64) * 256 + b[:, 0]                   # the box's first texel: closest point a
    pos = np.searchsorted(idx, corner)
    a = faces[np.arange(len(faces)), k0]
    assert np.array_equal(pts[pos], np.asarray(seen["vertices"], np.float32)[a])
    assert np.array_equal(tex.reshape(-1, 3)[corner], out["colors"][a][:, :3])
    (_, many), = images_to_meshes(z, tr, [x], [60], seed=5, resolution=R, target_faces=2000, texture_size=256, **STEPS)
    assert many["texture"].shape == (256, 256, 3) and many["uv"].shape == (len(many["triangles"]), 3, 2)


def test_run_py_writes_a_textured_glb_that_renders(tmp_path, monkeypatch):
    from PIL import Image
    import render_eval
    import run as run_cli
    from o2345 import mesh_io
    monkeypatch.chdir(tmp_path)
    img = str(tmp_path / "obj.png")
    Image.fromarray(_image(3)).save(img)
    out = run_cli.main(["--img_path", img, "--mesh_resolution", "64", "--seed", "2", "--target_faces", "2000",
                        "--texture_size", "512", "--output_format", ".glb"])
    assert out.endswith("mesh.glb")
    g = mesh_io.read_glb(out)
    assert g["textures"][0][0].shape == (512, 512, 4) and len(g["meshes"][0]["faces"]) in (2000, 1999)
    render_eval.main(["--object_path", out, "--output_dir", str(tmp_path / "views"), "--resolution", "128"])
    assert os.path.exists(tmp_path / "views" / "0.png")


def test_simplify_mesh_writes_textured_glb_and_obj(tmp_path):
    import simplify_mesh as SM
    from o2345 import mesh_io
    obj = _backpack_obj(str(tmp_path))
    for ext in (".glb", ".obj"):
        out = str(tmp_path / f"small{ext}")
        res = SM.main(["--in", obj, "--out", out, "--target_faces", "3000", "--texture_size", "512"])
        assert res[5].shape == (512, 512, 3)
    g = mesh_io.read_glb(str(tmp_path / "small.glb"))
    assert len(g["meshes"][0]["faces"]) in (3000, 2999) and g["textures"][0][0].shape == (512, 512, 4)
    assert (tmp_path / "small.mtl").exists() and (tmp_path / "small_albedo.png").exists()
    _, f, _ = mesh_io.read_obj(str(tmp_path / "small.obj"))
    assert len(f) in (3000, 2999)
