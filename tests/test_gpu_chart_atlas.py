"""GPU: the multi-face chart atlas (o2345_chart_atlas through ops / mesh_texture) bit-identical to the numpy oracle
(oracle/chart_atlas_oracle.py) on the hand meshes, the example mesh at 10 % and in full and a marching-cubes mesh;
determinism; an analytic colour round trip through the rasterizer; colour against the per-face atlas; the decoded
normal-map frame; simplify_mesh.py --atlas charts."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import chart_atlas_oracle as CA
from oracle import texture_oracle as TO
from test_chart_atlas_host import HAND, hand_case
from test_gpu_texture import _backpack_obj, _flat_textured, _sphere, dev_t, example6996  # noqa: F401 (fixture)
from test_simplify_host import ROOT, example_mesh

pytestmark = pytest.mark.gpu
PKG = os.path.join(ROOT, "one-2-3-45_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)


def gpu_charts(v, f, N):
    from o2345 import ops
    vt, ft = dev_t(v, np.float32).view(-1, 3), dev_t(f, np.int32).view(-1, 3)
    return vt, ft, ops.chart_atlas(vt, ft, N)


def same_charts(at, want):
    assert (at["j"], at["rho"], at["rounds"], at["charts"]) == (want["j"], want["rho"], want["rounds"], want["charts"])
    for k in ("label", "chart", "boxes", "owner"):
        assert np.array_equal(at[k].cpu().numpy(), want[k]), k
    uv = at["uv"].cpu().numpy()
    assert np.array_equal(uv.view(np.uint32), want["uv"].view(np.uint32))


def check(v, f, N, points=True):
    from o2345 import ops
    v, f = np.asarray(v, np.float32), np.asarray(f, np.int64)
    want = CA.atlas(v, f, N)
    vt, ft, at = gpu_charts(v, f, N)
    same_charts(at, want)
    if points:
        idx, pts, face = ops.texel_points(vt, ft, at["uv"], at["owner"], N)
        wi, wp, wf = TO.texel_points(v, f, want["uv"], want["owner"], N)
        assert np.array_equal(idx.cpu().numpy(), wi) and np.array_equal(face.cpu().numpy(), wf)
        assert np.array_equal(pts.cpu().numpy().view(np.uint32), wp.view(np.uint32))
    _, _, at2 = gpu_charts(v, f, N)      # two runs, the same bits
    assert all(torch.equal(at[k], at2[k]) for k in ("uv", "boxes", "owner", "label", "chart"))
    return want


@pytest.mark.parametrize("name", sorted(HAND))
def test_hand_cases_are_bit_identical_to_the_oracle(name):
    check(*hand_case(name))


def test_bad_input_is_refused():
    from o2345 import ops
    from o2345._lib import O2345Error
    v, f, _ = hand_case("cube")
    with pytest.raises(O2345Error):
        gpu_charts(v, np.array([[0, 1, 8]]), 64)
    bad = v.copy()
    bad[0, 0] = np.nan
    with pytest.raises(O2345Error):
        gpu_charts(bad, f, 64)
    with pytest.raises(O2345Error):
        gpu_charts(np.zeros((3, 3), np.float32), np.array([[0, 1, 2]]), 64)
    with pytest.raises(O2345Error):
        ops.chart_atlas(dev_t(v, np.float32), dev_t(f, np.int32), 100)


@pytest.mark.parametrize("N", [256, 512, 1024, 2048])
def test_example_mesh_is_bit_identical(example6996, N):
    v0, vi, f = example6996
    check(v0[vi], f, N, points=N == 1024)


def test_full_example_mesh_fits_where_the_face_atlas_refuses():
    from o2345 import ops
    from o2345._lib import O2345Error
    v, f, _ = example_mesh()
    want = check(v, f, 1024, points=False)
    print(f"full mesh ({len(f)} faces) at N = 1024: {want['charts']} charts, {want['rounds']} rounds, rho {want['rho']:.2f}")
    with pytest.raises(O2345Error):
        ops.texture_atlas(dev_t(v, np.float32), dev_t(f, np.int32), 1024)


def test_marching_cubes_mesh_is_bit_identical():
    from o2345.mesh_io import merge_vertices
    from oracle.recon_oracle import marching_cubes
    g = np.linspace(-1, 1, 48)
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    sdf = 0.5 - np.sqrt(x ** 2 + (1.6 * y) ** 2 + z ** 2) + 0.08 * np.sin(5 * x) * np.cos(4 * z)
    v, f, _ = marching_cubes(sdf, 0.0)
    v, f, _ = merge_vertices(v / 47 * 2 - 1, f)
    check(v.astype(np.float32), f, 1024)


def test_analytic_colour_round_trips_through_the_rasterizer():
    from o2345 import mesh_raster as MR
    from o2345.mesh_texture import bake
    v, f = _sphere()
    N, omega = 512, 6.0
    uv, tex, at = bake(v, f, N, lambda p: 0.5 + 0.5 * torch.sin(omega * p), return_atlas=True, atlas="charts")
    c2w, K = MR.rig_cameras(1.5, 256)
    lip, rho = 0.5 * omega, at["rho"]
    bound = lip * 2 ** 0.5 * 3 ** 0.5 / rho + 1 / 255

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
    print(f"charts analytic round trip: {at['charts']} charts, rho {rho:.1f}, bound {bound:.4f}, worst {good:.4f}, "
          f"v flipped {bad:.4f}")
    assert good <= bound + 2e-4
    assert bad > bound


def test_decoded_normal_frame_round_trips_through_tangent_frames():
    """The chart atlas's normal map decodes, in the frame mesh_io writes (TANGENT = T, w = sign((N x T) . B)), to the
    normal it was given."""
    from o2345 import mesh_io
    from o2345.mesh_texture import bake
    v, f = _sphere()
    N = 512
    _, _, nmap, at = bake(v, f, N, lambda p: torch.full_like(p, 0.5), return_atlas=True, atlas="charts",
                          normal_fn=lambda p: p)
    T, B, Nn = mesh_io.tangent_frames(v, f, at["uv"].cpu().numpy())
    w = np.where(np.einsum("ij,ij->i", np.cross(Nn, T), B) < 0, -1.0, 1.0)
    face = at["texel_face"].cpu().numpy()
    t = at["tangent_normals"].cpu().numpy().astype(np.float64)
    Bd = w[face, None] * np.cross(Nn[face], T[face])
    dec = t[:, :1] * T[face] + t[:, 1:2] * Bd + t[:, 2:] * Nn[face]
    p = at["points"].cpu().numpy().astype(np.float64)
    cos = np.einsum("ij,ij->i", dec, p) / np.linalg.norm(dec, axis=1) / np.linalg.norm(p, axis=1)
    worst = np.degrees(np.arccos(np.clip(cos.min(), -1, 1)))
    print(f"decoded frame: worst angle {worst:.5f} deg over {len(p)} texels")
    assert worst < 1e-3
    assert nmap.shape == (N, N, 3)


# measured on an H100 80GB HBM3 at 700 W (DESIGN §2): PSNR against the 69 960-face original of the 10 % example's
# transfer bake, 24 rig views at 512^2; per-face atlas / charts: 35.80 / 43.11 dB at N = 512, 44.40 / 44.91 dB at 1024
CHARTS_MARGIN, PSNR_SLACK = {512: 7.31, 1024: 0.51}, 0.3


@pytest.mark.parametrize("N", [512, 1024])
def test_charts_beat_the_face_atlas_on_colour(example6996, tmp_path, N):
    from o2345 import mesh_io
    from o2345 import mesh_raster as MR
    from o2345.mesh_texture import bake, transfer_fn
    v0, vi, f = example6996
    obj = _backpack_obj(str(tmp_path))
    _, f0, c0 = mesh_io.read_obj(obj)
    flat0 = MR.flatten(MR.normalize_scene(MR.load_scene(obj)))
    rig = flat0["verts"]
    c2w, K = MR.rig_cameras(1.5, 512)
    ref = MR.render(flat0, c2w, K, 512, 512)

    def psnr(atlas):
        uv, tex = bake(v0[vi], f, N, transfer_fn(v0, f0, c0, texture_size=N), atlas=atlas)
        r = MR.render(_flat_textured(rig[vi], f, uv, tex), c2w, K, 512, 512)
        m = (ref["alpha"] > 0) & (r["alpha"] > 0)
        return 10 * np.log10(1.0 / float(((r["color"] - ref["color"]) ** 2)[m].mean()))
    p_faces, p_charts = psnr("faces"), psnr("charts")
    print(f"N = {N}: PSNR faces {p_faces:.3f} dB, charts {p_charts:.3f} dB")
    assert p_charts - p_faces > CHARTS_MARGIN[N] - PSNR_SLACK



def test_simplify_mesh_writes_chart_textured_glb_and_obj(tmp_path):
    import simplify_mesh as SM
    from o2345 import mesh_io
    from o2345 import mesh_raster as MR
    obj = _backpack_obj(str(tmp_path))
    for ext in (".glb", ".obj"):
        out = str(tmp_path / f"full{ext}")
        res = SM.main(["--in", obj, "--out", out, "--target_faces", "1000000", "--texture_size", "1024",
                       "--atlas", "charts", "--normal_map"])
        assert res[5].shape == (1024, 1024, 3)
    g = mesh_io.read_glb(str(tmp_path / "full.glb"))
    assert len(g["meshes"][0]["faces"]) == 69960
    r = MR.render_rig(str(tmp_path / "full.glb"), resolution=128)
    assert (r["alpha"] > 0).sum() > 1000
    assert (tmp_path / "full.mtl").exists() and (tmp_path / "full_albedo.png").exists()


def test_run_py_writes_chart_textured_glb_and_obj_without_simplifying(tmp_path, monkeypatch):
    from PIL import Image
    import render_eval
    import run as run_cli
    from o2345 import mesh_io
    from test_gpu_texture import _image
    monkeypatch.chdir(tmp_path)
    img = str(tmp_path / "obj.png")
    Image.fromarray(_image(3)).save(img)
    for fmt in (".glb", ".obj"):
        out = run_cli.main(["--img_path", img, "--mesh_resolution", "64", "--seed", "2", "--texture_size", "512",
                            "--atlas", "charts", "--output_format", fmt])
        assert out.endswith(f"mesh{fmt}")
    g = mesh_io.read_glb(str(tmp_path / "exp" / "obj" / "mesh.glb"))
    assert g["textures"][0][0].shape == (512, 512, 4)
    assert (tmp_path / "exp" / "obj" / "mesh_albedo.png").exists()
    render_eval.main(["--object_path", str(tmp_path / "exp" / "obj" / "mesh.glb"), "--output_dir", str(tmp_path / "views"),
                      "--resolution", "128"])
    assert os.path.exists(tmp_path / "views" / "0.png")
