"""GPU: normal-map baking (csrc/texture.cu tangent encode, quantise, vertex normals) and the normal-mapped branch of the
rasterizer (csrc/raster.cu) bit-identical to oracle/normal_map_oracle.py; an analytic normal field baked onto a sphere
and read back through the rasterizer; normals transferred from the full example mesh; the field path (SDF gradient)
through image_to_mesh, run.py and simplify_mesh.py."""
import os

import numpy as np
import pytest
import torch

from oracle import normal_map_oracle as NO
from oracle import texture_oracle as TO
from test_gpu_texture import _backpack_obj, _image, _sphere, dev_t, example6996, gpu_atlas  # noqa: F401

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


# ----------------------------------------------------------------------------- kernels against the oracle
def hand_cases():
    rng = np.random.default_rng(0)
    tet_v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    tet_f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    cube = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    cube_f = np.array([t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))])
    soup = rng.normal(size=(40, 3)).astype(np.float32)
    soup_f = rng.integers(0, 40, (60, 3))
    return {"tetrahedron": (tet_v, tet_f), "cube": (cube, cube_f), "soup": (soup, soup_f),
            "degenerate": (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0], [5, 5, 5]], np.float32),
                           np.array([[0, 1, 2], [0, 1, 3], [0, 0, 1], [2, 1, 0]]))}


@pytest.mark.parametrize("name", sorted(hand_cases()))
def test_hand_cases_are_bit_identical_to_the_oracle(name):
    from o2345 import ops
    v, f = hand_cases()[name]
    vt, ft = dev_t(v, np.float32), dev_t(f, np.int32)
    assert np.array_equal(bits(ops.vertex_normals(vt, ft).cpu().numpy()), bits(NO.vertex_normals(v, f)))
    rng = np.random.default_rng(len(f))
    uv = rng.random((len(f), 3, 2)).astype(np.float32)
    uv[0] = uv[0, :1]                                              # a face with det = 0
    tf = rng.integers(0, len(f), 500)
    n = rng.normal(size=(500, 3)).astype(np.float32)
    n[:3] = [[0, 0, 0], [np.nan, 1, 0], [0, np.inf, 0]]
    got = ops.tangent_normals(vt, ft, dev_t(uv, np.float32), dev_t(tf, np.int32), dev_t(n, np.float32)).cpu().numpy()
    want = NO.tangent_normals(v, f, uv, tf, n)
    assert np.array_equal(bits(got), bits(want))
    tex = rng.normal(size=(64, 64, 3)).astype(np.float32)
    tex[0, :4] = [[0, 0, 0], [np.nan, 0, 0], [np.inf, 1, 1], [1e-30, 0, 0]]
    assert np.array_equal(ops.normal_quantise(dev_t(tex, np.float32)).cpu().numpy(), NO.quantise_normals(tex))


@pytest.mark.parametrize("N", [1024, 2048])
def test_example_mesh_normal_bake_is_bit_identical(example6996, tmp_path, N):
    from o2345 import mesh_io, ops
    from o2345.mesh_texture import bake, normal_transfer_fn
    v0, vi, f = example6996
    _, f0, _ = mesh_io.read_obj(_backpack_obj(str(tmp_path)))
    vn = ops.vertex_normals(dev_t(v0, np.float32), dev_t(f0, np.int32)).cpu().numpy()
    assert np.array_equal(bits(vn), bits(NO.vertex_normals(v0, f0)))
    v = v0[vi]
    nfn = normal_transfer_fn(v0, f0, texture_size=N)
    uv, _, nmap, at = bake(v, f, N, lambda p: torch.zeros_like(p), normal_fn=nfn, return_atlas=True)
    normals = nfn(at["points"]).cpu().numpy()
    tn = NO.tangent_normals(v, f, uv, at["texel_face"].cpu().numpy(), normals)
    assert np.array_equal(bits(at["tangent_normals"].cpu().numpy()), bits(tn))
    filled = TO.fill(at["texel_index"].cpu().numpy(), tn, at["owner"].cpu().numpy(), N)
    assert np.array_equal(bits(at["normal_fill"].cpu().numpy()), bits(filled))
    assert np.array_equal(nmap, NO.quantise_normals(filled))
    _, _, again = bake(v, f, N, lambda p: torch.zeros_like(p), normal_fn=nfn)
    assert np.array_equal(nmap, again)                             # two runs, the same bytes
    owned = nmap.reshape(-1, 3)[at["texel_index"].cpu().numpy()]
    assert (owned[:, 2] > 128).mean() > 0.99                      # the source's normals agree with the faces' winding


# ----------------------------------------------------------------------------- the rasterizer's normal-map branch
def _mapped_scene(seed=0, flip_w=False):
    """A small closed mesh split per corner, with face normals, (T, w) of its atlas frame and a random normal map."""
    from o2345.mesh_io import tangent_frames
    v, f = _sphere(300)
    rng = np.random.default_rng(seed)
    uv = rng.random((len(f), 3, 2)).astype(np.float32)
    T, B, N = tangent_frames(v, f, uv)
    w = np.where(np.einsum("ij,ij->i", np.cross(N, T), B) < 0, -1.0, 1.0) * (-1 if flip_w else 1)
    fi = f.reshape(-1)
    tex = rng.integers(0, 256, (32, 32, 4), dtype=np.uint8)
    col = rng.integers(0, 256, (16, 16, 4), dtype=np.uint8)
    return {"verts": np.ascontiguousarray(v[fi]), "faces": np.arange(len(fi), dtype=np.int32).reshape(-1, 3),
            "colors": rng.random((len(fi), 3)).astype(np.float32), "uvs": uv.reshape(-1, 2),
            "face_tex": np.where(rng.random(len(f)) < 0.5, 0, -1).astype(np.int32),
            "texels": np.concatenate([col.reshape(-1), tex.reshape(-1)]),
            "tex_info": np.array([[0, 16, 16, 0, 0], [256, 32, 32, 1, 2]], np.int32),
            "normals": np.repeat(N, 3, 0).astype(np.float32),
            "tangents": np.repeat(np.concatenate([T, w[:, None]], 1), 3, 0).astype(np.float32),
            "face_ntex": np.where(rng.random(len(f)) < 0.8, 1, np.where(rng.random(len(f)) < 0.5, -1, 7)).astype(np.int32)}


@pytest.mark.parametrize("shading", [0, 1])
def test_normal_mapped_raster_is_bit_identical_to_the_oracle(shading):
    from o2345 import mesh_raster as MR
    scene = _mapped_scene()
    scene["normals"][:3] = 0                                      # a face whose interpolated normal has no direction
    c2w, K = MR.rig_cameras(1.5, 96)
    c2w, K = c2w[::5], K
    out = MR.render(scene, c2w, K, 96, 96, shading=["unlit", "lambert"][shading])
    w2c, intr = MR.camera_arrays(c2w, K)
    want = NO.render(scene["verts"], scene["faces"], w2c, intr, 96, 96, shading=shading,
                     **{k: scene[k] for k in ("colors", "uvs", "face_tex", "texels", "tex_info", "normals", "tangents",
                                              "face_ntex")})
    for k in ("color", "normal", "depth", "alpha"):
        assert np.array_equal(bits(out[k].cpu().numpy()), bits(want[k])), k
    assert np.array_equal(out["tri"].cpu().numpy(), want["tri"])
    plain = MR.render(dict(scene, normals=None, tangents=None, face_ntex=None), c2w, K, 96, 96,
                      shading=["unlit", "lambert"][shading])
    changed = (out["normal"] != plain["normal"]).any(-1)
    assert changed.sum() > 1000                                   # the map really is applied


def test_normals_and_tangents_without_a_normal_map_render_as_before(tmp_path):
    from o2345 import mesh_io
    from o2345 import mesh_raster as MR
    p = os.path.join(os.path.dirname(__file__), "golden", "render_eval", "backpack_gt.glb")
    flat = MR.flatten(MR.normalize_scene(MR.load_scene(p)))
    scene = MR.normalize_scene(MR.load_scene(p))
    nv = len(flat["verts"])
    c2w, K = MR.rig_cameras(1.5, 128)
    base = MR.render(flat, c2w[:6], K, 128, 128, shading="lambert")
    # the file's own NORMAL / TANGENT given to the kernel, with no face pointing at a normal map
    nrm = np.concatenate([m["normals"] if m["normals"] is not None else np.zeros((len(m["verts"]), 3))
                          for m in scene["meshes"]]).astype(np.float32)
    tan = np.concatenate([m["tangents"] if m["tangents"] is not None else np.zeros((len(m["verts"]), 4))
                          for m in scene["meshes"]]).astype(np.float32)
    assert len(nrm) == nv
    for face_ntex in (None, np.full(len(flat["faces"]), -1, np.int32)):
        out = MR.render(dict(flat, normals=nrm, tangents=tan, face_ntex=face_ntex), c2w[:6], K, 128, 128, shading="lambert")
        for k in base:
            assert torch.equal(out[k], base[k]), k
    # the same mesh written with a normal map that codes (0, 0, 1) everywhere: geometry and coverage unchanged
    v, f = flat["verts"], flat["faces"]
    uv = np.random.default_rng(0).random((len(f), 3, 2)).astype(np.float32)
    q = str(tmp_path / "flat.glb")
    mesh_io.write_textured_glb(q, v, f, uv, np.full((8, 8, 3), 200, np.uint8), np.tile([[[128, 128, 255]]], (8, 8, 1)).astype(np.uint8))
    a = MR.render_rig(q, resolution=128)
    assert (a["alpha"] > 0).sum() > 1000


# ----------------------------------------------------------------------------- analytic round trip
def _outward(v, f):
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    return f if (np.einsum("ij,ij->i", n, v[f].mean(1)) > 0).mean() > 0.5 else f[:, ::-1].copy()


def test_analytic_normal_round_trips_through_the_rasterizer(tmp_path):
    from o2345 import mesh_io
    from o2345 import mesh_raster as MR
    from o2345.mesh_texture import bake
    v, f = _sphere()
    f = _outward(v, f)
    N = 512
    uv, tex, nmap, at = bake(v, f, N, lambda p: torch.full_like(p, 0.5), normal_fn=lambda p: p, return_atlas=True)
    rho, rmin = at["rho"], float(np.linalg.norm(at["points"].cpu().numpy(), axis=1).min())
    # worst angle: the four texels of a bilinear sample hold the normal of surface points up to one texel diagonal
    # (sqrt(2) / rho) from the pixel's point, and p / |p| turns by at most that distance over |p| >= rmin; the 8-bit
    # code moves each component by at most 1/255, i.e. the unit vector by sqrt(3) / 255 (radians, to first order)
    bound = np.sqrt(2) / (rho * rmin) + np.sqrt(3) / 255
    c2w, K = MR.rig_cameras(1.5, 256)

    def errors(path):
        """Per view: the angle between the rendered normal and p / |p| at every covered pixel, and p / |p|."""
        out = MR.render_rig(path, resolution=256)
        nrm, alpha, depth = (out[k].cpu().numpy() for k in ("normal", "alpha", "depth"))
        flat = MR.flatten(MR.normalize_scene(MR.load_scene(path)))
        centre = flat["verts"].astype(np.float64).mean(0)         # the sphere's centre in the rig frame
        res = []
        for i in range(len(c2w)):
            yy, xx = np.nonzero(alpha[i] > 0)
            zc = depth[i, yy, xx].astype(np.float64)
            pc = np.stack([(xx + 0.5 - K[0, 2]) / K[0, 0] * zc, (yy + 0.5 - K[1, 2]) / K[1, 1] * zc, zc, np.ones_like(zc)], 1)
            pw = (pc @ c2w[i].T)[:, :3] - centre
            want = pw / np.linalg.norm(pw, axis=1, keepdims=True)
            res.append((np.arccos(np.clip(np.einsum("ij,ij->i", nrm[i, yy, xx], want), -1, 1)), yy, xx))
        return res

    def worst(path):
        # pixels whose winning facet faces the camera (its flat normal within 90 deg of p / |p|): on the silhouette a
        # facet of the far side can win the depth tie, and its camera-facing normal is rightly the opposite one
        return max(e[front[i][y, x]].max() for i, (e, y, x) in enumerate(errors(path)))

    def write(name, nt, flip_w=False):
        p = str(tmp_path / name)
        v2, f2, uv2 = mesh_io.to_viewer_frame(v, f, uv)
        mesh_io.write_textured_glb(p, v2, f2, uv2, tex, nt)
        if flip_w:                                                # TANGENT w negated in the file
            import json
            import struct
            raw = bytearray(open(p, "rb").read())
            jl = struct.unpack_from("<I", raw, 12)[0]
            doc = json.loads(bytes(raw[20:20 + jl]))
            acc = doc["accessors"][doc["meshes"][0]["primitives"][0]["attributes"]["TANGENT"]]
            bv = doc["bufferViews"][acc["bufferView"]]
            start = 20 + jl + 8 + bv["byteOffset"]
            t = np.frombuffer(bytes(raw[start:start + bv["byteLength"]]), np.float32).reshape(-1, 4).copy()
            t[:, 3] *= -1
            raw[start:start + bv["byteLength"]] = t.tobytes()
            open(p, "wb").write(bytes(raw))
        return p
    flat_path = write("flat.glb", None)
    front = []
    for e, y, x in errors(flat_path):
        m = np.zeros((256, 256), bool)
        m[y, x] = e < np.pi / 2
        front.append(m)
    good = worst(write("good.glb", nmap))
    green = nmap.copy()
    green[..., 1] = 255 - green[..., 1]
    controls = {"no map": worst(flat_path), "green flipped": worst(write("green.glb", green)),
                "w negated": worst(write("w.glb", nmap, flip_w=True))}
    print(f"analytic normal round trip: rho {rho:.1f}, |p| >= {rmin:.3f}, bound {np.degrees(bound):.3f} deg, "
          f"worst {np.degrees(good):.3f} deg, " + ", ".join(f"{k} {np.degrees(e):.2f} deg" for k, e in controls.items()))
    assert good <= bound + 1e-3                                   # 1e-3 rad: the point recovered from fp32 depth
    for k, e in controls.items():
        assert e > bound, k


# ----------------------------------------------------------------------------- real normals from the full mesh
# measured on an H100 80GB HBM3 at 700 W (DESIGN §2): mean angle between the rendered normals of the 6 996-face mesh and
# the 69 960-face original's over pixels covered in both, 24 rig views at 512^2.  Against the original's facets: flat
# 3.218 deg, with the transferred N = 2048 normal map 2.417 deg; against its vertex normals: 3.703 and 0.543 deg.  The
# computation is deterministic; the slack only absorbs a change of GPU model.
MARGIN_DEG = {"facets": 0.801, "vertex normals": 3.160}
SLACK_DEG = 0.2


def _smooth(flat, normals):
    """flatten()'s arrays shaded with the given vertex normals: a 1 x 1 map coding (128, 128, 255) decodes to the
    interpolated normal tilted by atan(sqrt(2) (128 / 127.5 - 1)) < 0.32 deg."""
    n = normals / np.linalg.norm(normals, axis=1, keepdims=True)
    a = np.where(np.abs(n[:, :1]) < 0.9, [[1.0, 0.0, 0.0]], [[0.0, 1.0, 0.0]])
    t = np.cross(n, a)
    t /= np.linalg.norm(t, axis=1, keepdims=True)
    return dict(flat, uvs=np.zeros((len(n), 2), np.float32), face_tex=np.full(len(flat["faces"]), -1, np.int32),
                texels=np.array([128, 128, 255, 255], np.uint8), tex_info=np.array([[0, 1, 1, 1, 1]], np.int32),
                normals=n.astype(np.float32), tangents=np.concatenate([t, np.ones((len(n), 1))], 1).astype(np.float32),
                face_ntex=np.zeros(len(flat["faces"]), np.int32))


def test_transferred_normal_map_is_closer_to_the_original(example6996, tmp_path):
    from o2345 import mesh_io, ops
    from o2345 import mesh_raster as MR
    from o2345.mesh_texture import bake, normal_transfer_fn
    v0, vi, f = example6996
    obj = _backpack_obj(str(tmp_path))
    _, f0, _ = mesh_io.read_obj(obj)
    N = 2048
    uv, tex, nmap = bake(v0[vi], f, N, lambda p: torch.full_like(p, 0.5), normal_fn=normal_transfer_fn(v0, f0, texture_size=N))
    c2w, K = MR.rig_cameras(1.5, 512)
    # the original as the rasterizer shades it (flat facets), and shaded by its own surface normal (its vertex normals in
    # the rig frame: the loader's frame change is a rotation and a uniform scale, so they are the same field)
    flat0 = MR.flatten(MR.normalize_scene(MR.load_scene(obj)))
    vn = ops.vertex_normals(dev_t(flat0["verts"], np.float32), dev_t(flat0["faces"], np.int32)).cpu().numpy()
    refs = {"facets": MR.render(flat0, c2w, K, 512, 512), "vertex normals": MR.render(_smooth(flat0, vn), c2w, K, 512, 512)}
    res = {}
    for name, nt in (("plain", None), ("mapped", nmap)):
        p = str(tmp_path / f"{name}.glb")
        mesh_io.write_textured_glb(p, v0[vi], f, uv, tex, nt)          # the OBJ's own frame, as the original is loaded
        r = MR.render_rig(p, resolution=512)
        for rn, ref in refs.items():
            m = (ref["alpha"] > 0) & (r["alpha"] > 0)
            cos = (r["normal"] * ref["normal"]).sum(-1).clamp(-1, 1)
            res[name, rn] = float(torch.rad2deg(torch.arccos(cos[m])).mean())
    for rn in refs:
        margin = res["plain", rn] - res["mapped", rn]
        print(f"mean normal angle against the original's {rn}: flat {res['plain', rn]:.3f} deg, normal map "
              f"{res['mapped', rn]:.3f} deg, margin {margin:.3f} deg")
        assert margin > MARGIN_DEG[rn] - SLACK_DEG, rn


# ----------------------------------------------------------------------------- the field path
STEPS = dict(ddim_steps=4, stage2_steps=2)
R = 64


def test_image_to_mesh_bakes_the_sdf_gradient(tmp_path, monkeypatch):
    from o2345 import mesh_texture as MT
    from o2345 import synthetic as S
    from o2345.pipeline import build_networks, image_to_mesh
    from o2345.zero123 import build_zero123
    dev = torch.device("cuda:0")
    z = build_zero123(dev, seed=0, clip=True).half()
    tr = build_networks(dev, vol_dim=96, states=S.all_states(0), perturb=0.0)
    seen = {}
    real = MT.bake

    def spy(vertices, faces, n, colour_fn, device=None, normal_fn=None):
        uv, tex, nmap, at = real(vertices, faces, n, colour_fn, device, return_atlas=True, normal_fn=normal_fn)
        seen.update(at=at, normal_fn=normal_fn, vertices=vertices)
        return uv, tex, nmap
    monkeypatch.setattr(MT, "bake", spy)
    torch.cuda.manual_seed(5)
    out = image_to_mesh(z, tr, _image(), polar_angle=60, resolution=R, target_faces=2000, texture_size=256,
                        normal_map=True, **STEPS)
    nmap, at = out["normal_texture"], seen["at"]
    assert nmap.shape == (256, 256, 3) and nmap.dtype == np.uint8
    idx = at["texel_index"].cpu().numpy()
    g = seen["normal_fn"](at["points"]).cpu().numpy().astype(np.float64)
    T, B, Nf, ok = NO.frames(seen["vertices"], out["triangles"], out["uv"])
    tf = at["texel_face"].cpu().numpy()
    t = nmap.reshape(-1, 3)[idx].astype(np.float64) / 127.5 - 1
    dec = t[:, :1] * T[tf] + t[:, 1:2] * B[tf] + t[:, 2:] * Nf[tf]
    dec /= np.linalg.norm(dec, axis=1, keepdims=True)
    gl = np.linalg.norm(g, axis=1)
    use = ok[tf] & (gl > 0)
    ang = np.arccos(np.clip(np.einsum("ij,ij->i", dec[use], g[use] / gl[use, None]), -1, 1))
    bound = np.sqrt(3) / 255 + 1e-4                               # the 8-bit code; owned texels are not touched by the fill
    print(f"field path: {use.sum()} texels, worst decoded angle {np.degrees(ang.max()):.3f} deg")
    assert use.mean() > 0.99 and ang.max() <= bound


def test_run_py_writes_a_normal_mapped_glb_that_renders(tmp_path, monkeypatch):
    from PIL import Image
    import render_eval
    import run as run_cli
    from o2345 import mesh_io
    monkeypatch.chdir(tmp_path)
    img = str(tmp_path / "obj.png")
    Image.fromarray(_image(3)).save(img)
    out = run_cli.main(["--img_path", img, "--mesh_resolution", "64", "--seed", "2", "--target_faces", "2000",
                        "--texture_size", "512", "--normal_map", "--output_format", ".glb"])
    g = mesh_io.read_glb(out)
    assert len(g["textures"]) == 2 and (g["meshes"][0]["face_ntex"] == 1).all()
    render_eval.main(["--object_path", out, "--output_dir", str(tmp_path / "views"), "--resolution", "128"])
    nrm = np.load(tmp_path / "views" / "normal.npy")
    cov = np.abs(nrm).sum(-1) > 0
    assert cov.sum() > 1000
    np.testing.assert_allclose(np.linalg.norm(nrm[cov], axis=-1), 1, atol=1e-5)


def test_simplify_mesh_writes_normal_mapped_glb_and_obj(tmp_path):
    import simplify_mesh as SM
    from o2345 import mesh_io
    obj = _backpack_obj(str(tmp_path))
    for ext in (".glb", ".obj"):
        res = SM.main(["--in", obj, "--out", str(tmp_path / f"small{ext}"), "--target_faces", "3000", "--texture_size", "512",
                       "--normal_map"])
        assert res[6].shape == (512, 512, 3)
    g = mesh_io.read_glb(str(tmp_path / "small.glb"))
    assert len(g["textures"]) == 2 and set(np.unique(g["meshes"][0]["tangents"][:, 3])) <= {-1.0, 1.0}
    assert (tmp_path / "small_normal.png").exists()
    assert "norm small_normal.png" in open(tmp_path / "small.mtl").read()
