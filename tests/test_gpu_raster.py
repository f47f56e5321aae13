"""GPU: the mesh rasterizer (csrc/raster.cu through ops.raster / mesh_raster) against the numpy oracle
(oracle/raster_oracle.py): triangle ids bit-identical, depth / colour / texture colour within 1e-6 relative, on analytic
scenes and on the reference's example pair (backpack_gt.glb, backpack_ours.obj) from all 24 rig views; determinism;
analytic depth and texture; the silhouette IoU of the pair; the render_eval.py command line.  The pair's provenance and
what was trimmed from backpack_gt.glb (only images the renderer ignores): tests/golden/render_eval/README.md."""
import gzip
import math
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from o2345 import mesh_raster as MR
from o2345 import ops
from oracle import raster_oracle as RO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "render_eval")
PLANE_W2C = np.array([[[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]]], np.float32)


def gpu(flat, w2c, intr, W, H, shading=0):
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out = ops.raster(t(flat["verts"]), t(flat["faces"]), t(w2c), t(intr), W, H, shading=shading, colors=t(flat.get("colors")),
                     uvs=t(flat.get("uvs")), face_tex=t(flat.get("face_tex")), texels=t(flat.get("texels")),
                     tex_info=t(flat.get("tex_info")))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def compare(flat, w2c, intr, W, H, shading=0):
    ref = RO.render(flat["verts"], flat["faces"], w2c, intr, W, H, shading=shading, colors=flat.get("colors"),
                    uvs=flat.get("uvs"), face_tex=flat.get("face_tex"), texels=flat.get("texels"), tex_info=flat.get("tex_info"))
    out = gpu(flat, w2c, intr, W, H, shading)
    assert np.array_equal(out["tri"], ref["tri"])
    assert np.array_equal(out["alpha"], ref["alpha"])
    np.testing.assert_allclose(out["depth"], ref["depth"], rtol=1e-6, atol=0)
    np.testing.assert_allclose(out["color"], ref["color"], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(out["normal"], ref["normal"], rtol=1e-6, atol=1e-6)
    return out, ref


def plane(xy, z=1.0):
    xy = np.asarray(xy, np.float32)
    return np.concatenate([xy * np.float32(z), np.full((len(xy), 1), z, np.float32)], 1)


ANALYTIC = {
    "shared_edge": (plane([[0.5, 0.5], [6.5, 0.5], [0.5, 6.5], [6.5, 6.5]]), [[0, 1, 2], [1, 3, 2]], 8, [1, 1, 0, 0]),
    "fan": (plane([[3.5, 3.5]] + [[3.5 + 3 * math.cos(a), 3.5 + 3 * math.sin(a)] for a in np.linspace(0, 2 * math.pi, 9)[:-1]]),
            [[0, 1 + k, 1 + (k + 1) % 8] for k in range(8)], 8, [1, 1, 0, 0]),
    "coplanar": (np.concatenate([plane([[0.2, 0.3], [7.1, 0.9], [1.0, 6.8]]), plane([[0.2, 0.3], [7.1, 0.9], [1.0, 6.8]], 0.5)]),
                 [[0, 1, 2], [0, 1, 2], [3, 4, 5], [3, 4, 5]], 8, [1, 1, 0, 0]),
}


@pytest.mark.parametrize("name", sorted(ANALYTIC) + ["convex"])
def test_analytic_scenes_match_the_oracle(name):
    if name == "convex":
        from scipy.spatial import ConvexHull
        rng = np.random.default_rng(3)
        p = rng.normal(size=(60, 3))
        v = (p / np.linalg.norm(p, axis=1, keepdims=True) + [0, 0, 4]).astype(np.float32)
        f, W, K = ConvexHull(v).simplices, 32, [40, 40, 16, 16]
    else:
        v, f, W, K = ANALYTIC[name]
    rng = np.random.default_rng(0)
    flat = {"verts": v, "faces": np.asarray(f, np.int32), "colors": rng.uniform(size=(len(v), 3)).astype(np.float32)}
    out, _ = compare(flat, PLANE_W2C, np.array([K], np.float32), W, W)
    if name == "coplanar":
        assert set(np.unique(out["tri"])) == {-1, 2}


@pytest.fixture(scope="module")
def pair(tmp_path_factory):
    d = tmp_path_factory.mktemp("pair")
    obj = str(d / "backpack_ours.obj")
    with gzip.open(os.path.join(GOLD, "backpack_ours.obj.gz"), "rb") as src, open(obj, "wb") as dst:
        shutil.copyfileobj(src, dst)
    return {"gt": os.path.join(GOLD, "backpack_gt.glb"), "ours": obj}


@pytest.mark.parametrize("which", ["gt", "ours"])
@pytest.mark.parametrize("shading", ["unlit", "lambert"])
def test_example_pair_matches_the_oracle_at_all_24_views(pair, which, shading):
    flat = MR.flatten(MR.normalize_scene(MR.load_scene(pair[which])))
    w2c, intr = MR.camera_arrays(*MR.rig_cameras(1.3, 128))
    out, _ = compare(flat, w2c, intr, 128, 128, MR.SHADINGS[shading])
    assert 0.1 < out["alpha"].mean() < 0.6
    if which == "gt":
        assert flat["tex_info"] is not None and out["color"][out["alpha"] > 0].std() > 0.02


def test_two_runs_are_bit_identical(pair):
    flat = MR.flatten(MR.normalize_scene(MR.load_scene(pair["gt"])))
    c2w, K = MR.rig_cameras(1.3, 512)
    a = {k: v.cpu().numpy() for k, v in MR.render(flat, c2w, K, 512, 512, shading="lambert").items()}
    b = {k: v.cpu().numpy() for k, v in MR.render(flat, c2w, K, 512, 512, shading="lambert").items()}
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def test_plane_at_known_distance_gives_its_depth():
    d = 2.75
    v = np.array([[-5, -5, d], [5, -5, d], [5, 5, d], [-5, 5, d]], np.float32)
    flat = {"verts": v, "faces": np.array([[0, 1, 2], [0, 2, 3]], np.int32)}
    out = gpu(flat, PLANE_W2C, np.array([[50, 50, 32, 32]], np.float32), 64, 64)
    assert (out["tri"] >= 0).all()
    np.testing.assert_allclose(out["depth"], d, rtol=1e-6, atol=0)
    np.testing.assert_array_equal(out["normal"], np.broadcast_to([0, 0, -1], (1, 64, 64, 3)))


def test_textured_quad_reproduces_its_texture():
    W, H = 24, 16
    tex = np.random.default_rng(5).integers(0, 256, size=(H, W, 4)).astype(np.uint8)
    v = plane([[0, 0], [W, 0], [W, H], [0, H]], 1.0)
    flat = {"verts": v, "faces": np.array([[0, 1, 2], [0, 2, 3]], np.int32), "uvs": np.array([[0, 0], [1, 0], [1, 1], [0, 1]], np.float32),
            "face_tex": np.zeros(2, np.int32), "texels": tex.reshape(-1), "tex_info": np.array([[0, W, H, 1, 1]], np.int32)}
    out, _ = compare(flat, PLANE_W2C, np.array([[1, 1, 0, 0]], np.float32), W, H)
    np.testing.assert_allclose(out["color"][0], tex[..., :3] / 255.0, atol=1e-5)


# oracle/raster_oracle.py at 128^2, camera_dist 1.3: mean silhouette IoU over the 24 views of backpack_gt.glb and
# backpack_ours.obj = 0.8004; with the OBJ loaded without the Y-up -> Z-up change = 0.6040.  The threshold keeps a margin
# of 0.05 below the measured value; the wrong-axis control falls 0.15 short of it.
IOU_MEASURED, IOU_THRESHOLD = 0.8004, 0.75


def mean_iou(a, b):
    return float(((a & b).sum((1, 2)) / (a | b).sum((1, 2))).mean())


def test_silhouette_iou_of_the_pair(pair):
    c2w, K = MR.rig_cameras(1.3, 128)
    sil = lambda path, y_up=None: (MR.render(MR.flatten(MR.normalize_scene(MR.load_scene(path, y_up=y_up))), c2w, K, 128, 128)
                                   ["tri"] >= 0).cpu().numpy()
    gt = sil(pair["gt"])
    iou = mean_iou(gt, sil(pair["ours"]))
    assert abs(iou - IOU_MEASURED) < 1e-4 and iou > IOU_THRESHOLD
    assert mean_iou(gt, sil(pair["ours"], y_up=False)) < IOU_THRESHOLD      # negative control: the wrong axis convention


def test_command_line_writes_24_rgba_views(pair, tmp_path, capsys):
    sys.path.insert(0, os.path.join(ROOT, "one-2-3-45_b200"))
    import render_eval
    from PIL import Image
    out_dir = str(tmp_path / "views")
    render_eval.main(["--object_path", pair["gt"], "--output_dir", out_dir, "--resolution", "96", "--engine", "CYCLES"])
    assert "ignored" in capsys.readouterr().err
    ref = MR.render_rig(pair["gt"], 1.5, 96)["tri"].cpu().numpy()
    for i in range(24):
        img = np.asarray(Image.open(os.path.join(out_dir, f"{i}.png")))
        assert img.shape == (96, 96, 4)
        assert np.array_equal(img[..., 3] == 255, ref[i] >= 0) and set(np.unique(img[..., 3])) <= {0, 255}
    assert np.load(os.path.join(out_dir, "depth.npy")).shape == (24, 96, 96)
    assert np.load(os.path.join(out_dir, "normal.npy")).shape == (24, 96, 96, 3)
