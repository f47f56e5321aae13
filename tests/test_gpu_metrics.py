"""GPU: mesh scoring (csrc/metrics.cu through ops / mesh_metrics) against the numpy oracle (oracle/metrics_oracle.py):
surface samples and nearest neighbours bit-identical, F-Score counts equal and Chamfer within 1e-9 on the reference's
example pair, determinism, the CLIP-similarity plumbing with synthetic weights, and the eval_mesh.py command line."""
import gzip
import json
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from o2345 import mesh_metrics as MM
from o2345 import mesh_raster as MR
from o2345 import ops
from oracle import metrics_oracle as MO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "render_eval")
N_PAIR, TAU = 20000, 0.05


@pytest.fixture(scope="module")
def pair(tmp_path_factory):
    obj = str(tmp_path_factory.mktemp("pair") / "backpack_ours.obj")
    with gzip.open(os.path.join(GOLD, "backpack_ours.obj.gz"), "rb") as src, open(obj, "wb") as dst:
        shutil.copyfileobj(src, dst)
    gt = os.path.join(GOLD, "backpack_gt.glb")
    return {"gt": gt, "ours": obj, "flat_gt": MM.load_flat(gt), "flat_ours": MM.load_flat(obj)}


def gpu_sample(verts, faces, n, seed):
    p, f = ops.surface_sample(torch.from_numpy(np.asarray(verts, np.float32)).cuda(),
                              torch.from_numpy(np.asarray(faces, np.int32)).cuda(), n, seed)
    return p.cpu().numpy(), f.cpu().numpy()


def gpu_nearest(query, ref):
    d2, idx = ops.nearest(torch.from_numpy(np.asarray(query, np.float32)).cuda(), torch.from_numpy(np.asarray(ref, np.float32)).cuda())
    return d2.cpu().numpy(), idx.cpu().numpy()


def analytic_meshes():
    from scipy.spatial import ConvexHull
    rng = np.random.default_rng(4)
    tri = (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32), [[0, 1, 2]])
    # areas 1 : 3, plus a zero-area face, a repeated index and out-of-range / negative indices
    v2 = np.array([[0, 0, 0], [1, 0, 0], [0, 2, 0], [5, 0, 0], [8, 0, 0], [5, 2, 0], [9, 9, 9]], np.float32)
    two = (v2, [[0, 0, 1], [0, 1, 2], [6, 7, 1], [3, 4, 5], [-1, 2, 3], [0, 3, 4]])
    p = rng.normal(size=(3000, 3))
    hull_v = (p / np.linalg.norm(p, axis=1, keepdims=True) * [0.3, 0.2, 0.1]).astype(np.float32)
    hull_f = ConvexHull(hull_v).simplices.astype(np.int32)      # ~6000 faces: several CDF chunks
    hull_f[::97] = hull_f[::97, [0, 0, 1]]                       # zero-area faces inside the chunks
    hull_f[5::211, 2] = len(hull_v) + 3                          # bad indices
    return {"triangle": tri, "two": two, "hull": (hull_v, hull_f)}


@pytest.mark.parametrize("name", ["triangle", "two", "hull"])
@pytest.mark.parametrize("n,seed", [(1, 0), (12345, 7), (20000, 2 ** 64 - 1)])
def test_sampling_is_bit_identical_to_the_oracle_on_analytic_meshes(name, n, seed):
    v, f = analytic_meshes()[name]
    p, fid = gpu_sample(v, f, n, seed)
    rp, rf = MO.surface_sample(v, f, n, seed)
    assert np.array_equal(fid, rf) and p.tobytes() == rp.tobytes()
    assert (MO.surface_weights(v, f)[fid] > 0).all()


@pytest.mark.parametrize("which", ["gt", "ours"])
def test_sampling_is_bit_identical_to_the_oracle_on_the_example_meshes(pair, which):
    flat = pair["flat_" + which]                  # backpack_gt.glb: 53 objects flattened into one mesh
    p, fid = gpu_sample(flat["verts"], flat["faces"], 50000, 11)
    rp, rf = MO.surface_sample(flat["verts"], flat["faces"], 50000, 11)
    assert np.array_equal(fid, rf) and p.tobytes() == rp.tobytes()


def test_sampling_without_area_is_refused():
    from o2345 import _lib
    with pytest.raises(_lib.O2345Error, match="no area"):
        gpu_sample(np.zeros((3, 3), np.float32), [[0, 1, 2], [0, 1, 5]], 10, 0)


def nn_cases():
    rng = np.random.default_rng(8)
    cube = rng.uniform(-0.4, 0.4, size=(1999, 3)).astype(np.float32)
    # reference on a 9^3 lattice over [0, 1]: grid side 14, so lattice points, cell faces (k / 14) and the bbox corners
    # are all query points
    g = np.arange(9, dtype=np.float32) / np.float32(8)
    lat = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    b = np.arange(15, dtype=np.float32) / np.float32(14)
    bq = np.stack(np.meshgrid(b, b[::3], b[::2], indexing="ij"), -1).reshape(-1, 3)
    corners = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32)
    dup = np.repeat(rng.uniform(size=(400, 3)).astype(np.float32), 3, 0)[rng.permutation(1200)]
    d = rng.normal(size=(500, 3))
    far = (d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(2, 1000, size=(500, 1))).astype(np.float32)
    plane = np.concatenate([rng.uniform(-1, 1, size=(3000, 2)), np.zeros((3000, 1))], 1).astype(np.float32)
    return {
        "random": (rng.uniform(-0.5, 0.5, size=(3001, 3)).astype(np.float32), cube),
        "lattice_boundaries": (np.concatenate([lat, bq, corners, lat + np.float32(1 / 16)]), lat),
        "duplicates": (np.concatenate([rng.uniform(size=(700, 3)).astype(np.float32), dup[:300]]), dup),
        "far": (np.concatenate([far, far + 0.3]), cube),
        "planar": (rng.uniform(-1.5, 1.5, size=(2500, 3)).astype(np.float32), plane),
        "single_point": (rng.normal(size=(777, 3)).astype(np.float32), np.array([[0.25, -1, 3]], np.float32)),
        "one_place": (rng.normal(size=(300, 3)).astype(np.float32), np.tile(np.float32([[1, 2, 3]]), (64, 1))),
        "n1": (np.array([[0.1, 0.2, 0.3]], np.float32), cube),
        "n1_both": (np.array([[0.1, 0.2, 0.3]], np.float32), np.array([[-5, 0, 5]], np.float32)),
    }


@pytest.mark.parametrize("name", sorted(nn_cases()))
def test_nearest_is_bit_identical_to_brute_force(name):
    q, r = nn_cases()[name]
    d2, idx = gpu_nearest(q, r)
    rd2, ridx = MO.nearest(q, r)
    assert np.array_equal(idx, ridx) and d2.tobytes() == rd2.tobytes()


def test_nearest_on_the_example_pair_samples_both_ways(pair):
    p, _ = MO.surface_sample(pair["flat_ours"]["verts"], pair["flat_ours"]["faces"], N_PAIR, 0)
    g, _ = MO.surface_sample(pair["flat_gt"]["verts"], pair["flat_gt"]["faces"], N_PAIR, 1)
    for q, r in ((p, g), (g, p)):
        d2, idx = gpu_nearest(q, r)
        rd2, ridx = MO.nearest(q, r)
        assert np.array_equal(idx, ridx) and d2.tobytes() == rd2.tobytes()


@pytest.fixture(scope="module")
def pair_oracle(pair):
    return MO.score(pair["flat_ours"], pair["flat_gt"], N_PAIR, (TAU, 0.02), seed=0)


def test_fscore_chamfer_of_the_pair_equals_the_oracle(pair, pair_oracle):
    a = MM.fscore_chamfer(pair["flat_ours"], pair["flat_gt"], N_PAIR, (TAU, 0.02), seed=0)
    for tau in (TAU, 0.02):
        assert a["fscore"][tau] == pair_oracle["fscore"][tau]
    assert abs(a["chamfer"] - pair_oracle["chamfer"]) <= 1e-9 * pair_oracle["chamfer"]
    b = MM.fscore_chamfer(pair["flat_ours"], pair["flat_gt"], N_PAIR, (TAU, 0.02), seed=0)
    assert a == b


def test_clip_similarity_plumbing(pair):
    from o2345 import synthetic as S
    from o2345.zero123 import load_clip_image_embedder
    ckpt = {"state_dict": {"cond_stage_model." + k: torch.from_numpy(v) for k, v in S.clip_state(20).items()}}
    ckpt["state_dict"]["model.diffusion_model.out.2.bias"] = torch.zeros(4)       # ignored: only the tower is read
    emb = load_clip_image_embedder(ckpt, device="cuda")
    same = MM.clip_similarity(pair["gt"], pair["gt"], emb, resolution=128)
    assert len(same["per_view"]) == 24 and max(abs(c - 1) for c in same["per_view"]) < 1e-6
    s = MM.clip_similarity(pair["ours"], pair["gt"], emb, resolution=128)

    def views(path):
        out = MR.render_rig(path, 1.3, 128)
        a = out["alpha"][..., None]
        return ((out["color"].clamp(0, 1) * a + (1 - a)) * 2 - 1).permute(0, 3, 1, 2).contiguous()   # rgb * alpha + (1 - alpha)
    with torch.no_grad():
        ea, eb = emb(views(pair["ours"])).double(), emb(views(pair["gt"])).double()
    cos = ((ea * eb).sum(1) / (ea.norm(dim=1) * eb.norm(dim=1))).tolist()
    np.testing.assert_allclose(s["per_view"], cos, rtol=0, atol=1e-6)
    assert abs(s["mean"] - np.mean(cos)) < 1e-6
    del ckpt["state_dict"]["cond_stage_model.model.visual.proj"]
    with pytest.raises(KeyError):
        load_clip_image_embedder(ckpt)


def test_command_line_on_the_pair(pair, pair_oracle, tmp_path, capsys):
    sys.path.insert(0, os.path.join(ROOT, "one-2-3-45_b200"))
    import eval_mesh
    out = str(tmp_path / "scores.json")
    eval_mesh.main(["--pred", pair["ours"], "--gt", pair["gt"], "--n_points", str(N_PAIR), "--out", out])
    lines = capsys.readouterr().out.strip().splitlines()
    o = pair_oracle["fscore"][TAU]
    expect = f"F@0.05={o['fscore']:.6f} P={o['precision']:.6f} R={o['recall']:.6f} chamfer={pair_oracle['chamfer']:.6f}"
    assert lines[0] == f"{pair['ours']} vs {pair['gt']}: {expect}"
    assert lines[1] == f"mean over 1 pairs: {expect}"
    doc = json.load(open(out))
    assert doc["protocol"]["n_points"] == N_PAIR and doc["protocol"]["thresholds"] == [TAU] and doc["protocol"]["clip"] is None
    assert doc["pairs"][0]["fscore"]["0.05"]["n_precise"] == o["n_precise"]
    assert doc["mean"]["fscore"]["0.05"]["fscore"] == o["fscore"]
