"""GPU: the lod-1 refinement path (num_lods = 2) against the golden vectors frozen from the REAL reference
(tests/golden/lod1_mini.npz, oracle/pin_lod1_against_reference.py) and the CPU restatement of oracle/lod1_oracle.py at
the mini configuration (D0 = 24 -> D1 = 48), full-size properties (32 views of 256^2, 96^3 -> 192^3, R = 256), the
reconstruction CLI with a num_lods = 2 conf, and the argument checks of the new entry points.

Tolerances as in test_gpu_parity.py: sdf 5e-5, cost rows 5e-4, dense volume 5e-4; flags and survivors bit-exact.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch

from helpers import MINI, OracleMini
from oracle import lod1_oracle as L1
from oracle import recon_oracle as O
from oracle.pin_lod1_against_reference import PRUNE_CASES, PRUNE_SEED

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D0, D1 = MINI["D"], 2 * MINI["D"]


def maxerr(a, b):
    return float((torch.as_tensor(a).double().cpu() - torch.as_tensor(b).double().cpu()).abs().max())


BLEND_TOL = {0: 2e-4, 1: 5e-4}          # fp32 / tensor-core blend kernels, as in test_gpu_parity.py


@pytest.fixture(scope="module")
def g1():
    return np.load(os.path.join(ROOT, "tests", "golden", "lod1_mini.npz"))


def lattice_mask(coords, D):
    c = coords[:, 1:].long().cpu()
    m = np.zeros(D ** 3, bool)
    m[((c[:, 0] * D + c[:, 1]) * D + c[:, 2]).numpy()] = True
    return m


def mask_coords(packed, D):
    lin = np.nonzero(np.unpackbits(packed)[:D ** 3])[0]
    xyz = np.stack([lin // (D * D), (lin // D) % D, lin % D], 1)
    return torch.from_numpy(np.concatenate([np.zeros((len(lin), 1)), xyz], 1)).float()


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def om():
    return OracleMini()


@pytest.fixture(scope="module")
def st1():
    from o2345 import synthetic as S
    return {k: O.to_torch_state(v) for k, v in S.lod1_states(0).items()}


@pytest.fixture(scope="module")
def tr(dev):
    from o2345 import synthetic as S
    from o2345.pipeline import build_networks
    states = {**S.all_states(0), **S.lod1_states(0)}
    return build_networks(dev, vol_dim=D0, states=states, perturb=0.0, num_lods=2)


@pytest.fixture(scope="module")
def lod0(om, tr, dev):
    """lod-0 volume and SDF volume computed by the CUDA path."""
    fm = tr.obtain_pyramid_feature_maps(om.imgs.to(dev))
    cond = tr.sdf_network_lod0.get_conditional_volume(fm[None], om.origin.to(dev)[None], om.proj.to(dev)[None],
                                                      sizeH=MINI["H"], sizeW=MINI["W"])
    sdf = tr.sdf_network_lod0.get_sdf_volume(cond["dense_volume_scale0"], cond["valid_mask_volume_scale0"],
                                             cond["coords_scale0"], om.origin.to(dev)[None])
    return {"cond": cond, "sdf": sdf}


def test_sdf_volume(om, tr, lod0, dev, g1, golden):
    assert np.array_equal(lod0["cond"]["valid_mask_volume_scale0"].cpu().numpy().astype(np.int8).reshape(-1), golden["occ"])
    assert maxerr(lod0["sdf"].reshape(-1), g1["sdf0"]) < 1e-4            # the reference's get_sdf_volume
    from o2345 import _lib, ops
    vol, occ = lod0["cond"]["dense_volume_scale0"], lod0["cond"]["valid_mask_volume_scale0"]
    ref = L1.sdf_volume(vol.cpu(), occ.cpu(), om.origin, tr.sdf_network_lod0.voxel_size, om.st["sdf_network_lod0"])
    assert lod0["sdf"].shape == (1, 1, D0, D0, D0)
    assert maxerr(lod0["sdf"], ref) < 5e-5
    outside = occ.reshape(-1) == 0
    assert outside.any() and bool((lod0["sdf"].reshape(-1)[outside] == 1.0).all())
    fp32 = ops.sdf_voxels(occ.reshape(-1), vol._o2345_cl[1], om.origin.to(dev), tr.sdf_network_lod0.voxel_size,
                          tr.sdf_network_lod0.sdf_layer.packed(), precision=_lib.SDF_FP32)
    assert maxerr(fp32, ref.reshape(-1)) < 5e-5


@pytest.mark.parametrize("case", PRUNE_CASES)
def test_prune_bit_exact(tr, lod0, g1, dev, case):
    """The kernel fed the reference's own lod-0 SDF volume keeps exactly the reference's survivors at the default budget,
    part-way down the threshold ladder and through the seeded subsample."""
    vol, occ = lod0["cond"]["dense_volume_scale0"], lod0["cond"]["valid_mask_volume_scale0"]
    sdf = torch.from_numpy(g1["sdf0"]).to(dev).reshape(1, D0, D0, D0)
    max_pts = int(g1["prune_max_pts"][PRUNE_CASES.index(case)])
    np.random.seed(PRUNE_SEED)
    coords, feats = tr.sdf_renderer_lod0.get_valid_sparse_coords_by_sdf(sdf, lod0["cond"]["coords_scale0"][0], occ[0],
                                                                        vol[0], maximum_pts=max_pts)
    assert np.array_equal(np.packbits(lattice_mask(coords, D0)), g1[f"prune_{case}_mask"])
    assert torch.equal(coords.cpu(), mask_coords(g1[f"prune_{case}_mask"], D0))          # lattice order, batch column 0
    assert maxerr(feats.flatten()[::7], g1[f"prune_{case}_feat_s"]) < 5e-4
    # the same call on the CPU restatement, same volume
    np.random.seed(PRUNE_SEED)
    rc, rf, _, rthr = L1.prune(sdf.cpu(), occ.cpu()[0], vol.cpu()[0], maximum_pts=max_pts)
    assert torch.equal(coords.cpu(), rc) and torch.equal(feats.cpu(), rf)
    last = tr.sdf_renderer_lod0._last_prune
    assert last["ladder"][last["rung"]] == np.float32(rthr)
    if case == "subsample":
        assert coords.shape[0] == max_pts and last["rung"] == len(last["ladder"]) - 1
    if case == "ladder":
        assert last["rung"] >= 1 and last["counts"][last["rung"]] <= max_pts < last["counts"][last["rung"] - 1]


def test_prune_rejects_a_coords_volume_that_is_not_the_lattice(tr, lod0):
    vol, occ = lod0["cond"]["dense_volume_scale0"], lod0["cond"]["valid_mask_volume_scale0"]
    with pytest.raises(ValueError):
        tr.sdf_renderer_lod0.get_valid_sparse_coords_by_sdf(lod0["sdf"][0], lod0["cond"]["coords_scale0"][0] * 2, occ[0],
                                                            vol[0])


@pytest.fixture(scope="module")
def lod1(om, tr, lod0, st1, g1, dev):
    """lod-1 volume from the reference's default-budget survivors (features from this path's lod-0 volume)."""
    vol, occ = lod0["cond"]["dense_volume_scale0"], lod0["cond"]["valid_mask_volume_scale0"]
    sdf = torch.from_numpy(g1["sdf0"]).to(dev).reshape(1, D0, D0, D0)
    pre_c, pre_f = tr.sdf_renderer_lod0.get_valid_sparse_coords_by_sdf(sdf, lod0["cond"]["coords_scale0"][0], occ[0], vol[0])
    pre_c[:, 1:] = pre_c[:, 1:] * 2
    fm1 = tr.obtain_pyramid_feature_maps(om.imgs.to(dev), lod=1)
    net = tr.sdf_network_lod1
    cond = net.get_conditional_volume(fm1[None], om.origin.to(dev)[None], om.proj.to(dev)[None], sizeH=MINI["H"],
                                      sizeW=MINI["W"], pre_coords=pre_c, pre_feats=pre_f)
    fm1_ref = O.pyramid_feature_maps(om.imgs, st1["pyramid_feature_network_lod1"])
    ref = L1.conditional_volume(fm1_ref, om.origin, om.proj, st1["sdf_network_lod1"], D1, net.voxel_size, MINI["H"],
                                MINI["W"], pre_c.cpu(), pre_f.cpu())
    return {"cond": cond, "last": net._last, "ref": ref, "fm1": fm1, "fm1_ref": fm1_ref, "n_pre": pre_c.shape[0]}


def test_lod1_children_bit_exact(lod1, g1):
    last, ref = lod1["last"], lod1["ref"]
    assert np.array_equal(np.packbits(last["keep"].cpu().numpy().astype(bool)), g1["lod1_keep"])
    n = int(last["count"].item())
    xyz = ref["xyz"].long()
    lin = ((xyz[:, 0] * D1 + xyz[:, 1]) * D1 + xyz[:, 2]).numpy()
    keep = np.zeros(D1 ** 3, bool)
    keep[lin] = True
    assert np.array_equal(last["keep"].cpu().numpy().astype(bool), keep)
    assert n == len(lin) <= 8 * lod1["n_pre"]
    assert np.array_equal(last["rows"][:n].cpu().numpy(), np.sort(lin))


def test_lod1_cost_and_volume(lod1, g1):
    last, ref = lod1["last"], lod1["ref"]
    n = int(last["count"].item())
    assert maxerr(last["cost"][:n].flatten()[::11], g1["lod1_cost_s"]) < 5e-4
    assert np.array_equal(np.packbits(lod1["cond"]["valid_mask_volume_scale1"].cpu().numpy().reshape(-1) > 0), g1["lod1_occ"])
    assert maxerr(lod1["cond"]["dense_volume_scale1"].flatten()[::13], g1["lod1_dense_s"]) < 5e-4
    assert maxerr(lod1["fm1"], lod1["fm1_ref"]) < 5e-5
    n = int(last["count"].item())
    xyz = ref["xyz"].long()
    order = np.argsort(((xyz[:, 0] * D1 + xyz[:, 1]) * D1 + xyz[:, 2]).numpy())
    assert last["cost"].shape[1] == 32
    assert maxerr(last["cost"][:n], ref["cost"][order]) < 5e-4
    vol, occ = lod1["cond"]["dense_volume_scale1"], lod1["cond"]["valid_mask_volume_scale1"]
    assert vol.shape == (1, 16, D1, D1, D1) and lod1["cond"]["coords_scale1"].shape == (1, 3, D1, D1, D1)
    assert torch.equal(occ.cpu(), ref["occ"])
    assert maxerr(vol, ref["dense"]) < 5e-4


def test_lod1_sdf_and_grid(om, tr, lod1, st1, g1):
    vol = lod1["cond"]["dense_volume_scale1"]
    out = tr.sdf_network_lod1.sdf(om.pts.to(vol.device), vol, 1)
    ref = O.sdf_query(om.pts, vol.cpu(), st1["sdf_network_lod1"])
    assert maxerr(out["sdf_pts_scale1"], ref[0]) < 5e-5
    assert maxerr(out["sdf_pts_scale1"], g1["lod1_sdf"]) < 1e-4
    R = MINI["R"]
    v, t, u = tr.sdf_renderer_lod1.extract_geometry(tr.sdf_network_lod1, -torch.ones(3), torch.ones(3), R, 0.0, vol.device,
                                                    conditional_volume=vol, lod=1)
    assert maxerr(u, O.sdf_grid(vol.cpu(), st1["sdf_network_lod1"], R)) < 5e-5
    assert maxerr(u, g1["lod1_u_grid"]) < 1e-4
    assert v.dtype == np.float64 and np.all(np.abs(v) <= 1.0 + 1e-9) and t.min() >= 0 and t.max() < len(v)


def test_lod1_marching_cubes_vertex_set(dev, g1):
    """Marching cubes on the reference's lod-1 grid: bit-exact case grid and vertices, same triangle set."""
    from o2345 import ops
    u = torch.from_numpy(g1["lod1_u_grid"]).to(dev)
    verts, tris, cases = ops.marching_cubes(u, 0.0)
    v_ref, t_ref, c_ref = O.marching_cubes(g1["lod1_u_grid"], 0.0)
    assert len(v_ref) > 0
    assert np.array_equal(cases.cpu().numpy(), c_ref) and np.array_equal(verts.cpu().numpy(), v_ref)
    key = lambda a: np.sort(np.sort(a, 1).view([("a", a.dtype), ("b", a.dtype), ("c", a.dtype)]).ravel())
    assert np.array_equal(key(np.ascontiguousarray(tris.cpu().numpy().astype(np.int64))), key(np.ascontiguousarray(t_ref)))


@pytest.mark.parametrize("precision", [0, 1])
def test_lod1_vertex_colors(om, tr, lod1, st1, g1, dev, precision):
    """The lod-1 mesh is coloured with rendering_network_lod1, the lod-1 volume and the LOD-0 feature maps."""
    vol, occ = lod1["cond"]["dense_volume_scale1"], lod1["cond"]["valid_mask_volume_scale1"]
    r = tr.sdf_renderer_lod1
    prev, r.blend_precision = r.blend_precision, precision
    try:
        rgb, _ = r.blend_points(om.verts.to(dev), tr.sdf_network_lod1, tr.rendering_network_lod1, vol, occ,
                                om.fmaps.to(dev), om.imgs.to(dev), om.w2cs.to(dev), om.intr.to(dev), [MINI["W"], MINI["H"]])
    finally:
        r.blend_precision = prev
    col, _ = O.vertex_colors(om.verts, vol.cpu(), occ.cpu(), om.fmaps, om.imgs, om.w2cs, om.intr, st1["sdf_network_lod1"],
                             st1["rendering_network_lod1"], W=MINI["W"], H=MINI["H"])
    assert maxerr(rgb, col) < 1e-3 + BLEND_TOL[precision]
    assert maxerr(rgb, g1["lod1_vert_color"]) < 2e-3 + BLEND_TOL[precision]


def test_export_mesh_mini(om, tr, st1, dev):
    """export_mesh at num_lods = 2 extracts and colours the lod-1 surface."""
    from o2345.pipeline import _sample_from
    imgs = om.imgs.numpy()
    sample = _sample_from(om.cams, np.concatenate([imgs[:1], imgs]), dev, MINI["H"], MINI["W"])[0]
    mesh = tr(sample, mode="export_mesh", resolution=MINI["R"])
    assert len(mesh["vertices"]) > 0 and np.isfinite(mesh["vertices"]).all() and mesh["colors"].shape[1] == 3
    n = int(tr.sdf_network_lod1._last["count"].item())
    vol = torch.zeros(D1 ** 3, 16)
    vol[tr.sdf_network_lod1._last["rows"][:n].long().cpu()] = tr.sdf_network_lod1._last["reg"][:n].cpu()
    vol = vol.reshape(D1, D1, D1, 16).permute(3, 0, 1, 2)[None]
    assert maxerr(mesh["fields"], O.sdf_grid(vol, st1["sdf_network_lod1"], MINI["R"])) < 5e-5
    # vertex set: the CPU marching cubes on the same lod-1 grid, mapped to world units and merged as the mesh tail does
    from o2345.mesh_io import merge_vertices
    R = MINI["R"]
    v_ref, t_ref, _ = O.marching_cubes(mesh["fields"].cpu().numpy(), 0.0)
    v_ref = v_ref / (R - 1.0) * 2.0 - 1.0
    sm, tm = sample["scale_mat"].cpu().numpy(), sample["trans_mat"].cpu().numpy().reshape(-1, 4, 4)[0]
    v_ref = v_ref * sm[0][0, 0] + sm[0][:3, 3][None]
    v_ref = (np.concatenate([v_ref, np.ones_like(v_ref[:, :1])], 1) @ tm.T)[:, :3]
    v_ref, t_ref, _ = merge_vertices(v_ref, t_ref)
    assert mesh["vertices"].shape == v_ref.shape and np.allclose(mesh["vertices"], v_ref, rtol=0, atol=1e-9)
    key = lambda a: np.sort(np.sort(a, 1).view([("a", a.dtype), ("b", a.dtype), ("c", a.dtype)]).ravel())
    assert np.array_equal(key(np.ascontiguousarray(np.asarray(mesh["triangles"], np.int64))),
                          key(np.ascontiguousarray(np.asarray(t_ref, np.int64))))


def test_full_size_bit_identical(dev):
    """32 views of 256^2, 96^3 -> 192^3, R = 256: survivors within the budget, a mesh, and two runs bit-identical."""
    from o2345 import synthetic as S
    from o2345.pipeline import build_networks, synthetic_sample
    tr = build_networks(dev, vol_dim=96, states={**S.all_states(0), **S.lod1_states(0)}, perturb=0.0, num_lods=2)
    sample = synthetic_sample(dev)
    runs = []
    for _ in range(2):
        mesh = tr(sample, mode="export_mesh", resolution=256)
        n_pre = tr.sdf_renderer_lod0._last_prune["counts"][tr.sdf_renderer_lod0._last_prune["rung"]]
        n_rows = int(tr.sdf_network_lod1._last["count"].item())
        runs.append((mesh, min(n_pre, 110000), n_rows))
    (m0, n_pre, n_rows), (m1, _, _) = runs
    assert 0 < n_pre <= 110000 and 0 < n_rows <= 8 * n_pre
    assert len(m0["vertices"]) > 0 and len(m0["triangles"]) > 0 and np.isfinite(m0["vertices"]).all()
    for k in ("vertices", "triangles", "colors"):
        assert np.array_equal(m0[k], m1[k]), k


CONF2 = """
general { base_exp_dir = %s }
model {
  num_lods = 2
  sdf_network_lod0 { lod = 0, ch_in = 56, voxel_size = 0.02105263, vol_dims = [96, 96, 96], hidden_dim = 128,
    cost_type = variance_mean, d_pyramid_feature_compress = 16, regnet_d_out = 16, num_sdf_layers = 4, multires = 6 }
  sdf_network_lod1 { lod = 1, ch_in = 56, voxel_size = 0.0104712, vol_dims = [192, 192, 192], hidden_dim = 128,
    cost_type = variance_mean, d_pyramid_feature_compress = 8, regnet_d_out = 16, num_sdf_layers = 4, multires = 6 }
  variance_network { init_val = 0.2 }
  variance_network_lod1 { init_val = 0.2 }
  rendering_network { in_geometry_feat_ch = 16, in_rendering_feat_ch = 56, anti_alias_pooling = True }
  rendering_network_lod1 { in_geometry_feat_ch = 16, in_rendering_feat_ch = 56, anti_alias_pooling = True }
  trainer { n_samples_lod0 = 64, n_importance_lod0 = 64, n_samples_lod1 = 64, n_importance_lod1 = 64, n_outside = 0,
    perturb = 1.0, alpha_type = div }
}
"""


def test_cli_num_lods_2(tmp_path, monkeypatch):
    from PIL import Image
    from o2345 import synthetic as S
    sys.path.insert(0, os.path.join(ROOT, "one-2-3-45_b200"))
    import exp_runner_generic_blender_val as runner
    exp = tmp_path / "scene"
    (exp / "stage1_8").mkdir(parents=True)
    (exp / "stage2_8").mkdir()
    meta = S.pose_json(60.0)
    ids = list(meta["c2ws"])
    imgs = S.images(33, 256, 256, seed=7)
    u8 = lambda a: Image.fromarray(np.round(a.transpose(1, 2, 0) * 255).astype(np.uint8))
    u8(imgs[0]).save(exp / "stage1_8" / ids[0])
    for v in range(32):
        u8(imgs[1 + v]).save(exp / "stage2_8" / ids[8 + v])
    (exp / "pose.json").write_text(json.dumps(meta))
    conf = tmp_path / "lod1.conf"
    conf.write_text(CONF2 % str(tmp_path / "base"))
    monkeypatch.chdir(tmp_path)
    mesh = runner.main(["--specific_dataset_name", str(exp), "--mode", "export_mesh", "--resolution", "64", "--conf", str(conf)])
    assert (exp / "mesh.ply").read_bytes().startswith(b"ply") and len(mesh["vertices"]) > 0
    out = runner.main(["--specific_dataset_name", str(exp), "--mode", "val", "--conf", str(conf)])
    for name in ("val_color.png", "val_color_lod1.png", "val_depth_lod1.npy", "val_normal_lod1.npy"):
        assert (exp / name).exists(), name
    assert np.load(exp / "val_depth_lod1.npy").shape == (256, 256)
    assert np.isfinite(out["color_lod1"]).all() and np.isfinite(out["normal_lod1"]).all()


def test_new_entry_points_reject_bad_arguments():
    import ctypes as C
    from o2345 import _lib
    lib = _lib.load()
    fake = C.c_void_p(0x1000)
    lad = (C.c_float * 17)(*([0.01] * 17))
    cases = [
        lambda: lib.o2345_sdf_voxels(fake, fake, 1, fake, 0.1, fake, 0, fake, None),                  # D < 2
        lambda: lib.o2345_sdf_voxels(fake, fake, 8, fake, 0.1, fake, 5, fake, None),                  # precision
        lambda: lib.o2345_prune_by_sdf(fake, fake, 8, lad, 17, fake, fake, fake, None),               # > 16 rungs
        lambda: lib.o2345_prune_by_sdf(fake, fake, 8, lad, 0, fake, fake, fake, None),                # no rung
        lambda: lib.o2345_prune_by_sdf(fake, fake, 8, lad, 4, fake, fake, fake, None),                # scratch aliases
        lambda: lib.o2345_lod_children(fake, 0, 48, fake, fake, fake, fake, None),                    # no parent
        lambda: lib.o2345_lod_children(None, 4, 48, fake, fake, fake, fake, None),                    # null
        lambda: lib.o2345_costvol_gather_lod(fake, 12, 4, 8, 8, 8, 8, fake, fake, 0.1, 8, fake, fake, 8, fake,
                                             None, None, fake, None),                                 # C = 12
        lambda: lib.o2345_costvol_gather_lod(fake, 8, 4, 8, 8, 8, 8, fake, fake, 0.1, 8, fake, fake, 8, fake,
                                             fake, None, fake, None),                                 # parent w/o feats
    ]
    for i, call in enumerate(cases):
        assert call() == -1, (i, _lib.last_error())


def test_lod_children_rejects_bad_coordinates(dev):
    from o2345 import _lib, ops
    fkeep = torch.ones(D1 ** 3, dtype=torch.uint8, device=dev)
    good = torch.tensor([[0, 2, 4, 6], [0, 10, 10, 10]], dtype=torch.float32, device=dev)
    keep, parent = ops.lod_children(good, D1, fkeep)
    assert int(keep.sum()) == 16 and int((parent >= 0).sum()) == 16
    for bad in ([[0, 2, 4, 6], [0, 2, 4, 6]],               # duplicate parent
                [[0, D1 - 1, 0, 0]],                        # child outside the lattice
                [[0, -2, 0, 0]],
                [[0, 2.5, 0, 0]]):                          # not an integer
        with pytest.raises(_lib.O2345Error):
            ops.lod_children(torch.tensor(bad, dtype=torch.float32, device=dev), D1, fkeep)
