"""CPU: the lod-1 restatement of oracle/lod1_oracle.py reproduces the golden vectors frozen from the REAL reference
(tests/golden/lod1_mini.npz, written by oracle/pin_lod1_against_reference.py).  The oracle's lod-0 volume differs from
the reference's by ~1.5e-5 (BatchNorm summation order), which bounds the float tolerances below."""
import os

import numpy as np
import pytest
import torch

from helpers import MINI, OracleMini
from oracle import lod1_oracle as L1
from oracle import recon_oracle as O
from oracle.pin_lod1_against_reference import PRUNE_CASES, PRUNE_SEED

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D0, D1 = MINI["D"], 2 * MINI["D"]


@pytest.fixture(scope="module")
def g1():
    return np.load(os.path.join(ROOT, "tests", "golden", "lod1_mini.npz"))


@pytest.fixture(scope="module")
def om():
    return OracleMini()


@pytest.fixture(scope="module")
def st1():
    from o2345 import synthetic as S
    return {k: O.to_torch_state(v) for k, v in S.lod1_states(0).items()}


def close(a, b, tol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    assert np.max(np.abs(a - b)) <= tol, float(np.max(np.abs(a - b)))


def mask_coords(packed, D):
    """Packed lattice mask -> [N,4] (0, x, y, z) float coordinates in lattice order."""
    lin = np.nonzero(np.unpackbits(packed)[:D ** 3])[0]
    xyz = np.stack([lin // (D * D), (lin // D) % D, lin % D], 1)
    return torch.from_numpy(np.concatenate([np.zeros((len(lin), 1)), xyz], 1)).float()


def test_sdf_volume(om, g1):
    s = L1.sdf_volume(om.volume, om.occ, om.origin, om.voxel, om.st["sdf_network_lod0"])
    close(s.reshape(-1), g1["sdf0"], 5e-5)


@pytest.mark.parametrize("case", PRUNE_CASES)
def test_prune_on_the_golden_sdf_volume(om, g1, case):
    sdf0 = torch.from_numpy(g1["sdf0"]).reshape(1, D0, D0, D0)
    max_pts = int(g1["prune_max_pts"][PRUNE_CASES.index(case)])
    np.random.seed(PRUNE_SEED)
    coords, feats, mask, _ = L1.prune(sdf0, om.occ[0], om.volume[0], maximum_pts=max_pts)
    assert np.array_equal(np.packbits(mask.numpy()), g1[f"prune_{case}_mask"])       # bit-exact survivors
    assert torch.equal(coords, mask_coords(g1[f"prune_{case}_mask"], D0))
    close(feats.flatten()[::7], g1[f"prune_{case}_feat_s"], 5e-5)


@pytest.fixture(scope="module")
def lod1(om, g1, st1):
    pre_c = mask_coords(g1["prune_default_mask"], D0)
    xyz = pre_c[:, 1:].long()
    pre_f = om.volume[0].reshape(16, -1).t()[(xyz[:, 0] * D0 + xyz[:, 1]) * D0 + xyz[:, 2]]
    pre_c[:, 1:] *= 2
    fm1 = O.pyramid_feature_maps(om.imgs, st1["pyramid_feature_network_lod1"])
    return L1.conditional_volume(fm1, om.origin, om.proj, st1["sdf_network_lod1"], D1, 2.0 / (D1 - 1), MINI["H"],
                                 MINI["W"], pre_c, pre_f)


def test_lod1_children_cost_volume(lod1, g1):
    xyz = lod1["xyz"].long()
    lin = (xyz[:, 0] * D1 + xyz[:, 1]) * D1 + xyz[:, 2]
    keep = np.zeros(D1 ** 3, bool)
    keep[lin.numpy()] = True
    assert np.array_equal(np.packbits(keep), g1["lod1_keep"])
    close(lod1["cost"][torch.argsort(lin)].flatten()[::11], g1["lod1_cost_s"], 2e-4)
    assert np.array_equal(np.packbits(lod1["occ"].reshape(-1).numpy() > 0), g1["lod1_occ"])
    close(lod1["dense"].flatten()[::13], g1["lod1_dense_s"], 2e-4)


def test_lod1_sdf_grid_and_vertex_colours(om, lod1, g1, st1):
    vol, occ = lod1["dense"], lod1["occ"]
    close(O.sdf_query(om.pts, vol, st1["sdf_network_lod1"])[0], g1["lod1_sdf"], 1e-4)
    close(O.sdf_grid(vol, st1["sdf_network_lod1"], MINI["R"]), g1["lod1_u_grid"], 1e-4)
    col, _ = O.vertex_colors(om.verts, vol, occ, om.fmaps, om.imgs, om.w2cs, om.intr, st1["sdf_network_lod1"],
                             st1["rendering_network_lod1"], W=MINI["W"], H=MINI["H"])
    close(col, g1["lod1_vert_color"], 1e-3)
