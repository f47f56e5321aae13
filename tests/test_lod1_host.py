"""CPU: host side of the lod-1 refinement path (num_lods = 2): network assembly, synthetic weights, checkpoint keys, and
the CPU restatement of the pruning rule the kernels implement as a window minimum."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from o2345 import synthetic as S


def test_lod1_states_match_the_modules_and_leave_lod0_draws_alone():
    from o2345.sparse_sdf_network import SparseSdfNetwork
    st = S.lod1_states(0)
    net = SparseSdfNetwork(lod=1, ch_in=56, voxel_size=2 / 191, vol_dims=[192] * 3, d_pyramid_feature_compress=8,
                           regnet_d_out=16)
    assert net.sparse_costreg_net.d_in == 2 * 8 + 16
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items() if "num_batches_tracked" not in k}
    assert shapes == {k: v.shape for k, v in st["sdf_network_lod1"].items()}
    a, b = S.all_states(0), S.all_states(0)
    assert set(a) == {"sdf_network_lod0", "pyramid_feature_network", "rendering_network_lod0", "variance_network_lod0"}
    assert all(np.array_equal(a[n][k], b[n][k]) for n in a for k in a[n])


def test_build_networks_num_lods_2_on_cpu():
    from o2345.pipeline import build_networks
    tr = build_networks("cpu", vol_dim=24, states={**S.all_states(0), **S.lod1_states(0)}, num_lods=2)
    assert tr.num_lods == 2 and tr.sdf_renderer_lod1 is not None
    assert tr.sdf_network_lod1.vol_dims.tolist() == [48] * 3 and tr.sdf_network_lod1.voxel_size == 2.0 / 47
    assert tr.sdf_network_lod1.d_pyramid_feature_compress == 8
    with pytest.raises(KeyError):
        build_networks("cpu", vol_dim=24, states=S.all_states(0), num_lods=2)
    assert build_networks("cpu", vol_dim=24, states=S.all_states(0)).sdf_renderer_lod1 is None


def test_build_networks_checks_the_lod1_conf():
    from o2345.checkpoints import parse_conf
    from o2345.pipeline import build_networks
    conf = """
model { num_lods = 2
  sdf_network_lod0 { lod = 0, ch_in = 56, voxel_size = 0.1, vol_dims = [24, 24, 24], regnet_d_out = 16 }
  sdf_network_lod1 { lod = 1, ch_in = 56, voxel_size = 0.05, vol_dims = [%d, %d, %d], d_pyramid_feature_compress = 8,
                     regnet_d_out = 16 }
  variance_network { init_val = 0.2 }
  rendering_network { in_geometry_feat_ch = 16, in_rendering_feat_ch = 56 }
  rendering_network_lod1 { in_geometry_feat_ch = 16, in_rendering_feat_ch = 56 }
  trainer { n_samples_lod0 = 8, n_importance_lod0 = 8, n_samples_lod1 = 8, n_importance_lod1 = 8, n_outside = 0,
            perturb = 0.0, alpha_type = div }
}
general { base_exp_dir = x }
"""
    states = {**S.all_states(0), **S.lod1_states(0)}
    tr = build_networks("cpu", states=states, conf=parse_conf(conf % (48, 48, 48)))
    assert tr.num_lods == 2 and tr.sdf_network_lod1.voxel_size == 0.05
    with pytest.raises(ValueError):
        build_networks("cpu", states=states, conf=parse_conf(conf % (40, 40, 40)))
    with pytest.raises(ValueError):
        build_networks("cpu", states=states, conf=parse_conf(conf % (48, 48, 48)), num_lods=1)
    bad = parse_conf(conf % (48, 48, 48))
    bad["model"]["prune_depth_filter"] = True
    with pytest.raises(NotImplementedError):
        build_networks("cpu", states=states, conf=bad)


def test_recon_states_lod1_keys():
    from o2345.checkpoints import recon_states
    ck = {k: {"w": torch.zeros(1)} for k in ("pyramid_feature_network", "sdf_network_lod0", "rendering_network_lod0",
                                               "variance_network_lod0")}
    said = []
    assert set(recon_states(ck, report=said.append)) == set(ck) and said == []
    with pytest.raises(KeyError):
        recon_states(ck, num_lods=2)
    ck1 = {**ck, **{k: {"w": torch.ones(1)} for k in ("pyramid_feature_network_lod1", "sdf_network_lod1",
                                                       "rendering_network_lod1", "variance_network_lod1")}}
    assert set(recon_states(ck1, num_lods=2)) == set(ck1)


def test_window_minimum_is_the_dilated_threshold_mask():
    """avg_pool3d(|sdf| < t, 7, 1, 3) > 0 equals (min of |sdf| over the clipped 7^3 window) < t for every t: the rule
    o2345_prune_by_sdf evaluates once for the whole threshold ladder."""
    g = torch.Generator().manual_seed(0)
    D = 13
    sdf = torch.randn(1, 1, D, D, D, generator=g) * 0.05
    m = (-F.max_pool3d(-sdf.abs(), kernel_size=7, stride=1, padding=3))       # window minimum, border clipped
    for t in [0.02 - 0.002 * k for k in range(10)]:
        pooled = F.avg_pool3d((sdf.abs() < t).float(), kernel_size=7, stride=1, padding=3) > 0
        assert torch.equal(pooled, m < t)
