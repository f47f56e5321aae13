"""CPU: host-side logic that needs no GPU -- case tables, seeded inputs, state-dict layout, PLY writer."""
import os

import numpy as np
import torch

from o2345 import mc_tables, synthetic as S


def test_mc_tables_are_consistent():
    mask, tri, ntri = mc_tables.tables()
    assert ntri[0] == 0 and ntri[255] == 0 and ntri.max() <= 5
    for c in range(256):
        used = set(int(e) for e in tri[c] if e >= 0)
        want = {e for e in range(12) if ((c >> mc_tables.EDGE_ENDS[e, 0]) & 1) != ((c >> mc_tables.EDGE_ENDS[e, 1]) & 1)}
        assert used == want and mask[c] == sum(1 << e for e in want)
        # complementary cases cut the same edges with the same number of triangles or a re-pairing of them
        assert mask[c] == mask[255 - c]


def test_marching_cubes_sphere_is_closed_and_outward():
    from oracle import recon_oracle as O
    R = 24
    g = np.linspace(-1, 1, R)
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    u = 0.6 - np.sqrt(x * x + y * y + z * z)          # u > 0 inside (u = -sdf)
    v, t, _ = O.marching_cubes(u.astype(np.float32), 0.0)
    e = np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), 1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    assert np.all(cnt == 2)                              # watertight
    assert len(v) - len(cnt) + len(t) == 2               # Euler characteristic of a sphere
    p = v[t]
    vol = np.einsum("ij,ij->i", p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6.0
    assert vol > 0                                       # normals point outwards


def test_synthetic_is_deterministic_and_shaped():
    a, b = S.all_states(0), S.all_states(0)
    for k in a:
        for kk in a[k]:
            assert np.array_equal(a[k][kk], b[k][kk])
    sd = a["sdf_network_lod0"]
    assert sd["sdf_layer.lin0.weight_v"].shape == (128, 39) and sd["sdf_layer.lin2.weight_v"].shape == (128, 144)
    assert sd["sparse_costreg_net.conv6.net.0.kernel"].shape == (27, 64, 64)
    cams = S.scene_cameras()
    assert cams["affine_mats"].shape == (32, 4, 4) and cams["query_near_far"][0] < 0 < cams["query_near_far"][1]


def test_host_modules_accept_reference_state_dicts():
    from o2345.pipeline import build_networks
    tr = build_networks("cpu", vol_dim=24, states=S.all_states(0))
    keys = set(tr.sdf_network_lod0.state_dict().keys())
    for k in S.sdf_network_state(0):
        assert k in keys
    assert set(S.feature_net_state(1)) <= set(tr.pyramid_feature_network_geometry_lod0.state_dict().keys())
    assert set(S.rendering_network_state(2)) == set(tr.rendering_network_lod0.state_dict().keys())
    w = tr.sdf_network_lod0.sdf_layer.lin1.effective()
    v, g = torch.from_numpy(S.sdf_network_state(0)["sdf_layer.lin1.weight_v"]), torch.from_numpy(S.sdf_network_state(0)["sdf_layer.lin1.weight_g"])
    assert torch.allclose(w, v * (g / v.norm(dim=1, keepdim=True)))


def test_rendering_network_pack_layout():
    from o2345.rendering_network import GeneralRenderingNetwork
    from o2345 import _lib
    net = GeneralRenderingNetwork(16, 56, True)
    net.load_state_dict({k: torch.as_tensor(v) for k, v in S.rendering_network_state(2).items()})
    p = net.packed()
    assert p.numel() == _lib.RNET_PACK_FLOATS
    # base_fc.0 block starts after ray_dir_fc: [193][64] stored input-major
    off = 64 + 16 + 1024 + 64
    assert torch.equal(p[off:off + 193 * 64].view(193, 64), net.base_fc[0].weight.t())
    assert float(p[-4]) == abs(float(net.s))


def test_ply_writer(tmp_path):
    from o2345.trainer_generic import write_ply
    v = np.random.rand(5, 3)
    f = np.array([[0, 1, 2], [2, 3, 4]])
    c = (np.random.rand(5, 3) * 255).astype(np.uint8)
    path = os.path.join(tmp_path, "m.ply")
    write_ply(path, v, f, c)
    raw = open(path, "rb").read()
    head, body = raw.split(b"end_header\n")
    assert b"element vertex 5" in head and b"element face 2" in head
    assert len(body) == 5 * 16 + 2 * 13


def test_modules_refuse_autograd_calls():
    """SURVEY.md 8(b) note 2: the kernels are inference-only; a grad-enabled call on trainable parameters must fail loudly
    (before any kernel launch), and the same call is accepted under no_grad or with frozen parameters up to the point
    where it needs the GPU."""
    import pytest
    import torch
    from o2345.featurenet import FeatureNet
    from o2345.unet import UNetModel
    net = FeatureNet()
    with pytest.raises(RuntimeError, match="inference-only"):
        net(torch.zeros(1, 3, 16, 16))
    unet = UNetModel.__new__(UNetModel)          # no 859 M-parameter allocation: the guard only looks at parameters()
    torch.nn.Module.__init__(unet)
    unet.w = torch.nn.Parameter(torch.zeros(1))
    with pytest.raises(RuntimeError, match="inference-only"):
        unet.forward(torch.zeros(1, 8, 8, 8), torch.zeros(1), torch.zeros(1, 1, 768))
    net.requires_grad_(False)
    from o2345 import _lib
    with pytest.raises(_lib.O2345Error):          # past the guard: now it is the missing GPU that stops the CPU call
        net(torch.zeros(1, 3, 16, 16))


def test_geglu_pack_matches_the_epilogue_contract():
    """ops_a.geglu_pack reorders the GEGLU projection so that every 32-column chunk holds 16 values followed by their 16
    gates (what the ACT_GEGLU GEMM epilogue consumes); emulated here in torch."""
    import torch
    from o2345 import ops_a
    g = torch.Generator().manual_seed(0)
    I, K, M = 64, 40, 9
    w, b = torch.randn(2 * I, K, generator=g), torch.randn(2 * I, generator=g)
    x = torch.randn(M, K, generator=g)
    wp, bp = ops_a.geglu_pack(w, b)
    y = (x @ wp.t() + bp).view(M, -1, 2, 16)                     # [M, chunk, {value, gate}, 16]
    got = (y[:, :, 0] * torch.nn.functional.gelu(y[:, :, 1])).reshape(M, I)
    full = x @ w.t() + b
    want = full[:, :I] * torch.nn.functional.gelu(full[:, I:])
    assert torch.allclose(got, want, atol=1e-5)


def test_command_lines_parse_the_reference_arguments():
    import os
    import sys
    import pytest
    pkg = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "one-2-3-45_b200")
    sys.path.insert(0, pkg)
    import exp_runner_generic_blender_val as runner
    import run as run_cli
    import torch
    if torch.cuda.is_available():
        pytest.skip("argument handling without a GPU is what this checks")
    with pytest.raises(SystemExit, match="CUDA"):                 # parses the reference's flags, then refuses to run on the CPU
        run_cli.main(["--img_path", "x.png", "--gpu_idx", "0", "--half_precision", "--mesh_resolution", "128", "--output_format", ".ply"])
    with pytest.raises(SystemExit, match="CUDA"):
        runner.main(["--specific_dataset_name", "/tmp/x", "--mode", "export_mesh", "--conf", "confs/one2345_lod0_val_demo.conf",
                     "--resolution", "256"])
    with pytest.raises(SystemExit, match="only 'export_mesh' and 'val'"):
        runner.main(["--mode", "train"])


def test_ddim_iteration_counts():
    """76 / 49 UNet iterations for S = 75 / 50 (reference ddim.py:126-131 drops the schedule's last entry)."""
    from o2345.zero123 import ddim_iterations
    assert ddim_iterations(75) == 76 and ddim_iterations(50) == 49 and ddim_iterations(5) == 4


def test_ddim_direction_coefficient_stays_positive():
    """The DDIM update takes sqrt(1 - a_prev - sigma^2) of fp32 schedule values (o2345_cfg_ddim_update).  For the Zero123
    schedules (5, 50 and 75 steps, eta 0 and 1, the fp32 alphas_cumprod and its fp16 rounding of a `.half()` model) that
    difference stays positive at every iteration, in fp32 arithmetic and with room for its rounding.  Its smallest value,
    at the last step with eta = 1, is 6.5e-6 for 5 steps and above 1e-4 for 50 and 75 steps: far above a few fp32 ulps of 1."""
    from types import SimpleNamespace

    from o2345.ddim import DDIMSampler
    from oracle import ldm_oracle as LO
    ac = torch.from_numpy(LO.linear_beta_alphas_cumprod())
    for a in (ac, ac.half()):
        for S in (5, 50, 75):
            for eta in (0.0, 1.0):
                smp = DDIMSampler(SimpleNamespace(num_timesteps=1000, device=torch.device("cpu"), alphas_cumprod=a))
                smp.make_schedule(S, ddim_eta=eta, verbose=False)
                steps = len(smp.ddim_timesteps) - 1
                ap, sig = smp.ddim_alphas_prev[:steps].numpy(), smp.ddim_sigmas[:steps].numpy()
                term32 = np.float32(1.0) - ap - sig * sig
                exact = 1.0 - ap.astype(np.float64) - sig.astype(np.float64) ** 2
                assert term32.dtype == np.float32 and (term32 > 0).all(), (a.dtype, S, eta, term32.min())
                assert exact.min() > 64 * 2.0 ** -24, (a.dtype, S, eta, exact.min())


def test_upsample_conv_weight_decomposition_is_exact_algebra():
    """nearest 2x + 3x3 conv (pad 1) == four 2x2 convolutions of the low-resolution map with the collapsed kernel rows / columns
    summed (o2345.unet._Packed.conv_up, consumed by o2345_conv_up2x_f16): checked in fp64 on the CPU with torch's own conv2d,
    borders included.  Phase (a, b) writes output pixels (2y + a, 2x + b); its tap (ty, tx) reads input (y + ty + a - 1,
    x + tx + b - 1)."""
    import torch
    import torch.nn.functional as F
    from o2345.unet import _Packed
    g = torch.Generator().manual_seed(3)
    C, N, H, W = 8, 5, 6, 7
    conv = torch.nn.Conv2d(C, N, 3, padding=1)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(N, C, 3, 3, generator=g))
        conv.bias.copy_(torch.randn(N, generator=g))
    x = torch.randn(2, C, H, W, generator=g, dtype=torch.float64)
    want = F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), conv.weight.double(), conv.bias.double(), padding=1)
    pk = _Packed(conv)
    w4, b4 = pk.conv_up(conv)
    assert w4.shape == (4, N, 4 * C) and w4.dtype == torch.float16 and torch.equal(b4, conv.bias.detach().float())
    # the packed fp16 sums against the same sums in fp64: only the final rounding separates them
    w = conv.weight.detach().double()
    rows = {0: (w[:, :, 0], w[:, :, 1] + w[:, :, 2]), 1: (w[:, :, 0] + w[:, :, 1], w[:, :, 2])}
    got = torch.empty_like(want)
    xp = F.pad(x, (1, 1, 1, 1))
    for a in (0, 1):
        for b in (0, 1):
            k = torch.empty(N, C, 2, 2, dtype=torch.float64)
            for ty in (0, 1):
                r = rows[a][ty]
                cols = (r[:, :, 0], r[:, :, 1] + r[:, :, 2]) if b == 0 else (r[:, :, 0] + r[:, :, 1], r[:, :, 2])
                k[:, :, ty, 0], k[:, :, ty, 1] = cols
            packed = w4[2 * a + b].double().reshape(N, 2, 2, C).permute(0, 3, 1, 2)          # (ty, tx, c) order -> [N, C, 2, 2]
            assert float((packed - k).abs().max()) <= 2.0 ** -10 * float(k.abs().max())      # fp16 rounding of the sums
            full = F.conv2d(xp, k, conv.bias.double())                                        # [.., H + 1, W + 1] over the padded map
            got[:, :, a::2, b::2] = full[:, :, a:a + H, b:b + W]
    assert float((got - want).abs().max()) < 1e-10
