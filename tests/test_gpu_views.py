"""GPU: rendering a reconstruction from any camera (GenericTrainer.render_cameras, pipeline.render_turntable, the
`--mode turntable` command line) at the mini configuration of test_gpu_parity.py (24^3 volume, 6 source views of 64^2).

Rays of several cameras share one launch group through render_blend dir_mode 2 (direction from each ray's own origin)
and o2345_ray_midpoints_per_ray; every camera must still get exactly the bits of the one-camera path (val_step / render
at perturb 0).  The sparse cost-volume network reduces batch statistics with atomics, so the bit-for-bit comparisons
share one volume between the two sides.  Tolerances against the reference golden are those of
test_render_end_to_end_against_reference_golden.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch

from helpers import MINI, OracleMini, mini_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLEND_TOL = {0: 2e-4, 1: 5e-4}          # fp32 / tensor-core blend kernels, as in test_gpu_parity.py
H, W = MINI["H"], MINI["W"]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def om():
    return OracleMini()


@pytest.fixture(scope="module", params=[1, 2], ids=["lod0", "lod1"])
def tr(request, dev):
    from o2345 import synthetic as S
    from o2345.pipeline import build_networks
    states = {**S.all_states(0), **(S.lod1_states(0) if request.param == 2 else {})}
    return build_networks(dev, vol_dim=MINI["D"], states=states, perturb=0.0, num_lods=request.param)


@pytest.fixture(scope="module")
def sample(dev):
    from o2345.pipeline import _sample_from
    cams, imgs = mini_scene()
    # _sample_from drops image 0 (the query image): the source views are the mini scene's six images
    return _sample_from(cams, np.concatenate([imgs[:1], imgs]), dev, H, W)[0]


@pytest.fixture(params=[0, 1], ids=["blend_fp32", "blend_tc_fp16"])
def precision(request, tr):
    rs = [r for r in (tr.sdf_renderer_lod0, tr.sdf_renderer_lod1) if r is not None]
    old = [r.blend_precision for r in rs]
    for r in rs:
        r.blend_precision = request.param
    yield request.param
    for r, p in zip(rs, old):
        r.blend_precision = p


@pytest.fixture
def frozen(tr, monkeypatch):
    """Builds the volumes once and hands the same tensors to every later call."""
    memo = {}

    def once(name):
        fn = getattr(tr, name)

        def f(*a):
            if name not in memo:
                memo[name] = fn(*a)
            return memo[name]
        monkeypatch.setattr(tr, name, f)
    once("_conditional_features")
    once("_lod1_volume")
    return tr


def mini_meta():
    from o2345 import synthetic as S
    meta = S.pose_json(60.0)
    k = np.array(meta["intrinsics"])
    k[:2] *= W / 256.0
    meta["intrinsics"] = k.tolist()
    return meta


def four_cameras(om):
    """View 0, stage-1 view 3, and two orbit cameras moved to distances 0.5 (inside the volume: near < 0) and 1.8."""
    from o2345 import synthetic as S
    meta = mini_meta()
    poses = np.array(list(meta["c2ws"].values()))
    orbit = S.orbit_cameras(meta, 8)
    c2w, K, nf = S.normalise_cameras(om.cams, np.concatenate([poses[[0, 3]], orbit[[2, 5]]]), meta["intrinsics"])
    for i, d in ((2, 0.5), (3, 1.8)):
        c2w[i, :3, 3] *= np.float32(d / np.linalg.norm(c2w[i, :3, 3]))
        nf[i] = [0.95 * (d - 1), 1.05 * (d + 1)]
    assert nf[2, 0] < 0 < nf[3, 0] and len(set(nf[:, 0].tolist())) == 4
    return c2w, K, nf


def with_query_camera(sample, c2w, K, nf):
    from o2345 import synthetic as S
    dev = sample["query_c2w"].device
    o, v = S.query_rays(K, c2w, H, W)
    s = dict(sample)
    s["query_c2w"] = torch.from_numpy(c2w)[None].to(dev)
    s["query_near_far"] = torch.from_numpy(nf)[None].to(dev)
    s["rays"] = {"rays_o": torch.from_numpy(o)[None].to(dev), "rays_v": torch.from_numpy(v)[None].to(dev)}
    return s


def test_batched_cameras_equal_one_camera_renders(om, frozen, sample, precision):
    tr = frozen
    c2w, K, nf = four_cameras(om)
    assert np.array_equal(c2w[0], sample["query_c2w"][0].cpu().numpy())
    # 1536-ray launch groups: every group but the first holds rays of two cameras
    out = tr.render_cameras(sample, c2w, K, nf, chunk_size=1536)
    suffix = "_lod1" if tr.num_lods > 1 else ""
    assert out["color"].shape == (4, H, W, 3) and out["depth"].shape == (4, H, W) and out["weights_sum"].shape == (4, H, W)
    for c in range(4):
        ref = tr.val_step(with_query_camera(sample, c2w[c], K[c], nf[c]), perturb_overwrite=0)
        assert np.array_equal(out["color"][c].reshape(-1, 3).cpu().numpy(), ref["color" + suffix]), c
        assert np.array_equal(out["depth"][c].reshape(-1, 1).cpu().numpy(), ref["depth" + suffix]), c
        assert np.array_equal(out["normal"][c].reshape(-1, 3).cpu().numpy(), ref["normal" + suffix]), c
    assert 0.5 < float(out["weights_sum"].max()) <= 1.0 + 1e-5                # fp32 sum of weights that add up to <= 1


def test_view0_equals_val_step(frozen, sample):
    tr = frozen
    state = torch.get_rng_state()
    out = tr.render_cameras(sample, sample["query_c2w"][0], sample["intrinsics"][0][0], sample["query_near_far"][0])
    assert torch.equal(torch.get_rng_state(), state)                       # nothing drawn from the host generator
    ref = tr.val_step(sample, perturb_overwrite=0)
    suffix = "_lod1" if tr.num_lods > 1 else ""
    for k, shape in (("color", (-1, 3)), ("depth", (-1, 1)), ("normal", (-1, 3))):
        assert np.array_equal(out[k][0].reshape(shape).cpu().numpy(), ref[k + suffix]), k


def test_novel_view_against_reference_golden(om, tr, sample, precision):
    if tr.num_lods > 1:
        pytest.skip("the reference golden renders the lod-0 level")
    from o2345 import synthetic as S
    gv = np.load(os.path.join(ROOT, "tests", "golden", "views_mini.npz"))
    meta = mini_meta()
    poses = np.array(list(meta["c2ws"].values()))
    c2w, K, nf = S.normalise_cameras(om.cams, poses[int(gv["novel_view"])], meta["intrinsics"])
    np.testing.assert_allclose(c2w[0], gv["novel_c2w"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(nf[0], gv["novel_near_far"], rtol=0, atol=1e-5)
    out = tr.render_cameras(sample, c2w, K, nf, background_rgb=1.0, alpha_inter_ratio=1.0)
    sel = gv["novel_sel"]
    err = lambda a, b: float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())
    assert err(out["color"][0].reshape(-1, 3)[sel].cpu().numpy(), gv["novel_color"]) < 2e-3 + BLEND_TOL[precision]
    assert err(out["depth"][0].reshape(-1, 1)[sel].cpu().numpy(), gv["novel_depth"]) < 5e-3
    assert err(out["weights_sum"][0].reshape(-1, 1)[sel].cpu().numpy(), gv["novel_weights_sum"]) < 5e-3


@pytest.mark.parametrize("prec", [0, 1], ids=["blend_fp32", "blend_tc_fp16"])
def test_ray_origin_direction_equals_query_center_per_camera(om, dev, prec):
    """Kernel level: dir_mode 2 on rays of two cameras gives each ray the bits of dir_mode 0 with its camera's centre, and
    the per-ray last section gives the bits of the scalar one."""
    from o2345 import ops
    from o2345 import synthetic as S
    from o2345.pipeline import build_networks
    from o2345.sparse_neus_renderer import channel_last_volume
    tr = build_networks(dev, vol_dim=MINI["D"], states=S.all_states(0), perturb=0.0)
    c2w, K, nf = four_cameras(om)
    rays = [tuple(a[::5] for a in S.query_rays(K[c], c2w[c], H, W)) for c in (0, 3)]
    n = 700
    ro = torch.from_numpy(np.concatenate([o[:n] for o, _ in rays])).to(dev)
    rd = torch.from_numpy(np.concatenate([v[:n] for _, v in rays])).to(dev)
    near = torch.from_numpy(np.repeat(nf[[0, 3], 0], n)).to(dev)[:, None]
    far = torch.from_numpy(np.repeat(nf[[0, 3], 1], n)).to(dev)[:, None]
    z = (near + (far - near) * torch.linspace(0.0, 1.0, 128).to(dev)[None, :]).contiguous()
    vol, occ = om.volume.to(dev), om.occ.to(dev)
    sd = ((far - near) / 128).view(-1).contiguous()
    mid, dists, act = ops.ray_midpoints(ro, rd, z, sd, occ)
    views = tr.sdf_renderer_lod0._source_views(om.fmaps.to(dev), om.imgs.to(dev), om.w2cs.to(dev), om.intr.to(dev), [W, H])
    pack, vol_cl = tr.rendering_network_lod0.packed(), channel_last_volume(vol)
    rgb, nval = ops.render_blend(ops.PointSource.rays(ro, rd, mid), act, vol_cl, occ, views, pack, precision=prec, ray_origins=True)
    S_ = z.shape[1]
    for k, c in enumerate((0, 3)):
        r = slice(k * n, (k + 1) * n)
        m1, d1, a1 = ops.ray_midpoints(ro[r], rd[r], z[r].contiguous(), float(sd[k * n]), occ)
        assert torch.equal(m1, mid[r]) and torch.equal(d1, dists[r]) and torch.equal(a1, act[k * n * S_:(k + 1) * n * S_])
        rgb1, nval1 = ops.render_blend(ops.PointSource.rays(ro[r], rd[r], m1), a1, vol_cl, occ, views, pack,
                                       query_center=torch.from_numpy(c2w[c, :3, 3]).to(dev), precision=prec)
        assert torch.equal(rgb1, rgb[k * n * S_:(k + 1) * n * S_]) and torch.equal(nval1, nval[k * n * S_:(k + 1) * n * S_])
    assert int((nval > 0).sum()) > 1000                                   # the rays do see the object
    with pytest.raises(Exception, match="ray points"):
        ops.render_blend(ops.PointSource.explicit(om.pts[:64].to(dev)), None, vol_cl, occ, views, pack, ray_origins=True)


def test_turntable_from_a_sample(tr, sample):
    from o2345.pipeline import render_turntable
    out = render_turntable(tr, sample, n_frames=4, chunk_size=5000)
    assert out["color"].shape == (4, H, W, 3) and out["c2ws"].shape == (4, 4, 4) and out["near_far"].shape == (4, 2)
    # frame 0 is the input view
    np.testing.assert_allclose(out["c2ws"][0], sample["query_c2w"][0].cpu().numpy(), atol=1e-5)
    assert bool(torch.isfinite(out["depth"]).all()) and float(out["weights_sum"].amax(dim=(1, 2)).min()) > 0.5


def test_turntable_command_line(tmp_path, monkeypatch):
    """`exp_runner_generic_blender_val.py --mode turntable` on a folder laid out like run.py's output."""
    from PIL import Image
    from o2345 import synthetic as S
    sys.path.insert(0, os.path.join(ROOT, "one-2-3-45_b200"))
    import exp_runner_generic_blender_val as runner
    monkeypatch.chdir(tmp_path)
    exp = tmp_path / "exp"
    (exp / "stage1_8").mkdir(parents=True), (exp / "stage2_8").mkdir()
    meta = mini_meta()
    json.dump(meta, open(exp / "pose.json", "w"))
    names = list(meta["c2ws"].keys())
    imgs = (S.images(33, H, W, seed=7) * 255).round().astype(np.uint8).transpose(0, 2, 3, 1)
    Image.fromarray(imgs[0]).save(exp / "stage1_8" / names[0])
    for i, name in enumerate(names[8:40]):
        Image.fromarray(imgs[i + 1]).save(exp / "stage2_8" / name)
    out = runner.main(["--specific_dataset_name", str(exp), "--mode", "turntable"])
    pngs = sorted(os.listdir(exp / "turntable"))
    assert pngs == [f"{i:03d}.png" for i in range(36)]
    first = Image.open(exp / "turntable" / "000.png")
    assert first.mode == "RGBA" and first.size == (W, H)
    gif = Image.open(exp / "turntable.gif")
    assert gif.n_frames == 36 and gif.size == (W, H)
    assert np.load(exp / "turntable_depth.npy").shape == (36, H, W)
    assert out["color"].shape == (36, H, W, 3)
