"""Scene samples (row B0) and network assembly for the reconstruction path.

`load_sample` mirrors BlenderPerView.__getitem__ (reference data/One2345_eval_new_data.py:139-377)
for a folder written by run.py (pose.json, stage1_8/0.png, stage2_8/*.png); `synthetic_sample`
builds the same dict from seeded inputs.  `build_networks` mirrors Runner.__init__ (reference
exp_runner_generic_blender_val.py:93-151) for the demo configuration, with one level (num_lods = 1) or two.
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from . import synthetic as S
from .featurenet import FeatureNet
from .rendering_network import GeneralRenderingNetwork, SingleVarianceNetwork
from .sparse_sdf_network import SparseSdfNetwork
from .trainer_generic import GenericTrainer


from .checkpoints import Conf  # noqa: E402,F401


def build_networks(device, vol_dim=96, states=None, n_samples=64, n_importance=64, perturb=1.0, base_exp_dir=None,
                   variance_init=0.3, conf=None, num_lods=None):
    """FeatureNet, SparseSdfNetwork, SingleVarianceNetwork, GeneralRenderingNetwork, GenericTrainer on `device`, assembled
    like Runner.__init__ (reference exp_runner_generic_blender_val.py:93-132).  With `conf` (a parsed
    confs/one2345_lod0_val_demo.conf) the constructor arguments come from it, exactly as the reference passes
    `**conf['model.sdf_network_lod0']` etc. -- including its 8-digit voxel_size 0.02105263; without it the same
    constants are built in (voxel_size = 2 / (D - 1) in full precision).

    num_lods = 2 (from the conf's model.num_lods, or the keyword without a conf) adds the lod-1 FeatureNet, SDF network,
    variance network (built from model.variance_network, as the reference does) and rendering network; without a conf
    the lod-1 volume has 2 D cells per side, voxel_size 2 / (2 D - 1) and 8 compressed channels (the demo conf's
    sdf_network_lod1).  `states` must then also hold the lod-1 networks (o2345.synthetic.lod1_states)."""
    if conf is not None:
        if num_lods is not None and num_lods != conf.get_int('model.num_lods'):
            raise ValueError(f"num_lods={num_lods} contradicts the conf's model.num_lods={conf.get_int('model.num_lods')}")
        num_lods = conf.get_int('model.num_lods')
    num_lods = 1 if num_lods is None else num_lods
    if num_lods not in (1, 2):
        raise NotImplementedError(f"num_lods={num_lods}: 1 or 2 levels are on the accelerated path")
    fnet = FeatureNet()
    lod1 = {}
    if conf is not None:
        sdf = SparseSdfNetwork(**conf['model.sdf_network_lod0'])
        var = SingleVarianceNetwork(**conf['model.variance_network'])
        rnet = GeneralRenderingNetwork(**conf['model.rendering_network'])
        tk = dict(conf['model.trainer'])
        if num_lods > 1:
            lod1 = {"sdf_network_lod1": SparseSdfNetwork(**conf['model.sdf_network_lod1']),
                    "variance_network_lod1": SingleVarianceNetwork(**conf['model.variance_network']),
                    "rendering_network_lod1": GeneralRenderingNetwork(**conf['model.rendering_network_lod1'])}
    else:
        sdf = SparseSdfNetwork(lod=0, ch_in=56, voxel_size=2.0 / (vol_dim - 1), vol_dims=[vol_dim] * 3, hidden_dim=128,
                               cost_type='variance_mean', d_pyramid_feature_compress=16, regnet_d_out=16,
                               num_sdf_layers=4, multires=6)
        var = SingleVarianceNetwork(variance_init)
        rnet = GeneralRenderingNetwork(in_geometry_feat_ch=16, in_rendering_feat_ch=56, anti_alias_pooling=True)
        tk = dict(n_samples_lod0=n_samples, n_importance_lod0=n_importance, n_samples_lod1=64, n_importance_lod1=64,
                  n_outside=0, perturb=perturb, alpha_type='div')
        if num_lods > 1:
            D1 = 2 * vol_dim
            lod1 = {"sdf_network_lod1": SparseSdfNetwork(lod=1, ch_in=56, voxel_size=2.0 / (D1 - 1), vol_dims=[D1] * 3,
                                                         hidden_dim=128, cost_type='variance_mean', d_pyramid_feature_compress=8,
                                                         regnet_d_out=16, num_sdf_layers=4, multires=6),
                    "variance_network_lod1": SingleVarianceNetwork(variance_init),
                    "rendering_network_lod1": GeneralRenderingNetwork(in_geometry_feat_ch=16, in_rendering_feat_ch=56,
                                                                      anti_alias_pooling=True)}
    if num_lods > 1:
        lod1["pyramid_feature_network_lod1"] = FeatureNet()
        d0, d1 = sdf.vol_dims.tolist(), lod1["sdf_network_lod1"].vol_dims.tolist()
        if d1 != [2 * d for d in d0]:
            raise ValueError(f"the lod-1 vol_dims {d1} must be twice the lod-0 vol_dims {d0}")
    if states is not None:
        load = lambda m, sd: m.load_state_dict({k: torch.as_tensor(np.asarray(v)) for k, v in sd.items()}, strict=False)
        for m, key in ((fnet, "pyramid_feature_network"), (sdf, "sdf_network_lod0"), (rnet, "rendering_network_lod0"),
                       (var, "variance_network_lod0"), *((m1, k1) for k1, m1 in lod1.items())):
            if key not in states:
                raise KeyError(f"no weights for {key!r} (num_lods = {num_lods})")
            res = load(m, states[key])
            assert not res.unexpected_keys, res.unexpected_keys
            assert all("num_batches_tracked" in k for k in res.missing_keys), res.missing_keys
    for m in (fnet, sdf, var, rnet, *lod1.values()):
        m.to(device)
        for p in m.parameters():
            p.requires_grad_(False)
    if conf is None:
        conf = Conf({"general": Conf({"base_exp_dir": base_exp_dir}), "model": Conf({"num_lods": num_lods})})
    trainer = GenericTrainer(None, fnet, lod1.get("pyramid_feature_network_lod1"), sdf, lod1.get("sdf_network_lod1"), var,
                             lod1.get("variance_network_lod1"), rnet, lod1.get("rendering_network_lod1"),
                             tk["n_samples_lod0"], tk["n_importance_lod0"],
                             tk["n_samples_lod1"], tk["n_importance_lod1"], tk["n_outside"], tk["perturb"],
                             alpha_type=tk["alpha_type"], conf=conf, base_exp_dir=base_exp_dir)
    return trainer


def _sample_from(cams, imgs, device, H, W, pin=False):
    """Adds the batch dimension the reference's DataLoader adds and moves everything to `device`."""
    t = lambda x: x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x))     # device-resident views pass through
    rays_o, rays_v = S.query_rays(cams["query_intrinsic"], cams["query_c2w"], H, W)
    host = {
        "images": t(imgs[1:])[None], "query_image": t(imgs[0])[None], "w2cs": t(cams["w2cs"])[None],
        "c2ws": t(cams["c2ws"])[None], "intrinsics": t(cams["intrinsics"])[None],
        "affine_mats": t(cams["affine_mats"])[None], "query_c2w": t(cams["query_c2w"])[None],
        "query_w2c": t(cams["query_w2c"])[None], "query_near_far": t(cams["query_near_far"])[None],
        "scale_mat": t(cams["scale_mat"])[None], "trans_mat": t(cams["trans_mat"])[None],
        "partial_vol_origin": t(cams["partial_vol_origin"])[None], "img_wh": torch.tensor([[W, H]]),
    }
    rays = {"rays_o": t(rays_o)[None], "rays_v": t(rays_v)[None]}
    if pin:
        host = {k: (v if v.is_cuda else v.pin_memory()) for k, v in host.items()}
        rays = {k: v.pin_memory() for k, v in rays.items()}
    sample = {k: v.to(device, non_blocking=pin) for k, v in host.items()}
    sample["rays"] = {k: v.to(device, non_blocking=pin) for k, v in rays.items()}
    sample["batch_idx"], sample["meta"] = torch.tensor([0]), ["synthetic"]
    return sample, host, rays


def synthetic_sample(device, n_views=32, H=256, W=256, seed=1234, elev=60.0):
    """One scene with seeded images: 1 query view + n_views source views."""
    meta = S.pose_json(elev)
    k = np.array(meta["intrinsics"])
    k[:2] *= W / 256.0
    meta["intrinsics"] = k.tolist()
    cams = S.scene_cameras(meta, n_src=n_views, img_wh=(W, H))
    imgs = S.images(n_views + 1, H, W, seed=seed)
    return _sample_from(cams, imgs, device, H, W)[0]


def load_sample(folder, device):
    """Reads <folder>/pose.json, stage1_8/<first id>, stage2_8/<ids 8..39> like the reference dataset."""
    from PIL import Image
    meta = json.load(open(os.path.join(folder, "pose.json")))
    ids = list(meta["c2ws"].keys())

    def read(path):
        a = np.asarray(Image.open(path), np.float32) / 255.0
        a = a.transpose(2, 0, 1)
        if a.shape[0] == 4:
            a = a[:3] * a[-1:] + (1 - a[-1:])
        return a

    imgs = [read(os.path.join(folder, "stage1_8", ids[0]))]
    imgs += [read(os.path.join(folder, "stage2_8", ids[v])) for v in range(8, 40)]
    imgs = np.stack(imgs).astype(np.float32)
    H, W = imgs.shape[2:]
    cams = S.scene_cameras(meta, n_src=32, img_wh=(W, H))
    return _sample_from(cams, imgs, device, H, W)[0]


# --------------------------------------------------------------------------------------
# turntable: the reconstruction rendered from a circle of cameras around the object
# --------------------------------------------------------------------------------------
@torch.no_grad()
def render_turntable(trainer, sample_or_dir, n_frames=36, out_dir=None, chunk_size=65536):
    """Volume-renders n_frames views on the circle of the input view (synthetic.orbit_cameras: its elevation and radius,
    azimuths 0, 360 / n, ...) through trainer.render_cameras, with alpha_inter_ratio 1.0 as `--mode val` renders.

    sample_or_dir: an experiment folder (pose.json, stage1_8/, stage2_8/: read like load_sample) or a sample dict (its
    trans_mat / scale_mat give the frame).  With out_dir, writes out_dir/turntable/NNN.png (RGBA: colour over opacity,
    opacity = weights_sum), out_dir/turntable.gif (on white) and out_dir/turntable_depth.npy [n,H,W].
    Returns render_cameras' dict (device tensors) plus the cameras: c2ws [n,4,4], intrinsics [n,3,3], near_far [n,2]."""
    dev = next(trainer.parameters()).device
    if isinstance(sample_or_dir, (str, os.PathLike)):
        meta = json.load(open(os.path.join(sample_or_dir, "pose.json")))
        sample = load_sample(sample_or_dir, dev)
        W, H = (int(v) for v in sample['img_wh'][0])
        scene = S.scene_cameras(meta, n_src=32, img_wh=(W, H))
        K = scene["query_intrinsic"]
    else:
        sample = sample_or_dir
        trans_mat = sample['trans_mat'][0].cpu().numpy().astype(np.float64)
        scene = {"trans_mat": trans_mat, "scale_mat": sample['scale_mat'][0].cpu().numpy()}
        meta = {"c2ws": {"0": trans_mat @ np.diag([1.0, -1.0, -1.0, 1.0])}}     # view 0 back in pose.json's convention
        K = sample['intrinsics'][0][0].cpu().numpy()
    c2ws, intr, near_far = S.normalise_cameras(scene, S.orbit_cameras(meta, n_frames), K)
    out = trainer.render_cameras(sample, c2ws, intr, near_far, chunk_size=chunk_size, alpha_inter_ratio=1.0)
    out.update(c2ws=c2ws, intrinsics=intr, near_far=near_far)
    if out_dir is not None:
        write_turntable(out, out_dir)
    return out


def write_turntable(frames, out_dir):
    """out_dir/turntable/NNN.png, turntable.gif and turntable_depth.npy from render_cameras' dict."""
    from PIL import Image
    alpha = frames["weights_sum"].clamp(0, 1)[..., None]
    # the composited colour is premultiplied by the opacity (no background): PNG wants it straight
    rgba = torch.cat([(frames["color"] / alpha.clamp_min(1e-6)).clamp(0, 1) * (alpha > 0), alpha], -1)
    on_white = (frames["color"] + (1 - alpha)).clamp(0, 1)
    to_u8 = lambda x: (x * 255).round().to(torch.uint8).cpu().numpy()
    rgba, on_white = to_u8(rgba), to_u8(on_white)
    os.makedirs(os.path.join(out_dir, "turntable"), exist_ok=True)
    for i, f in enumerate(rgba):
        Image.fromarray(f, "RGBA").save(os.path.join(out_dir, "turntable", f"{i:03d}.png"))
    gif = [Image.fromarray(f, "RGB") for f in on_white]
    gif[0].save(os.path.join(out_dir, "turntable.gif"), save_all=True, append_images=gif[1:], duration=80, loop=0)
    np.save(os.path.join(out_dir, "turntable_depth.npy"), frames["depth"].cpu().numpy())


# --------------------------------------------------------------------------------------
# run.py end to end (reference run.py:79-119): image -> 8 + 32 generated views -> mesh
# --------------------------------------------------------------------------------------
def sample_from_views(stage1, stage2, pose, device, pin=False):
    """The batch dict of BlenderPerView built from in-memory views instead of PNG files (SURVEY.md 8(f) item 1)."""
    ids = list(pose["c2ws"].keys())
    first = int(ids[0].split(".")[0])
    views = [stage1[first]] + [stage2[ids[v].split(".")[0]] for v in range(8, 40)]
    if torch.is_tensor(views[0]):      # uint8 [H, W, 3] on the device (generate_views(keep_on_device=True)): the same u8 / 255 there
        imgs = (torch.stack(views).to(torch.float32) / 255.0).permute(0, 3, 1, 2).contiguous()
    else:
        imgs = np.stack([(u8.astype(np.float32) / 255.0).transpose(2, 0, 1) for u8 in views]).astype(np.float32)
    H, W = imgs.shape[2:]
    cams = S.scene_cameras(pose, n_src=32, img_wh=(W, H))
    return _sample_from(cams, imgs, device, H, W, pin=pin)[0]


def _simplify_kw(target_faces, texture_size=None, normal_map=False, atlas="faces", project_view=None, min_component=None,
                 ambient_occlusion=False, remesh=False):
    # the keywords only when they are set: a trainer without mesh simplification or texture baking is called as before
    if atlas != "faces" and texture_size is None:
        raise ValueError("atlas needs texture_size")
    if remesh and target_faces is None:
        raise ValueError("remesh needs target_faces")
    kw = {} if target_faces is None else {"target_faces": target_faces}
    kw = kw if texture_size is None else dict(kw, texture_size=texture_size)
    kw = kw if atlas == "faces" else dict(kw, atlas=atlas)
    kw = kw if project_view is None else dict(kw, project_view=project_view)
    kw = kw if min_component is None else dict(kw, min_component=min_component)
    kw = dict(kw, ambient_occlusion=True) if ambient_occlusion else kw
    kw = dict(kw, remesh=True) if remesh else kw
    return dict(kw, normal_map=True) if normal_map else kw


@torch.no_grad()
def image_to_mesh(zero123, trainer, input_u8, polar_angle=60, resolution=256, ddim_steps=75, stage2_steps=50, scale=3.0,
                  exp_dir=None, batched=True, target_faces=None, texture_size=None, normal_map=False, atlas="faces",
                  project_view=None, min_component=None, ambient_occlusion=False, remesh=False):
    """`python run.py --img_path X --half_precision` without SAM / elevation estimation: Zero123 stage 1 + stage 2
    (the reference's 10 DDIM sampler calls, run as two batched ones unless batched=False), camera set-up, cost volume, SDF grid, marching cubes, vertex colours.
    Returns dict(vertices, triangles, colors) as host numpy arrays (and writes mesh.ply when exp_dir is given); with
    target_faces the mesh is simplified to that many faces first (GenericTrainer.export_mesh_step); with texture_size N its
    colours are also baked into an N x N texture (the dict gains uv and texture, o2345/mesh_texture.py), and with
    normal_map its SDF gradient into a tangent-space normal map (normal_texture).  atlas: "faces" (one chart per face) or
    "charts" (multi-face charts, mesh_texture.bake); it needs texture_size.  project_view: dict(photo uint8 [H,W,3] on
    white, alpha uint8 [H,W] or None), the input photo at any resolution (run.py load_photo), projected onto the final
    mesh from the input camera (GenericTrainer.export_mesh_step); the dict gains project_weight.  min_component: 0 < F
    <= 1, the components smaller than F times the largest one's area, or enclosed by it, are dropped after the vertex
    merge and before everything else (o2345/mesh_clean.py); the dict gains clean (the counts).  ambient_occlusion (needs
    texture_size): the full mesh's vertex AO baked into an occlusion map in the same uv (occlusion_texture).  remesh (needs
    target_faces): an isotropic remesh to about target_faces faces replaces the simplification (o2345/mesh_remesh.py);
    everything after it, colours included, is taken on the remeshed mesh."""
    from .zero123 import generate_views
    dev = next(trainer.parameters()).device
    stage1, stage2, pose = generate_views(zero123, input_u8, polar_angle, ddim_steps, stage2_steps, scale, exp_dir, dev, batched=batched,
                                          keep_on_device=exp_dir is None)
    sample = sample_from_views(stage1, stage2, pose, dev)
    trainer.base_exp_dir = exp_dir
    return trainer(sample, mode="export_mesh", resolution=resolution,
                   **_simplify_kw(target_faces, texture_size, normal_map, atlas, project_view, min_component,
                                  ambient_occlusion, remesh))


# --------------------------------------------------------------------------------------
# many images -> many meshes: Zero123 calls of several images packed into one sampler batch
# --------------------------------------------------------------------------------------
# Images per pack: the sampler runs stage 1 at batch 16 K and stage 2 at batch 64 K.  Chosen from tools/throughput.py
# (DESIGN.md section 5): the largest K measured (1, 2, 4, 8) whose UNet time per image still falls by more than the
# run-to-run spread; K = 8 peaks at 14.7 GB allocated.
MAX_PACK = 8


def pack_slices(n, max_pack):
    """Consecutive packs of at most max_pack of n images, in input order: [(start, stop), ...]."""
    if max_pack < 1:
        raise ValueError(f"max_pack must be >= 1, got {max_pack}")
    return [(s, min(s + max_pack, n)) for s in range(0, n, max_pack)]


@torch.no_grad()
def images_to_meshes(zero123, trainer, inputs_u8, polar_angles, seed=0, resolution=256, exp_dirs=None, *, max_pack=None,
                     indices=None, ddim_steps=75, stage2_steps=50, scale=3.0, target_faces=None, texture_size=None,
                     normal_map=False, atlas="faces", project_views=None, min_component=None, ambient_occlusion=False,
                     remesh=False):
    """image_to_mesh for a list of images: a generator of (index, mesh) in input order.  The images go through Zero123 in
    packs of at most MAX_PACK (zero123.generate_views_multi: two sampler calls per pack), then each is reconstructed on its
    own (sample_from_views + trainer(..., mode="export_mesh")).

    polar_angles: one per image or one for all.  Image i's noise comes from seed + indices[i] (indices: the images'
    positions in the caller's full list, default 0..n-1; a process that renders a share of a list passes the share's
    positions), so a mesh does not depend on the pack size, the number of processes or which one renders it; `index` is
    indices[i].  exp_dirs (one per image): stage1_8/, stage2_8/, pose.json and mesh.ply are written there.  max_pack
    overrides MAX_PACK.  target_faces, texture_size, normal_map, atlas, min_component, ambient_occlusion, remesh: as in
    image_to_mesh.
    project_views: one image_to_mesh project_view per image."""
    from .zero123 import generate_views_multi
    n = len(inputs_u8)
    polars = list(polar_angles) if np.ndim(polar_angles) else [polar_angles] * n
    indices = list(range(n)) if indices is None else list(indices)
    if len(polars) != n or len(indices) != n or (exp_dirs is not None and len(exp_dirs) != n):
        raise ValueError(f"{n} images need as many polar angles ({len(polars)}), indices ({len(indices)}) and exp_dirs")
    if project_views is not None and len(project_views) != n:
        raise ValueError(f"{n} images need as many project_views ({len(project_views)})")
    dev = next(trainer.parameters()).device
    for a, b in pack_slices(n, MAX_PACK if max_pack is None else max_pack):
        dirs = None if exp_dirs is None else exp_dirs[a:b]
        views = generate_views_multi(zero123, inputs_u8[a:b], polars[a:b], ddim_steps, stage2_steps, scale, seed=seed,
                                     indices=indices[a:b], exp_dirs=dirs, device=dev, keep_on_device=dirs is None)
        for i, (stage1, stage2, pose) in enumerate(views):
            sample = sample_from_views(stage1, stage2, pose, dev)
            trainer.base_exp_dir = None if dirs is None else dirs[i]
            yield indices[a + i], trainer(sample, mode="export_mesh", resolution=resolution,
                                          **_simplify_kw(target_faces, texture_size, normal_map, atlas,
                                                         None if project_views is None else project_views[a + i],
                                                         min_component, ambient_occlusion, remesh))
        del views
