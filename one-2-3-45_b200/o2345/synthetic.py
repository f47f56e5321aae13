"""Seeded synthetic weights, cameras and images for the reconstruction hot path.

No checkpoints or real images exist offline (SURVEY.md section 8(d)), so every test, the
smoke run and bench.py draw their inputs from here.  Everything is generated with
``numpy.random.default_rng`` so the same arrays can be rebuilt on the GPU box, inside
the oracle tests and inside ``tests/golden/make_golden.py`` (which feeds them to the
real reference modules) without shipping weight files.

State-dict keys and shapes mirror the reference modules so a real checkpoint loads the
same way (reference: reconstruction/exp_runner_generic_blender_val.py:435-512):

* ``sdf_network_lod0``      -> reconstruction/models/sparse_sdf_network.py:145-196
* ``pyramid_feature_network`` -> reconstruction/models/featurenet.py:40-72
* ``rendering_network_lod0`` -> reconstruction/models/rendering_network.py:26-72
* ``variance_network_lod0``  -> reconstruction/models/fields.py:179-185
"""
from __future__ import annotations

import math

import numpy as np

# channel plan of the sparse cost-regularisation U-Net (reference tsparse/modules.py:259-285)
def costreg_channels(d_in: int, d_out: int):
    """(name, cin, cout) for the ten sparse convolutions, in execution order."""
    return [("conv0", d_in, d_out), ("conv1", d_out, 16), ("conv2", 16, 16), ("conv3", 16, 32),
            ("conv4", 32, 32), ("conv5", 32, 64), ("conv6", 64, 64), ("conv7", 64, 32),
            ("conv9", 32, 16), ("conv11", 16, d_out)]


def _uniform(rng, shape, bound):
    return rng.uniform(-bound, bound, size=shape).astype(np.float32)


def _normal(rng, shape, mean, std):
    return (mean + std * rng.standard_normal(size=shape)).astype(np.float32)


def _bn(rng, c, prefix, sd, spread=0.15):
    # gamma deliberately takes both signs far from zero in a few channels so the
    # |gamma| rule of InPlaceABN (SURVEY.md appendix C) is exercised.
    gamma = _normal(rng, (c,), 1.0, spread)
    gamma[:: max(1, c // 4)] *= -1.0
    sd[prefix + ".weight"] = gamma
    sd[prefix + ".bias"] = _normal(rng, (c,), 0.0, spread)
    sd[prefix + ".running_mean"] = np.zeros((c,), np.float32)
    sd[prefix + ".running_var"] = np.ones((c,), np.float32)


def sdf_network_state(seed=0, ch_in=56, d_compress=16, regnet_d_out=16, hidden=128,
                      multires=6, d_latent=16, perturb=0.05, parent_ch=0):
    """Weights of SparseSdfNetwork (compress conv + sparse U-Net + weight-normed SDF MLP).  parent_ch = 16 for a lod > 0
    network, whose U-Net input also carries the parent voxel's features."""
    rng = np.random.default_rng(seed)
    sd = {}
    fan = ch_in * 9
    sd["compress_layer.conv.weight"] = _uniform(rng, (d_compress, ch_in, 3, 3), 1.0 / math.sqrt(fan))
    _bn(rng, d_compress, "compress_layer.bn", sd)
    for name, cin, cout in costreg_channels(2 * d_compress + parent_ch, regnet_d_out):
        bound = 1.0 / math.sqrt((cout if name in ("conv7", "conv9", "conv11") else cin) * 27)
        sd[f"sparse_costreg_net.{name}.net.0.kernel"] = _uniform(rng, (27, cin, cout), bound)
        _bn(rng, cout, f"sparse_costreg_net.{name}.net.1", sd, spread=0.1)
        # sparse BatchNorm keeps gamma positive in every released checkpoint we know of;
        # nn.BatchNorm1d has no abs() so the sign is free either way.
    d_pe = 3 * (2 * multires + 1)
    dims_in = [d_pe, hidden + d_latent, hidden + d_latent]
    dims_out = [hidden, hidden, hidden]
    for l, (din, dout) in enumerate(zip(dims_in, dims_out)):
        w = np.zeros((dout, din), np.float32)
        b = np.zeros((dout,), np.float32)
        if l == 2:  # geometric init of the output layer (sparse_sdf_network.py:75-81)
            w = _normal(rng, (dout, din), math.sqrt(math.pi) / math.sqrt(din), 1e-4)
            b[:] = -0.5
            w[:, -d_latent:] = 0.0
            b[-d_latent:] = 0.0
        elif l == 0:  # (sparse_sdf_network.py:83-88)
            w[:, :3] = _normal(rng, (dout, 3), 0.0, math.sqrt(2) / math.sqrt(dout))
        else:  # (sparse_sdf_network.py:94-98)
            w = _normal(rng, (dout, din), 0.0, math.sqrt(2) / math.sqrt(dout))
            w[:, -d_latent:] = 0.0
        if perturb > 0:  # make every input column matter, as in a trained checkpoint
            if l == 0:
                # column 3+6k+j belongs to frequency 2^k: damp by 1/2^k so |grad sdf| stays O(1)
                damp = np.repeat(0.5 ** np.arange(multires), 6).astype(np.float32)
                w[:, 3:] += _normal(rng, (dout, din - 3), 0.0, perturb * 0.3) * damp[None]
            else:
                # latent features are O(5) after BN+ReLU+skip adds: keep their pull on the SDF gentle
                w[:, -d_latent:] += _normal(rng, (dout, d_latent), 0.0, perturb * 0.1)
            b += _normal(rng, (dout,), 0.0, perturb * 0.2)
        g = np.linalg.norm(w.astype(np.float64), axis=1, keepdims=True).astype(np.float32)
        if perturb > 0:
            g = (g * (1.0 + _normal(rng, g.shape, 0.0, perturb))).astype(np.float32)
        sd[f"sdf_layer.lin{l}.bias"] = b
        sd[f"sdf_layer.lin{l}.weight_g"] = g
        sd[f"sdf_layer.lin{l}.weight_v"] = w
    return sd


def feature_net_state(seed=1):
    """Weights of FeatureNet (reference featurenet.py:45-68)."""
    rng = np.random.default_rng(seed)
    sd = {}
    plan = [("conv0.0", 3, 8, 3), ("conv0.1", 8, 8, 3),
            ("conv1.0", 8, 16, 5), ("conv1.1", 16, 16, 3), ("conv1.2", 16, 16, 3),
            ("conv2.0", 16, 32, 5), ("conv2.1", 32, 32, 3), ("conv2.2", 32, 32, 3)]
    for name, cin, cout, k in plan:
        sd[name + ".conv.weight"] = _uniform(rng, (cout, cin, k, k), 1.0 / math.sqrt(cin * k * k))
        _bn(rng, cout, name + ".bn", sd)
    for name, cin, cout, k in [("toplayer", 32, 32, 1), ("lat1", 16, 32, 1), ("lat0", 8, 32, 1),
                               ("smooth1", 32, 16, 3), ("smooth0", 32, 8, 3)]:
        bound = 1.0 / math.sqrt(cin * k * k)
        sd[name + ".weight"] = _uniform(rng, (cout, cin, k, k), bound)
        sd[name + ".bias"] = _uniform(rng, (cout,), bound)
    return sd


def rendering_network_state(seed=2, geo_ch=16, feat_ch=56):
    """Weights of GeneralRenderingNetwork (reference rendering_network.py:31-72)."""
    rng = np.random.default_rng(seed)
    sd = {"s": np.array(0.2, np.float32)}
    c = feat_ch + 3

    def lin(name, din, dout, kaiming):
        if kaiming:
            sd[name + ".weight"] = _normal(rng, (dout, din), 0.0, math.sqrt(2.0 / din))
            sd[name + ".bias"] = _normal(rng, (dout,), 0.0, 0.02)
        else:
            b = 1.0 / math.sqrt(din)
            sd[name + ".weight"] = _uniform(rng, (dout, din), b)
            sd[name + ".bias"] = _uniform(rng, (dout,), b)

    lin("ray_dir_fc.0", 4, 16, False)
    lin("ray_dir_fc.2", 16, c, False)
    lin("base_fc.0", 3 * c + geo_ch, 64, True)
    lin("base_fc.2", 64, 32, True)
    lin("vis_fc.0", 32, 32, True)
    lin("vis_fc.2", 32, 33, True)
    lin("vis_fc2.0", 32, 32, True)
    lin("vis_fc2.2", 32, 1, True)
    lin("rgb_fc.0", 32 + 1 + 4, 16, True)
    lin("rgb_fc.2", 16, 8, True)
    lin("rgb_fc.4", 8, 1, True)
    return sd


def variance_network_state(init_val=0.3):
    return {"variance": np.array(init_val, np.float32)}


def all_states(seed=0):
    return {
        "sdf_network_lod0": sdf_network_state(seed),
        "pyramid_feature_network": feature_net_state(seed + 1),
        "rendering_network_lod0": rendering_network_state(seed + 2),
        "variance_network_lod0": variance_network_state(),
    }


def lod1_states(seed=0):
    """Weights of the four lod-1 networks of the demo conf (sdf_network_lod1: 8 compressed channels).  Separate from
    all_states so that every lod-0 draw stays as it is."""
    return {
        "sdf_network_lod1": sdf_network_state(seed + 10, d_compress=8, parent_ch=16),
        "pyramid_feature_network_lod1": feature_net_state(seed + 11),
        "rendering_network_lod1": rendering_network_state(seed + 12),
        "variance_network_lod1": variance_network_state(),
    }


# --------------------------------------------------------------------------------------
# cameras: pose.json content (reference utils/utils.py:80-145) and the per-scene camera
# normalisation of BlenderPerView (reference data/One2345_eval_new_data.py:139-377).
# --------------------------------------------------------------------------------------

def _look_at_poses(elev, azim, radius=1.2):
    """c2w [n,3,4] float32 (reference utils/utils.py:80-104, Blender convention)."""
    th = np.asarray(azim, np.float32)
    ph = np.asarray(elev, np.float32)
    r = np.float32(radius)
    centers = np.stack([r * np.sin(th) * np.sin(ph), -r * np.cos(th) * np.sin(ph), r * np.cos(ph)], -1)

    def nrm(v):
        return (v / (np.linalg.norm(v, axis=-1, keepdims=True) + np.float32(1e-10))).astype(np.float32)

    fwd = nrm(centers)
    up = np.tile(np.array([[0, 0, 1]], np.float32), (len(th), 1))
    right = nrm(np.cross(up, fwd))
    up = nrm(np.cross(fwd, right))
    poses = np.zeros((len(th), 3, 4), np.float32)
    poses[:, :, 0], poses[:, :, 1], poses[:, :, 2], poses[:, :, 3] = right, up, fwd, centers
    return poses


def pose_json(init_elev=60.0):
    """The dict ``gen_poses`` serialises to pose.json: 40 c2w matrices, K, near/far."""
    mid, deg = init_elev, 10
    if init_elev <= 75:
        other = init_elev + 30
        first = list(range(8))
    else:
        other = init_elev - 30
        first = list(range(4)) + list(range(8, 12))
    elev = np.radians([mid] * 4 + [other] * 4 + [mid - deg, mid + deg, mid, mid] * 4
                      + [other - deg, other + deg, other, other] * 4)
    ids = [f"{n}.png" for n in first] + [f"{n}_{v}.png" for n in first for v in range(4)]
    over = [30 + x * 90 for x in range(4)]
    eye = [60 + x * 90 for x in range(4)]
    delta = [0, 0, -deg, deg]
    azim = np.radians(over + eye + [t + d for t in over for d in delta] + [t + d for t in eye for d in delta])
    poses = _look_at_poses(elev, azim)
    c2ws = {}
    for i, name in enumerate(ids):
        p = poses[i].astype(np.float64)
        c2ws[name] = np.concatenate([p, [[0, 0, 0, 1]]], 0).tolist()
    focal, hw = 560 / 2, 256
    return {"intrinsics": [[focal, 0, hw / 2], [0, focal, hw / 2], [0, 0, 1]],
            "near_far": [1.2 - 0.7, 1.2 + 0.6], "c2ws": c2ws}


def scene_cameras(meta=None, n_src=32, img_wh=(256, 256), factor=1.1):
    """Cameras of one scene as ``BlenderPerView.__getitem__`` hands them to the trainer.

    Closed-form restatement: the reference re-expresses every camera relative to view 0,
    fits a cube around the union of the view frusta and decomposes ``K [R|t] S`` with
    cv2; for a uniform scale ``S`` that decomposition is ``c2w' = [R^T | (C - c)/r]``.
    Returns float32 arrays shaped like the sample dict entries (query view removed).
    """
    meta = pose_json() if meta is None else meta
    W, H = img_wh
    poses = np.array(list(meta["c2ws"].values()), np.float64)
    K4 = np.eye(4)
    K4[:3, :3] = np.array(meta["intrinsics"], np.float64)
    nf = np.array(meta["near_far"], np.float64)
    flip = np.diag([1.0, -1.0, -1.0, 1.0])
    c2w_all = poses @ flip
    w2c_all = np.linalg.inv(c2w_all)
    ref_inv = np.linalg.inv(w2c_all[0])               # trans_mat (= c2w of view 0)
    ids = [0] + list(range(8, 8 + n_src))
    ext = np.stack([w2c_all[i] @ ref_inv for i in ids])  # world := camera-0 frame

    # union of frusta -> centre / radius (reference data/scene.py:16-101), float32 like torch
    K = K4[:3, :3].astype(np.float32)
    lo = np.full(3, np.inf, np.float32)
    hi = np.full(3, -np.inf, np.float32)
    dmin, dmax = np.float32(nf[0]), np.float32(nf[1])
    for e in ext:
        c2w = np.linalg.inv(e.astype(np.float32)).astype(np.float32)
        d = np.array([dmin] * 4 + [dmax] * 4, np.float32)
        xs = (np.array([0, 0, W, W, 0, 0, W, W], np.float32) - K[0, 2]) * d / K[0, 0]
        ys = (np.array([0, H, 0, H, 0, H, 0, H], np.float32) - K[1, 2]) * d / K[1, 1]
        pts = np.stack([xs, ys, d, np.ones(8, np.float32)], 0)
        pw = (c2w @ pts)[:3]
        lo, hi = np.minimum(lo, pw.min(1)), np.maximum(hi, pw.max(1))
    center = ((hi + lo) / 2).astype(np.float32)
    radius = np.float32((hi - lo).max() / 2) * np.float32(factor)
    scale_mat = np.diag([radius, radius, radius, 1.0]).astype(np.float32)
    scale_mat[:3, 3] = center

    w2cs, c2ws, affine, near_fars = zip(*[_normalised_camera(e, K4[:3, :3], scale_mat) for e in ext])
    f32 = lambda x: np.asarray(x, np.float32)
    w2cs, c2ws, affine, near_fars = f32(w2cs), f32(c2ws), f32(affine), f32(near_fars)
    intr = np.tile(K[None], (len(ids), 1, 1))
    return {
        "w2cs": w2cs[1:], "c2ws": c2ws[1:], "affine_mats": affine[1:], "intrinsics": intr[1:],
        "near_fars": near_fars, "query_c2w": c2ws[0], "query_w2c": w2cs[0],
        "query_intrinsic": intr[0], "query_near_far": near_fars[0],
        "scale_mat": scale_mat, "trans_mat": f32(ref_inv), "scale_factor": np.float32(1.0 / radius),
        "partial_vol_origin": np.array([-1.0, -1.0, -1.0], np.float32), "img_wh": np.array([W, H]),
        "ref_inv": ref_inv,   # float64 trans_mat: normalise_cameras reproduces the scene's own cameras bit for bit with it
    }


def _normalised_camera(ext, K, scale_mat):
    """One camera of BlenderPerView.__getitem__'s loop (reference :256-274): ext is its view-0-relative w2c (float64),
    K [3,3] its intrinsics.  -> (w2c float64, c2w float32, affine K w2c float64, [near, far])."""
    R = ext[:3, :3]
    cam_center = -R.T @ ext[:3, 3]
    c2w = np.eye(4, dtype=np.float32)
    c2w[:3, :3] = R.T
    c2w[:3, 3] = (cam_center - scale_mat[:3, 3].astype(np.float64)) / float(scale_mat[0, 0])
    w2c = np.linalg.inv(c2w)
    a = np.eye(4)
    a[:3, :4] = np.asarray(K, np.float64) @ w2c[:3, :4]
    dist = math.sqrt(float(np.sum(c2w[:3, 3].astype(np.float64) ** 2)))
    return w2c, c2w, a, [0.95 * (dist - 1), 1.05 * (dist + 1)]


_BLENDER2OPENCV = np.diag([1.0, -1.0, -1.0, 1.0])


def normalise_cameras(scene, c2ws_blender, intrinsics):
    """Cameras given in pose.json's frame (Blender c2w [n,4,4] or [4,4]) -> the normalised frame the scene's volume
    lives in, with the dataset's arithmetic: blender2opencv, then relative to view 0 (w2c @ w2c_ref_inv), then
    K w2c scale_mat decomposed, near / far from the camera distance (reference BlenderPerView.__getitem__ :172-274).

    scene: scene_cameras' dict (its float64 "ref_inv" reproduces the scene's own cameras bit for bit; a sample's float32
    "trans_mat" is used when there is none).  intrinsics [3,3] or [n,3,3].
    Returns float32 (c2w [n,4,4] OpenCV, intrinsics [n,3,3], near_far [n,2])."""
    poses = np.asarray(c2ws_blender, np.float64).reshape(-1, 4, 4)
    n = len(poses)
    K = np.broadcast_to(np.asarray(intrinsics, np.float64).reshape(-1, 3, 3), (n, 3, 3))
    ref_inv = np.asarray(scene.get("ref_inv", scene["trans_mat"]), np.float64).reshape(4, 4)
    scale_mat = np.asarray(scene["scale_mat"], np.float32).reshape(4, 4)
    c2ws, near_fars = [], []
    for pose, k in zip(poses, K):
        _, c2w, _, nf = _normalised_camera(np.linalg.inv(pose @ _BLENDER2OPENCV) @ ref_inv, k, scale_mat)
        c2ws.append(c2w), near_fars.append(nf)
    return np.asarray(c2ws, np.float32), K.astype(np.float32), np.asarray(near_fars, np.float32)


def orbit_cameras(meta, n_frames):
    """n_frames Blender c2w [n,4,4] on the circle of the input view (view 0 of pose.json): its elevation and radius, at
    azimuths 0, 360 / n, ... degrees from it, looking at the origin (reference utils/utils.py:80-145, _look_at_poses)."""
    c = np.asarray(next(iter(meta["c2ws"].values())), np.float64)[:3, 3]
    radius = float(np.linalg.norm(c))
    polar = math.acos(max(-1.0, min(1.0, c[2] / radius)))
    azim0 = math.atan2(c[0], -c[1])
    azim = azim0 + 2 * math.pi * np.arange(n_frames) / n_frames
    poses = _look_at_poses(np.full(n_frames, polar), azim, radius)
    out = np.tile(np.eye(4, dtype=np.float32), (n_frames, 1, 1))
    out[:, :3, :] = poses
    return out


def query_rays(intrinsic, c2w, H=256, W=256):
    """rays_o / rays_v [H*W,3] (reference models/rays.py:11-54): pixel centres at integer
    coordinates, unit-norm directions, row-major pixel order."""
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
    p = np.stack([xs, ys, np.ones_like(ys)], -1).reshape(-1, 3)
    kinv = np.linalg.inv(intrinsic.astype(np.float32)).astype(np.float32)
    p = (p @ kinv.T).astype(np.float32)
    v = p / np.linalg.norm(p, axis=-1, keepdims=True)
    v = (v @ c2w[:3, :3].T).astype(np.float32)
    o = np.broadcast_to(c2w[:3, 3][None], v.shape).astype(np.float32).copy()
    return o, v


def images(n_views=32, H=256, W=256, seed=1234):
    """uint8-quantised RGB views in [0,1], float32 [V,3,H,W]: smooth colour blobs on white."""
    rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.linspace(-1, 1, H, dtype=np.float32), np.linspace(-1, 1, W, dtype=np.float32),
                         indexing="ij")
    out = np.ones((n_views, 3, H, W), np.float32)
    for v in range(n_views):
        cx, cy = rng.uniform(-0.15, 0.15, 2)
        rad = rng.uniform(0.45, 0.6)
        inside = (xs - cx) ** 2 + (ys - cy) ** 2 < rad * rad
        ph = rng.uniform(0, 2 * np.pi, 3)
        fr = rng.uniform(2.0, 6.0, 3)
        for c in range(3):
            tex = 0.5 + 0.4 * np.sin(fr[c] * xs + ph[c]) * np.cos(fr[(c + 1) % 3] * ys - ph[c])
            out[v, c][inside] = tex[inside]
    return (np.round(out * 255.0) / 255.0).astype(np.float32)


# --------------------------------------------------------------------------------------
# path A: seeded Zero123 UNet weights (860 M parameters, generated on the fly -- never stored)
# --------------------------------------------------------------------------------------

def unet_state(seed=0, gain=0.7):
    """State dict of the Zero123 UNet (reference keys / shapes, openaimodel.py:414-735): weights
    N(0, gain / sqrt(fan_in)), small biases, norm scales around 1.  The reference zero-initialises several
    output convolutions (`zero_module`); they get the same random treatment here so that every layer matters."""
    import torch
    from .unet import UNetModel
    with torch.device("meta"):
        shapes = {k: tuple(v.shape) for k, v in UNetModel().state_dict().items()}
    rng = np.random.default_rng(seed)
    sd = {}
    for k, shp in shapes.items():
        if len(shp) >= 2:
            fan_in = int(np.prod(shp[1:]))
            sd[k] = (rng.standard_normal(shp, dtype=np.float32) * np.float32(gain / math.sqrt(fan_in)))
        elif ".norm" in k or "in_layers.0" in k or "out_layers.0" in k or k.startswith("out.0"):
            sd[k] = (1.0 + 0.1 * rng.standard_normal(shp, dtype=np.float32)) if k.endswith("weight") else \
                (0.05 * rng.standard_normal(shp, dtype=np.float32))
        else:
            sd[k] = 0.02 * rng.standard_normal(shp, dtype=np.float32)
    return sd


def vae_state(seed=10, gain=0.7):
    """State dict of the AutoencoderKL (reference keys, 83.7 M parameters), same recipe as unet_state."""
    import torch
    from .autoencoder import AutoencoderKL
    with torch.device("meta"):
        shapes = {k: tuple(v.shape) for k, v in AutoencoderKL().state_dict().items()}
    rng = np.random.default_rng(seed)
    sd = {}
    for k, shp in shapes.items():
        if len(shp) >= 2:
            sd[k] = rng.standard_normal(shp, dtype=np.float32) * np.float32(gain / math.sqrt(int(np.prod(shp[1:]))))
        elif "norm" in k:
            sd[k] = (1.0 + 0.1 * rng.standard_normal(shp, dtype=np.float32)) if k.endswith("weight") else \
                (0.05 * rng.standard_normal(shp, dtype=np.float32))
        else:
            sd[k] = 0.02 * rng.standard_normal(shp, dtype=np.float32)
    return sd


def clip_state(seed=20, gain=0.7):
    """State dict of FrozenCLIPImageEmbedder (OpenAI CLIP ViT-L/14 vision tower, 304 M parameters, keys
    `model.visual.*`), same recipe as unet_state; embeddings N(0, 0.02) like CLIP's own initialisation scale."""
    import torch
    from .clip_image import FrozenCLIPImageEmbedder
    with torch.device("meta"):
        shapes = {k: tuple(v.shape) for k, v in FrozenCLIPImageEmbedder().state_dict().items()}
    rng = np.random.default_rng(seed)
    sd = {}
    for k, shp in shapes.items():
        if k.endswith(("class_embedding", "positional_embedding")):
            sd[k] = 0.02 * rng.standard_normal(shp, dtype=np.float32)
        elif k.endswith("visual.proj"):
            sd[k] = rng.standard_normal(shp, dtype=np.float32) * np.float32(gain / math.sqrt(shp[0]))
        elif len(shp) >= 2:
            sd[k] = rng.standard_normal(shp, dtype=np.float32) * np.float32(gain / math.sqrt(int(np.prod(shp[1:]))))
        elif ".ln_" in k:
            sd[k] = (1.0 + 0.1 * rng.standard_normal(shp, dtype=np.float32)) if k.endswith("weight") else \
                (0.05 * rng.standard_normal(shp, dtype=np.float32))
        else:
            sd[k] = 0.02 * rng.standard_normal(shp, dtype=np.float32)
    return sd
