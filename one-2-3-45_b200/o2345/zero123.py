"""Zero123 multi-view generation on the o2345 kernels: LatentDiffusion (inference subset) + the run.py stage logic.

Mirrors, with the same call signatures:
  * LatentDiffusion.apply_model / encode_first_stage / decode_first_stage / get_learned_conditioning /
    cc_projection / ema_scope / register_schedule     (reference ldm/models/diffusion/ddpm.py:126-193,526,619-630,
    763-860,888-984,1441-1474) -- the `hybrid` conditioning of configs/sd-objaverse-finetune-c_concat-256.yaml;
  * sample_model_batch, predict_stage1_gradio, zero123_infer            (reference utils/zero123_utils.py:60-178);
  * stage1_run / stage2_run view bookkeeping                             (reference run.py:18-54).
The CLIP image tower (row A8) lives in o2345/clip_image.py (`FrozenCLIPImageEmbedder`); `cond_stage_model` is pluggable and
build_zero123(clip=True) attaches it (default: a seeded stand-in embedding, which is what bench.py times in round 1).
Out of scope here (SURVEY.md section 8(f)): the LoFTR elevation search (the polar angle is an input).
Checkpoint keys: `model.diffusion_model.*`, `first_stage_model.*`, `cc_projection.*`, `cond_stage_model.*` load directly.
"""
from __future__ import annotations

import contextlib
import json
import os

import numpy as np
import torch
import torch.nn as nn

from . import ops_a as A
from . import synthetic as S
from .autoencoder import AutoencoderKL
from .ddim import DDIMSampler, make_ddim_timesteps
from .unet import UNetModel


class _DiffusionWrapper(nn.Module):
    def __init__(self, unet):
        super().__init__()
        self.diffusion_model = unet
        self.conditioning_key = "hybrid"


class LatentDiffusion(nn.Module):
    def __init__(self, unet_config=None, first_stage_config=None, scale_factor=0.18215, timesteps=1000,
                 linear_start=0.00085, linear_end=0.0120, cond_stage_model=None):
        super().__init__()
        self.model = _DiffusionWrapper(UNetModel(**(unet_config or {})))
        self.first_stage_model = AutoencoderKL(**(first_stage_config or {}))
        self.cc_projection = nn.Linear(772, 768)
        self.scale_factor, self.num_timesteps, self.parameterization = scale_factor, timesteps, "eps"
        self.cond_stage_model = cond_stage_model
        # register_schedule('linear'), reference ddpm.py:126-178 + util.py:21-25: fp64 math, fp32 buffers
        betas = np.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=np.float64) ** 2
        ac = np.cumprod(1.0 - betas, axis=0)
        f32 = lambda a: torch.tensor(a, dtype=torch.float32)
        self.register_buffer("betas", f32(betas))
        self.register_buffer("alphas_cumprod", f32(ac))
        self.register_buffer("alphas_cumprod_prev", f32(np.append(1.0, ac[:-1])))
        self._cc = None

    @property
    def device(self):
        return self.betas.device

    def half(self):
        """`model.half()` in the reference (zero123_utils.py:45) also rounds the schedule buffers to fp16, and the
        sampler then reads those (SURVEY.md row A9).  Weights are already consumed as fp16 by the kernels."""
        for n in ("betas", "alphas_cumprod", "alphas_cumprod_prev"):
            getattr(self, n).data = getattr(self, n).data.half()
        return self

    @contextlib.contextmanager
    def ema_scope(self, context=None):
        yield None  # EMA weights are what gets loaded; there is nothing to swap at inference

    @torch.no_grad()
    def apply_model(self, x_noisy, t, cond, return_ids=False):
        xc = torch.cat([x_noisy] + cond["c_concat"], dim=1)
        cc = cond["c_crossattn"][0] if len(cond["c_crossattn"]) == 1 else torch.cat(cond["c_crossattn"], 1)
        return self.model.diffusion_model(xc, t, context=cc)

    @torch.no_grad()
    def encode_first_stage(self, x):
        return self.first_stage_model.encode(x)

    @torch.no_grad()
    def decode_first_stage(self, z, predict_cids=False, force_not_quantize=False):
        return self.first_stage_model.decode(1. / self.scale_factor * z)

    @torch.no_grad()
    def get_learned_conditioning(self, c):
        if self.cond_stage_model is None:
            g = torch.Generator().manual_seed(7)            # no conditioning encoder attached: a fixed embedding
            return torch.randn(1, 1, 768, generator=g).expand(c.shape[0], -1, -1).contiguous().to(c.device)
        enc = getattr(self.cond_stage_model, "encode", None)   # reference ddpm.py:619-626
        return enc(c) if callable(enc) else self.cond_stage_model(c)

    @torch.no_grad()
    def project_condition(self, c):
        """cc_projection: Linear(772 -> 768) on [n,1,772] (reference ddpm.py:526)."""
        w = self.cc_projection.weight
        key = (w.data_ptr(), w._version)
        if self._cc is None or self._cc[0] != key:
            wp = torch.zeros(768, 776, dtype=torch.float16, device=w.device)
            wp[:, :772] = w.detach().half()
            self._cc = (key, wp, self.cc_projection.bias.detach().float().contiguous())
        n = c.shape[0]
        cp = torch.zeros(n, 776, dtype=torch.float16, device=c.device)
        cp[:, :772] = c.reshape(n, 772).half()
        return A.gemm(cp, self._cc[1], bias=self._cc[2]).float().view(n, 1, 768)


@torch.no_grad()
def sample_model_batch(model, sampler, input_im, xs, ys, n_samples=4, precision='autocast', ddim_eta=1.0, ddim_steps=75,
                       scale=3.0, h=256, w=256, x_T=None, step_noise=None, decode_chunk=8, to_host=True):
    """reference utils/zero123_utils.py:60-98; returns images in [0,1], float32, on the host (to_host=False: on the device).

    Beyond the reference: `input_im` may hold G conditioning images; then n_samples views are sampled for EACH of them in
    one batch of G * n_samples (xs / ys list the G * n_samples relative poses, image-major), which is G reference calls
    run as one; `x_T` / `step_noise` carry the noise those calls would have drawn (see generate_views)."""
    with model.ema_scope():
        G = input_im.shape[0]
        total = G * n_samples
        assert len(xs) == total and len(ys) == total, "one relative pose per sampled view"
        c = model.get_learned_conditioning(input_im)
        c = c.tile(n_samples, 1, 1) if G == 1 else c.repeat_interleave(n_samples, 0)
        T = [[np.radians(x), np.sin(np.radians(y)), np.cos(np.radians(y)), 0] for x, y in zip(xs, ys)]
        T = torch.tensor(np.array(T))[:, None, :].float().to(c.device)
        c = model.project_condition(torch.cat([c, T], dim=-1))
        z = model.encode_first_stage(input_im).mode().detach()
        cond = {'c_crossattn': [c],
                'c_concat': [z.repeat(n_samples, 1, 1, 1) if G == 1 else z.repeat_interleave(n_samples, 0)]}
        uc = None
        if scale != 1.0:
            uc = {'c_concat': [torch.zeros(total, 4, h // 8, w // 8).to(c.device)], 'c_crossattn': [torch.zeros_like(c)]}
        samples, _ = sampler.sample(S=ddim_steps, conditioning=cond, batch_size=total, shape=[4, h // 8, w // 8],
                                    verbose=False, unconditional_guidance_scale=scale, unconditional_conditioning=uc,
                                    eta=ddim_eta, x_T=x_T, step_noise=step_noise)
        x = torch.cat([model.decode_first_stage(samples[i:i + decode_chunk]) for i in range(0, total, decode_chunk)])
        x = torch.clamp((x + 1.0) / 2.0, min=0.0, max=1.0)
        return x.cpu() if to_host else x


DELTA_X_1_8 = [0] * 4 + [30] * 4 + [-30] * 4
DELTA_Y_1_8 = [0 + 90 * (i % 4) if i < 4 else 30 + 90 * (i % 4) for i in range(8)] + [30 + 90 * (i % 4) for i in range(4)]
DELTA_X_2, DELTA_Y_2 = [-10, 10, 0, 0], [0, 0, -10, 10]


def _to_uint8(img):
    """(x * 255).astype(uint8): the PNG the reference writes between the stages (zero123_utils.py:125-129)."""
    return (255.0 * img.numpy().transpose(1, 2, 0)).astype(np.uint8)


def _to_uint8_device(imgs):
    """The same quantisation for a batch [n, 3, H, W] that stays on the device: fp32 multiply, truncation -> [n, H, W, 3] uint8."""
    return (255.0 * imgs.permute(0, 2, 3, 1)).to(torch.uint8).contiguous()


def _as_input_device(u8, whiten):
    """_as_input for device-resident uint8 views [n, H, W, 3] -> [n, 3, H, W] in [-1, 1]."""
    a = u8.to(torch.float32)
    if whiten:
        a = torch.where(a >= 253.0, torch.full_like(a, 255.0), a)
    return (a / 255.0).permute(0, 3, 1, 2) * 2 - 1


def _as_input(u8, whiten):
    a = u8.astype(np.float32)
    if whiten:                       # stage-2 inputs: >= 253 -> 255 (zero123_utils.py:145-147)
        a[a >= 253.0] = 255.0
    return torch.from_numpy(a / 255.0).permute(2, 0, 1)[None] * 2 - 1


def ddim_iterations(ddim_steps, num_timesteps=1000):
    """UNet iterations of one sampler call: the uniform schedule minus its last entry (76 / 49 for S = 75 / 50)."""
    return len(make_ddim_timesteps(ddim_steps, num_timesteps)) - 1


@torch.no_grad()
def generate_views(model, input_u8, polar_angle=60, ddim_steps=75, stage2_steps=50, scale=3.0, exp_dir=None, device="cuda",
                   batched=True, keep_on_device=False):
    """run.py's stage1_run + stage2_run (reference run.py:18-54) with the elevation given instead of estimated: the
    reference's 10 sampler calls (2 x 76 + 8 x 49 UNet iterations at batch 8 = 4 views x CFG).  Returns (stage1 dict
    id -> uint8 image, stage2 dict 'i_j' -> uint8 image, pose dict).  With exp_dir the same PNG files and pose.json are
    written.

    batched=True (default): with the elevation known the two stage-1 calls are independent of each other, and so are the
    eight stage-2 calls once their stage-1 view exists, so they run as TWO sampler calls -- 76 iterations at batch 16
    (8 views x CFG) and 49 iterations at batch 64 (32 views x CFG): the same 40 views and the same arithmetic per view,
    but every weight is streamed from HBM 125 times instead of 544 and the GEMMs have 2x / 8x the rows.  The noise is
    drawn FIRST, call by call in the reference's order and shapes (x_T, then one tensor per iteration), so every view
    sees exactly the numbers it would have seen in the sequential run.  batched=False runs the ten calls one after the
    other, as the reference does.

    The views pass through uint8 between the stages and on the way to the reconstruction exactly as the reference's PNG files
    make them (x * 255 truncated; stage-2 inputs whitened at >= 253), but the quantisation runs on the device and stage 2 is
    fed from device memory: the host copies (numpy uint8 [H, W, 3], what the dicts hold) are made once at the end -- or not at
    all with keep_on_device=True (dict values are then uint8 device tensors; `pipeline.image_to_mesh` uses that when no files
    are to be written)."""
    dev = torch.device(device)
    inp = _as_input(input_u8, False).to(dev)
    stage1, stage2 = {}, {}
    first = list(range(4))
    second = list(range(4, 8)) if polar_angle <= 75 else list(range(8, 12))
    pose = S.pose_json(float(polar_angle))

    def stage1_call(adjust, x_T=None, step_noise=None):
        sampler = DDIMSampler(model)
        imgs = sample_model_batch(model, sampler, inp, [DELTA_X_1_8[i] for i in adjust], [DELTA_Y_1_8[i] for i in adjust],
                                  n_samples=len(adjust), ddim_steps=ddim_steps, scale=scale, x_T=x_T, step_noise=step_noise,
                                  to_host=False)
        u8 = _to_uint8_device(imgs)
        for k, i in enumerate(adjust):
            stage1[i] = u8[k]

    def stage2_call(anchors, x_T=None, step_noise=None):
        sampler = DDIMSampler(model)
        ims = _as_input_device(torch.stack([stage1[i] for i in anchors]), True)
        imgs = sample_model_batch(model, sampler, ims, DELTA_X_2 * len(anchors), DELTA_Y_2 * len(anchors), n_samples=4,
                                  ddim_steps=stage2_steps, scale=scale, x_T=x_T, step_noise=step_noise, to_host=False)
        u8 = _to_uint8_device(imgs)
        for a, i in enumerate(anchors):
            for j in range(4):
                stage2[f"{i}_{j}"] = u8[4 * a + j]

    if not batched:
        stage1_call(first)
        stage2_call([0])
        stage1_call(second)
        for i in ([1, 2, 3] + second):
            stage2_call([i])
    else:
        draws = _draw_view_noise(second, ddim_iterations(ddim_steps, model.num_timesteps),
                                 ddim_iterations(stage2_steps, model.num_timesteps), dev)
        stage1_call(first + second, *_gather_noise([draws], [[("s1", 0), ("s1", 1)]]))
        anchors = first + second
        stage2_call(anchors, *_gather_noise([draws], [[("s2", i) for i in anchors]]))
    return _finish_views(stage1, stage2, pose, exp_dir, keep_on_device)


def _stage1_ids(polar_angle):
    """The 8 stage-1 view ids of run.py's stage1_run: 0-3, then 4-7 (polar <= 75) or 8-11 (reference run.py:18-35)."""
    return list(range(4)) + (list(range(4, 8)) if polar_angle <= 75 else list(range(8, 12)))


def _draw_view_noise(second, n1, n2, dev):
    """The noise of one image's ten reference sampler calls, drawn from the default generator of `dev` in the reference's order of
    calls (stage 1 views 0-3, stage 2 of view 0, stage 1 of `second`, stage 2 of views 1-3 and `second`); inside a call x_T
    first, then one draw per iteration (ddim.py:137,223).  -> {(kind, key): (x_T, [noise per iteration])}."""
    draws = {}
    for kind, key in [("s1", 0), ("s2", 0), ("s1", 1)] + [("s2", i) for i in [1, 2, 3] + second]:
        x_T = torch.randn(4, 4, 32, 32, device=dev)
        draws[(kind, key)] = (x_T, [torch.randn(4, 4, 32, 32, device=dev) for _ in range(n1 if kind == "s1" else n2)])
    return draws


def image_noise(seed, index, polar_angle, n1, n2, device):
    """The noise contract of generate_views_multi for the image at position `index` of the caller's list: the generator of
    `device` (the CUDA generator of that device; the CPU generator for a CPU device) seeded with seed + index, then the
    draws of generate_views(batched=True) for n1 stage-1 and n2 stage-2 iterations."""
    dev = torch.device(device)
    if dev.type == "cuda":
        with torch.cuda.device(dev):
            torch.cuda.manual_seed(seed + index)
    else:
        torch.manual_seed(seed + index)
    return _draw_view_noise(_stage1_ids(polar_angle)[4:], n1, n2, dev)


def _gather_noise(draws, keys):
    """x_T and the per-iteration noise of one batched sampler call: draws[i][k] for k in keys[i], image-major."""
    parts = [d[k] for d, ks in zip(draws, keys) for k in ks]
    return torch.cat([p[0] for p in parts]), [torch.cat([p[1][i] for p in parts]) for i in range(len(parts[0][1]))]


def _finish_views(stage1, stage2, pose, exp_dir, keep_on_device):
    """Host copies of the device-resident uint8 views (unless keep_on_device) and, with exp_dir, stage1_8/*.png,
    stage2_8/*.png and pose.json as run.py writes them."""
    if not keep_on_device or exp_dir is not None:
        host1, host2 = torch.stack([stage1[i] for i in stage1]).cpu().numpy(), torch.stack([stage2[k] for k in stage2]).cpu().numpy()
        if not keep_on_device:
            stage1 = {i: host1[n] for n, i in enumerate(stage1)}
            stage2 = {k: host2[n] for n, k in enumerate(stage2)}
        files1, files2 = {i: host1[n] for n, i in enumerate(stage1)}, {k: host2[n] for n, k in enumerate(stage2)}
    if exp_dir is not None:
        from PIL import Image
        os.makedirs(os.path.join(exp_dir, "stage1_8"), exist_ok=True)
        os.makedirs(os.path.join(exp_dir, "stage2_8"), exist_ok=True)
        for i, im in files1.items():
            Image.fromarray(im).save(os.path.join(exp_dir, "stage1_8", f"{i}.png"))
        for k, im in files2.items():
            Image.fromarray(im).save(os.path.join(exp_dir, "stage2_8", f"{k}.png"))
        json.dump(pose, open(os.path.join(exp_dir, "pose.json"), "w"), indent=4)
    return stage1, stage2, pose


@torch.no_grad()
def generate_views_multi(model, inputs_u8, polar_angles, ddim_steps=75, stage2_steps=50, scale=3.0, seed=0, indices=None,
                         exp_dirs=None, device="cuda", keep_on_device=False):
    """generate_views for K images in two sampler calls: stage 1 at batch 16 K (8 views x CFG per image) for the stage-1
    iterations, then stage 2 at batch 64 K (32 views x CFG per image).  Every image gets the view ids, pose.json and
    uint8 quantisation generate_views gives it; polar_angles (one per image, or one for all) may differ, so one call can
    mix the two stage-1 id sets.

    Noise: before image i's draws the CUDA generator of `device` is seeded with seed + indices[i] (indices: each image's
    position in the caller's full list, default 0..K-1), then the image's noise is drawn exactly as
    generate_views(batched=True) draws it.  An image's noise, and so its views up to the rounding of the GEMM shapes, does
    not depend on K, on the other images or on which process renders it; with K = 1 the result is bit-identical to
    `torch.cuda.manual_seed(seed + indices[0]); generate_views(...)`.

    Returns a list of K (stage1, stage2, pose) triples as generate_views returns them; exp_dirs (one per image, or None)
    receive the same files."""
    dev = torch.device(device)
    K = len(inputs_u8)
    polars = [float(p) for p in polar_angles] if np.ndim(polar_angles) else [float(polar_angles)] * K
    indices = list(range(K)) if indices is None else [int(i) for i in indices]
    if K == 0 or len(polars) != K or len(indices) != K or (exp_dirs is not None and len(exp_dirs) != K):
        raise ValueError(f"{K} images need as many polar angles ({len(polars)}), indices ({len(indices)}) and exp_dirs")
    ids = [_stage1_ids(p) for p in polars]
    n1, n2 = ddim_iterations(ddim_steps, model.num_timesteps), ddim_iterations(stage2_steps, model.num_timesteps)
    draws = [image_noise(seed, indices[i], polars[i], n1, n2, dev) for i in range(K)]
    inp = torch.cat([_as_input(u8, False) for u8 in inputs_u8]).to(dev)

    x_T, noise = _gather_noise(draws, [[("s1", 0), ("s1", 1)]] * K)
    sampler = DDIMSampler(model)
    imgs = sample_model_batch(model, sampler, inp, [DELTA_X_1_8[j] for v in ids for j in v], [DELTA_Y_1_8[j] for v in ids for j in v],
                              n_samples=8, ddim_steps=ddim_steps, scale=scale, x_T=x_T, step_noise=noise, to_host=False)
    u8 = _to_uint8_device(imgs)
    stage1 = [{j: u8[8 * i + k] for k, j in enumerate(v)} for i, v in enumerate(ids)]

    x_T, noise = _gather_noise(draws, [[("s2", j) for j in v] for v in ids])
    sampler = DDIMSampler(model)
    ims = _as_input_device(torch.stack([stage1[i][j] for i, v in enumerate(ids) for j in v]), True)
    imgs = sample_model_batch(model, sampler, ims, DELTA_X_2 * (8 * K), DELTA_Y_2 * (8 * K), n_samples=4, ddim_steps=stage2_steps,
                              scale=scale, x_T=x_T, step_noise=noise, to_host=False)
    u8 = _to_uint8_device(imgs)
    out = []
    for i, v in enumerate(ids):
        stage2 = {f"{j}_{q}": u8[32 * i + 4 * a + q] for a, j in enumerate(v) for q in range(4)}
        out.append(_finish_views(stage1[i], stage2, S.pose_json(polars[i]), None if exp_dirs is None else exp_dirs[i], keep_on_device))
    return out


def _checkpoint_state(ckpt):
    """The state dict of a Zero123 checkpoint given as a path or as loaded: a Lightning file's `state_dict`, or the file itself."""
    sd = torch.load(ckpt, map_location="cpu") if isinstance(ckpt, (str, os.PathLike)) else ckpt
    return sd.get("state_dict", sd)


def load_clip_image_embedder(ckpt, device="cpu"):
    """FrozenCLIPImageEmbedder (the CLIP ViT-L/14 image tower) from a Zero123 checkpoint: only its
    `cond_stage_model.model.visual.*` tensors are read and no UNet is built.  A missing tower tensor is an error."""
    from .clip_image import FrozenCLIPImageEmbedder
    prefix = "cond_stage_model."
    sd = {k[len(prefix):]: v for k, v in _checkpoint_state(ckpt).items() if k.startswith(prefix + "model.visual.")}
    m = FrozenCLIPImageEmbedder()
    missing = m.load_state_dict(sd, strict=False).missing_keys
    if missing:
        raise KeyError(f"checkpoint lacks {len(missing)} tensors of the CLIP image tower, e.g. {missing[:3]}")
    return m.requires_grad_(False).to(device)


def load_zero123_checkpoint(ckpt, device="cpu", use_ema=True, unet_config=None, first_stage_config=None, clip=True,
                            report=print):
    """LatentDiffusion from a Zero123 checkpoint (`zero123-xl.ckpt`: a Lightning file with a `state_dict`, or the state
    dict itself), ready to sample the way the reference does (utils/zero123_utils.py:31-47, 60-98):
      * the UNet weights are the EMA shadow `model_ema.*` (the reference samples inside `ema_scope()`);
      * the CLIP ViT-L/14 image tower is attached and `cond_stage_model.*` loaded (text-side CLIP keys are ignored);
      * anything the sampling path needs and the file lacks is an ERROR, not a silent default."""
    from .checkpoints import zero123_sampling_state
    sd = _checkpoint_state(ckpt)
    m = LatentDiffusion(unet_config=unet_config, first_stage_config=first_stage_config)
    if clip:
        from .clip_image import FrozenCLIPImageEmbedder
        m.cond_stage_model = FrozenCLIPImageEmbedder()
    names = [n for n, _ in m.model.named_parameters()]
    sd = zero123_sampling_state(sd, names, use_ema=use_ema, report=report)
    res = m.load_state_dict(sd, strict=False)
    needed = ("model.diffusion_model.", "first_stage_model.", "cc_projection.") + (("cond_stage_model.model.visual.",) if clip else ())
    missing = [k for k in res.missing_keys if k.startswith(needed)]
    if missing:
        raise KeyError(f"checkpoint lacks {len(missing)} tensors the sampling path needs, e.g. {missing[:3]}")
    ignored = [k for k in res.unexpected_keys if not k.startswith(("cond_stage_model.model.", "first_stage_model.loss", "model_ema."))
               and k not in _SCHEDULE_KEYS]
    if ignored and report is not None:
        report(f"zero123 checkpoint: {len(ignored)} unused keys, e.g. {ignored[:3]}")
    for p in m.parameters():
        p.requires_grad_(False)
    return m.to(device)


# buffers of the reference's DDPM.register_schedule that the sampler does not read (ddpm.py:150-178)
_SCHEDULE_KEYS = {"sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod", "log_one_minus_alphas_cumprod", "sqrt_recip_alphas_cumprod",
                  "sqrt_recipm1_alphas_cumprod", "posterior_variance", "posterior_log_variance_clipped", "posterior_mean_coef1",
                  "posterior_mean_coef2", "logvar"}


def build_zero123(device, seed=0, clip=False):
    """LatentDiffusion with seeded random weights (no checkpoint exists offline).  clip=True attaches the CLIP ViT-L/14
    image tower (row A8, o2345/clip_image.py) as cond_stage_model instead of the fixed stand-in embedding."""
    m = LatentDiffusion()
    if clip:
        from .clip_image import FrozenCLIPImageEmbedder
        m.cond_stage_model = FrozenCLIPImageEmbedder()
        m.cond_stage_model.load_state_dict({k: torch.from_numpy(v) for k, v in S.clip_state(seed + 20).items()})
    m.model.diffusion_model.load_state_dict({k: torch.from_numpy(v) for k, v in S.unet_state(seed).items()})
    m.first_stage_model.load_state_dict({k: torch.from_numpy(v) for k, v in S.vae_state(seed + 10).items()})
    # cc_projection is seeded too (nn.Linear's own initialisation draws from the unseeded global generator: every process would
    # build a different model): the reference's initialisation (ddpm.py:526-528: identity on the CLIP embedding, zero bias)
    # and nn.Linear's uniform bound for the four pose columns
    g = torch.Generator().manual_seed(seed + 30)
    with torch.no_grad():
        w = m.cc_projection.weight
        w.zero_()
        w[:, :768] = torch.eye(768)
        w[:, 768:] = (torch.rand(768, 4, generator=g) * 2 - 1) / 772 ** 0.5
        m.cc_projection.bias.zero_()
    for p in m.parameters():
        p.requires_grad_(False)
    return m.to(device)
