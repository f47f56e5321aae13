"""GPU: Zero123 UNet on the wgmma path and the DDIM sampler, against the reference goldens.

Tolerance: the reference itself runs this model in fp16 under autocast (fp32 GroupNorm / LayerNorm / softmax); the
golden vector is the reference's fp32 CPU output.  fp16 storage of ~60 layers gives ~1e-2 relative deviations, so
the bar is 3x the measured deviation: max |err| < 6.5e-3 and mean |err| < 1.2e-3 on an output of std 0.38 (measured: 2.1e-3 / 3.9e-4;
a missing bias in one layer moves the output by > 1e-2, a wrong layer by O(1))."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "ldm_mini.npz"))


@pytest.fixture(scope="module")
def unet():
    from o2345 import synthetic as S
    from o2345.unet import UNetModel
    net = UNetModel()
    net.load_state_dict({k: torch.from_numpy(v) for k, v in S.unet_state(0).items()})
    return net.cuda().requires_grad_(False)      # the o2345 modules are inference-only and refuse grad-enabled calls


def test_unet_matches_reference_golden(unet, gold):
    from oracle.pin_ldm_against_reference import unet_inputs
    x, t, ctx = unet_inputs()
    e = unet(torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda(), torch.from_numpy(ctx).cuda())
    torch.cuda.synchronize()
    assert e.shape == (2, 4, 32, 32) and e.dtype == torch.float32
    err = (e.cpu() - torch.from_numpy(gold["unet_eps"])).abs()
    print("unet: max err", float(err.max()), "mean err", float(err.mean()))
    assert float(err.max()) < 6.5e-3 and float(err.mean()) < 1.2e-3     # 3x the measured 2.1e-3 / 3.9e-4


def test_unet_batch8_is_consistent_with_batch2(unet):
    """CFG batch of 8 (4 views x 2): rows are independent, so a batch-8 pass equals two batch-4 passes."""
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(8, 8, 32, 32, device="cuda", generator=g)
    t = torch.full((8,), 501, device="cuda")
    ctx = torch.randn(8, 1, 768, device="cuda", generator=g)
    full = unet(x, t, ctx).clone()          # graph replays reuse one static output buffer per input shape
    half = torch.cat([unet(x[:4], t[:4], ctx[:4]).clone(), unet(x[4:], t[4:], ctx[4:]).clone()])
    # batch 8 and batch 4 pick different split-K factors (M differs), so partial sums are ordered differently and a
    # few fp16 roundings of intermediate activations flip: agreement to ~fp16 resolution of an O(1) output
    assert float((full - half).abs().max()) < 1e-2
    unet.use_cuda_graph = False              # eager launches and graph replay run the same kernels with the same tile choices;
    eager = unet(x, t, ctx)                  # split-K planes are summed in a fixed order, but the GroupNorm group sums are
    unet.use_cuda_graph = True               # fp32 atomics (shared memory, and global for the strided convs): rounding only
    assert float((eager - full).abs().max()) < 1e-2


def test_ddim_sampler_matches_reference_trajectory(gold):
    from o2345.ddim import DDIMSampler
    from oracle import ldm_oracle as LO
    toy = LO.ToyModel().to("cuda")
    B = 2
    g = np.random.default_rng(5)
    cond = {"c_crossattn": [torch.from_numpy(g.standard_normal((B, 1, 768), dtype=np.float32)).cuda()],
            "c_concat": [torch.from_numpy(g.standard_normal((B, 4, 32, 32), dtype=np.float32)).cuda()]}
    uc = {"c_crossattn": [torch.zeros(B, 1, 768, device="cuda")], "c_concat": [torch.zeros(B, 4, 32, 32, device="cuda")]}
    torch.manual_seed(123)
    x_T = torch.randn(B, 4, 32, 32)
    noises = [torch.randn(B, 4, 32, 32) for _ in range(4)]
    sampler = DDIMSampler(toy)
    # inject the reference's noise draws: patch torch.randn for the duration of the call
    it = iter(noises)
    real = torch.randn
    torch.randn = lambda *a, **k: next(it).cuda()
    try:
        out, inter = sampler.sample(S=5, batch_size=B, shape=[4, 32, 32], conditioning=cond, verbose=False, eta=1.0,
                                    x_T=x_T.cuda(), unconditional_guidance_scale=3.0, unconditional_conditioning=uc)
    finally:
        torch.randn = real
    assert np.array_equal(sampler.ddim_timesteps, gold["ddim_timesteps"])
    assert float((out.cpu() - torch.from_numpy(gold["ddim_out"])).abs().max()) < 2e-4
    assert "x_inter" in inter and "pred_x0" in inter


def test_ddim_step_noise_is_the_global_generator_stream_drawn_early():
    """Two sampler calls that draw from torch's CUDA generator as they go (the reference's behaviour), against ONE call over
    the concatenated batch fed with the same draws made up front in the same order (zero123.generate_views, batched):
    the same latents per view with a model that treats the images of a batch independently."""
    from o2345.ddim import DDIMSampler
    from oracle import ldm_oracle as LO
    torch.backends.cudnn.allow_tf32 = False
    toy = LO.ToyModel().to("cuda")
    g = np.random.default_rng(9)
    B = 2

    def conds(n):
        c = {"c_crossattn": [torch.from_numpy(g.standard_normal((n, 1, 768), dtype=np.float32)).cuda()],
             "c_concat": [torch.from_numpy(g.standard_normal((n, 4, 32, 32), dtype=np.float32)).cuda()]}
        u = {"c_crossattn": [torch.zeros(n, 1, 768, device="cuda")], "c_concat": [torch.zeros(n, 4, 32, 32, device="cuda")]}
        return c, u
    (c0, u0), (c1, u1) = conds(B), conds(B)
    torch.cuda.manual_seed(77)
    seq = []
    for c, u in ((c0, u0), (c1, u1)):
        out, _ = DDIMSampler(toy).sample(S=5, batch_size=B, shape=[4, 32, 32], conditioning=c, verbose=False, eta=1.0,
                                         unconditional_guidance_scale=3.0, unconditional_conditioning=u)
        seq.append(out)
    torch.cuda.manual_seed(77)
    draws = []
    for _ in range(2):
        x_T = torch.randn(B, 4, 32, 32, device="cuda")
        draws.append((x_T, [torch.randn(B, 4, 32, 32, device="cuda") for _ in range(4)]))
    cat = lambda a, b: {k: [torch.cat([a[k][0], b[k][0]])] for k in a}
    out, _ = DDIMSampler(toy).sample(S=5, batch_size=2 * B, shape=[4, 32, 32], conditioning=cat(c0, c1), verbose=False, eta=1.0,
                                     unconditional_guidance_scale=3.0, unconditional_conditioning=cat(u0, u1),
                                     x_T=torch.cat([draws[0][0], draws[1][0]]),
                                     step_noise=[torch.cat([draws[0][1][i], draws[1][1][i]]) for i in range(4)])
    # the toy model is a cuDNN convolution, whose algorithm may change with the batch size: equal up to fp32 summation order
    assert float((out[:B] - seq[0]).abs().max()) < 1e-5 and float((out[B:] - seq[1]).abs().max()) < 1e-5
    with pytest.raises(ValueError):
        DDIMSampler(toy).sample(S=5, batch_size=B, shape=[4, 32, 32], conditioning=c0, verbose=False, eta=1.0,
                                unconditional_guidance_scale=3.0, unconditional_conditioning=u0, step_noise=draws[0][1][:3])
