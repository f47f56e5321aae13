"""GPU: the glue kernels of the Zero123 UNet / VAE / CLIP tower (csrc/unet_ops.cu) checked one by one.

Conversions, copies and single-rounding additions are compared bit for bit with torch doing the same rounding.  The
kernels with arithmetic (softmax_rows, the VAE's unfused attention chain, timestep_embedding, cfg_ddim_update, silu, geglu)
are compared with float64 references computed from the same fp16 / fp32 inputs, each against a bound derived in its
docstring; every test prints the largest measured error as a fraction of its bound."""
import math
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu

U16 = 2.0 ** -11            # fp16 unit roundoff
U32 = 2.0 ** -24            # fp32 unit roundoff
SUB16 = 2.0 ** -25          # half the smallest fp16 subnormal: the absolute rounding error below the normal range
DEV = "cuda"
F16_MAX = 65504.0


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _assert_within(name, err, tol):
    """err <= tol everywhere; prints the worst err / tol."""
    ratio = float((err / tol).max())
    print(f"{name}: max err {float(err.max()):.3e}, worst err / bound {ratio:.3f}")
    assert ratio <= 1.0, (name, ratio)


# ---------------------------------------------------------------------------------------------------- softmax_rows
def _score_rows(n, g):
    """13 rows of fp16 scores (not a multiple of the 8 rows a CTA takes): random, wide, flat, peaked, and rows holding
    +-65504."""
    s = torch.randn(13, n, device=DEV, generator=g) * 3.0
    s[4] = 1.5                                                    # flat
    s[5, n // 2] += 25.0                                          # peaked
    s[6, n - 1] = F16_MAX                                         # one +65504: the others get exactly 0
    s[7, ::2] = -F16_MAX                                          # half the row at -65504
    s[8] = -F16_MAX                                               # all -65504: uniform
    s[9, 0] = F16_MAX
    s[9, n // 3] = F16_MAX                                        # +65504 twice (once if n == 1)
    s[10, 0] = -F16_MAX
    s[10, n - 1] = F16_MAX
    s[11:] *= 8.0
    return s.half()


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 77, 257, 1000, 1023, 1024])
def test_softmax_rows_matches_fp64(n):
    """softmax_rows (fp32 max / expf / sum, probabilities rounded to fp16) against float64 softmax of the same fp16 scores.

    Before the final rounding each probability carries a relative error eps = (n + 24) * 2^-24: the fp32 row sum (n
    additions), expf (2 ulp), the reciprocal and the product, and the fp32 difference s - max (exact unless the exponents
    differ by more than 13 bits, <= 18 * 2^-24 relative wherever p is above the fp16 range).  The fp16 rounding then adds
    2^-11 relative or 2^-25 absolute, so |p - want| <= (2^-11 (1 + eps) + eps) want + 2^-25, and each row sums to 1 within
    2^-11 (1 + eps) + eps + n 2^-25.  A row of length 1 is exactly 1.  Measured on an H100 80GB HBM3 (700 W): up to 0.999
    of the bound, which the final rounding alone nearly reaches (a half-ulp error on a probability just above a power of
    two)."""
    from o2345 import ops_a as A
    s = _score_rows(n, _gen(n))
    p = A.softmax_rows(s)
    want = torch.softmax(s.double(), -1)
    assert bool(torch.isfinite(p).all())
    eps = (n + 24) * U32
    _assert_within(f"softmax_rows n={n}", (p.double() - want).abs(), (U16 * (1 + eps) + eps) * want + SUB16)
    row_err = (p.double().sum(-1) - 1.0).abs()
    assert float(row_err.max()) <= U16 * (1 + eps) + eps + n * SUB16, float(row_err.max())
    if n == 1:
        assert bool((p == 1.0).all())
    # 3-D input ([B, N, N] as the VAE issues it) goes through the same rows
    p3 = A.softmax_rows(s[:12].reshape(3, 4, n))
    assert torch.equal(_bits(p3.reshape(12, n)), _bits(p[:12]))


# ------------------------------------------------------------------------------------ unfused attention (VAE mid block)
@pytest.mark.parametrize("N", [64, 256, 1024])
def test_vae_mid_block_attention_chain(N):
    """The VAE's single-head mid-block attention exactly as autoencoder.py issues it (bgemm QK^T * C^-1/2 -> softmax_rows ->
    transpose_tokens -> bgemm), C = 512, B = 2, against float64 softmax(Q K^T / sqrt(C)) V.

    The scores are rounded to fp16 (2^-11 |s| absolute in the logits, which moves each softmax weight by <= 2 * 2^-11 max|s|
    relative), the probabilities are rounded to fp16 (<= 2^-11 relative, weights no longer summing exactly to one) and the
    output is rounded to fp16: |o - want| <= 2^-11 max|v| (1 + 2 max|s| + N 2^-14) + 2^-11 |want|.  Measured on an H100
    80GB HBM3 (700 W): at most 0.043 of that bound (max error 8.3e-4 at N = 64)."""
    from o2345 import ops_a as A
    B, C = 2, 512
    g = _gen(N)
    q, k, v = (torch.randn(B * N, C, device=DEV, generator=g).half() for _ in range(3))
    s = torch.empty(B, N, N, dtype=torch.float16, device=DEV)
    A.bgemm(q, k, s, 1, B, (0, N * C), (0, N * C), (0, N * N), N, N, C, C, C, N, alpha=int(C) ** -0.5)
    p = A.softmax_rows(s)
    vt = A.transpose_tokens(v, B, N, C)
    o = torch.empty(B * N, C, dtype=torch.float16, device=DEV)
    A.bgemm(p, vt, o, 1, B, (0, N * N), (0, C * N), (0, N * C), N, C, N, N, N, C)
    qd, kd, vd = (t.double().view(B, N, C) for t in (q, k, v))
    sd = qd @ kd.transpose(1, 2) / math.sqrt(C)
    want = (torch.softmax(sd, -1) @ vd).reshape(B * N, C)
    vmax, smax = float(v.abs().max()), float(sd.abs().max())
    tol = U16 * vmax * (1 + 2 * smax + N * 2.0 ** -14) + U16 * want.abs()
    _assert_within(f"VAE attention chain N={N}", (o.double() - want).abs(), tol)


@pytest.mark.parametrize("N,C", [(77, 72), (1, 8), (257, 1024), (64, 512)])
def test_transpose_tokens_is_exact(N, C):
    from o2345 import ops_a as A
    B = 2
    x = torch.randn(B * N, C, device=DEV, generator=_gen(N * C)).half()
    y = A.transpose_tokens(x, B, N, C)
    assert torch.equal(_bits(y), _bits(x.view(B, N, C).transpose(1, 2)))


# ------------------------------------------------------------------------------------------------- layout converters
def _with_specials(x):
    """Puts values at the edges of fp16 into the first elements of an fp32 tensor: overflow to inf, the largest finite
    value, subnormals, a tie and signed zero."""
    sp = torch.tensor([70000.0, -65519.0, 65520.0, 1e-8, -3e-5, 2.0 ** -25, 1.0 + 2.0 ** -11, -0.0, 6e-5, 1e5],
                      device=x.device)
    flat = x.view(-1)
    m = min(flat.numel(), sp.numel())
    flat[:m] = sp[:m]
    return x


@pytest.mark.parametrize("C,ldy,off", [(3, 16, 5), (4, 8, 4), (8, 24, 8), (320, 336, 7)])
def test_nchw_to_cl_into_a_column_slice(C, ldy, off):
    """[B, C, H, W] fp32 -> rows (b, y, x) of a channel-last fp16 buffer, columns off .. off + C of rows ldy wide, with one
    rounding: bit-equal to x.permute(0, 2, 3, 1).half(); the other columns keep their sentinel.  H * W = 35 is odd."""
    from o2345 import ops_a as A
    B, H, W = 2, 5, 7
    x = _with_specials(torch.randn(B, C, H, W, device=DEV, generator=_gen(C)) * 4.0)
    sentinel = -31.25
    out = torch.full((B * H * W, ldy), sentinel, dtype=torch.float16, device=DEV)
    A.nchw_to_cl(x, out, off)
    want = x.permute(0, 2, 3, 1).reshape(B * H * W, C).half()
    assert torch.equal(_bits(out[:, off:off + C]), _bits(want))
    keep = torch.ones(ldy, dtype=torch.bool, device=DEV)
    keep[off:off + C] = False
    assert bool((out[:, keep] == sentinel).all())


@pytest.mark.parametrize("C,ldx,off", [(3, 8, 4), (8, 24, 8), (320, 648, 320)])
def test_cl_to_nchw_from_a_column_slice(C, ldx, off):
    """Channel-last fp16 rows read from a column slice (ldx > C) -> [B, C, H, W] fp32: exact."""
    from o2345 import ops_a as A
    B, H, W = 2, 5, 7
    big = torch.randn(B * H * W, ldx, device=DEV, generator=_gen(ldx)).half()
    x = big[:, off:off + C]
    y = A.cl_to_nchw(x, B, C, H, W)
    assert torch.equal(_bits(y), _bits(x.float().view(B, H, W, C).permute(0, 3, 1, 2)))


@pytest.mark.parametrize("M,C,ldd,off", [(1, 8, 24, 8), (37, 320, 648, 320), (1003, 64, 136, 72)])
def test_copy_channels_into_a_column_slice(M, C, ldd, off):
    from o2345 import ops_a as A
    src = torch.randn(M, C, device=DEV, generator=_gen(M + C)).half()
    sentinel = 5.5
    dst = torch.full((M, ldd), sentinel, dtype=torch.float16, device=DEV)
    A.copy_channels(src, dst, off)
    assert torch.equal(_bits(dst[:, off:off + C]), _bits(src))
    keep = torch.ones(ldd, dtype=torch.bool, device=DEV)
    keep[off:off + C] = False
    assert bool((dst[:, keep] == sentinel).all())


@pytest.mark.parametrize("B,HW,C,ld,off", [(3, 63, 40, 104, 24), (2, 81, 320, 1920, 640), (4, 9, 1280, 2568, 1288)])
def test_add_channel_bias_from_a_column_slice(B, HW, C, ld, off):
    """y[b, p, c] += e[b, c] with e a column slice of a wider [B, ld] matrix (as the UNet's stacked timestep projections
    are): bit-equal to (y.float() + e.float()).half().  The first two element counts are not multiples of 256."""
    from o2345 import ops_a as A
    g = _gen(B * HW * C)
    y = torch.randn(B * HW, C, device=DEV, generator=g).half()
    emb = (torch.randn(B, ld, device=DEV, generator=g) * 2.0).half()
    e = emb[:, off:off + C]
    want = (y.float().view(B, HW, C) + e.float()[:, None, :]).half().view(B * HW, C)
    A.add_channel_bias(y, e, B, HW, C)
    assert torch.equal(_bits(y), _bits(want))


def test_clip_add_positions():
    """Row 0 of every image becomes cls + pos[0], every other row tok + pos[n], each one fp32 addition rounded once to fp16
    (B = 3 images of N = 257 tokens, ViT-L width)."""
    from o2345 import ops_a as A
    B, N, d = 3, 257, 1024
    g = _gen(257)
    tok = torch.randn(B * N, d, device=DEV, generator=g).half()
    cls = torch.randn(d, device=DEV, generator=g)
    pos = torch.randn(N, d, device=DEV, generator=g) * 0.5
    want = (tok.float().view(B, N, d) + pos).half()
    want[:, 0] = (cls + pos[0]).half()
    A.clip_add_positions(tok, cls, pos, B, N, d)
    assert torch.equal(_bits(tok), _bits(want.view(B * N, d)))


# -------------------------------------------------------------------------------------------------- timestep_embedding
@pytest.mark.parametrize("dim", [320, 1280])
def test_timestep_embedding_matches_fp64(dim):
    """[cos(t f_k) | sin(t f_k)], f_k = exp(-ln(10000) k / half), against float64 cos / sin of the argument the reference
    forms in fp32 (util.py:151-171).  The kernel's fp32 frequency may differ from the reference's by a few ulp, which
    moves the argument by about |t| 2^-23; the fp16 rounding adds half an ulp of the value.  Bound: one fp16 ulp of the
    value + |t| 2^-23.  Measured on an H100 80GB HBM3 (700 W): at most 0.51 of the bound."""
    from o2345 import ops_a as A
    t = torch.tensor([0.0, 1.0, 500.0, 981.0, 999.0])
    out = A.timestep_embedding(t.to(DEV), dim)
    half = dim // 2
    freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32) / half)
    args = (t[:, None].float() * freqs[None]).double()
    want = torch.cat([torch.cos(args), torch.sin(args)], -1).to(DEV)
    ulp = torch.exp2(torch.floor(torch.log2(want.abs())).clamp(min=-14) - 10)
    tol = ulp + t.double().to(DEV)[:, None].abs() * 2.0 ** -23
    _assert_within(f"timestep_embedding dim={dim}", (out.double() - want).abs(), tol)


# ----------------------------------------------------------------------------------------------------- cfg_ddim_update
def _zero123_samplers():
    """DDIMSampler schedules of the Zero123 model: 75 and 50 steps, eta 0 and 1, from the fp32 alphas_cumprod table and from
    its fp16 rounding (the schedule a `.half()` model hands the sampler)."""
    from o2345.ddim import DDIMSampler
    from oracle import ldm_oracle as LO
    ac = torch.from_numpy(LO.linear_beta_alphas_cumprod())
    for table, a in (("fp32", ac), ("fp16", ac.half())):
        for S in (75, 50):
            for eta in (0.0, 1.0):
                smp = DDIMSampler(SimpleNamespace(num_timesteps=1000, device=torch.device("cpu"), alphas_cumprod=a))
                smp.make_schedule(S, ddim_eta=eta, verbose=False)
                yield f"{table} S={S} eta={eta:g}", smp


def test_cfg_ddim_update_every_step_of_the_zero123_schedules():
    """The fused CFG + DDIM update against a float64 restatement of p_sample_ddim (reference ddim.py:212-243) from the same
    fp32 inputs and the same fp32 schedule values, at every iteration of each schedule, guidance 1 and 3; every other step
    without noise, every third without pred_x0; n = 2 * 4 * 11 * 13 (not a multiple of 256).

    fp32 error model (u = 2^-24), with E = |e_u| + s (|e_c| + |e_u|) bounding e_t and its rounding, and
    P = (|x| + sqrt(1 - a_t) E) / sqrt(a_t) bounding pred_x0 (the 1 / sqrt(a_t) amplification, ~14 at t = 981):
      pred_x0:  8 u P;
      x_prev:   sqrt(a') (11 u P) + 6 u c E + 3 u E / c + 3 u sigma |noise|, with c = sqrt(1 - a' - sigma^2); the fp32
                difference 1 - a' - sigma^2 (down to 1.1e-4 at the last step) carries an absolute error of a few u,
                hence the E / c term.
    The assertions use 16 u times the sum of those magnitudes (a margin over the derived 11).  Measured on an H100 80GB
    HBM3 (700 W): at most 2.6 u (x_prev) and 3.0 u (pred_x0) times those magnitudes."""
    from o2345 import ops_a as A
    g = _gen(981)
    shape = (2, 4, 11, 13)
    n = math.prod(shape)
    x = torch.randn(shape, device=DEV, generator=g)
    eps2 = torch.randn((2 * shape[0],) + shape[1:], device=DEV, generator=g)
    noise = torch.randn(shape, device=DEV, generator=g)
    xd, nd = x.double().view(-1), noise.double().view(-1)
    eu, ec = eps2.double().view(-1)[:n], eps2.double().view(-1)[n:]
    worst = {"x_prev": 0.0, "pred_x0": 0.0}
    for name, smp in _zero123_samplers():
        steps = len(smp.ddim_timesteps) - 1                    # the sampler's iterations (t_start = -1)
        for scale in (1.0, 3.0):
            E = eu.abs() + scale * (ec.abs() + eu.abs())
            e = eu + scale * (ec - eu)
            for idx in range(steps):
                a_t, a_p = float(smp.ddim_alphas[idx]), float(smp.ddim_alphas_prev[idx])
                sig, s1m = float(smp.ddim_sigmas[idx]), float(smp.ddim_sqrt_one_minus_alphas[idx])
                use_noise, want_x0 = idx % 2 == 0, idx % 3 != 0
                x_prev, pred = A.cfg_ddim_update(x, eps2, noise if use_noise else None, scale, a_t, a_p, sig, s1m, want_x0)
                p0 = (xd - s1m * e) / math.sqrt(a_t)
                c = math.sqrt(1.0 - a_p - sig * sig)
                nz = sig * nd if use_noise else torch.zeros_like(nd)
                want = math.sqrt(a_p) * p0 + c * e + nz
                P = (xd.abs() + s1m * E) / math.sqrt(a_t)
                mag = math.sqrt(a_p) * P + c * E + E / c + nz.abs()
                where = f"{name} scale={scale:g} index={idx}"
                assert bool(torch.isfinite(x_prev).all()), where
                r = float(((x_prev.double().view(-1) - want).abs() / (U32 * mag)).max())
                worst["x_prev"] = max(worst["x_prev"], r)
                assert r <= 16.0, (where, "x_prev", r)
                if want_x0:
                    assert bool(torch.isfinite(pred).all()), where
                    r = float(((pred.double().view(-1) - p0).abs() / (U32 * P)).max())
                    worst["pred_x0"] = max(worst["pred_x0"], r)
                    assert r <= 16.0, (where, "pred_x0", r)
                else:
                    assert pred is None
    print(f"cfg_ddim_update: worst err / (u * magnitude): x_prev {worst['x_prev']:.2f}, pred_x0 {worst['pred_x0']:.2f} (bar 16)")


# ------------------------------------------------------------------------------------------------------ silu and geglu
def _extremes():
    return torch.tensor([F16_MAX, -F16_MAX, 20.0, -20.0, 88.0, -88.0, 0.0, -0.0, 6e-5, -6e-5, 11.0, -11.0, 2.0 ** -24, 1.0],
                        dtype=torch.float16, device=DEV)


def test_silu_matches_fp64():
    """silu(x) = x / (1 + __expf(-x)) in fp32, rounded to fp16.  __expf(y) is within (2 + 1.2 |y|) ulp, which reaches the
    result as relative error; with the fp32 sum and quotient eps = (6 + 1.2 |x|) 2^-23, and the bound is
    (2^-11 + eps) |want| + 2^-25.  Inputs include +-65504 and +-20; no NaN may appear.  Measured on an H100 80GB HBM3
    (700 W): the worst case is the bound itself, at x = 2^-24, whose silu 2^-25 is a tie that rounds to 0."""
    from o2345 import ops_a as A
    x = (torch.randn(1037, device=DEV, generator=_gen(1037)) * 4.0).half()
    x[:14] = _extremes()
    y = A.silu(x)
    assert not bool(torch.isnan(y).any())
    xd = x.double()
    want = xd * torch.sigmoid(xd)
    eps = (6 + 1.2 * xd.abs()) * 2.0 ** -23
    _assert_within("silu", (y.double() - want).abs(), (U16 + eps) * want.abs() + SUB16)


def test_geglu_matches_fp64():
    """geglu: a * 0.5 g (1 + erff(g / sqrt 2)) in fp32, rounded to fp16, I = 640 and M = 77 rows (M * I / 8 is not a
    multiple of the 256-thread block).  erff is within 2 ulp, so 1 + erf carries an absolute error <= 2^-23 that the
    cancellation at negative g turns relative; hence |y - want| <= (2^-11 + 2^-20) |want| + |a| |g| (1 + |g|) 2^-23 + 2^-25.
    Extreme inputs (+-65504 and +-20) give finite values or, where the exact product exceeds the fp16 range, inf of the
    right sign; never NaN.  Measured on an H100 80GB HBM3 (700 W): at most 0.994 of the bound."""
    from o2345 import ops_a as A
    M, I = 77, 640
    g = _gen(640)
    x = torch.randn(M, 2 * I, device=DEV, generator=g) * 2.0
    ex = _extremes().float()
    x[0, :14] = ex                          # extreme values, gates in the normal range
    x[1, I:I + 14] = ex                     # extreme gates
    x[2, :14] = ex
    x[2, I:I + 14] = ex.flip(0)             # both extreme
    x = x.half()
    y = A.geglu(x)
    assert not bool(torch.isnan(y).any())
    a, gt = x[:, :I].double(), x[:, I:].double()
    want = a * 0.5 * gt * (1 + torch.erf(gt / math.sqrt(2.0)))
    over = want.abs() >= 65520.0                                  # rounds to inf in fp16
    assert torch.equal(y[over], want[over].half())
    err = (y.double() - want).abs()[~over]
    tol = ((U16 + 2.0 ** -20) * want.abs() + a.abs() * gt.abs() * (1 + gt.abs()) * 2.0 ** -23 + SUB16)[~over]
    _assert_within("geglu", err, tol)
