"""GPU: the fused self-attention kernel (o2345_attention_f16) against softmax(q k^T * scale) v computed in float64 from the
same fp16 inputs the kernel received.

Error model.  The kernel forms the scores in fp32 (fp16 products, fp32 accumulation), takes p = 2^((s - m) * scale * log2 e)
in fp32 and rounds p to fp16 for the P V product; O and the row sums l accumulate those same rounded p in fp32, and O / l is
rounded to fp16.  Rounding p (relative error <= 2^-11, or 2^-25 absolute below the fp16 normal range) moves each softmax
weight by <= 2^-11 relative, and because numerator and denominator use the same rounded p the weights still sum to one: the
weighted mean of V moves by <= 2 * 2^-11 * max|v| (plus N * 2^-25 * max|v| from subnormal weights).  The fp32 score and
exponent errors are ~2^-20 relative to the weights even at the off-centre scores of +-60, and the output rounding adds
2^-11 |want|.  Hence

    |out - want| <= C1 * 2^-11 * max|v| + 2^-11 * |want|.

C1 = 0.55 is about three times the largest value measured on an H100 80GB HBM3 (700 W power limit): 0.175 on the random
rows (off-centre 0.131, late maximum 0.057, peaked 0.0: there the output error stays below 2^-11 |want|).  With q = 0 (the
flat regime) every p is exactly 1, so only the fp32 sums and the output rounding remain:
|out - want| <= N * 2^-23 * max|v| + 2^-11 |want|; the largest error measured there is 2^-10, half an ulp of an output
in [2, 4)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U16 = 2.0 ** -11            # fp16 unit roundoff
C1 = 0.55                   # 3x the 0.175 measured on an H100 80GB HBM3 (700 W)
KT = 64                     # keys per tile of the kernel

NS = [1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 511, 512, 513, 1024]     # key-tile edges, and the 4 / 8-warp switch at 512
DS = [40, 64, 80, 160]
REGIMES = ["flat", "random", "peaked", "late_max", "off_centre"]


def _call(q, k, v, B, N, H, d, out, scale):
    from o2345 import _lib as L, ops_a as A
    L.call("o2345_attention_f16", A._v(q), A._v(k), A._v(v), B, N, H, d, q.stride(0), A._v(out), out.stride(0), float(scale),
           A._stream())


def _reference(q, k, v, B, N, H, d, scale):
    """float64 softmax(q k^T * scale) v per (batch, head) -> ([B*N, H*d], scaled scores [B, H, N, N])."""
    f = lambda t: t.double().reshape(B, N, H, d).transpose(1, 2)
    s = f(q) @ f(k).transpose(-1, -2) * scale
    o = torch.softmax(s, -1) @ f(v)
    return o.transpose(1, 2).reshape(B * N, H * d), s


def _fill(buf, regime, B, N, H, d, scale, g):
    """Writes q, k, v of one input regime into the column blocks 0, C, 2C of buf [B*N, >= 3C] (fp16)."""
    C, dev = H * d, buf.device
    rn = lambda *shape: torch.randn(*shape, device=dev, generator=g)
    q, k, v = (buf[:, i * C:(i + 1) * C].view(B, N, H, d) for i in range(3))
    if regime == "flat":                      # all scores 0: the output is the mean of V's rows (offset, so a lost or
        q.zero_()                             # extra key changes it by ~2 / N)
        k.copy_(rn(B, N, H, d))
        v.copy_(0.5 * rn(B, N, H, d) + 2.0)
    elif regime == "random":
        for t in (q, k, v):
            t.copy_(0.8 * rn(B, N, H, d))
    elif regime == "peaked":
        # min(d, N) orthogonal "special" keys A * e_m at random positions; query i points at one of them with weight lam, so
        # its special key scores scale * lam * A and every other key at most scale * lam * max|k_j[m]| (<~ 4.5 lam scale)
        A = 16.0
        kk = rn(B, N, H, d)
        nsp = min(d, N)
        pos = torch.randperm(N, device=dev, generator=g)[:nsp]
        kk[:, pos] = 0.0
        kk[:, pos, :, torch.arange(nsp, device=dev)] = A
        lam = 30.0 / (scale * (A - 4.5))
        m = torch.randint(0, nsp, (B, N, H), device=dev, generator=g)
        q.copy_(lam * torch.nn.functional.one_hot(m, d).float() + 0.05 * rn(B, N, H, d))
        k.copy_(kk)
        v.copy_(rn(B, N, H, d))
    elif regime == "late_max":
        # q[..., 0] = 4 and k[j, ..., 0] = bonus(j) / (4 scale): the scaled score carries bonus(j) = 0.5 * tile(j), + 3 in the
        # last tile, over noise of std 0.25.  The running maximum rises at every tile (an a0 < 1 rescale of O and l each
        # time) and the row maximum lies in the last tile.
        tile = torch.arange(N, device=dev) // KT
        bonus = 0.5 * tile.float() + 3.0 * (tile == tile[-1]).float()
        r = math.sqrt(0.25 / (scale * math.sqrt(d)))
        qq, kk = r * rn(B, N, H, d), r * rn(B, N, H, d)
        qq[..., 0] = 4.0
        kk[..., 0] = (bonus / (4.0 * scale))[None, :, None]
        q.copy_(qq), k.copy_(kk), v.copy_(rn(B, N, H, d))
    elif regime == "off_centre":
        # one shared vector mu added to every key: the scaled scores of a row sit near scale * q_i . mu ~ +-60 while their
        # spread across keys stays O(1) (softmax ignores the per-row shift; the kernel's running maximum does not)
        mu = rn(H, d)
        mu = mu / mu.norm(dim=-1, keepdim=True) * (60.0 / (0.8 * scale))
        q.copy_(0.8 * rn(B, N, H, d))
        k.copy_(0.5 * rn(B, N, H, d) + mu)
        v.copy_(rn(B, N, H, d))
    else:
        raise ValueError(regime)


def _check_inputs(regime, s, N):
    """The regime's defining property holds for the fp16-rounded inputs (float64 scaled scores s [B, H, N, N])."""
    if regime == "peaked" and N > 1:
        top = s.topk(2, dim=-1).values
        assert float((top[..., 0] - top[..., 1]).min()) >= 20.0
    if regime == "late_max":
        assert bool((s.argmax(-1) // KT == (N - 1) // KT).all())
    if regime == "off_centre":
        assert float(s.abs().amax()) > 30.0


def _bound(regime, want, v, N):
    vmax = float(v.float().abs().max())
    if regime == "flat":
        return N * 2.0 ** -23 * vmax + U16 * want.abs()
    return C1 * U16 * vmax + U16 * want.abs()


def _measured_c1(err, want, v):
    return float(((err - U16 * want.abs()) / (U16 * float(v.float().abs().max()))).max())


def _bh(N):
    return (2, 2) if N < 512 else (1, 2)


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("d", DS)
def test_attention_matches_fp64(d, N, regime):
    """Every head dim on both sides of the 4 / 8-warp switch and at every key-tile tail, in five input regimes, through
    ops_a.attention (row stride 3C, scale d^-0.5); a second call on the same inputs is bit-identical."""
    from o2345 import ops_a
    if regime == "late_max" and N <= KT:
        pytest.skip("one key tile: no later tile to hold the maximum")
    B, H = _bh(N)
    C, scale = H * d, d ** -0.5
    g = torch.Generator(device="cuda").manual_seed(1000 * d + N + 7 * REGIMES.index(regime))
    buf = torch.empty(B * N, 3 * C, dtype=torch.float16, device="cuda")
    _fill(buf, regime, B, N, H, d, scale, g)
    q, k, v = buf[:, :C], buf[:, C:2 * C], buf[:, 2 * C:]
    out = ops_a.attention(q, k, v, B, N, H, d)
    want, s = _reference(q, k, v, B, N, H, d, scale)
    _check_inputs(regime, s, N)
    err = (out.double() - want).abs()
    print(f"attention d={d} N={N} {regime}: max err {float(err.max()):.3e} c1 {_measured_c1(err, want, v):.3f}")
    assert bool(torch.isfinite(out).all())
    bad = err > _bound(regime, want, v, N)
    assert not bool(bad.any()), (float(err.max()), int(bad.sum()))
    again = ops_a.attention(q, k, v, B, N, H, d)
    assert torch.equal(out.view(torch.int16), again.view(torch.int16))


@pytest.mark.parametrize("regime", ["random", "peaked", "late_max", "off_centre"])
@pytest.mark.parametrize("scale", [None, 1.0, 0.02])
@pytest.mark.parametrize("pad", [8, 64])
@pytest.mark.parametrize("d,N", [(40, 65), (64, 17), (80, 513), (160, 129)])
def test_attention_strides_slices_and_scales(d, N, pad, scale, regime):
    """q, k, v as column blocks of a [B*N, 3C + pad] buffer (ld = 3C + pad), the output written into a column slice of a
    wider buffer (ldo = C + 24, starting at column 8), and scales 1.0 and 0.02 besides d^-0.5.  Every column outside the
    slice and the rows past B*N keep their sentinel."""
    if regime == "late_max" and N <= KT:
        pytest.skip("one key tile: no later tile to hold the maximum")
    B, H = 2, 2
    C = H * d
    scale = d ** -0.5 if scale is None else scale
    g = torch.Generator(device="cuda").manual_seed(7 * d + N + pad)
    sentinel = torch.tensor(-31.25, dtype=torch.float16)
    buf = torch.empty(B * N, 3 * C + pad, dtype=torch.float16, device="cuda")
    buf[:, 3 * C:] = 7.0
    _fill(buf, regime, B, N, H, d, scale, g)
    q, k, v = buf[:, :C], buf[:, C:2 * C], buf[:, 2 * C:3 * C]
    wide = torch.full((B * N + 3, C + 24), float(sentinel), dtype=torch.float16, device="cuda")
    out = wide[:B * N, 8:8 + C]
    _call(q, k, v, B, N, H, d, out, scale)
    want, s = _reference(q, k, v, B, N, H, d, scale)
    _check_inputs(regime, s, N)
    err = (out.double() - want).abs()
    print(f"attention strided d={d} N={N} ld={3 * C + pad} scale={scale:.4g} {regime}: max err {float(err.max()):.3e} "
          f"c1 {_measured_c1(err, want, v):.3f}")
    bad = err > _bound(regime, want, v, N)
    assert not bool(bad.any()), (float(err.max()), int(bad.sum()))
    keep = torch.ones_like(wide, dtype=torch.bool)
    keep[:B * N, 8:8 + C] = False
    assert bool((wide[keep].view(torch.int16) == sentinel.view(torch.int16).item()).all())


@pytest.mark.parametrize("B,N,H,d", [(2, 1024, 8, 40), (8, 256, 8, 80), (3, 64, 8, 160), (2, 16, 8, 160), (1, 100, 2, 40), (1, 640, 4, 80),
                                     (1, 1000, 2, 160), (2, 257, 16, 64), (1, 577, 3, 64)])
def test_attention_matches_reference(B, N, H, d):
    """The UNet / CLIP head counts (8, 16) at a few sizes, against torch in fp32 (3e-3 abs on outputs of O(1))."""
    from o2345 import ops_a
    g = torch.Generator(device="cuda").manual_seed(N + d)
    C = H * d
    qkv = (torch.randn(B * N, 3 * C, device="cuda", generator=g) * 0.8).half()
    out = ops_a.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], B, N, H, d)
    torch.cuda.synchronize()
    q, k, v = (qkv[:, i * C:(i + 1) * C].float().view(B, N, H, d).permute(0, 2, 1, 3) for i in range(3))
    want = torch.softmax(q @ k.transpose(-1, -2) * d ** -0.5, -1) @ v
    want = want.permute(0, 2, 1, 3).reshape(B * N, C)
    err = (out.float() - want).abs().max().item()
    assert err < 3e-3, err
