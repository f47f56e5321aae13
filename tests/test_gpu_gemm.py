"""GPU: the wgmma GEMM against torch.matmul in fp32 on the same fp16 inputs (fp32 accumulate on both sides)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def ref(a, b, bias=None, residual=None, act=0, alpha=1.0):
    y = alpha * (a.float() @ b.float().t())
    if bias is not None:
        y = y + bias
    if act == 1:
        y = torch.nn.functional.silu(y)
    if act == 2:
        y = torch.nn.functional.gelu(y)
    if residual is not None:
        y = y + residual.float()
    return y


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 128, 256), (8192, 320, 2880), (100, 72, 40), (512, 1280, 11520),
                                   (64, 2560, 320), (1, 1280, 320), (333, 200, 136)])
def test_gemm_matches_matmul(M, N, K):
    from o2345 import ops_a
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).half()
    b = (torch.randn(N, K, device="cuda", generator=g) * 0.5).half()
    out = ops_a.gemm(a, b, out_dtype=torch.float32)
    torch.cuda.synchronize()
    want = ref(a, b)
    err = (out - want).abs().max().item()
    assert err <= 2e-3 * (K ** 0.5), (err, M, N, K)          # fp32 accumulation: only summation order differs


def test_gemm_epilogues_and_fp16_out():
    from o2345 import ops_a
    g = torch.Generator(device="cuda").manual_seed(1)
    a = (torch.randn(300, 192, device="cuda", generator=g) * 0.3).half()
    b = (torch.randn(160, 192, device="cuda", generator=g) * 0.3).half()
    bias = torch.randn(160, device="cuda", generator=g)
    res = torch.randn(300, 160, device="cuda", generator=g).half()
    for act in (0, 1, 2):
        out = ops_a.gemm(a, b, bias=bias, residual=res, act=act, alpha=0.5)
        want = ref(a, b, bias, res, act, 0.5)
        assert out.dtype == torch.float16
        assert (out.float() - want).abs().max().item() < 2e-2
    # strided A (a column slice of a wider matrix), as the attention q/k/v views use
    wide = (torch.randn(256, 3 * 64, device="cuda", generator=g) * 0.3).half()
    q = wide[:, 64:128]
    out = ops_a.gemm(q, b[:, :64].contiguous(), out_dtype=torch.float32)
    assert (out - ref(q, b[:, :64])).abs().max().item() < 1e-2


def test_batched_gemm_heads_inside_a_token_tensor():
    """q, k live as column blocks of a [B, N, 3*H*d] tensor (fused qkv projection); scores per (b, h)."""
    from o2345 import ops_a
    g = torch.Generator(device="cuda").manual_seed(2)
    B, N, H, d = 2, 256, 8, 40
    Cc = H * d
    qkv = (torch.randn(B, N, 3 * Cc, device="cuda", generator=g) * 0.5).half()
    q, k = qkv[:, :, :Cc], qkv[:, :, Cc:2 * Cc]
    out = torch.empty(B * H, N, N, dtype=torch.float16, device="cuda")
    ops_a.bgemm(q, k, out, H, B, (d, N * 3 * Cc), (d, N * 3 * Cc), (N * N, H * N * N), N, N, d, 3 * Cc, 3 * Cc, N, alpha=d ** -0.5)
    want = torch.einsum("bihd,bjhd->bhij", q.float().view(B, N, H, d), k.float().view(B, N, H, d)) * d ** -0.5
    assert (out.float().view(B, H, N, N) - want).abs().max().item() < 2e-2
    # P @ V with V^T [B, C, N] and the result written back into [B, N, C]
    p = torch.softmax(want, -1).half().contiguous().view(B * H, N, N)
    v = qkv[:, :, 2 * Cc:]
    vt = ops_a.transpose_tokens(v.contiguous(), B, N, Cc)
    o = torch.zeros(B, N, Cc, dtype=torch.float16, device="cuda")
    ops_a.bgemm(p, vt, o, H, B, (N * N, H * N * N), (d * N, Cc * N), (d, N * Cc), N, d, N, N, N, Cc)
    want_o = torch.einsum("bhij,bjhd->bihd", p.float().view(B, H, N, N), v.float().view(B, N, H, d)).reshape(B, N, Cc)
    assert (o.float() - want_o).abs().max().item() < 2e-2


@pytest.mark.parametrize("B,H,W,C,N", [(8, 32, 32, 320, 320), (8, 16, 16, 640, 640), (8, 8, 8, 1280, 1280), (8, 4, 4, 1280, 1280),
                                       (2, 64, 64, 512, 512), (1, 256, 256, 128, 128), (3, 8, 8, 72, 40), (1, 128, 128, 256, 3)])
def test_implicit_conv3x3_matches_conv2d(B, H, W, C, N):
    """The TMA shifted-window convolution against F.conv2d (fp32) on the same fp16 operands."""
    from o2345 import ops_a
    g = torch.Generator(device="cuda").manual_seed(H + C)
    x = (torch.randn(B, H, W, C, device="cuda", generator=g) * 0.5).half()
    w = (torch.randn(N, C, 3, 3, device="cuda", generator=g) * (2.0 / (9 * C)) ** 0.5).half()
    bias = torch.randn(N, device="cuda", generator=g)
    wk = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    out = ops_a.conv3x3(x.view(-1, C), B, H, W, C, wk, bias=bias, out_dtype=torch.float32)
    want = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias, padding=1).permute(0, 2, 3, 1).reshape(-1, N)
    err = (out - want).abs().max().item()
    assert err < 5e-3, err


@pytest.mark.parametrize("M,N,K", [(8192, 2560, 320), (2048, 640, 5760), (512, 10240, 1280), (128, 1280, 11520), (8, 20160, 1280),
                                   (8192, 960, 320), (2048, 1920, 640), (4096, 512, 1152), (1000, 256, 192), (300, 192, 72),
                                   (257, 160, 64), (129, 3840, 1280)])
def test_pair_kernel_shapes(M, N, K):
    """Every tile width of the kernel (160 / 256 / 128 / 64), M tails inside the second warpgroup, split-K shapes."""
    from o2345 import ops_a
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).half()
    b = (torch.randn(N, K, device="cuda", generator=g) * 0.5).half()
    out = ops_a.gemm(a, b, out_dtype=torch.float32)
    again = ops_a.gemm(a, b, out_dtype=torch.float32)        # the split-K workspace must come back zeroed
    want = ref(a, b)
    assert (out - want).abs().max().item() <= 2e-3 * (K ** 0.5)
    assert (again - want).abs().max().item() <= 2e-3 * (K ** 0.5)


def test_rowbias_and_geglu_epilogues():
    from o2345 import ops_a
    g = torch.Generator(device="cuda").manual_seed(5)
    Bn, HW, K, N = 4, 96, 320, 640
    a = (torch.randn(Bn * HW, K, device="cuda", generator=g) * 0.3).half()
    b = (torch.randn(N, K, device="cuda", generator=g) * 0.3).half()
    bias = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(Bn * HW, N, device="cuda", generator=g).half()
    emb = torch.randn(Bn, 3 * N, device="cuda", generator=g).half()
    rb = emb[:, N:2 * N]                                       # a column block of a wider matrix, as emb_all is
    out = ops_a.gemm(a, b, bias=bias, residual=res, act=1, rowbias=rb, rows_per_group=HW)
    want = torch.nn.functional.silu(a.float() @ b.float().t() + bias + rb.float().repeat_interleave(HW, 0)) + res.float()
    assert (out.float() - want).abs().max().item() < 2e-2
    # GEGLU: value * gelu(gate) with the projection rows interleaved by geglu_pack
    I = N // 2
    wp, bp = ops_a.geglu_pack(b, bias)
    out = ops_a.gemm(a, wp, bias=bp, act=ops_a.ACT_GEGLU)
    y = a.float() @ b.float().t() + bias
    want = y[:, :I] * torch.nn.functional.gelu(y[:, I:])
    assert out.shape == (Bn * HW, I)
    assert (out.float() - want).abs().max().item() < 2e-2
    assert (ops_a.geglu((y.half())).float() - (y.half().float()[:, :I] * torch.nn.functional.gelu(y.half().float()[:, I:]))).abs().max() < 2e-2


def test_conv_rowbias_split_k():
    """ResBlock first conv: per-image embedding bias in the epilogue, on a shape that takes the split-K route."""
    from o2345 import ops_a
    g = torch.Generator(device="cuda").manual_seed(6)
    B, H, W, C, N = 8, 8, 8, 1280, 1280
    x = (torch.randn(B, H, W, C, device="cuda", generator=g) * 0.5).half()
    w = (torch.randn(N, C, 3, 3, device="cuda", generator=g) * (2.0 / (9 * C)) ** 0.5).half()
    bias = torch.randn(N, device="cuda", generator=g)
    emb = torch.randn(B, N, device="cuda", generator=g).half()
    wk = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    out = ops_a.conv3x3(x.view(-1, C), B, H, W, C, wk, bias=bias, rowbias=emb, out_dtype=torch.float32)
    want = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias, padding=1) + emb.float()[:, :, None, None]
    assert (out - want.permute(0, 2, 3, 1).reshape(-1, N)).abs().max().item() < 5e-3


@pytest.mark.parametrize("B,HW,C", [(8, 1024, 320), (8, 256, 1920), (8, 16, 2560), (2, 4096, 128), (3, 64, 512), (1, 65536, 256)])
def test_groupnorm_affine_matches_torch(B, HW, C):
    from o2345 import ops_a
    g = torch.Generator(device="cuda").manual_seed(C)
    x = (torch.randn(B, HW, C, device="cuda", generator=g) * 2 + 0.5).half()
    gamma, beta = torch.randn(C, device="cuda", generator=g), torch.randn(C, device="cuda", generator=g)
    for _ in range(2):                                         # second call: the scratch must have been left zeroed
        scale, shift = ops_a.groupnorm_stats(x.view(-1, C), B, HW, C, 32, 1e-5, gamma, beta)
        y, _, _ = ops_a.norm_act_im2col(x.view(-1, C), B, HW, 1, C, 1, 1, False, (scale, shift), True)
        want = torch.nn.functional.silu(torch.nn.functional.group_norm(x.float().permute(0, 2, 1), 32, gamma, beta, 1e-5)).permute(0, 2, 1)
        assert (y.float().view(B, HW, C) - want).abs().max().item() < 2e-2
        # the one-kernel cluster version (statistics exchanged through distributed shared memory): same numbers
        y1 = ops_a.groupnorm_apply(x.view(-1, C), B, HW, C, 32, 1e-5, gamma, beta, True)
        assert (y1.float().view(B, HW, C) - want).abs().max().item() < 2e-2
        assert (y1.float() - y.float()).abs().max().item() < 4e-3      # fp16 rounding of values up to ~8: one ulp either way


@pytest.fixture
def persistent_everywhere():
    """Forces the persistent launch of the GEMM kernel wherever it is available (staged fp16 epilogue, no split-K), whatever
    the tile count; restores the heuristic afterwards."""
    from o2345 import _lib
    lib = _lib.load()
    lib.o2345_debug_gemm_persist(1, 0)
    yield lib
    lib.o2345_debug_gemm_persist(0, 0)
    lib.o2345_debug_gemm_force(0, 0, 0)


@pytest.mark.parametrize("bn", [128, 160, 256])
@pytest.mark.parametrize("M,N,K", [(65536, 320, 320), (16384, 640, 640), (40000, 960, 328), (300, 192, 72), (8192, 2560, 64),
                                   (33000, 1280, 1280)])
def test_persistent_kernel_matches_matmul(persistent_everywhere, bn, M, N, K):
    """At most one CTA per SM walking many tiles, the operand ring's stages and phases running on across tiles: every tile
    width, one to ~8 tiles per CTA, M tails inside the second warpgroup, N tails, K tails, a single k-block (then only the
    ring hand-over is between two tiles), bias + residual + activation and GEGLU epilogues."""
    from o2345 import ops_a
    persistent_everywhere.o2345_debug_gemm_force(2, bn, 1)
    g = torch.Generator(device="cuda").manual_seed(M + N + K + bn)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).half()
    b = (torch.randn(N, K, device="cuda", generator=g) * 0.5).half()
    bias = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g).half()
    tol = 4e-3 * (K ** 0.5) + 2e-2                                  # fp16 output rounding + summation order
    out = ops_a.gemm(a, b)
    assert out.dtype == torch.float16
    assert (out.float() - ref(a, b)).abs().max().item() <= tol
    for act in (0, 1):
        out = ops_a.gemm(a, b, bias=bias, residual=res, act=act)
        assert (out.float() - ref(a, b, bias, res, act)).abs().max().item() <= tol
    if N % 64 == 0:
        wp, bp = ops_a.geglu_pack(b, bias)
        out = ops_a.gemm(a, wp, bias=bp, act=ops_a.ACT_GEGLU)
        y = a.float() @ b.float().t() + bias
        want = y[:, :N // 2] * torch.nn.functional.gelu(y[:, N // 2:])
        assert ((out.float() - want).abs() - 2e-3 * want.abs()).max().item() <= tol          # fp16 output: relative on the large values


@pytest.mark.parametrize("B,H,W,C,N", [(64, 32, 32, 320, 320), (16, 16, 16, 640, 640), (64, 8, 8, 1280, 1280), (3, 64, 64, 128, 128)])
def test_persistent_kernel_implicit_conv(persistent_everywhere, B, H, W, C, N):
    """The implicit 3x3 convolution (nine shifted TMA boxes per channel block) through the persistent launch, with the
    ResBlock epilogue: bias + per-image embedding row bias, then the skip connection."""
    from o2345 import ops_a
    g = torch.Generator(device="cuda").manual_seed(B + H + C)
    x = (torch.randn(B, H, W, C, device="cuda", generator=g) * 0.5).half()
    w = (torch.randn(N, C, 3, 3, device="cuda", generator=g) * (2.0 / (9 * C)) ** 0.5).half()
    bias = torch.randn(N, device="cuda", generator=g)
    emb = torch.randn(B, N, device="cuda", generator=g).half()
    res = torch.randn(B * H * W, N, device="cuda", generator=g).half()
    wk = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    conv = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias, padding=1).permute(0, 2, 3, 1).reshape(-1, N)
    out = ops_a.conv3x3(x.view(-1, C), B, H, W, C, wk, bias=bias, rowbias=emb)
    assert (out.float() - (conv + emb.float().repeat_interleave(H * W, 0))).abs().max().item() < 2e-2
    out = ops_a.conv3x3(x.view(-1, C), B, H, W, C, wk, bias=bias, residual=res)
    assert (out.float() - (conv + res.float())).abs().max().item() < 2e-2


@pytest.mark.parametrize("B,H,W,C,N", [(8, 4, 4, 1280, 1280), (16, 8, 8, 1280, 1280), (64, 16, 16, 640, 640), (4, 32, 32, 512, 512),
                                       (2, 128, 128, 256, 256), (3, 16, 16, 64, 72)])
def test_upsampling_conv_as_four_phase_convolutions(B, H, W, C, N):
    """nearest 2x + 3x3 conv (the UNet / VAE Upsample layers) as four 2x2 implicit convolutions of the low-resolution map with
    pre-summed weights, against F.interpolate + F.conv2d in fp32 on the same fp16 inputs -- borders (zero padding of the
    UP-SAMPLED map), every phase, split-K (4x4, 8x8 maps) and persistent (large maps) routes."""
    from o2345 import ops_a
    from o2345.unet import _Packed
    g = torch.Generator(device="cuda").manual_seed(B * 31 + H + C)
    conv = torch.nn.Conv2d(C, N, 3, padding=1).cuda()
    with torch.no_grad():
        conv.weight.copy_(torch.randn(N, C, 3, 3, device="cuda", generator=g) * (2.0 / (9 * C)) ** 0.5)
        conv.bias.copy_(torch.randn(N, device="cuda", generator=g))
    conv = conv.half()
    x = (torch.randn(B, H, W, C, device="cuda", generator=g) * 0.5).half()
    pk = _Packed(conv)
    w4, b4 = pk.conv_up(conv)
    out = ops_a.conv_up2x(x.view(-1, C), B, H, W, C, w4, bias=b4)
    up = torch.nn.functional.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2.0, mode="nearest")
    want = torch.nn.functional.conv2d(up, conv.weight.float(), conv.bias.float(), padding=1).permute(0, 2, 3, 1).reshape(-1, N)
    assert out.shape == want.shape
    err = (out.float() - want).abs()
    assert err.max().item() < 2e-2 and err.mean().item() < 1.5e-3, (err.max().item(), err.mean().item())
    # the gather route (what round 2 replaced) agrees too
    a, Ho, Wo = ops_a.norm_act_im2col(x.view(-1, C), B, H, W, C, 3, 1, True, None, False)
    w9 = conv.weight.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    old = ops_a.gemm(a, w9, bias=conv.bias.float())
    assert (out.float() - old.float()).abs().max().item() < 2e-2


@pytest.mark.parametrize("M,C", [(4096, 320), (1000, 640), (257, 1280), (77, 1024), (50, 768), (33, 72), (9, 100)])
def test_layernorm_rows_matches_torch(M, C):
    """16-byte vectorised rows (2 / 3 / 5 chunks per lane) and the scalar fallback (C not a multiple of 8), fp32 statistics."""
    from o2345 import ops_a
    g = torch.Generator(device="cuda").manual_seed(M + C)
    x = (torch.randn(M, C, device="cuda", generator=g) * 2.0 + 0.5).half()
    gamma = torch.randn(C, device="cuda", generator=g)
    beta = torch.randn(C, device="cuda", generator=g)
    out = ops_a.layernorm(x, gamma, beta, eps=1e-5)
    want = torch.nn.functional.layer_norm(x.float(), (C,), gamma, beta, 1e-5)
    assert out.dtype == torch.float16 and out.shape == x.shape
    assert (out.float() - want).abs().max().item() < 1.5e-2          # fp16 output rounding on values up to ~10
    assert (out.float() - want).abs().mean().item() < 1e-3
