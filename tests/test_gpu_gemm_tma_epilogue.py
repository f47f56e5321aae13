"""GPU: the staged GEMM epilogue (fp16 output through TMA stores from each consumer warpgroup's half tile, residual loaded by
TMA into that half tile) against fp64 references, with the persistent launch forced on and every tile width forced: M and
N tails, column-slice outputs (ldc > N), residual + row-group bias over several groups per tile, GEGLU, the up-sampling
conv's phase scatter, and more tiles than SMs so that every CTA runs several tiles back to back."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BNS = [64, 128, 160, 256]


@pytest.fixture
def persistent_bn():
    """Forces the persistent launch wherever it is available; the test forces its tile width; restores the heuristic."""
    from o2345 import _lib
    lib = _lib.load()
    lib.o2345_debug_gemm_persist(1, 0)
    yield lib
    lib.o2345_debug_gemm_persist(0, 0)
    lib.o2345_debug_gemm_force(0, 0, 0)


def _act(y, act):
    if act == 1:
        return torch.nn.functional.silu(y)
    if act == 2:
        return torch.nn.functional.gelu(y)
    return y


def _rand(shape, g, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).half()


@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("M,N,K,rpg,act", [(40000, 200, 320, 40, 0), (9000, 328, 136, 5, 1), (333, 72, 64, 100, 2),
                                           (20000, 640, 200, 1000, 0)])
def test_slice_output_residual_rowbias(persistent_bn, bn, M, N, K, rpg, act):
    """out = act(a b^T + bias + rowbias[row // rpg]) + residual written into columns [8, 8 + N) of a wider tensor (the
    neighbouring columns must stay untouched); rpg 5 spans more groups per warpgroup than the shared-memory copy holds."""
    from o2345 import ops_a
    persistent_bn.o2345_debug_gemm_force(2, bn, 1)
    g = torch.Generator(device="cuda").manual_seed(M + N + K + bn)
    a, b = _rand((M, K), g, 0.5), _rand((N, K), g, 0.5)
    bias = torch.randn(N, device="cuda", generator=g)
    groups = (M + rpg - 1) // rpg
    rowbias = _rand((groups, N + 8), g)[:, :N]                     # row stride N + 8: a multiple of 8, not N
    ldc = N + 24
    wide = torch.full((M, ldc), 7.0, device="cuda", dtype=torch.float16)
    res_wide = _rand((M, ldc), g)
    out = ops_a.gemm(a, b, bias=bias, residual=res_wide[:, 8:8 + N], act=act, out=wide[:, 8:8 + N], rowbias=rowbias,
                     rows_per_group=rpg)
    y = a.double() @ b.double().t() + bias.double() + rowbias.double().repeat_interleave(rpg, 0)[:M]
    want = _act(y, act).half().double() + res_wide[:, 8:8 + N].double()
    err = (out.double() - want).abs() - 2e-3 * want.abs()
    assert err.max().item() <= 4e-3 * K ** 0.5 + 2e-2
    assert bool((wide[:, :8] == 7.0).all()) and bool((wide[:, 8 + N:] == 7.0).all())


@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("M,I,K", [(30000, 160, 320), (1000, 80, 128), (65, 16, 64)])
def test_geglu(persistent_bn, bn, M, I, K):
    """GEGLU: a value column and its gate 16 columns later, out has I = N / 2 columns (80: the 16-column TMA boxes)."""
    from o2345 import ops_a
    persistent_bn.o2345_debug_gemm_force(2, bn, 1)
    g = torch.Generator(device="cuda").manual_seed(M + I + K + bn)
    a, w = _rand((M, K), g, 0.5), _rand((2 * I, K), g, 0.5)
    bias = torch.randn(2 * I, device="cuda", generator=g)
    wp, bp = ops_a.geglu_pack(w, bias)
    out = ops_a.gemm(a, wp, bias=bp, act=ops_a.ACT_GEGLU)
    y = a.double() @ w.double().t() + bias.double()
    want = y[:, :I] * torch.nn.functional.gelu(y[:, I:])
    assert out.shape == (M, I)
    err = (out.double() - want).abs() - 2e-3 * want.abs()
    assert err.max().item() <= 4e-3 * K ** 0.5 + 2e-2


@pytest.mark.parametrize("bn", BNS)
@pytest.mark.parametrize("B,H,W,C,N", [(16, 32, 32, 64, 96), (3, 4, 4, 32, 40), (1, 4, 256, 64, 64)])
def test_upsampling_conv_phase_scatter(persistent_bn, bn, B, H, W, C, N):
    """Nearest 2x + 3x3 conv as four phase convolutions, each written through the 5-D output map: many tiles per CTA,
    half tiles of several image rows (W < 64), of part of a row (W = 256), and an M tail inside the first warpgroup."""
    from o2345 import ops_a
    from o2345.unet import _Packed
    persistent_bn.o2345_debug_gemm_force(2, bn, 1)
    g = torch.Generator(device="cuda").manual_seed(B * 31 + H + W + C + bn)
    conv = torch.nn.Conv2d(C, N, 3, padding=1).cuda()
    with torch.no_grad():
        conv.weight.copy_(torch.randn(N, C, 3, 3, device="cuda", generator=g) * (2.0 / (9 * C)) ** 0.5)
        conv.bias.copy_(torch.randn(N, device="cuda", generator=g))
    conv = conv.half()
    x = _rand((B, H, W, C), g, 0.5)
    w4, b4 = _Packed(conv).conv_up(conv)
    out = ops_a.conv_up2x(x.view(-1, C), B, H, W, C, w4, bias=b4, act=1)
    up = torch.nn.functional.interpolate(x.permute(0, 3, 1, 2).double(), scale_factor=2.0, mode="nearest")
    y = torch.nn.functional.conv2d(up, conv.weight.double(), conv.bias.double(), padding=1).permute(0, 2, 3, 1).reshape(-1, N)
    want = torch.nn.functional.silu(y)
    assert out.shape == want.shape
    err = (out.double() - want).abs()
    assert err.max().item() < 2e-2 and err.mean().item() < 1.5e-3, (err.max().item(), err.mean().item())


@pytest.mark.parametrize("bn", BNS)
def test_conv_residual_rowbias(persistent_bn, bn):
    """The ResBlock conv epilogue: bias + per-image embedding (a 128-row tile spans two images of 64 pixels) + skip."""
    from o2345 import ops_a
    B, H, W, C, N = 40, 8, 8, 64, 200
    persistent_bn.o2345_debug_gemm_force(2, bn, 1)
    g = torch.Generator(device="cuda").manual_seed(bn)
    x = _rand((B, H, W, C), g, 0.5)
    w = (torch.randn(N, C, 3, 3, device="cuda", generator=g) * (2.0 / (9 * C)) ** 0.5).half()
    bias = torch.randn(N, device="cuda", generator=g)
    emb = _rand((B, N), g)
    res = _rand((B * H * W, N), g)
    wk = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()
    out = ops_a.conv3x3(x.view(-1, C), B, H, W, C, wk, bias=bias, rowbias=emb, residual=res)
    y = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), bias.double(), padding=1)
    y = y.permute(0, 2, 3, 1).reshape(-1, N) + emb.double().repeat_interleave(H * W, 0)
    want = y.half().double() + res.double()
    assert (out.double() - want).abs().max().item() < 2e-2
