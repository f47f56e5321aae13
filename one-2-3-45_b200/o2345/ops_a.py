"""Path A (Zero123 DDIM / UNet / VAE / CLIP) tensor-level wrappers over the C-ABI: fp16 activations, fp32 norms.

The split-K workspace and the GroupNorm scratch are one buffer per device, handed to the C-ABI by these wrappers (the
entry points themselves own no memory): calls that may use them must be issued on ONE stream per device at a time, which
is how the UNet / VAE / CLIP executors run.  Callers that want concurrent streams pass their own workspaces to
o2345_gemm_f16 / o2345_groupnorm_stats."""
from __future__ import annotations

import ctypes as C
import ctypes as C_

import torch

from . import _lib as L
from .ops import _p, _stream

_f16, _f32 = torch.float16, torch.float32


def _v(t):
    """Raw device pointer of a tensor for the C-ABI (None stays NULL).  No CPU path and no cross-device launches: the library
    runs on the current device's current stream."""
    if t is None:
        return None
    if not t.is_cuda or t.device.index != torch.cuda.current_device():
        raise L.O2345Error(f"expected a tensor on the current CUDA device, got one on {t.device}")
    return C.c_void_p(t.data_ptr())


_WS = {}
WS_FLOATS = 8 << 20   # 32 MB of split-K partial planes (e.g. 4 planes of 2048 x 1024)


def _splitk_ws(dev):
    """fp32 workspace for the split-K partial planes (needs no initialisation)."""
    k = str(dev)
    if k not in _WS:
        _WS[k] = torch.empty(WS_FLOATS, dtype=_f32, device=dev)
    return _WS[k]


def _epilogue(bias=None, residual=None, rowbias=None, rows_per_group=1, act=0, alpha=1.0, out_f32=False):
    """o2345_epilogue; the tensors must stay alive until the call returns (they are arguments of the caller)."""
    if rowbias is not None:
        assert rowbias.dtype == _f16 and rowbias.stride(-1) == 1
    return L.Epilogue(bias=_p(bias, _f32), residual=None if residual is None else residual.data_ptr(),
                      rowbias=None if rowbias is None else rowbias.data_ptr(),
                      rowbias_ld=0 if rowbias is None else rowbias.stride(0), rows_per_group=int(rows_per_group),
                      act=int(act), alpha=float(alpha), out_f32=int(out_f32))


ACT_NONE, ACT_SILU, ACT_GELU, ACT_GEGLU, ACT_QUICKGELU = 0, 1, 2, 3, 4


def gemm(a, b, bias=None, residual=None, act=0, alpha=1.0, out_dtype=_f16, out=None, rowbias=None, rows_per_group=1):
    """out[M,N] = act(alpha * a[M,K] @ b[N,K]^T + bias + rowbias[row // rows_per_group]) + residual.  a, b fp16 with
    contiguous K; rows may be strided.  act = ACT_GEGLU: b's rows are interleaved 16 values / 16 gates (geglu_pack) and
    out has N/2 columns."""
    assert a.dtype == _f16 and b.dtype == _f16 and a.stride(-1) == 1 and b.stride(-1) == 1
    M, K = a.shape
    N = b.shape[0]
    assert b.shape[1] == K, (a.shape, b.shape)
    if out is None:
        out = torch.empty(M, N // 2 if act == ACT_GEGLU else N, dtype=out_dtype, device=a.device)
    assert out.stride(-1) == 1
    if residual is not None:
        assert residual.dtype == _f16 and residual.stride(0) == out.stride(0) and residual.stride(-1) == 1
    ep = _epilogue(bias, residual, rowbias, rows_per_group, act, alpha, out.dtype == _f32)
    L.call("o2345_gemm_f16", _v(a), _v(b), _v(out), M, N, K, a.stride(0), b.stride(0), out.stride(0), 0, 0, 0, 0, 0, 0, 0, 0,
           C.byref(ep), _v(_splitk_ws(a.device)), WS_FLOATS, _stream())
    return out


def geglu_pack(w, bias):
    """Reorders the rows of a GEGLU projection ([2I, K]: I values then I gates) into chunks of 16 values + their 16 gates,
    the column order the ACT_GEGLU epilogue expects."""
    I = w.shape[0] // 2
    assert I % 16 == 0
    idx = torch.arange(I, device=w.device).reshape(-1, 16)
    perm = torch.cat([idx, idx + I], 1).reshape(-1)
    return w[perm].contiguous(), None if bias is None else bias[perm].contiguous()


def bgemm(a, b, out, nh, nb, sa, sb, sc, M, N, K, lda, ldb, ldc, alpha=1.0):
    """nh*nb products; sa/sb/sc = (stride_h, stride_b) element offsets of the operand for batch z = b*nh + h."""
    ep = _epilogue(alpha=alpha, out_f32=out.dtype == _f32)
    L.call("o2345_gemm_f16", _v(a), _v(b), _v(out), M, N, K, lda, ldb, ldc, nh, nb, sa[0], sa[1], sb[0], sb[1], sc[0], sc[1],
           C.byref(ep), None, 0, _stream())
    return out


_GN_SCRATCH = {}


def groupnorm_stats(x, B, HW, C, G=32, eps=1e-5, gamma=None, beta=None):
    """GroupNorm as a per-(image, channel) affine: returns (scale, shift) fp32 [B, C] with GN(x) = x * scale + shift."""
    k = (str(x.device), B, G)
    if k not in _GN_SCRATCH:
        _GN_SCRATCH[k] = torch.zeros(int(L.load().o2345_groupnorm_scratch_floats(B, G)), dtype=_f32, device=x.device)
    scale = torch.empty(B, C, dtype=_f32, device=x.device)
    shift = torch.empty_like(scale)
    L.call("o2345_groupnorm_stats", _v(x), B, HW, C, G, float(eps), _p(gamma, _f32), _p(beta, _f32), _v(_GN_SCRATCH[k]),
           _v(scale), _v(shift), _stream())
    return scale, shift


def groupnorm_apply_pays(B, HW, C):
    """The one-kernel GroupNorm spreads an image over at most 16 CTAs: it wins while a CTA's slab stays small (the UNet's
    activations: <= 123 KB); the VAE's 128-channel 256 x 256 maps keep the many-CTA statistics kernel + apply."""
    return HW * C * 2 <= 16 * 131072


def groupnorm_apply(x, B, HW, C, G, eps, gamma, beta, act):
    """GroupNorm (+SiLU) of x [B*HW, C] in one cluster kernel (statistics exchanged through distributed shared memory)."""
    out = torch.empty(B * HW, C, dtype=_f16, device=x.device)
    L.call("o2345_groupnorm_apply", _v(x), B, HW, C, int(G), float(eps), _p(gamma, _f32), _p(beta, _f32), int(act), _v(out), _stream())
    return out


def norm_act_im2col(x, B, H, W, C, ksize=3, stride=1, upsample=False, gn=None, act=False, pad_lo=-1):
    """gn = (scale, shift) from groupnorm_stats or None.  Returns ([B*Ho*Wo, k*k*C] fp16, Ho, Wo)."""
    Hin, Win = (2 * H, 2 * W) if upsample else (H, W)
    pad_hi = ksize // 2
    pad = pad_hi if pad_lo < 0 else pad_lo
    Ho, Wo = (Hin + pad + pad_hi - ksize) // stride + 1, (Win + pad + pad_hi - ksize) // stride + 1
    out = torch.empty(B * Ho * Wo, ksize * ksize * C, dtype=_f16, device=x.device)
    scale, shift = gn if gn is not None else (None, None)
    L.call("o2345_norm_act_im2col", _v(x), B, H, W, C, ksize, stride, int(upsample), int(pad_lo), _v(scale), _v(shift),
           int(act), _v(out), _stream())
    return out, Ho, Wo


def layernorm(x, gamma, beta, eps=1e-5):
    M, Cc = x.shape
    y = torch.empty_like(x)
    L.call("o2345_layernorm_rows", _v(x), M, Cc, float(eps), _v(gamma), _v(beta), _v(y), _stream())
    return y


def softmax_rows(s):
    rows, n = s.numel() // s.shape[-1], s.shape[-1]
    p = torch.empty_like(s)
    L.call("o2345_softmax_rows", _v(s), rows, n, _v(p), _stream())
    return p


def geglu(x):
    M, I2 = x.shape
    y = torch.empty(M, I2 // 2, dtype=_f16, device=x.device)
    L.call("o2345_geglu", _v(x), M, I2 // 2, _v(y), _stream())
    return y


def transpose_tokens(x, B, N, Cc):
    y = torch.empty(B, Cc, N, dtype=_f16, device=x.device)
    L.call("o2345_transpose_tokens", _v(x), B, N, Cc, _v(y), _stream())
    return y


def timestep_embedding(t, dim):
    t = t.to(_f32).contiguous()
    out = torch.empty(t.shape[0], dim, dtype=_f16, device=t.device)
    L.call("o2345_timestep_embedding", _v(t), t.shape[0], dim, _v(out), _stream())
    return out


def add_channel_bias(y, e, B, HW, Cc):
    """y[b, p, c] += e[b, c]; e may be a column slice of a wider [B, ld] matrix."""
    L.call("o2345_add_channel_bias", _v(y), _v(e), B, HW, Cc, e.stride(0), _stream())
    return y


def copy_channels(src, dst, off):
    M, Cc = src.shape
    L.call("o2345_copy_channels", _v(src), M, Cc, _v(dst), dst.stride(0), off, _stream())


def nchw_to_cl(x, out=None, off=0):
    B, Cc, H, W = x.shape
    x = x.to(_f32).contiguous()
    if out is None:
        out = torch.zeros(B * H * W, Cc, dtype=_f16, device=x.device)
    L.call("o2345_nchw_f32_to_cl_f16", _v(x), B, Cc, H * W, _v(out), out.stride(0), off, _stream())
    return out


def cl_to_nchw(x, B, Cc, H, W):
    y = torch.empty(B, Cc, H, W, dtype=_f32, device=x.device)
    L.call("o2345_cl_f16_to_nchw_f32", _v(x), B, Cc, H * W, x.stride(0), _v(y), _stream())
    return y


def cfg_ddim_update(x, eps2, noise, scale, a_t, a_prev, sigma_t, sqrt_one_minus_at, want_x0=True):
    n = x.numel()
    x_prev = torch.empty_like(x)
    pred = torch.empty_like(x) if want_x0 else None
    L.call("o2345_cfg_ddim_update", _v(x), _v(eps2), _v(noise), n, float(scale), float(a_t), float(a_prev), float(sigma_t),
           float(sqrt_one_minus_at), _v(x_prev), _v(pred), _stream())
    return x_prev, pred


def silu(x):
    y = torch.empty_like(x)
    L.call("o2345_silu", _v(x), x.numel(), _v(y), _stream())
    return y


def attention(q, k, v, B, N, H, d, out=None):
    """softmax(q k^T / sqrt(d)) v per (batch, head); q/k/v are [B*N, >=H*d] views sharing one row stride."""
    assert q.stride(0) == k.stride(0) == v.stride(0) and q.stride(1) == 1
    if out is None:
        out = torch.empty(B * N, H * d, dtype=_f16, device=q.device)
    L.call("o2345_attention_f16", _v(q), _v(k), _v(v), B, N, H, d, q.stride(0), _v(out), out.stride(0), float(d) ** -0.5, _stream())
    return out


USE_CONV_UP2X = True   # tools/unet_ab.py switches the four-phase up-sampling convolution off to measure the gather route


def conv_up2x(x, B, H, W, C, weight4, bias=None, act=0):
    """Nearest-neighbour 2x up-sampling followed by a 3x3 convolution (pad 1) of the channel-last x [B*H*W, C], as four 2x2
    convolutions of the LOW-resolution map (weight4 [4, N, 4*C] from _Packed.conv_up).  -> [B*2H*2W, N] fp16."""
    N = weight4.shape[1]
    assert weight4.shape == (4, N, 4 * C) and weight4.dtype == _f16 and weight4.is_contiguous()
    out = torch.empty(B * 4 * H * W, N, dtype=_f16, device=x.device)
    ep = _epilogue(bias, None, None, 1, act, 1.0, False)
    L.call("o2345_conv_up2x_f16", _v(x), B, H, W, C, _v(weight4), N, _v(out), N, C_.byref(ep), _v(_splitk_ws(x.device)), WS_FLOATS, _stream())
    return out


def conv3x3(x, B, H, W, C, weight, bias=None, residual=None, act=0, out_dtype=_f16, rowbias=None):
    """Implicit-GEMM 3x3 convolution (stride 1, pad 1) of a channel-last activation x [B*H*W, C]; weight [N, 9*C] in
    (ky, kx, c) order.  No im2col buffer: TMA fetches the nine shifted windows, zero-filling outside the image.
    rowbias [B, >=N] fp16: per-image channel bias (the ResBlock's timestep embedding)."""
    N = weight.shape[0]
    out = torch.empty(B * H * W, N, dtype=out_dtype, device=x.device)
    ep = _epilogue(bias, residual, rowbias, H * W, act, 1.0, out_dtype == _f32)
    L.call("o2345_conv3x3_f16", _v(x), B, H, W, C, _v(weight), N, _v(out), out.stride(0), C_.byref(ep),
           _v(_splitk_ws(x.device)), WS_FLOATS, _stream())
    return out


def conv3x3_supported(H, W, C):
    """Shapes the implicit 3x3 conv takes (the same rule o2345_conv3x3_f16 enforces): a 128-pixel output tile must be one
    TMA box of whole row segments / whole rows / whole images.  Everything else goes through norm_act_im2col + gemm."""
    if C % 8 or C < 64:
        return False
    if W % 128 == 0:
        return True
    if 128 % W:
        return False
    return (H % (128 // W) == 0) if H * W >= 128 else (128 % (H * W) == 0)


def clip_patches(x, res, patch, mean, std, kp):
    """[-1,1] images [B,3,H,W] -> fp16 [B*(res/patch)^2, kp]: bicubic resize + CLIP normalisation + patch gather."""
    B, _, H, W = x.shape
    x = x.to(_f32).contiguous()
    g = res // patch
    out = torch.empty(B * g * g, kp, dtype=_f16, device=x.device)
    m3 = (C.c_float * 3)(*[float(v) for v in mean])       # host constants (no device read-back)
    s3 = (C.c_float * 3)(*[float(v) for v in std])
    L.call("o2345_clip_patches", _v(x), B, H, W, int(res), int(patch), m3, s3, int(kp), _v(out), _stream())
    return out


def clip_add_positions(tok, cls, pos, B, N, d):
    L.call("o2345_clip_add_positions", _v(tok), _p(cls, _f32), _p(pos, _f32), B, N, d, _stream())
    return tok
