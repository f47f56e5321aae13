"""AutoencoderKL (VAE) encode / decode on the o2345 tensor-core path (SURVEY.md rows A6, A7).

Mirror of reference ldm/models/autoencoder.py:285-333 and ldm/modules/diffusionmodules/model.py:33-202,368-568
for the first_stage_config of configs/sd-objaverse-finetune-c_concat-256.yaml:45-66 (ch 128, ch_mult 1-2-4-4,
two ResnetBlocks per level, attention only in the middle, z_channels 4, double_z).  The module tree reproduces the
reference state-dict keys (`encoder.down.0.block.0.norm1.weight`, `decoder.up.3.upsample.conv.weight`, ...).
`encode(x)` returns a DiagonalGaussianDistribution-like object (`.mode()`, `.mean`), `decode(z)` an image batch.
Same primitives as the UNet: GroupNorm(eps 1e-6)+swish fused into the conv patch gather, wgmma GEMMs, and a
single-head 512-channel attention in the middle block.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ._lib import inference_only
from . import ops_a as A
from .unet import _Packed

_f16, _f32 = torch.float16, torch.float32


def Normalize(c):
    return nn.GroupNorm(32, c, eps=1e-6, affine=True)


class ResnetBlock(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.in_channels, self.out_channels = cin, cout
        self.norm1, self.conv1 = Normalize(cin), nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2, self.conv2 = Normalize(cout), nn.Conv2d(cout, cout, 3, padding=1)
        if cin != cout:
            self.nin_shortcut = nn.Conv2d(cin, cout, 1)


class AttnBlock(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.in_channels = c
        self.norm = Normalize(c)
        self.q, self.k, self.v, self.proj_out = (nn.Conv2d(c, c, 1) for _ in range(4))


class _Resample(nn.Module):
    def __init__(self, c, stride):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=stride, padding=1 if stride == 1 else 0)


class _Level(nn.Module):
    pass


class Decoder(nn.Module):
    def __init__(self, ch=128, out_ch=3, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=4, **unused):
        super().__init__()
        self.num_resolutions, self.num_res_blocks = len(ch_mult), num_res_blocks
        bi = ch * ch_mult[-1]
        self.conv_in = nn.Conv2d(z_channels, bi, 3, padding=1)
        self.mid = _Level()
        self.mid.block_1, self.mid.attn_1, self.mid.block_2 = ResnetBlock(bi, bi), AttnBlock(bi), ResnetBlock(bi, bi)
        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            up = _Level()
            up.block, up.attn = nn.ModuleList(), nn.ModuleList()
            bo = ch * ch_mult[i_level]
            for _ in range(num_res_blocks + 1):
                up.block.append(ResnetBlock(bi, bo))
                bi = bo
            if i_level != 0:
                up.upsample = _Resample(bi, 1)
            self.up.insert(0, up)
        self.norm_out, self.conv_out = Normalize(bi), nn.Conv2d(bi, out_ch, 3, padding=1)


class Encoder(nn.Module):
    def __init__(self, ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, in_channels=3, z_channels=4, double_z=True, **unused):
        super().__init__()
        self.num_resolutions, self.num_res_blocks = len(ch_mult), num_res_blocks
        self.conv_in = nn.Conv2d(in_channels, ch, 3, padding=1)
        in_mult = (1,) + tuple(ch_mult)
        self.down = nn.ModuleList()
        for i_level in range(self.num_resolutions):
            d = _Level()
            d.block, d.attn = nn.ModuleList(), nn.ModuleList()
            bi, bo = ch * in_mult[i_level], ch * ch_mult[i_level]
            for _ in range(num_res_blocks):
                d.block.append(ResnetBlock(bi, bo))
                bi = bo
            if i_level != self.num_resolutions - 1:
                d.downsample = _Resample(bi, 2)
            self.down.append(d)
        self.mid = _Level()
        self.mid.block_1, self.mid.attn_1, self.mid.block_2 = ResnetBlock(bi, bi), AttnBlock(bi), ResnetBlock(bi, bi)
        self.norm_out = Normalize(bi)
        self.conv_out = nn.Conv2d(bi, 2 * z_channels if double_z else z_channels, 3, padding=1)


class Posterior:
    """DiagonalGaussianDistribution surface used at inference (reference distributions.py:24-61)."""

    def __init__(self, moments):
        self.mean, self.logvar = torch.chunk(moments, 2, dim=1)

    def mode(self):
        return self.mean


class AutoencoderKL(nn.Module):
    def __init__(self, ddconfig=None, lossconfig=None, embed_dim=4, **unused):
        super().__init__()
        dd = dict(ch=128, out_ch=3, ch_mult=(1, 2, 4, 4), num_res_blocks=2, in_channels=3, z_channels=4, double_z=True)
        dd.update(ddconfig or {})
        dd = {k: v for k, v in dd.items() if k in ("ch", "out_ch", "ch_mult", "num_res_blocks", "in_channels", "z_channels", "double_z")}
        self.encoder = Encoder(**{k: v for k, v in dd.items() if k != "out_ch"})
        self.decoder = Decoder(**{k: v for k, v in dd.items() if k not in ("in_channels", "double_z")})
        self.quant_conv = nn.Conv2d(2 * dd["z_channels"], 2 * embed_dim, 1)
        self.post_quant_conv = nn.Conv2d(embed_dim, dd["z_channels"], 1)
        self.embed_dim = embed_dim
        self._packed = None

    # ------------------------------------------------------------------ executor
    def _pk(self):
        key = tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._packed is None or self._packed.key != key:
            self._packed = _Packed(self)
        return self._packed

    @staticmethod
    def _conv(pk, x, B, H, W, C, conv, gn=None, stride=1, up=False, residual=None, pad_lo=-1, ksize=3):
        g = None if gn is None else A.groupnorm_stats(x, B, H * W, C, 32, gn.eps, *pk.norm(gn))
        w, b = pk.conv(conv)
        if ksize == 3 and stride == 1 and not up and pad_lo < 0 and A.conv3x3_supported(H, W, C):
            a = x if g is None else A.norm_act_im2col(x, B, H, W, C, 1, 1, False, g, True)[0]
            return A.conv3x3(a, B, H, W, C, w, bias=b, residual=residual), H, W
        if A.USE_CONV_UP2X and ksize == 3 and stride == 1 and up and g is None and residual is None and pad_lo < 0 and A.conv3x3_supported(H, W, C):
            w4, b4 = pk.conv_up(conv)       # nearest 2x + 3x3 conv as four 2x2 convs of the low-resolution map
            return A.conv_up2x(x, B, H, W, C, w4, bias=b4), 2 * H, 2 * W
        a, Ho, Wo = A.norm_act_im2col(x, B, H, W, C, ksize, stride, up, g, gn is not None and ksize == 3, pad_lo=pad_lo)
        return A.gemm(a, w, bias=b, residual=residual), Ho, Wo

    def _res(self, pk, blk, x, B, H, W):
        ci, co = blk.in_channels, blk.out_channels
        h, _, _ = self._conv(pk, x, B, H, W, ci, blk.conv1, gn=blk.norm1)
        skip = x
        if ci != co:
            ws, bs = pk.conv(blk.nin_shortcut)
            skip = A.gemm(x, ws, bias=bs)
        out, _, _ = self._conv(pk, h, B, H, W, co, blk.conv2, gn=blk.norm2, residual=skip)
        return out, co

    def _attn(self, pk, at, x, B, H, W):
        C, N = at.in_channels, H * W
        g = A.groupnorm_stats(x, B, N, C, 32, at.norm.eps, *pk.norm(at.norm))
        xn, _, _ = A.norm_act_im2col(x, B, H, W, C, 1, 1, False, g, False)
        q = A.gemm(xn, *pk.conv(at.q)[:1], bias=pk.conv(at.q)[1])
        k = A.gemm(xn, *pk.conv(at.k)[:1], bias=pk.conv(at.k)[1])
        v = A.gemm(xn, *pk.conv(at.v)[:1], bias=pk.conv(at.v)[1])
        s = torch.empty(B, N, N, dtype=_f16, device=x.device)
        A.bgemm(q, k, s, 1, B, (0, N * C), (0, N * C), (0, N * N), N, N, C, C, C, N, alpha=int(C) ** -0.5)
        p = A.softmax_rows(s)
        vt = A.transpose_tokens(v, B, N, C)
        o = torch.empty(B * N, C, dtype=_f16, device=x.device)
        A.bgemm(p, vt, o, 1, B, (0, N * N), (0, C * N), (0, N * C), N, C, N, N, N, C)
        wo, bo = pk.conv(at.proj_out)
        return A.gemm(o, wo, bias=bo, residual=x)

    @inference_only
    def decode(self, z):
        """z [B,4,h,w] -> image [B,3,8h,8w] fp32 (reference autoencoder.py:330-333, model.py:535-568)."""
        pk = self._pk()
        B, Cz, H, W = z.shape
        zc = A.nchw_to_cl(z, torch.zeros(B * H * W, 8, dtype=_f16, device=z.device))
        # post_quant_conv is a 1x1 conv on 4 channels: fold it as a GEMM with K padded to 8
        wq, bq = pk.conv(self.post_quant_conv)
        h8 = torch.zeros(B * H * W, 8, dtype=_f16, device=z.device)
        A.gemm(zc, wq, bias=bq, out=h8[:, :Cz])
        d = self.decoder
        h, _, _ = self._conv(pk, h8, B, H, W, 8, d.conv_in)
        C = d.conv_in.out_channels
        h, C = self._res(pk, d.mid.block_1, h, B, H, W)
        h = self._attn(pk, d.mid.attn_1, h, B, H, W)
        h, C = self._res(pk, d.mid.block_2, h, B, H, W)
        for i_level in reversed(range(d.num_resolutions)):
            for blk in d.up[i_level].block:
                h, C = self._res(pk, blk, h, B, H, W)
            if i_level != 0:
                h, H, W = self._conv(pk, h, B, H, W, C, d.up[i_level].upsample.conv, up=True)
        out, _, _ = self._conv(pk, h, B, H, W, C, d.conv_out, gn=d.norm_out)
        return A.cl_to_nchw(out, B, d.conv_out.out_channels, H, W)

    @inference_only
    def encode(self, x):
        """x [B,3,H,W] in [-1,1] -> Posterior over z [B,4,H/8,W/8] (reference autoencoder.py:324-328, model.py:434-459)."""
        pk = self._pk()
        B, Ci, H, W = x.shape
        e = self.encoder
        h = A.nchw_to_cl(x, torch.zeros(B * H * W, 8, dtype=_f16, device=x.device))
        h, _, _ = self._conv(pk, h, B, H, W, 8, e.conv_in)
        C = e.conv_in.out_channels
        for i_level in range(e.num_resolutions):
            for blk in e.down[i_level].block:
                h, C = self._res(pk, blk, h, B, H, W)
            if i_level != e.num_resolutions - 1:
                h, H, W = self._conv(pk, h, B, H, W, C, e.down[i_level].downsample.conv, stride=2, pad_lo=0)
        h, C = self._res(pk, e.mid.block_1, h, B, H, W)
        h = self._attn(pk, e.mid.attn_1, h, B, H, W)
        h, C = self._res(pk, e.mid.block_2, h, B, H, W)
        m, _, _ = self._conv(pk, h, B, H, W, C, e.conv_out, gn=e.norm_out)          # [M, 8]
        wq, bq = pk.conv(self.quant_conv)
        moments = A.gemm(m, wq, bias=bq)
        return Posterior(A.cl_to_nchw(moments, B, moments.shape[1], H, W))
