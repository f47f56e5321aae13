"""Zero123 UNetModel on the o2345 tensor-core path (SURVEY.md rows A2-A5).

Mirror of reference ldm/modules/diffusionmodules/openaimodel.py:414-777 for the configuration that
configs/sd-objaverse-finetune-c_concat-256.yaml:28-43 instantiates (spatial transformers, depth 1,
legacy=False): the module tree below reproduces the reference's state-dict keys
(`input_blocks.{i}.{j}.in_layers.0.weight`, `...transformer_blocks.0.attn1.to_q.weight`, ...), so a
`model.diffusion_model.*` checkpoint loads directly; `forward(x, timesteps, context)` has the reference
signature and returns the epsilon prediction [N,4,H,W] in fp32 (values rounded through fp16 exactly where
autocast would round them).

Execution: activations are channel-last fp16 [N*H*W, C].  Every Linear / 1x1 conv is one wgmma GEMM and every
3x3 stride-1 conv an implicit GEMM whose nine shifted windows are fetched by TMA (csrc/gemm_tc.cu: 128 x BN wgmma
tiles, operand tiles multicast over a 2 x 2 CTA cluster, split-K for small grids); the strided / up-sampling convs
gather patches first (csrc/unet_ops.cu).  GroupNorm (+SiLU) is one cluster kernel, or statistics kernel + apply for the
large maps; the ResBlock's `h + emb`, the attention / feed-forward residuals, the GEGLU gate and the single-token
cross-attention term ride in GEMM epilogues.  Self-attention is the fused mma.sync kernel (csrc/attention.cu; scores
never leave the SM); the batched-GEMM -> softmax -> batched-GEMM route remains for other head sizes.
Cross-attention: Zero123 conditions on ONE token, so softmax over a single key is exactly 1 and
attn2(x) = to_out(to_v(context)) broadcast over the image (SURVEY.md row A4) -- computed as two [N,C] GEMMs once per
sampling call; contexts with more than one token use the general path.  One forward is ~660 launches captured in a CUDA
graph per input shape.
`use_checkpoint` is accepted and ignored (inference).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ._lib import inference_only
from . import ops_a as A

_f16, _f32 = torch.float16, torch.float32


# ----------------------------------------------------------------------------- parameter holders
def _gn(c, eps=1e-5):
    return nn.GroupNorm(32, c, eps=eps)


class ResBlock(nn.Module):
    def __init__(self, ch, emb_ch, out_ch):
        super().__init__()
        self.channels, self.out_channels = ch, out_ch
        self.in_layers = nn.Sequential(_gn(ch), nn.SiLU(), nn.Conv2d(ch, out_ch, 3, padding=1))
        self.emb_layers = nn.Sequential(nn.SiLU(), nn.Linear(emb_ch, out_ch))
        self.out_layers = nn.Sequential(_gn(out_ch), nn.SiLU(), nn.Dropout(0.0), nn.Conv2d(out_ch, out_ch, 3, padding=1))
        self.skip_connection = nn.Identity() if ch == out_ch else nn.Conv2d(ch, out_ch, 1)


class CrossAttention(nn.Module):
    def __init__(self, query_dim, context_dim, heads, dim_head):
        super().__init__()
        inner = heads * dim_head
        self.heads, self.dim_head = heads, dim_head
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(context_dim or query_dim, inner, bias=False)
        self.to_v = nn.Linear(context_dim or query_dim, inner, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner, query_dim), nn.Dropout(0.0))


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.net = nn.Sequential(GEGLU(dim, dim * 4), nn.Dropout(0.0), nn.Linear(dim * 4, dim))


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, heads, dim_head, context_dim):
        super().__init__()
        self.attn1 = CrossAttention(dim, None, heads, dim_head)
        self.ff = FeedForward(dim)
        self.attn2 = CrossAttention(dim, context_dim, heads, dim_head)
        self.norm1, self.norm2, self.norm3 = nn.LayerNorm(dim), nn.LayerNorm(dim), nn.LayerNorm(dim)


class SpatialTransformer(nn.Module):
    def __init__(self, ch, heads, dim_head, context_dim):
        super().__init__()
        inner = heads * dim_head
        self.norm = _gn(ch, eps=1e-6)
        self.proj_in = nn.Conv2d(ch, inner, 1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(inner, heads, dim_head, context_dim)])
        self.proj_out = nn.Conv2d(inner, ch, 1)


class Downsample(nn.Module):
    def __init__(self, ch):
        super().__init__()
        self.op = nn.Conv2d(ch, ch, 3, stride=2, padding=1)


class Upsample(nn.Module):
    def __init__(self, ch):
        super().__init__()
        self.conv = nn.Conv2d(ch, ch, 3, padding=1)


# ----------------------------------------------------------------------------- packed fp16 weights
class _Packed:
    """fp16 GEMM operands derived from the fp32 parameters (rebuilt when a parameter changes)."""

    def __init__(self, model):
        self.key = tuple((p.data_ptr(), p._version) for p in model.parameters())
        self.w = {}

    def conv(self, m):
        k = id(m)
        if k not in self.w:
            w = m.weight.detach()
            co, ci, kh, kw = w.shape
            if ci % 8:  # pad the input channels to a multiple of 8 (TMA needs 16-byte rows)
                w = torch.cat([w, w.new_zeros(co, 8 - ci % 8, kh, kw)], 1)
            self.w[k] = (w.permute(0, 2, 3, 1).reshape(co, -1).to(_f16).contiguous(),
                         None if m.bias is None else m.bias.detach().to(_f32).contiguous())
        return self.w[k]

    def conv_up(self, m):
        """Weights of `nearest 2x up-sampling -> 3x3 conv` as FOUR 2x2 convolutions of the low-resolution input, one per output
        phase (row parity a, column parity b): the three kernel rows collapse onto two input rows -- a = 0: (row y-1: k0,
        row y: k1 + k2), a = 1: (row y: k0 + k1, row y+1: k2) -- and the same along x.  Summed in fp32, rounded to fp16
        once.  -> ([4, Cout, 4 * Cin] fp16 in (phase, out, (ty, tx, cin)) order, bias fp32)."""
        k = ("up", id(m))
        if k not in self.w:
            w = m.weight.detach().float()                                     # [co, ci, 3, 3]
            co, ci = w.shape[:2]
            assert ci % 8 == 0 and w.shape[2:] == (3, 3)
            rows = {0: (w[:, :, 0], w[:, :, 1] + w[:, :, 2]), 1: (w[:, :, 0] + w[:, :, 1], w[:, :, 2])}   # [co, ci, 3 (kx)] each
            phases = []
            for a in (0, 1):
                for b in (0, 1):
                    taps = []
                    for ty in (0, 1):
                        r = rows[a][ty]
                        cols = (r[:, :, 0], r[:, :, 1] + r[:, :, 2]) if b == 0 else (r[:, :, 0] + r[:, :, 1], r[:, :, 2])
                        taps += [cols[0], cols[1]]                            # (ty, tx) order, each [co, ci]
                    phases.append(torch.stack(taps, 1).reshape(co, 4 * ci))
            self.w[k] = (torch.stack(phases).to(_f16).contiguous(), None if m.bias is None else m.bias.detach().to(_f32).contiguous())
        return self.w[k]

    def linear(self, m):
        k = id(m)
        if k not in self.w:
            self.w[k] = (m.weight.detach().to(_f16).contiguous(),
                         None if m.bias is None else m.bias.detach().to(_f32).contiguous())
        return self.w[k]

    def geglu(self, m):
        k = ("geglu", id(m))
        if k not in self.w:
            self.w[k] = A.geglu_pack(*self.linear(m))
        return self.w[k]

    def qkv(self, attn):
        k = ("qkv", id(attn))
        if k not in self.w:
            self.w[k] = torch.cat([attn.to_q.weight, attn.to_k.weight, attn.to_v.weight], 0).detach().to(_f16).contiguous()
        return self.w[k]

    def norm(self, m):
        k = id(m)
        if k not in self.w:
            self.w[k] = (m.weight.detach().to(_f32).contiguous(), m.bias.detach().to(_f32).contiguous())
        return self.w[k]


class UNetModel(nn.Module):
    def __init__(self, image_size=32, in_channels=8, out_channels=4, model_channels=320, attention_resolutions=(4, 2, 1),
                 num_res_blocks=2, channel_mult=(1, 2, 4, 4), num_heads=8, use_spatial_transformer=True,
                 transformer_depth=1, context_dim=768, use_checkpoint=True, legacy=False, **unused):
        super().__init__()
        if not use_spatial_transformer or transformer_depth != 1 or legacy:
            raise NotImplementedError("only the Zero123 configuration (spatial transformers, depth 1, legacy=False) is built")
        self.in_channels, self.out_channels, self.model_channels = in_channels, out_channels, model_channels
        self.num_heads, self.context_dim = num_heads, context_dim
        mc, ted = model_channels, model_channels * 4
        self.time_embed = nn.Sequential(nn.Linear(mc, ted), nn.SiLU(), nn.Linear(ted, ted))
        self.input_blocks = nn.ModuleList([nn.Sequential(nn.Conv2d(in_channels, mc, 3, padding=1))])
        chans, ch, ds = [mc], mc, 1
        st = lambda c: SpatialTransformer(c, num_heads, c // num_heads, context_dim)
        for level, mult in enumerate(channel_mult):
            for _ in range(num_res_blocks):
                layers = [ResBlock(ch, ted, mult * mc)]
                ch = mult * mc
                if ds in attention_resolutions:
                    layers.append(st(ch))
                self.input_blocks.append(nn.Sequential(*layers))
                chans.append(ch)
            if level != len(channel_mult) - 1:
                self.input_blocks.append(nn.Sequential(Downsample(ch)))
                chans.append(ch)
                ds *= 2
        self.middle_block = nn.Sequential(ResBlock(ch, ted, ch), st(ch), ResBlock(ch, ted, ch))
        self.output_blocks = nn.ModuleList()
        for level, mult in list(enumerate(channel_mult))[::-1]:
            for i in range(num_res_blocks + 1):
                layers = [ResBlock(ch + chans.pop(), ted, mc * mult)]
                ch = mc * mult
                if ds in attention_resolutions:
                    layers.append(st(ch))
                if level and i == num_res_blocks:
                    layers.append(Upsample(ch))
                    ds //= 2
                self.output_blocks.append(nn.Sequential(*layers))
        self.out = nn.Sequential(_gn(ch), nn.SiLU(), nn.Conv2d(mc, out_channels, 3, padding=1))
        self._packed = None
        self.use_cuda_graph = True
        self._graphs = {}
        self._ctx_ref, self._ctx_ver, self._ctx_pk, self._cross_out = None, None, None, {}
        self.gn_one_kernel = True    # GroupNorm statistics + apply in one cluster kernel (o2345_groupnorm_apply)

    # ------------------------------------------------------------------ executor
    def _pk(self):
        key = tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._packed is None or self._packed.key != key:
            self._packed = _Packed(self)
        return self._packed

    def _norm(self, pk, x, B, H, W, C, gn, act, ksize=1, stride=1, up=False):
        """GroupNorm(x) (+SiLU) as the K-major A operand of the following GEMM: one cluster kernel, or statistics kernel +
        apply / patch gather."""
        if ksize == 1 and stride == 1 and not up and self.gn_one_kernel and A.groupnorm_apply_pays(B, H * W, C):
            return A.groupnorm_apply(x, B, H * W, C, 32, gn.eps, *pk.norm(gn), act), H, W
        g = A.groupnorm_stats(x, B, H * W, C, 32, gn.eps, *pk.norm(gn))
        return A.norm_act_im2col(x, B, H, W, C, ksize, stride, up, g, act)

    def _conv3(self, pk, x, B, H, W, C, conv, gn=None, act=False, stride=1, up=False, residual=None, rowbias=None):
        """3x3 conv (optionally behind GroupNorm + SiLU).  -> (out, Ho, Wo)."""
        w, b = pk.conv(conv)
        Ho, Wo = ((2 * H, 2 * W) if up else ((H + 2 - 3) // stride + 1, (W + 2 - 3) // stride + 1))
        if stride == 1 and not up and A.conv3x3_supported(H, W, C):
            # implicit GEMM: normalise once ([M, C], not 9x) and let TMA fetch the nine shifted windows
            a = x if gn is None else self._norm(pk, x, B, H, W, C, gn, act)[0]
            return A.conv3x3(a, B, H, W, C, w, bias=b, residual=residual, rowbias=rowbias), H, W
        if A.USE_CONV_UP2X and up and stride == 1 and gn is None and residual is None and rowbias is None and A.conv3x3_supported(H, W, C):
            # nearest 2x + 3x3 conv = four 2x2 convs of the low-resolution map (no [M, 9C] gather, 4C instead of 9C per output)
            w4, b4 = pk.conv_up(conv)
            return A.conv_up2x(x, B, H, W, C, w4, bias=b4), Ho, Wo
        if gn is None:
            a, Ho, Wo = A.norm_act_im2col(x, B, H, W, C, 3, stride, up, None, act)
        else:
            a, Ho, Wo = self._norm(pk, x, B, H, W, C, gn, act, 3, stride, up)
        return A.gemm(a, w, bias=b, residual=residual, rowbias=rowbias, rows_per_group=Ho * Wo), Ho, Wo

    def _emb_pack(self, pk):
        """All 22 ResBlock `emb_layers` Linears as ONE [sum Cout, 1280] GEMM per iteration (they share the input)."""
        if "emb_all" not in pk.w:
            blocks = [m for m in self.modules() if isinstance(m, ResBlock)]
            ws, bs, off, o = [], [], {}, 0
            for b in blocks:
                w, bias = pk.linear(b.emb_layers[1])
                ws.append(w), bs.append(bias)
                off[id(b)] = o
                o += w.shape[0]
            pk.w["emb_all"] = (torch.cat(ws, 0).contiguous(), torch.cat(bs, 0).contiguous(), off)
        return pk.w["emb_all"]

    def _resblock(self, pk, blk, x, B, H, W, emb_all):
        C, Co = blk.channels, blk.out_channels
        off = self._emb_pack(pk)[2][id(blk)]
        # h + emb_out[..., None, None] (openaimodel.py:271) rides in the conv epilogue as a per-image channel bias
        h, _, _ = self._conv3(pk, x, B, H, W, C, blk.in_layers[2], gn=blk.in_layers[0], act=True, rowbias=emb_all[:, off:off + Co])
        if isinstance(blk.skip_connection, nn.Identity):
            skip = x
        else:
            ws, bs = pk.conv(blk.skip_connection)
            skip = A.gemm(x, ws, bias=bs)
        out, _, _ = self._conv3(pk, h, B, H, W, Co, blk.out_layers[3], gn=blk.out_layers[0], act=True, residual=skip)
        return out, Co

    def _attention(self, pk, attn, xn, B, N, C, residual, rowbias=None):
        """Self-attention on layer-normed tokens xn [B*N, C]; returns to_out(...) + residual (+ rowbias[image])."""
        H, d = attn.heads, attn.dim_head
        qkv = A.gemm(xn, pk.qkv(attn))                                   # [B*N, 3C]
        if d in (40, 80, 160):                                            # fused kernel: scores never leave the SM
            o = A.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], B, N, H, d)
            wo, bo = pk.linear(attn.to_out[0])
            return A.gemm(o, wo, bias=bo, residual=residual, rowbias=rowbias, rows_per_group=N)
        s = torch.empty(B * H, N, N, dtype=_f16, device=xn.device)
        q, k = qkv[:, :C], qkv[:, C:2 * C]
        A.bgemm(q, k, s, H, B, (d, N * 3 * C), (d, N * 3 * C), (N * N, H * N * N), N, N, d, 3 * C, 3 * C, N, alpha=d ** -0.5)
        p = A.softmax_rows(s)
        vt = A.transpose_tokens(qkv[:, 2 * C:].contiguous(), B, N, C)      # [B, C, N]
        o = torch.empty(B * N, C, dtype=_f16, device=xn.device)
        A.bgemm(p, vt, o, H, B, (N * N, H * N * N), (d * N, C * N), (d, N * C), N, d, N, N, N, C)
        wo, bo = pk.linear(attn.to_out[0])
        return A.gemm(o, wo, bias=bo, residual=residual, rowbias=rowbias, rows_per_group=N)

    def _ensure_context(self, context):
        """Single-token cross-attention depends on the context only: out = to_out(to_v(ctx)), constant over the image and
        over every DDIM step of a sampling call.  It is computed once per context TENSOR OBJECT (identity + version; a
        strong reference is kept so the address cannot be recycled) AND per set of packed weights (reloading a checkpoint
        while the same context tensor is reused must not keep the old projection) into static buffers the captured graph reads."""
        B, T = context.shape[0], context.shape[1]
        pk = self._pk()
        if T != 1 or (context is self._ctx_ref and context._version == self._ctx_ver and self._ctx_pk == pk.key):
            return
        ctx16 = context.reshape(B, -1).to(_f16).contiguous()
        for st in (m for m in self.modules() if isinstance(m, SpatialTransformer)):
            attn = st.transformer_blocks[0].attn2
            wv, _ = pk.linear(attn.to_v)
            wo, bo = pk.linear(attn.to_out[0])
            key = (id(st), B)
            if key not in self._cross_out:
                self._cross_out[key] = torch.empty(B, wo.shape[0], dtype=_f16, device=context.device)
            A.gemm(A.gemm(ctx16, wv), wo, bias=bo, out=self._cross_out[key])
        self._ctx_ref, self._ctx_ver, self._ctx_pk = context, context._version, pk.key

    def _cross_attention(self, pk, st, blk, h, ctx16, B, N, C):
        attn = blk.attn2
        T = ctx16.shape[0] // B
        wo, bo = pk.linear(attn.to_out[0])
        if T == 1:  # one key: softmax == 1, output = to_out(to_v(ctx)) for every query token (see _ensure_context)
            return A.add_channel_bias(h, self._cross_out[(id(st), B)], B, N, C)
        H, d = attn.heads, attn.dim_head
        xn = A.layernorm(h, *pk.norm(blk.norm2), eps=blk.norm2.eps)
        q = A.gemm(xn, pk.linear(attn.to_q)[0])
        k = A.gemm(ctx16, pk.linear(attn.to_k)[0])                          # [B*T, C]
        v = A.gemm(ctx16, pk.linear(attn.to_v)[0])
        s = torch.empty(B * H, N, T, dtype=_f16, device=h.device)
        A.bgemm(q, k, s, H, B, (d, N * C), (d, T * C), (N * T, H * N * T), N, T, d, C, C, T, alpha=d ** -0.5)
        p = A.softmax_rows(s)
        Tp = (T + 7) // 8 * 8                                               # TMA rows need 16-byte strides
        pp = torch.zeros(B * H, N, Tp, dtype=_f16, device=h.device)
        pp[:, :, :T] = p
        vt = torch.zeros(B, C, Tp, dtype=_f16, device=h.device)
        vt[:, :, :T] = A.transpose_tokens(v, B, T, C)
        o = torch.empty(B * N, C, dtype=_f16, device=h.device)
        A.bgemm(pp, vt, o, H, B, (N * Tp, H * N * Tp), (d * Tp, C * Tp), (d, N * C), N, d, Tp, Tp, Tp, C)
        return A.gemm(o, wo, bias=bo, residual=h)

    def _transformer(self, pk, st, x, B, H, W, C, ctx16):
        N = H * W
        a, _, _ = self._norm(pk, x, B, H, W, C, st.norm, False)
        wi, bi = pk.conv(st.proj_in)
        h = A.gemm(a, wi, bias=bi)
        blk = st.transformer_blocks[0]
        xn = A.layernorm(h, *pk.norm(blk.norm1), eps=blk.norm1.eps)
        if ctx16.shape[0] == B and (id(st), B) in self._cross_out:
            # one context token: attn2(h) = to_out(to_v(ctx)) is a per-image constant (see _ensure_context), so
            # h + attn1(...) + attn2(...) is ONE epilogue: residual h, row-group bias cross_out[image]
            h = self._attention(pk, blk.attn1, xn, B, N, C, h, rowbias=self._cross_out[(id(st), B)])
        else:
            h = self._attention(pk, blk.attn1, xn, B, N, C, h)
            h = self._cross_attention(pk, st, blk, h, ctx16, B, N, C)
        w1, b1 = pk.geglu(blk.ff.net[0].proj)        # GEGLU gate applied in the GEMM epilogue: [M, 4C], not [M, 8C], leaves the SM
        w2, b2 = pk.linear(blk.ff.net[2])
        gg = A.gemm(A.layernorm(h, *pk.norm(blk.norm3), eps=blk.norm3.eps), w1, bias=b1, act=A.ACT_GEGLU)
        h = A.gemm(gg, w2, bias=b2, residual=h)
        wo, bo = pk.conv(st.proj_out)
        return A.gemm(h, wo, bias=bo, residual=x)

    def _run_block(self, pk, seq, x, B, H, W, C, emb_act, ctx16):
        for layer in seq:
            if isinstance(layer, ResBlock):
                x, C = self._resblock(pk, layer, x, B, H, W, emb_act)
            elif isinstance(layer, SpatialTransformer):
                x = self._transformer(pk, layer, x, B, H, W, C, ctx16)
            elif isinstance(layer, Downsample):
                x, H, W = self._conv3(pk, x, B, H, W, C, layer.op, stride=2)
            elif isinstance(layer, Upsample):
                x, H, W = self._conv3(pk, x, B, H, W, C, layer.conv, up=True)
            elif isinstance(layer, nn.Conv2d):
                x, H, W = self._conv3(pk, x, B, H, W, C, layer)
                C = layer.out_channels
            else:
                raise TypeError(type(layer))
        return x, H, W, C

    @inference_only
    def forward(self, x, timesteps=None, context=None, y=None, **kwargs):
        """Epsilon prediction.  On CUDA the ~525 kernel launches of one pass are captured once per input shape in a
        CUDA graph and replayed (the pass is launch-bound from Python: 18 ms eager vs the device time of the graph);
        the returned tensor is a copy of the graph's static output buffer."""
        assert y is None, "the Zero123 UNet is not class-conditional"
        self._ensure_context(context)
        if not (self.use_cuda_graph and x.is_cuda) or torch.cuda.is_current_stream_capturing():
            return self._forward_impl(x, timesteps, context)
        from . import _lib
        key = (tuple(x.shape), tuple(context.shape), self._pk().key)
        g = self._graphs.get(key)
        if g is None:
            sx, st, sc = x.detach().float().clone(), timesteps.detach().clone(), context.detach().float().clone()
            self._forward_impl(sx, st, sc)                       # warm-up: packs weights, sets kernel attributes
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            n0 = _lib.launches()
            with torch.cuda.graph(graph):
                out = self._forward_impl(sx, st, sc)
            g = self._graphs[key] = (graph, sx, st, sc, out, _lib.launches() - n0)
        graph, sx, st, sc, out, n_kernels = g
        sx.copy_(x), st.copy_(timesteps), sc.copy_(context)
        graph.replay()
        _lib.add_launches(n_kernels)
        # a fresh tensor, as the reference returns: the graph's static output buffer is overwritten by the next call, and
        # code written for the reference keeps eps across calls (e_t = apply_model(x, t, c); e_uc = apply_model(x, t, uc))
        return out.clone()

    @torch.no_grad()
    def _forward_impl(self, x, timesteps, context):
        pk = self._pk()
        B, Cin, H, W = x.shape
        C = (Cin + 7) // 8 * 8
        h = A.nchw_to_cl(x, torch.zeros(B * H * W, C, dtype=_f16, device=x.device))
        t_emb = A.timestep_embedding(timesteps, self.model_channels)
        w0, b0 = pk.linear(self.time_embed[0])
        w2, b2 = pk.linear(self.time_embed[2])
        emb = A.gemm(A.gemm(t_emb, w0, bias=b0, act=1), w2, bias=b2)
        wa, ba, _ = self._emb_pack(pk)
        emb_act = A.gemm(A.silu(emb), wa, bias=ba)                          # [B, sum Cout]: emb_layers of every ResBlock
        ctx16 = context.reshape(-1, context.shape[-1]).to(_f16).contiguous()
        hs = []
        for seq in self.input_blocks:
            h, H, W, C = self._run_block(pk, seq, h, B, H, W, C, emb_act, ctx16)
            hs.append((h, C))
        h, H, W, C = self._run_block(pk, self.middle_block, h, B, H, W, C, emb_act, ctx16)
        for seq in self.output_blocks:
            skip, Cs = hs.pop()
            cat = torch.empty(B * H * W, C + Cs, dtype=_f16, device=h.device)
            A.copy_channels(h, cat, 0)
            A.copy_channels(skip, cat, C)
            h, H, W, C = self._run_block(pk, seq, cat, B, H, W, C + Cs, emb_act, ctx16)
        out, _, _ = self._conv3(pk, h, B, H, W, C, self.out[2], gn=self.out[0], act=True)
        return A.cl_to_nchw(out, B, self.out_channels, H, W)
