"""FrozenCLIPImageEmbedder on the o2345 kernels (SURVEY.md row A8: the conditioning encoder of Zero123).

Mirror of reference ldm/modules/encoders/modules.py:343-382: `preprocess` (bicubic 224 x 224 resize with
align_corners=True, [-1, 1] -> [0, 1], CLIP mean / std) and `model.encode_image`, where `model` is OpenAI CLIP ViT-L/14's
vision tower (github.com/openai/CLIP clip/model.py `VisionTransformer`, 304 M parameters: conv1 14 x 14 / 14 without
bias, class token, 257 positional embeddings, ln_pre, 24 x [ln_1, 16-head attention, ln_2, MLP 1024 -> 4096 -> 1024 with
QuickGELU], ln_post on the class token, projection 1024 -> 768).  The `clip` package is not vendored in /root/reference
(requirements.txt: git+https://github.com/openai/CLIP.git), so the parameter tree below follows its published state-dict
names (`model.visual.conv1.weight`, `model.visual.transformer.resblocks.{i}.attn.in_proj_weight`, ...): a Zero123
checkpoint's `cond_stage_model.*` keys load directly.

Execution: one kernel resizes, normalises and patchifies (the A operand of the patch-embedding GEMM); every Linear is
the wgmma GEMM (QuickGELU / residual in the epilogue); attention is the fused mma.sync kernel at head dim 64;
LayerNorms are fp32-statistics row kernels; activations fp16 (the reference runs this tower in fp16 under
--half_precision as well).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops_a as A
from ._lib import inference_only

_f16, _f32 = torch.float16, torch.float32
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


class _Attention(nn.Module):           # nn.MultiheadAttention's parameter names
    def __init__(self, d):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.empty(3 * d, d))
        self.in_proj_bias = nn.Parameter(torch.empty(3 * d))
        self.out_proj = nn.Linear(d, d)


class _Block(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.attn = _Attention(d)
        self.ln_1 = nn.LayerNorm(d)
        self.mlp = nn.Sequential()
        self.mlp.add_module("c_fc", nn.Linear(d, 4 * d))
        self.mlp.add_module("gelu", nn.Identity())       # QuickGELU, applied in the c_fc epilogue
        self.mlp.add_module("c_proj", nn.Linear(4 * d, d))
        self.ln_2 = nn.LayerNorm(d)


class _Transformer(nn.Module):
    def __init__(self, d, layers):
        super().__init__()
        self.resblocks = nn.Sequential(*[_Block(d) for _ in range(layers)])


class VisionTransformer(nn.Module):
    def __init__(self, input_resolution=224, patch_size=14, width=1024, layers=24, heads=16, output_dim=768):
        super().__init__()
        self.input_resolution, self.patch_size, self.width, self.heads, self.output_dim = input_resolution, patch_size, width, heads, output_dim
        self.conv1 = nn.Conv2d(3, width, patch_size, patch_size, bias=False)
        n = (input_resolution // patch_size) ** 2 + 1
        self.class_embedding = nn.Parameter(torch.empty(width))
        self.positional_embedding = nn.Parameter(torch.empty(n, width))
        self.ln_pre = nn.LayerNorm(width)
        self.transformer = _Transformer(width, layers)
        self.ln_post = nn.LayerNorm(width)
        self.proj = nn.Parameter(torch.empty(width, output_dim))


class _ClipModel(nn.Module):
    def __init__(self, **kw):
        super().__init__()
        self.visual = VisionTransformer(**kw)


class FrozenCLIPImageEmbedder(nn.Module):
    def __init__(self, model='ViT-L/14', jit=False, device='cpu', antialias=False, **vit_kwargs):
        super().__init__()
        if model != 'ViT-L/14' or antialias:
            raise NotImplementedError("only ViT-L/14 without antialiasing (the Zero123 configuration) is built")
        self.model = _ClipModel(**vit_kwargs)
        self.antialias = antialias
        self.register_buffer('mean', torch.tensor(CLIP_MEAN), persistent=False)
        self.register_buffer('std', torch.tensor(CLIP_STD), persistent=False)
        self._packed = None

    # ------------------------------------------------------------------ packed fp16 operands
    def _pk(self):
        key = tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._packed is None or self._packed[0] != key:
            v = self.model.visual
            h = lambda t: t.detach().to(_f16).contiguous()
            f = lambda t: t.detach().to(_f32).contiguous()
            kp = (3 * v.patch_size ** 2 + 7) // 8 * 8                        # 588 -> 592: TMA rows are 16-byte multiples
            w1 = v.conv1.weight.detach().reshape(v.width, -1)
            w1 = torch.cat([w1, w1.new_zeros(v.width, kp - w1.shape[1])], 1)
            blocks = [dict(ln1=(f(b.ln_1.weight), f(b.ln_1.bias)), ln2=(f(b.ln_2.weight), f(b.ln_2.bias)),
                           wqkv=h(b.attn.in_proj_weight), bqkv=f(b.attn.in_proj_bias),
                           wo=h(b.attn.out_proj.weight), bo=f(b.attn.out_proj.bias),
                           w1=h(b.mlp.c_fc.weight), b1=f(b.mlp.c_fc.bias), w2=h(b.mlp.c_proj.weight), b2=f(b.mlp.c_proj.bias))
                      for b in v.transformer.resblocks]
            self._packed = (key, dict(conv1=h(w1), kp=kp, cls=f(v.class_embedding), pos=f(v.positional_embedding),
                                      ln_pre=(f(v.ln_pre.weight), f(v.ln_pre.bias)), ln_post=(f(v.ln_post.weight), f(v.ln_post.bias)),
                                      proj=h(v.proj.detach().t()), blocks=blocks))
        return self._packed[1]

    @inference_only
    def forward(self, x):
        """x [B,3,H,W] in [-1, 1] -> CLIP image embedding [B, 768] fp32 (reference modules.py:372-379)."""
        if isinstance(x, list):                                              # [""] = condition dropout for ucg
            return torch.zeros(1, self.model.visual.output_dim, device=self.model.visual.conv1.weight.device)
        v, pk = self.model.visual, self._pk()
        B, d, H, N = x.shape[0], v.width, v.heads, (v.input_resolution // v.patch_size) ** 2 + 1
        patches = A.clip_patches(x, v.input_resolution, v.patch_size, CLIP_MEAN, CLIP_STD, pk["kp"])   # [B*(N-1), kp] fp16
        tok = torch.empty(B * N, d, dtype=_f16, device=x.device)
        for b in range(B):                                                   # patch rows of image b start one row after its class row
            A.gemm(patches[b * (N - 1):(b + 1) * (N - 1)], pk["conv1"], out=tok[b * N + 1:(b + 1) * N])
        A.clip_add_positions(tok, pk["cls"], pk["pos"], B, N, d)
        h = A.layernorm(tok, *pk["ln_pre"])
        for blk in pk["blocks"]:
            qkv = A.gemm(A.layernorm(h, *blk["ln1"]), blk["wqkv"], bias=blk["bqkv"])
            o = A.attention(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], B, N, H, d // H)
            h = A.gemm(o, blk["wo"], bias=blk["bo"], residual=h)
            m = A.gemm(A.layernorm(h, *blk["ln2"]), blk["w1"], bias=blk["b1"], act=A.ACT_QUICKGELU)
            h = A.gemm(m, blk["w2"], bias=blk["b2"], residual=h)
        cls = A.layernorm(h.view(B, N, d)[:, 0].contiguous(), *pk["ln_post"])
        return A.gemm(cls, pk["proj"], out_dtype=_f32)

    def encode(self, im):
        return self(im).unsqueeze(1)
