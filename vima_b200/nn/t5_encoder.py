"""T5PromptEncoder / WordEmbedding: the t5-base encoder stack over interleaved word / object prompt tokens.

Module surface and state-dict keys of /root/reference/vima/nn/prompt_encoder/prompt_encoder.py:22-58 (+ the vendored HF
T5 encoder :61-825) and word_embd.py:8-23, without depending on `transformers`: 12 pre-RMSNorm blocks, d_model 768,
12 heads x 64, d_ff 3072 ReLU, bias-free Linears, UNSCALED dot-product scores plus a shared relative-position bias
(32 buckets, max distance 128, bidirectional) with the key mask folded in (prompt_encoder.py:785-797).

Kernel plan: RMSNorm (warp-shuffle) -> fused [q;k;v] wgmma GEMM -> fused attention (bias looked up from a
[heads, 2*Lp-1] table in shared memory; the reference materialises a B*H*Lp*Lp tensor) -> o GEMM (+residual) ->
RMSNorm -> wi GEMM (ReLU epilogue) -> wo GEMM (+residual) -> ... -> final RMSNorm.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn as nn

from .. import _C
from .. import engine as eng

T5_BASE = dict(vocab_size=32128, d_model=768, d_kv=64, d_ff=3072, num_layers=12, num_heads=12, relative_attention_num_buckets=32,
               relative_attention_max_distance=128, layer_norm_epsilon=1e-6)


def relative_position_buckets(max_len: int, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """Bucket id for every relative position (memory - context) in [-(max_len-1), max_len-1] (int64), bidirectional.
    Restates HF `T5Attention._relative_position_bucket` (HF:modeling_t5.py) with the same float32 log arithmetic,
    on the host; tests pin it bit-exactly against HF."""
    rel = torch.arange(-(max_len - 1), max_len, dtype=torch.long)
    nb = num_buckets // 2
    ret = (rel > 0).to(torch.long) * nb
    n = rel.abs()
    max_exact = nb // 2
    large = max_exact + (torch.log(n.float() / max_exact) / math.log(max_distance / max_exact) * (nb - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, nb - 1))
    return ret + torch.where(n < max_exact, n, large)


class _T5LayerNorm(nn.Module):
    def __init__(self, d: int, eps: float):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(d))
        self.variance_epsilon = eps


class _T5Attention(nn.Module):
    def __init__(self, cfg, has_bias: bool):
        super().__init__()
        inner = cfg["num_heads"] * cfg["d_kv"]
        self.q = nn.Linear(cfg["d_model"], inner, bias=False)
        self.k = nn.Linear(cfg["d_model"], inner, bias=False)
        self.v = nn.Linear(cfg["d_model"], inner, bias=False)
        self.o = nn.Linear(inner, cfg["d_model"], bias=False)
        if has_bias:
            self.relative_attention_bias = nn.Embedding(cfg["relative_attention_num_buckets"], cfg["num_heads"])


class _T5LayerSelfAttention(nn.Module):
    def __init__(self, cfg, has_bias):
        super().__init__()
        self.SelfAttention = _T5Attention(cfg, has_bias)
        self.layer_norm = _T5LayerNorm(cfg["d_model"], cfg["layer_norm_epsilon"])


class _T5DenseReluDense(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.wi = nn.Linear(cfg["d_model"], cfg["d_ff"], bias=False)
        self.wo = nn.Linear(cfg["d_ff"], cfg["d_model"], bias=False)


class _T5LayerFF(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.DenseReluDense = _T5DenseReluDense(cfg)
        self.layer_norm = _T5LayerNorm(cfg["d_model"], cfg["layer_norm_epsilon"])


class _T5Block(nn.Module):
    def __init__(self, cfg, has_bias):
        super().__init__()
        self.layer = nn.ModuleList([_T5LayerSelfAttention(cfg, has_bias), _T5LayerFF(cfg)])


class _T5Stack(nn.Module):
    def __init__(self, cfg, embed_tokens):
        super().__init__()
        self.embed_tokens = embed_tokens
        self.block = nn.ModuleList([_T5Block(cfg, i == 0) for i in range(cfg["num_layers"])])
        self.final_layer_norm = _T5LayerNorm(cfg["d_model"], cfg["layer_norm_epsilon"])


class T5EncoderModel(nn.Module):
    """Holder with HF's key layout: `shared.weight` aliased as `encoder.embed_tokens.weight`."""

    def __init__(self, cfg=None):
        super().__init__()
        self.config = dict(T5_BASE if cfg is None else cfg)
        self.shared = nn.Embedding(self.config["vocab_size"], self.config["d_model"])
        self.encoder = _T5Stack(self.config, self.shared)


class T5PromptEncoder(nn.Module):
    def __init__(self, cfg=None):
        """The reference downloads t5-base here (prompt_encoder.py:26); weights arrive through `load_state_dict`
        (the VIMA checkpoints carry the whole T5), so construction is offline with a plain init."""
        super().__init__()
        self.t5 = T5EncoderModel(cfg)
        self.output_dim = self.t5.config["d_model"]
        self.input_dim = self.t5.config["d_model"]
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, std=m.in_features ** -0.5)
        self._wc = eng.WeightCache(self)
        self._bucket_cache = {}

    def _packed(self, ctx, p):
        def build():
            out = []
            for blk in self.t5.encoder.block:
                sa, ff = blk.layer[0].SelfAttention, blk.layer[1].DenseReluDense
                # "f16f8" operands throughout (2 tensor pass-equivalents).  The RMSNorms stay kernels here, unlike the decoder's /
                # ViT's folded LayerNorms: T5's pre-norm residual stream is unbounded (t5-base hidden states reach 1e3-1e4 with
                # real weights), and an un-normalised GEMM operand must stay below 1024 for the e4m3 cross terms (65504 for fp16)
                out.append({
                    "qkv": eng.pack_linear(ctx, torch.cat([sa.q.weight.detach(), sa.k.weight.detach(), sa.v.weight.detach()], 0), None, transposed=False,
                                           p=p, f8=True),
                    "o": eng.pack_linear(ctx, sa.o.weight, None, transposed=False, p=p, f8=True),
                    "wi": eng.pack_linear(ctx, ff.wi.weight, None, transposed=False, p=p, f8=True),
                    "wo": eng.pack_linear(ctx, ff.wo.weight, None, transposed=False, p=p, f8=True),
                })
            return out

        return self._wc.get("t5", tuple(self.t5.encoder.parameters()), build)

    def _bias_table(self, Lp: int, device) -> torch.Tensor:
        """[heads, 2*Lp-1] fp32: relative_attention_bias[bucket(j - i)] for every offset (HF compute_bias)."""
        if Lp not in self._bucket_cache:
            cfg = self.t5.config
            self._bucket_cache[Lp] = relative_position_buckets(Lp, cfg["relative_attention_num_buckets"], cfg["relative_attention_max_distance"])
        buckets = self._bucket_cache[Lp].to(device)
        w = self.t5.encoder.block[0].layer[0].SelfAttention.relative_attention_bias.weight.detach()
        return w.index_select(0, buckets).t().contiguous()  # tiny gather: 2*Lp-1 x heads

    def encode(self, x: torch.Tensor, attention_mask: Optional[torch.Tensor], *, want16: bool = False):
        """x (B,Lp,D) fp32 batch-first -> final-RMSNorm output [B*Lp, D] fp32 (and as operands when want16)."""
        ctx = eng.ctx_for(x)
        p = eng.prec()
        cfg = self.t5.config
        B, Lp, D = x.shape
        H, dkv = cfg["num_heads"], cfg["d_kv"]
        inner = H * dkv
        dev = x.device
        Mp = B * Lp
        W = self._packed(ctx, p)
        blocks = self.t5.encoder.block
        h32 = x.reshape(Mp, D).contiguous().clone()  # residual stream, updated in place by the GEMM epilogues
        kmask = None
        if attention_mask is not None:
            kmask = eng.as_u8(attention_mask.reshape(B, Lp) != 0)
        bias = self._bias_table(Lp, dev)
        eps = cfg["layer_norm_epsilon"]
        _, _, n16 = eng.norm(ctx, h32, p, rows=Mp, cols=D, w=blocks[0].layer[0].layer_norm.weight.detach(), eps=eps, rms=True, want16=True, out_f8=True)
        c16 = eng.Opnd(Mp, inner, dev, p.split, f8=p.f8)
        o8 = None if c16.lo8 is None else (c16.lo8, c16.hi8)
        out32 = out16 = None
        for i, (blk, Wb) in enumerate(zip(blocks, W)):
            _, qkv16 = eng.gemm(ctx, n16, Wb["qkv"], p, want16=True)
            ctx.attention(q=(qkv16.hi, qkv16.lo, qkv16.ld, 0), k=(qkv16.hi, qkv16.lo, qkv16.ld, inner), v=(qkv16.hi, qkv16.lo, qkv16.ld, 2 * inner),
                          o=(c16.hi, c16.lo, c16.ld, 0), B=B, H=H, Lq=Lp, Lk=Lp, D=dkv, scale=1.0, causal=False, key_mask=kmask, rel_bias=bias,
                          dtype=p.dtype, o8=o8)
            eng.gemm(ctx, c16, Wb["o"], p, residual=h32, out_f32=h32)
            _, _, n16 = eng.norm(ctx, h32, p, rows=Mp, cols=D, w=blk.layer[1].layer_norm.weight.detach(), eps=eps, rms=True, want16=True, out_f8=True)
            _, f16 = eng.gemm(ctx, n16, Wb["wi"], p, act=_C.ACT_RELU, want16=True, out_f8=True)
            eng.gemm(ctx, f16, Wb["wo"], p, residual=h32, out_f32=h32)
            del f16
            if i + 1 < len(blocks):
                _, _, n16 = eng.norm(ctx, h32, p, rows=Mp, cols=D, w=blocks[i + 1].layer[0].layer_norm.weight.detach(), eps=eps, rms=True, want16=True,
                                     out_f8=True)
            else:
                out32, _, out16 = eng.norm(ctx, h32, p, rows=Mp, cols=D, w=self.t5.encoder.final_layer_norm.weight.detach(), eps=eps, rms=True,
                                           want_f32=True, want16=want16)
        return out32, out16

    def forward(self, x: torch.Tensor, *, attention_mask: Optional[torch.Tensor] = None, batch_first: bool = False):
        """x: (L,B,E) if not batch_first else (B,L,E); attention_mask (B,L) or (B,1,L)  (prompt_encoder.py:30-58)."""
        if batch_first:
            B, L, E = x.shape
            xb = x
        else:
            L, B, E = x.shape
            xb = x.transpose(0, 1)
        if attention_mask is not None and attention_mask.dim() == 3:
            attention_mask = attention_mask.squeeze(dim=1)
        out32, _ = self.encode(xb.float(), attention_mask)
        out = out32.view(B, L, E)
        return out if batch_first else out.transpose(0, 1)


class WordEmbedding(nn.Module):
    def __init__(self):
        """Frozen copy of t5-base's input embedding (word_embd.py:8-23); filled by `load_state_dict`."""
        super().__init__()
        self._embed_layer = nn.Embedding(T5_BASE["vocab_size"], T5_BASE["d_model"])
        self._embed_layer.weight.requires_grad_(False)
        self.output_dim = T5_BASE["d_model"]

    def forward(self, x: torch.Tensor):
        """x: any shape of int64 ids -> (..., 768).  The policy's prompt assembly gathers rows in its own kernel;
        this standalone lookup is a plain index_select."""
        return self._embed_layer.weight.detach()[x]
