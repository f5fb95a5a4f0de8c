"""ObjectsPerceiverEncoder: the Perceiver resampler of the VIMA-Flamingo baseline (reference:
/root/reference/vima/nn/obj_encoder/perceiver/perceiver.py:11-41, which wraps `transformers` PerceiverModel).

Parameter tree and state-dict keys are those of HF's PerceiverModel (`model.embeddings.latents`,
`model.encoder.cross_attention.*`, `model.encoder.self_attends.N.*`); the arithmetic -- LayerNorms, the q / k|v / output /
MLP projections (wgmma GEMMs with GELU and residual epilogues) and the latent attention -- runs on the sm_90a kernels.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from .. import _C
from .. import engine as eng


class _SelfAttention(nn.Module):
    def __init__(self, E: int, cross: bool):
        super().__init__()
        self.layernorm1 = nn.LayerNorm(E)
        self.layernorm2 = nn.LayerNorm(E) if cross else nn.Identity()
        self.query = nn.Linear(E, E)
        self.key = nn.Linear(E, E)
        self.value = nn.Linear(E, E)


class _SelfOutput(nn.Module):
    def __init__(self, E: int):
        super().__init__()
        self.dense = nn.Linear(E, E)


class _Attention(nn.Module):
    def __init__(self, E: int, cross: bool):
        super().__init__()
        self.self = _SelfAttention(E, cross)
        self.output = _SelfOutput(E)


class _MLP(nn.Module):
    def __init__(self, E: int):
        super().__init__()
        self.dense1 = nn.Linear(E, E)  # widening factor 1 (PerceiverConfig default)
        self.dense2 = nn.Linear(E, E)


class _Layer(nn.Module):
    def __init__(self, E: int, cross: bool):
        super().__init__()
        self.attention = _Attention(E, cross)
        self.layernorm = nn.LayerNorm(E)
        self.mlp = _MLP(E)


class _Embeddings(nn.Module):
    def __init__(self, num_latents: int, E: int):
        super().__init__()
        self.latents = nn.Parameter(torch.randn(num_latents, E))


class _Encoder(nn.Module):
    def __init__(self, E: int, n_self: int):
        super().__init__()
        self.cross_attention = _Layer(E, True)
        self.self_attends = nn.ModuleList([_Layer(E, False) for _ in range(n_self)])


class _PerceiverModel(nn.Module):
    def __init__(self, E: int, num_latents: int, n_self: int):
        super().__init__()
        self.embeddings = _Embeddings(num_latents, E)
        self.encoder = _Encoder(E, n_self)


class ObjectsPerceiverEncoder(nn.Module):
    def __init__(self, embed_dim: int, *, num_latents: int, num_blocks: int, num_self_attends_per_block: int, num_self_attention_heads: int,
                 num_cross_attention_heads: int, attention_probs_dropout_prob: float):
        super().__init__()
        if embed_dim % num_self_attention_heads or embed_dim % num_cross_attention_heads:
            raise ValueError("embed_dim must be divisible by the head counts")
        if embed_dim // num_self_attention_heads > 128 or embed_dim // num_cross_attention_heads > 128:
            raise NotImplementedError("the latent attention kernel is built for head_dim <= 128")
        self.model = _PerceiverModel(embed_dim, num_latents, num_self_attends_per_block)
        self.output_dim = embed_dim
        self._num_queries = num_latents
        self._num_blocks = num_blocks
        self._heads_self, self._heads_cross = num_self_attention_heads, num_cross_attention_heads
        self._wc = eng.WeightCache(self)

    # -------------------------------------------------------------------------------------------------
    def _packed(self, ctx, p):
        def pack_layer(layer: _Layer, cross: bool):
            a = layer.attention.self
            d = {"q": eng.pack_linear(ctx, a.query.weight, a.query.bias, transposed=False, p=p),
                 "o": eng.pack_linear(ctx, layer.attention.output.dense.weight, layer.attention.output.dense.bias, transposed=False, p=p),
                 "m1": eng.pack_linear(ctx, layer.mlp.dense1.weight, layer.mlp.dense1.bias, transposed=False, p=p),
                 "m2": eng.pack_linear(ctx, layer.mlp.dense2.weight, layer.mlp.dense2.bias, transposed=False, p=p)}
            kv_w = torch.cat([a.key.weight.detach(), a.value.weight.detach()], dim=0)
            kv_b = torch.cat([a.key.bias.detach(), a.value.bias.detach()], dim=0)
            if cross:
                d["kv"] = eng.pack_linear(ctx, kv_w, kv_b, transposed=False, p=p)
            else:  # self-attention: q | k | v in one GEMM
                d["qkv"] = eng.pack_linear(ctx, torch.cat([a.query.weight.detach(), kv_w], dim=0), torch.cat([a.query.bias.detach(), kv_b], dim=0),
                                           transposed=False, p=p)
            return d

        enc = self.model.encoder
        return self._wc.get("perceiver", tuple(self.parameters()),
                            lambda: {"cross": pack_layer(enc.cross_attention, True), "self": [pack_layer(l, False) for l in enc.self_attends]})

    def _ffn(self, ctx, p, layer: _Layer, W, x32, rows, E):
        """x + dense2(gelu(dense1(LN(x))))   (PerceiverLayer.feed_forward_chunk + residual)."""
        ln = layer.layernorm
        _, _, h16 = eng.norm(ctx, x32, p, rows=rows, cols=E, w=ln.weight.detach(), b=ln.bias.detach(), eps=ln.eps, want16=True)
        _, g16 = eng.gemm(ctx, h16, W["m1"], p, act=_C.ACT_GELU, want16=True)
        out32, _ = eng.gemm(ctx, g16, W["m2"], p, residual=x32, want_f32=True)
        return out32

    def forward(self, x: torch.Tensor, mask: torch.Tensor = None):
        """x (N, L, E) image tokens, mask (N, L) (all ones in the reference, obj_encoder.py:199-203) -> (N, num_latents, E)."""
        ctx = eng.ctx_for(x)
        p = eng.prec()
        N, L, E = x.shape
        if mask is not None and mask.shape != (N, L):
            raise ValueError("mask must be (N, L)")
        if L > 16:
            raise NotImplementedError("the latent attention kernel takes at most 16 input tokens per image")
        W = self._packed(ctx, p)
        enc = self.model.encoder
        nl = self._num_queries
        dev = x.device
        xin = x.reshape(N * L, E).float().contiguous()
        lat = self.model.embeddings.latents.detach().float().contiguous()
        # ---- cross-attention: latents (shared by all images) attend to the image tokens ----
        ca = enc.cross_attention.attention.self
        _, _, hq16 = eng.norm(ctx, lat, p, rows=nl, cols=E, w=ca.layernorm1.weight.detach(), b=ca.layernorm1.bias.detach(), eps=ca.layernorm1.eps,
                              want16=True)
        q32, _ = eng.gemm(ctx, hq16, W["cross"]["q"], p, want_f32=True)  # (nl, E): the same queries for every image
        _, _, hk16 = eng.norm(ctx, xin, p, rows=N * L, cols=E, w=ca.layernorm2.weight.detach(), b=ca.layernorm2.bias.detach(), eps=ca.layernorm2.eps,
                              want16=True)
        kv32, _ = eng.gemm(ctx, hk16, W["cross"]["kv"], p, want_f32=True)  # (N*L, 2E): k | v
        ctx32 = torch.empty((N * nl, E), dtype=torch.float32, device=dev)
        dh = E // self._heads_cross
        ctx.latent_attention(q=q32, ldq=E, q_batch_stride=0, k=kv32, ldk=2 * E, v=kv32[:, E:], ldv=2 * E, o=ctx32, ldo=E, N=N, Lq=nl, Lk=L,
                             H=self._heads_cross, d=dh, scale=1.0 / math.sqrt(dh))
        res = lat.unsqueeze(0).expand(N, nl, E).reshape(N * nl, E).contiguous()  # use_query_residual: + the un-normalised latents
        x32, _ = eng.gemm(ctx, eng.to_operand(ctx, ctx32, p), W["cross"]["o"], p, residual=res, want_f32=True)
        x32 = self._ffn(ctx, p, enc.cross_attention, W["cross"], x32, N * nl, E)
        # ---- the same stack of self-attention layers, num_blocks times ----
        dh = E // self._heads_self
        for _ in range(self._num_blocks):
            for layer, Wl in zip(enc.self_attends, W["self"]):
                sa = layer.attention.self
                _, _, h16 = eng.norm(ctx, x32, p, rows=N * nl, cols=E, w=sa.layernorm1.weight.detach(), b=sa.layernorm1.bias.detach(),
                                     eps=sa.layernorm1.eps, want16=True)
                qkv32, _ = eng.gemm(ctx, h16, Wl["qkv"], p, want_f32=True)  # (N*nl, 3E)
                ctx.latent_attention(q=qkv32, ldq=3 * E, q_batch_stride=nl * 3 * E, k=qkv32[:, E:], ldk=3 * E, v=qkv32[:, 2 * E:], ldv=3 * E,
                                     o=ctx32, ldo=E, N=N, Lq=nl, Lk=nl, H=self._heads_self, d=dh, scale=1.0 / math.sqrt(dh))
                a32, _ = eng.gemm(ctx, eng.to_operand(ctx, ctx32, p), Wl["o"], p, residual=x32, want_f32=True)
                x32 = self._ffn(ctx, p, layer, Wl, a32, N * nl, E)
        return x32.view(N, nl, E)
