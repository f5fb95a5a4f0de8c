"""ObjEncoder: CLIP-style ViT over 32x32 object crops + bbox MLP -> object tokens.

Module surface / state-dict keys of /root/reference/vima/nn/obj_encoder/obj_encoder.py:11-99 and
vit/vit.py:13-46,137-236; preprocessing of vit/preprocess.py:9-43.  Kernel plan per call (both views share the ViT,
so their crops are batched through it together):

    patchify (uint8 -> normalised patch rows, fused /255, -mean, /std)  -> conv1 as wgmma GEMM -> +cls +pos
    -> ln_pre [+ ln_1 chained] -> 4 x { in_proj GEMM (+bias) -> 5-token fp32 attention -> out_proj GEMM (+bias
    +residual) -> ln_2 -> c_fc GEMM (+bias, QuickGELU) -> c_proj GEMM (+bias +residual) -> next ln_1 } -> ln_post on
    the CLS rows -> projection GEMM;   bbox: /[256,128,128,256] -> fp32 K=4 layer -> two wgmma GEMMs;
    per view Linear(1536 -> E) over the [vit | bbox] operand written in place by the two producers.
"""
from __future__ import annotations

import math
import os
from collections import OrderedDict
from typing import Dict, List

import torch
import torch.nn as nn

from .. import _C
from .. import engine as eng
from .basic import F32GroupRunner, build_mlp, simt_linear

VIMA_IMG_MEAN = (0.3471, 0.3429, 0.3383)
VIMA_IMG_STD = (0.3011, 0.2961, 0.2956)


class QuickGELU(nn.Module):
    def forward(self, x):  # only a marker module: the activation runs in the c_fc GEMM epilogue
        raise RuntimeError("QuickGELU is fused into the GEMM epilogue; call the enclosing encoder")


class ResidualAttentionBlock(nn.Module):
    """Parameter holder (vit.py:199-236): nn.MultiheadAttention in_proj/out_proj, ln_1, mlp.{c_fc,c_proj}, ln_2."""

    def __init__(self, d_model: int, n_head: int):
        super().__init__()
        self.attn = nn.MultiheadAttention(d_model, n_head)
        self.ln_1 = nn.LayerNorm(d_model)
        self.mlp = nn.Sequential(OrderedDict([("c_fc", nn.Linear(d_model, d_model * 4)), ("gelu", QuickGELU()), ("c_proj", nn.Linear(d_model * 4, d_model))]))
        self.ln_2 = nn.LayerNorm(d_model)


def pack_vit_blocks(ctx, blocks, p):
    """ln_1 / ln_2 are folded into in_proj / c_fc (engine.fold_layernorm): those GEMMs read the un-normalised residual stream."""
    return [{
        "in": eng.pack_linear(ctx, blk.attn.in_proj_weight, blk.attn.in_proj_bias, transposed=False, p=p, f8=True,
                              ln=(blk.ln_1.weight.detach(), blk.ln_1.bias.detach())),
        "out": eng.pack_linear(ctx, blk.attn.out_proj.weight, blk.attn.out_proj.bias, transposed=False, p=p),
        "fc": eng.pack_linear(ctx, blk.mlp.c_fc.weight, blk.mlp.c_fc.bias, transposed=False, p=p, f8=True,
                              ln=(blk.ln_2.weight.detach(), blk.ln_2.bias.detach())),
        "pr": eng.pack_linear(ctx, blk.mlp.c_proj.weight, blk.mlp.c_proj.bias, transposed=False, p=p, f8=True),
    } for blk in blocks]


def run_vit_blocks(ctx, p, blocks, Wblocks, x32, x16, st, N, S, Wm, heads):
    """Pre-LN residual blocks (vit.py:199-236). x32: residual stream [N*S, W] (updated in place by the GEMM epilogues), x16: the
    same rows as GEMM operands, st: their (mean, rstd) for the first block's ln_1.  No LayerNorm kernel runs inside the blocks: the
    residual-carrying GEMMs (out_proj, c_proj) emit operands + row sums, in_proj / c_fc apply ln_1 / ln_2 in their epilogues.
    Returns the final residual stream."""
    dev = x32.device
    M = N * S
    att16 = eng.Opnd(M, Wm, dev, p.split)
    for i, (blk, Wb) in enumerate(zip(blocks, Wblocks)):
        qkv32, _ = eng.gemm(ctx, x16, Wb["in"], p, want_f32=True, row_stats=st)
        ctx.small_attention(qkv32, N=N, S=S, H=heads, W=Wm, scale=1.0 / math.sqrt(Wm // heads), o_hi=att16.hi, o_lo=att16.lo, dtype=p.dtype)
        part = eng.stats_buffer(ctx, M, Wb["out"], dev)
        _, x16 = eng.gemm(ctx, att16, Wb["out"], p, residual=x32, out_f32=x32, want16=True, out_f8=True, stats_out=part)
        st2 = eng.row_stats_of(ctx, part, M, Wm, blk.ln_2.eps)
        _, h16 = eng.gemm(ctx, x16, Wb["fc"], p, act=_C.ACT_QUICKGELU, want16=True, out_f8=True, row_stats=st2)
        last = i + 1 == len(blocks)
        part = None if last else eng.stats_buffer(ctx, M, Wb["pr"], dev)
        _, x16 = eng.gemm(ctx, h16, Wb["pr"], p, residual=x32, out_f32=x32, want16=not last, out_f8=True, stats_out=part)
        if not last:
            st = eng.row_stats_of(ctx, part, M, Wm, blocks[i + 1].ln_1.eps)
    return x32


class VisionTransformer(nn.Module):
    def __init__(self, resolution, patch_size: int, width: int, layers: int, heads: int, output_dim: int):
        super().__init__()
        hw = (resolution, resolution) if isinstance(resolution, int) else tuple(resolution)
        self._img_hw, self._patch_size, self.output_dim = hw, patch_size, output_dim
        self.width, self.heads = width, heads
        if width // heads != 32:
            raise NotImplementedError("the fused 5-token attention kernel is built for head_dim 32 (all VIMA checkpoints)")
        self.conv1 = nn.Conv2d(3, width, kernel_size=patch_size, stride=patch_size, bias=False)
        scale = width ** -0.5
        self.cls_token = nn.Parameter(scale * torch.randn(width))
        self.pos_embed = nn.Parameter(scale * torch.randn((hw[0] // patch_size) * (hw[1] // patch_size) + 1, width))
        self.ln_pre = nn.LayerNorm(width)
        self.blocks = nn.Sequential(*[ResidualAttentionBlock(width, heads) for _ in range(layers)])
        self.ln_post = nn.LayerNorm(width)
        self.projection = nn.Parameter(scale * torch.randn(width, output_dim))
        self._wc = eng.WeightCache(self)

    def _packed(self, ctx, p):
        def build():
            W = {"conv": eng.pack_linear(ctx, self.conv1.weight.detach().reshape(self.width, -1), None, transposed=False, p=p),
                 "proj": eng.pack_linear(ctx, self.projection, None, transposed=True, p=p), "blocks": pack_vit_blocks(ctx, self.blocks, p)}
            return W

        return self._wc.get("vit", tuple(self.parameters()), build)

    def encode_u8(self, img_u8: torch.Tensor, out16: eng.Opnd = None, out16_ld: int = None):
        """img_u8 (N,3,H,W) uint8 -> CLS features after ln_post @ projection, as 16-bit operands [N, output_dim]
        (written into `out16`'s first columns when given)."""
        ctx = eng.ctx_for(img_u8)
        p = eng.prec()
        N, C, H, Wd = img_u8.shape
        P, Wm = self._patch_size, self.width
        assert C == 3 and (H, Wd) == self._img_hw
        dev = img_u8.device
        W = self._packed(ctx, p)
        n_patch = (H // P) * (Wd // P)
        S = n_patch + 1
        patches = eng.Opnd(N * n_patch, 3 * P * P, dev, p.split)
        ctx.patchify(img_u8.contiguous(), N, H, Wd, P, patches.hi, patches.lo, dtype=p.dtype)
        pe32, _ = eng.gemm(ctx, patches, W["conv"], p, want_f32=True)
        tok32 = torch.empty((N * S, Wm), dtype=torch.float32, device=dev)
        ctx.vit_tokens(pe32, self.cls_token.detach(), self.pos_embed.detach(), N, S, Wm, tok32)
        b0 = self.blocks[0]
        x32, _, x16, st = eng.norm(ctx, tok32, p, rows=N * S, cols=Wm, w=self.ln_pre.weight.detach(), b=self.ln_pre.bias.detach(), eps=self.ln_pre.eps,
                                   want_f32=True, want16=True, out_f8=True, stats_eps=b0.ln_1.eps)
        x32 = run_vit_blocks(ctx, p, self.blocks, W["blocks"], x32, x16, st, N, S, Wm, self.heads)
        # ln_post on the CLS rows (row stride S*width), then @ projection
        _, _, cls16 = eng.norm(ctx, x32, p, rows=N, cols=Wm, ldx=S * Wm, w=self.ln_post.weight.detach(), b=self.ln_post.bias.detach(),
                               eps=self.ln_post.eps, want16=True)
        _, feat16 = eng.gemm(ctx, cls16, W["proj"], p, want16=out16 is None, out16=out16)
        return feat16

    def forward(self, x: torch.Tensor):
        """x: (N,3,H,W) already-normalised float image, as the reference's VisionTransformer.forward takes it (vit.py:171)."""
        raise NotImplementedError(
            "vima_b200.VisionTransformer consumes uint8 crops through ViTEncoder (normalisation is fused into the patchify kernel)"
        )


class ViTEncoder(nn.Module):
    def __init__(self, *, output_dim: int, resolution: int, patch_size: int, width: int, layers: int, heads: int):
        super().__init__()
        self.output_dim = output_dim
        self.vit = VisionTransformer(resolution=resolution, patch_size=patch_size, width=width, layers=layers, heads=heads, output_dim=output_dim)
        self._check_range = os.environ.get("VIMA_B200_CHECK_INPUTS", "1") != "0"
        self._range_checked = False

    def _check(self, x):
        # preprocess.py:28 `assert img.max() > 2` is a host sync per call in the reference; here: first call only
        if self._check_range and not self._range_checked:
            mx = torch.zeros(1, dtype=torch.int32, device=x.device)
            eng.ctx_for(x).max_u8(x.contiguous().view(-1), mx)
            assert int(mx.item()) > 2, "img should be between [0, 255] before normalize"
            self._range_checked = True

    def forward(self, x: torch.Tensor):
        """x: (..., 3, H, W) uint8 in [0,255] -> (..., output_dim) fp32 (vit.py:36-46)."""
        assert x.dim() >= 4
        if x.dtype != torch.uint8:
            x = x.to(torch.uint8)
        self._check(x)
        lead = x.shape[:-3]
        feat16 = self.vit.encode_u8(x.reshape(-1, *x.shape[-3:]))
        return feat16.float(eng.prec()).view(*lead, self.output_dim)


class ObjEncoder(nn.Module):
    bbox_max_h = 128
    bbox_max_w = 256

    def __init__(self, *, transformer_emb_dim: int, views: List[str], vit_output_dim: int = 512, vit_resolution: int, vit_patch_size: int,
                 vit_width: int, vit_layers: int, vit_heads: int, bbox_mlp_hidden_dim: int, bbox_mlp_hidden_depth: int):
        super().__init__()
        views = sorted(views)
        self._views = views
        self._transformer_emb_dim = transformer_emb_dim
        self.cropped_img_encoder = ViTEncoder(output_dim=vit_output_dim, resolution=vit_resolution, patch_size=vit_patch_size, width=vit_width,
                                              layers=vit_layers, heads=vit_heads)
        self.bbox_mlp = nn.ModuleDict({v: build_mlp(4, hidden_dim=bbox_mlp_hidden_dim, hidden_depth=bbox_mlp_hidden_depth, output_dim=bbox_mlp_hidden_dim)
                                       for v in views})
        self.pre_transformer_layer = nn.ModuleDict({v: nn.Linear(self.cropped_img_encoder.output_dim + bbox_mlp_hidden_dim, transformer_emb_dim)
                                                    for v in views})
        self._wc = eng.WeightCache(self)

    @property
    def output_dim(self):
        return self._transformer_emb_dim

    def forward(self, cropped_img: Dict[str, torch.Tensor], bbox: Dict[str, torch.Tensor], mask=None):
        """out: (..., n_objs * n_views, E) fp32  (obj_encoder.py:66-95); `mask` is unused, as in the reference."""
        views = self._views
        x0 = cropped_img[views[0]]
        ctx = eng.ctx_for(x0)
        p = eng.prec()
        dev = x0.device
        vit_dim = self.cropped_img_encoder.output_dim
        imgs, counts, leads = [], [], []
        for v in views:
            im = cropped_img[v]
            if im.dtype != torch.uint8:
                im = im.to(torch.uint8)
            leads.append(im.shape[:-3])
            im = im.reshape(-1, *im.shape[-3:])
            imgs.append(im)
            counts.append(im.shape[0])
        all_img = imgs[0] if len(imgs) == 1 else torch.cat(imgs, dim=0)
        self.cropped_img_encoder._check(all_img)
        n_all = all_img.shape[0]
        bdim = self.bbox_mlp[views[0]][-1].out_features
        cat16 = eng.Opnd(n_all, vit_dim + bdim, dev, p.split)  # [vit features | bbox features] per crop
        self.cropped_img_encoder.vit.encode_u8(all_img, out16=cat16.sub(0, n_all, 0, vit_dim))
        outs, r0 = [], 0
        for v, n, lead in zip(views, counts, leads):
            bb = bbox[v].reshape(-1, 4).to(torch.int64).contiguous()
            bb32 = torch.empty((n, 4), dtype=torch.float32, device=dev)
            ctx.bbox_norm(bb, n, bb32)
            # the bbox MLP's last GEMM writes next to the ViT features of this view's rows
            self.bbox_mlp[v](bb32, out16=cat16.sub(r0, n, vit_dim, bdim))
            pw = self._wc.get(f"pre.{v}", (self.pre_transformer_layer[v].weight, self.pre_transformer_layer[v].bias),
                              lambda v=v: eng.pack_linear(ctx, self.pre_transformer_layer[v].weight, self.pre_transformer_layer[v].bias, transposed=False, p=p))
            a = cat16.sub(r0, n)
            o32, _ = eng.gemm(ctx, a, pw, p, want_f32=True)
            outs.append(o32.view(*lead, self._transformer_emb_dim))
            r0 += n
        return torch.cat(outs, dim=-2)


# ------------------------------------------------------------------------------------------------------------
# VIMA-Gato baseline encoder (BASELINE.json configs[4]): whole 64x128 views, 32x32 patches, every patch token kept
# ------------------------------------------------------------------------------------------------------------
class VisionTransformerRectangular(VisionTransformer):
    """vit.py:275-330: the CLS-token ViT on a rectangular image (VIMA-GPT baseline: 64x128, patch 32 -> 1 + 8 tokens)."""

    def __init__(self, img_size, patch_size: int, width: int, layers: int, heads: int, output_dim: int):
        super().__init__(tuple(img_size), patch_size, width, layers, heads, output_dim)


class ViTEncoderRectangular(nn.Module):
    """vit.py:239-272: (..., 3, H, W) uint8 -> (..., output_dim)."""

    def __init__(self, *, output_dim: int, img_size, patch_size: int, width: int, layers: int, heads: int):
        super().__init__()
        self.output_dim = output_dim
        self.vit = VisionTransformerRectangular(img_size=img_size, patch_size=patch_size, width=width, layers=layers, heads=heads,
                                                output_dim=output_dim)

    def forward(self, x: torch.Tensor):
        assert x.dim() >= 4
        if x.dtype != torch.uint8:
            x = x.to(torch.uint8)
        lead = x.shape[:-3]
        feat16 = self.vit.encode_u8(x.reshape(-1, *x.shape[-3:]))
        return feat16.float(eng.prec()).view(*lead, self.output_dim)


class MultiViewRGBEncoder(nn.Module):
    """obj_encoder.py:209-246: both views through the shared CLS ViT, features concatenated on the FEATURE axis (2 * emb_dim)."""

    def __init__(self, *, emb_dim: int, views, img_size, vit_patch_size=None, vit_width=None, vit_layers=None, vit_heads=None):
        super().__init__()
        self._views = sorted(views)
        self._transformer_emb_dim = emb_dim
        self.cropped_img_encoder = ViTEncoderRectangular(img_size=img_size, output_dim=emb_dim, patch_size=vit_patch_size, width=vit_width,
                                                         layers=vit_layers, heads=vit_heads)

    def encode16(self, rgb, pad_cols: int = 0) -> "eng.Opnd":
        """rgb {view: (..., 3, H, W) u8} -> 16-bit operands [rows, 2E (+pad)], one batched pass through the shared ViT."""
        xs = [rgb[v] if rgb[v].dtype == torch.uint8 else rgb[v].to(torch.uint8) for v in self._views]
        rows = int(xs[0].numel() // (xs[0].shape[-3] * xs[0].shape[-2] * xs[0].shape[-1]))
        E = self._transformer_emb_dim
        p = eng.prec()
        out = eng.Opnd(rows, len(xs) * E + pad_cols, xs[0].device, p.split)
        for i, x in enumerate(xs):
            self.cropped_img_encoder.vit.encode_u8(x.reshape(-1, *x.shape[-3:]), out16=out.sub(0, rows, i * E, E))
        return out

    def forward(self, rgb):
        lead = rgb[self._views[0]].shape[:-3]
        return self.encode16(rgb).float(eng.prec()).view(*lead, self.output_dim)

    @property
    def output_dim(self):
        return self._transformer_emb_dim * len(self._views)


class GatoVisionTransformerRectangular(nn.Module):
    """vit.py:85-134: no CLS token; ln_post and the projection apply to all patch tokens."""

    def __init__(self, img_size, patch_size: int, width: int, layers: int, heads: int, output_dim: int):
        super().__init__()
        self.output_dim, self.width, self.heads = output_dim, width, heads
        self._img_size, self._patch_size = tuple(img_size), patch_size
        if width // heads != 32:
            raise NotImplementedError("the fused small-sequence attention kernel is built for head_dim 32")
        self.conv1 = nn.Conv2d(3, width, kernel_size=patch_size, stride=patch_size, bias=False)
        scale = width ** -0.5
        nh, nw = img_size[0] // patch_size, img_size[1] // patch_size
        self.pos_embed = nn.Parameter(scale * torch.randn(nh * nw, width))
        self.ln_pre = nn.LayerNorm(width)
        self.blocks = nn.Sequential(*[ResidualAttentionBlock(width, heads) for _ in range(layers)])
        self.ln_post = nn.LayerNorm(width)
        self.projection = nn.Parameter(scale * torch.randn(width, output_dim))
        self.img_patch_len = nh * nw
        self._wc = eng.WeightCache(self)

    def encode_u8(self, img_u8: torch.Tensor) -> torch.Tensor:
        """(N,3,H,W) uint8 -> (N, n_patches, output_dim) fp32."""
        ctx = eng.ctx_for(img_u8)
        p = eng.prec()
        N, C, H, Wd = img_u8.shape
        assert (H, Wd) == self._img_size and C == 3
        P, Wm, S = self._patch_size, self.width, self.img_patch_len
        dev = img_u8.device
        W = self._wc.get("gvit", tuple(self.parameters()), lambda: {
            "conv": eng.pack_linear(ctx, self.conv1.weight.detach().reshape(Wm, -1), None, transposed=False, p=p),
            "proj": eng.pack_linear(ctx, self.projection, None, transposed=True, p=p), "blocks": pack_vit_blocks(ctx, self.blocks, p)})
        patches = eng.Opnd(N * S, 3 * P * P, dev, p.split)
        ctx.patchify(img_u8.contiguous(), N, H, Wd, P, patches.hi, patches.lo, dtype=p.dtype)
        pe32, _ = eng.gemm(ctx, patches, W["conv"], p, want_f32=True)
        tok32 = torch.empty((N * S, Wm), dtype=torch.float32, device=dev)
        ctx.vit_tokens(pe32, None, self.pos_embed.detach(), N, S, Wm, tok32)
        b0 = self.blocks[0]
        x32, _, x16, st = eng.norm(ctx, tok32, p, rows=N * S, cols=Wm, w=self.ln_pre.weight.detach(), b=self.ln_pre.bias.detach(), eps=self.ln_pre.eps,
                                   want_f32=True, want16=True, out_f8=True, stats_eps=b0.ln_1.eps)
        x32 = run_vit_blocks(ctx, p, self.blocks, W["blocks"], x32, x16, st, N, S, Wm, self.heads)
        _, _, post16 = eng.norm(ctx, x32, p, rows=N * S, cols=Wm, w=self.ln_post.weight.detach(), b=self.ln_post.bias.detach(), eps=self.ln_post.eps,
                                want16=True)
        out32, _ = eng.gemm(ctx, post16, W["proj"], p, want_f32=True)
        return out32.view(N, S, self.output_dim)


class GatoViTEncoder(nn.Module):
    def __init__(self, *, img_size, patch_size: int, width: int, layers: int, heads: int, output_dim: int):
        super().__init__()
        self.output_dim = output_dim
        self.vit = GatoVisionTransformerRectangular(img_size=img_size, patch_size=patch_size, width=width, layers=layers, heads=heads,
                                                    output_dim=output_dim)

    def forward(self, x: torch.Tensor):
        """x: (..., 3, H, W) uint8 -> (..., L, E)   (vit.py:71-82)."""
        assert x.dim() >= 4
        if x.dtype != torch.uint8:
            x = x.to(torch.uint8)
        lead = x.shape[:-3]
        out = self.vit.encode_u8(x.reshape(-1, *x.shape[-3:]))
        return out.view(*lead, *out.shape[-2:])


class MultiViewRGBPerceiverEncoder(nn.Module):
    """obj_encoder.py:150-206: the Gato ViT's patch tokens of both views (16 per image) resampled by the Perceiver to
    `perceiver_num_queries` tokens.  The reference spells the sub-module `peceiver`; the state-dict keys keep that spelling."""

    def __init__(self, *, emb_dim: int, views, img_size, vit_patch_size=None, vit_width=None, vit_layers=None, vit_heads=None,
                 perceiver_num_queries: int, perceiver_num_blocks: int, perceiver_num_self_attends_per_block: int,
                 perceiver_num_self_attention_heads: int, perceiver_num_cross_attention_heads: int, perceiver_attention_probs_dropout_prob: float):
        super().__init__()
        from .perceiver import ObjectsPerceiverEncoder

        self._views = sorted(views)
        self._transformer_emb_dim = emb_dim
        self.cropped_img_encoder = GatoViTEncoder(img_size=img_size, output_dim=emb_dim, patch_size=vit_patch_size, width=vit_width,
                                                  layers=vit_layers, heads=vit_heads)
        self.peceiver = ObjectsPerceiverEncoder(emb_dim, num_latents=perceiver_num_queries, num_blocks=perceiver_num_blocks,
                                                num_self_attends_per_block=perceiver_num_self_attends_per_block,
                                                num_self_attention_heads=perceiver_num_self_attention_heads,
                                                num_cross_attention_heads=perceiver_num_cross_attention_heads,
                                                attention_probs_dropout_prob=perceiver_attention_probs_dropout_prob)

    def forward(self, rgb):
        views = self._views
        xs = [rgb[v] if rgb[v].dtype == torch.uint8 else rgb[v].to(torch.uint8) for v in views]
        lead = xs[0].shape[:-3]
        n = int(xs[0].numel() // (xs[0].shape[-3] * xs[0].shape[-2] * xs[0].shape[-1]))
        allx = torch.cat([x.reshape(-1, *x.shape[-3:]) for x in xs], dim=0)  # one batched pass through the shared ViT
        feats = self.cropped_img_encoder.vit.encode_u8(allx)  # (n_views * n, L, E)
        tokens = torch.cat([feats[i * n:(i + 1) * n] for i in range(len(views))], dim=1)  # (n, n_views * L, E)
        out = self.peceiver(tokens, torch.ones(tokens.shape[:2], dtype=torch.bool, device=tokens.device))
        return out.view(*lead, *out.shape[-2:])

    @property
    def output_dim(self):
        return self._transformer_emb_dim


class GatoMultiViewRGBEncoder(nn.Module):
    """obj_encoder.py:102-147: both views through the shared Gato ViT, patch tokens concatenated on the token axis."""

    def __init__(self, *, emb_dim: int, views, img_size, vit_patch_size=None, vit_width=None, vit_layers=None, vit_heads=None):
        super().__init__()
        self._views = sorted(views)
        self.output_dim = emb_dim
        self.cropped_img_encoder = GatoViTEncoder(img_size=img_size, patch_size=vit_patch_size, width=vit_width, layers=vit_layers,
                                                  heads=vit_heads, output_dim=emb_dim)

    def forward(self, rgb):
        views = self._views
        xs = [rgb[v] if rgb[v].dtype == torch.uint8 else rgb[v].to(torch.uint8) for v in views]
        lead = xs[0].shape[:-3]
        n = [int(x.numel() // (x.shape[-3] * x.shape[-2] * x.shape[-1])) for x in xs]
        allx = torch.cat([x.reshape(-1, *x.shape[-3:]) for x in xs], dim=0)  # one batched pass through the shared ViT
        feats = self.cropped_img_encoder.vit.encode_u8(allx)
        outs, r0 = [], 0
        for k in n:
            outs.append(feats[r0:r0 + k].view(*lead, *feats.shape[-2:]))
            r0 += k
        return torch.cat(outs, dim=-2)

    @property
    def img_patch_len(self):
        return self.cropped_img_encoder.vit.img_patch_len * len(self._views)
