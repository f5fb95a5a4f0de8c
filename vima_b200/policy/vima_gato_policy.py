"""VIMAGatoPolicy: the decoder-only baseline (reference: /root/reference/vima/policy/vima_gato_policy.py:11-326).

One causal sequence [encoded prompt | separator | interleaved obs / action history] through `HFGPT` -- BASELINE.json
configs[4], the causal-only kernel path.  Same surface as the reference (constructor, sub-module names, methods);
the reference's `self.device` bug (:133) does not exist here -- the device comes from the inputs.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from .. import engine as eng
from .. import nn as vnn
from ..utils import *  # noqa: F401,F403
from .vima_policy import VIMAPolicy, history_cols, history_steps


class VIMAGatoPolicy(nn.Module):
    def __init__(self, *, embed_dim: int, vocab_size=40478, n_positions=512, n_layer=12, n_head=12, dropout: float = 0.1):
        super().__init__()
        self.embed_dim = embed_dim
        self.transformer = vnn.HFGPT(n_embd=embed_dim, use_geglu=True, vocab_size=vocab_size, n_positions=n_positions, n_layer=n_layer,
                                     n_head=n_head, dropout=dropout)
        self.prompt_sep_token = nn.Parameter(torch.zeros(embed_dim))
        self.obj_encoder = vnn.GatoMultiViewRGBEncoder(emb_dim=embed_dim, views=["front", "top"], img_size=(64, 128), vit_patch_size=32,
                                                       vit_width=768, vit_layers=4, vit_heads=24)
        self._obj_xf_num_queries = self.obj_encoder.img_patch_len
        self.end_effector_encoder = vnn.Embedding(num_embeddings=2, embedding_dim=2)
        obs_feat_dim = self.obj_encoder.output_dim + 2
        self.obs_fusion_layer = nn.Identity() if obs_feat_dim == embed_dim else vnn.Linear(obs_feat_dim, embed_dim)
        self.action_encoder = vnn.ActionEmbedding(
            output_dim=embed_dim,
            embed_dict={
                "pose0_position": vnn.ContinuousActionEmbedding(output_dim=256, input_dim=2, hidden_dim=256, hidden_depth=1),
                "pose0_rotation": vnn.ContinuousActionEmbedding(output_dim=256, input_dim=4, hidden_dim=256, hidden_depth=1),
                "pose1_position": vnn.ContinuousActionEmbedding(output_dim=256, input_dim=2, hidden_dim=256, hidden_depth=1),
                "pose1_rotation": vnn.ContinuousActionEmbedding(output_dim=256, input_dim=4, hidden_dim=256, hidden_depth=1),
            },
        )
        self.action_decoder = vnn.ActionDecoder(
            input_dim=embed_dim,
            action_dims={"pose0_position": [50, 100], "pose0_rotation": [50] * 4, "pose1_position": [50, 100], "pose1_rotation": [50] * 4},
            hidden_dim=512, hidden_depth=2, activation="relu", norm_type=None, last_layer_gain=0.01,
        )
        self.prompt_embedding = vnn.WordEmbedding()
        self.t5_prompt_encoder = vnn.T5PromptEncoder()
        self.t5_prompt_encoder_post_layer = (
            nn.Identity() if embed_dim == self.t5_prompt_encoder.output_dim else vnn.Linear(self.t5_prompt_encoder.output_dim, embed_dim, bias=False)
        )
        self.prompt_obj_post_layer = vnn.build_mlp(self.obj_encoder.output_dim, hidden_dim=768, output_dim=768, hidden_depth=2)
        self._views = ["front", "top"]
        self._n_discrete_x_bins = 50
        self._n_discrete_y_bins = 100
        self._n_discrete_z_bins = 50
        self._n_discrete_rot_bins = 50
        self._wc = eng.WeightCache(self)
        self._bins = {}

    @property
    def device(self):
        return next(self.parameters()).device

    # --------------------------------------------------------------------------------------------------
    def forward(self, obs_token: torch.Tensor, action_token: Optional[torch.Tensor], prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor):
        """obs_token (T,B,Q,E), action_token (T-1,B,E)|None, prompt_token (Lp,B,E), prompt_token_mask (B,Lp) -> (T,B,E)
        (vima_gato_policy.py:120-191)."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        ctx = eng.ctx_for(obs_token)
        T, B, Q, E = obs_token.shape
        assert Q == self._obj_xf_num_queries
        Lp = prompt_token.shape[0]
        La = 0 if action_token is None else action_token.shape[0]
        Ls = T * Q + La
        L = Lp + 1 + Ls
        dev = obs_token.device
        tokens = torch.empty((L, B, E), dtype=torch.float32, device=dev)
        tokens[:Lp].copy_(prompt_token)
        tokens[Lp].copy_(self.prompt_sep_token.detach().unsqueeze(0).expand(B, E))
        ones = torch.ones((T, B, Q), dtype=torch.uint8, device=dev)
        scratch_m = torch.empty((B, Ls), dtype=torch.uint8, device=dev)
        scratch_p = torch.empty((B, Ls), dtype=torch.int64, device=dev)
        ctx.assemble_history(obs_token.float().contiguous(), ones, None if action_token is None else action_token.float().contiguous(),
                             tokens[Lp + 1:], scratch_m, scratch_p)
        mask = torch.empty((B, L), dtype=torch.uint8, device=dev)
        position_ids = torch.empty((B, L), dtype=torch.int64, device=dev)
        ctx.gato_positions(eng.as_u8(prompt_token_mask), L, mask, position_ids)
        tokens_out = self.transformer(tokens, custom_mask=mask.view(torch.bool), batch_first=False, position_ids=position_ids)
        return tokens_out[Lp + 1 + Q - 1 :: Q + 1]

    # --------------------------------------------------------------------------------------------------
    # Cached decode (DESIGN.md 7 (f)1; not in the reference, which re-runs [prompt | separator | history] every step).  The prompt
    # and separator are prefilled once into the first Lp+1 columns of the self-attention cache; a step appends [a_{t-1}, o_t^1..Q].
    def _prompt_prefix(self, ctx, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor):
        """[prompt | separator] tokens (Lp+1,n,E), mask (n,Lp+1) uint8 and position ids (n,Lp+1): the first Lp+1 rows of `forward`."""
        Lp, n, E = prompt_token.shape
        dev = prompt_token.device
        tokens = torch.empty((Lp + 1, n, E), dtype=torch.float32, device=dev)
        tokens[:Lp].copy_(prompt_token)
        tokens[Lp].copy_(self.prompt_sep_token.detach().unsqueeze(0).expand(n, E))
        mask = torch.empty((n, Lp + 1), dtype=torch.uint8, device=dev)
        pos = torch.empty((n, Lp + 1), dtype=torch.int64, device=dev)
        ctx.gato_positions(eng.as_u8(prompt_token_mask).contiguous(), Lp + 1, mask, pos)
        return tokens, mask, pos

    def _check_prompt(self, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor, n: int, Lmax: int) -> None:
        Lp, nb, E = prompt_token.shape
        if nb != n or E != self.embed_dim or tuple(prompt_token_mask.shape) != (n, Lp):
            raise ValueError(f"expected prompt_token (Lp, {n}, {self.embed_dim}) and a ({n}, Lp) mask, got {tuple(prompt_token.shape)} / "
                             f"{tuple(prompt_token_mask.shape)}")
        if Lp + 1 >= Lmax:
            raise ValueError(f"a prompt of {Lp} tokens + separator leaves no room in max_tokens={Lmax}")

    def _decode_weights(self) -> "eng.WeightState":
        """What a decode cache's rows are computed from: the decoder and the separator token (the step's tokens are the caller's)."""
        return eng.WeightState([self.transformer], slots=[(self, "prompt_sep_token")])

    def _check_obs(self, Q: int) -> None:
        if Q != self._obj_xf_num_queries:
            raise ValueError(f"an observation is {self._obj_xf_num_queries} tokens, got {Q}")

    def start_decode(self, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor, *, max_tokens: Optional[int] = None):
        """Open a K/V cache for a batch of episodes and prefill [prompt | separator]: prompt_token (Lp,B,E), prompt_token_mask
        (B,Lp); `max_tokens` columns per episode, prompt and separator included (default: the decoder's n_positions, which bounds
        the whole sequence).  Feed it to `forward_step` once per environment step."""
        ctx = eng.ctx_for(prompt_token)
        Lp, B, E = prompt_token.shape
        n_pos = self.transformer.n_positions
        Lmax = n_pos if max_tokens is None else int(max_tokens)
        if Lmax > n_pos:
            raise ValueError(f"max_tokens={Lmax} exceeds n_positions={n_pos}")
        self._check_prompt(prompt_token, prompt_token_mask, B, Lmax)
        p = eng.prec()
        cache = vnn.DecodeCache(B=B, Lmax=Lmax, E=E, n_layer=self.transformer.n_layer, device=prompt_token.device, split=p.split,
                                precision=p.name, weights=self._decode_weights())
        cache.prefix = Lp + 1  # columns before the first step
        self.transformer.prefill(cache, list(range(B)), *self._prompt_prefix(ctx, prompt_token, prompt_token_mask))
        return cache

    def forward_step(self, cache, obs_token: torch.Tensor, prev_action_token: Optional[torch.Tensor]):
        """One environment step through the cache: obs_token (1,B,Q,E), prev_action_token (1,B,E) (None at the first step) ->
        predicted action token (1,B,E); equals `forward(...)[-1:]` over the whole history.  Every history token is valid, so the
        step's position ids are n_valid + arange (vima_gato_policy.py:172-183)."""
        ctx = eng.ctx_for(obs_token)
        _, B, Q, E = obs_token.shape
        self._check_obs(Q)
        if (prev_action_token is None) != (cache.L == cache.prefix):
            raise ValueError("forward_step: exactly one action token per previous step is required")
        L = Q + (0 if prev_action_token is None else 1)
        from ..nn.xattn_gpt import check_cache_append

        check_cache_append(cache, B, L, E, eng.prec())  # every refusal happens before the cache is touched
        new = obs_token[0].float()
        if prev_action_token is not None:
            new = torch.cat([prev_action_token[0].float().unsqueeze(1), new], dim=1)
        new = new.contiguous()
        dev = obs_token.device
        pos = cache.n_valid[:, None] + torch.arange(L, dtype=torch.int64, device=dev)[None, :]
        ones = torch.ones((B, L), dtype=torch.bool, device=dev)
        out = self.transformer(new, custom_mask=ones, position_ids=pos, batch_first=True, cache=cache)
        cache.n_valid += L
        return out[:, -1:].transpose(0, 1)

    # Slot decode: each row of the batch holds one episode at its own length (VIMAPolicy.open_slots ... capture_step_slots).  A
    # slot's columns [0, Lp+1) hold its prompt and separator; the step kernels are VIMAPolicy's with an all-ones obs mask, so their
    # position rule n_valid + cumsum - 1 is Gato's n_valid + arange.
    def open_slots(self, n_slots: int, *, max_tokens: Optional[int] = None, kv_pool_tokens: Optional[int] = None):
        """Allocate a SlotDecodeCache of `n_slots` slots (all inactive) of `max_tokens` columns each, prompt and separator included
        (default: the decoder's n_positions), in the current precision mode, its K/V in a pool of `kv_pool_tokens` tokens
        (VIMAPolicy.open_slots)."""
        w = self.transformer.lm.positions_embed.weight
        eng.ctx_for(w)
        n_pos = self.transformer.n_positions
        Lmax = n_pos if max_tokens is None else int(max_tokens)
        if not 2 < Lmax <= n_pos:
            raise ValueError(f"max_tokens={Lmax} outside (2, n_positions={n_pos}]")
        if n_slots < 1:
            raise ValueError("n_slots must be >= 1")
        p = eng.prec()
        return vnn.SlotDecodeCache(S=int(n_slots), Lmax=Lmax, Lp_cap=0, E=self.embed_dim, n_layer=self.transformer.n_layer, device=w.device,
                                   split=p.split, precision=p.name, weights=self._decode_weights(), kv_pool_tokens=kv_pool_tokens)

    def admit(self, cache, slots, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor) -> None:
        """Start a new episode in each of `slots` (replacing whatever they held): prompt_token (Lp,n,E), prompt_token_mask (n,Lp).
        Prefills the n new [prompt | separator] sequences only, on the current stream."""
        ctx = eng.ctx_for(prompt_token)
        s = cache.slot_index(slots)
        if cache.Lp_cap:
            raise ValueError("admit: this SlotDecodeCache was opened for a cross-attention decoder")
        self._check_prompt(prompt_token, prompt_token_mask, len(s), cache.Lmax)
        cache.check_precision(eng.prec())
        cache.check_prefix(s, prompt_token.shape[0] + 1)  # prompt + separator, in pages the prefill scatters into
        if not s:
            return
        self.transformer.prefill(cache, s, *self._prompt_prefix(ctx, prompt_token, prompt_token_mask))

    def admit_history(self, cache, slots, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor, obs_token: torch.Tensor,
                      action_token: torch.Tensor, steps) -> None:
        """VIMAPolicy.admit_history with every obs token valid: obs_token (T,n,Q,E), action_token (T,n,E), steps n host ints in
        [0, T].  Slot slots[j]'s columns become [prompt | separator | o_0, a_0, ..., o_{k-1}] (k = steps[j]), the first
        Lp + 1 + k(Q+1) - 1 tokens of `forward`, prefilled in one batched pass over the decoder."""
        s = cache.slot_index(slots)
        if cache.Lp_cap:
            raise ValueError("admit_history: this SlotDecodeCache was opened for a cross-attention decoder")
        self._check_prompt(prompt_token, prompt_token_mask, len(s), cache.Lmax)
        k, T, Q = history_steps(cache, s, obs_token, None, action_token, steps)
        self._check_obs(Q)
        Lp, n, E = prompt_token.shape
        lens = [Lp + 1 + history_cols(x, Q) for x in k]
        cache.check_precision(eng.prec())
        cache.check_admit_history(s, lens)
        if not s:
            return
        ctx = eng.ctx_for(prompt_token)
        dev = prompt_token.device
        cache.reserve_history(s, lens, [x > 0 for x in k])
        steps32 = cache.device_ints(k).to(torch.int32)
        act = action_token.float().contiguous()
        L = max(lens)
        tokens = torch.empty((L, n, E), dtype=torch.float32, device=dev)
        tokens[:Lp].copy_(prompt_token)
        tokens[Lp].copy_(self.prompt_sep_token.detach().unsqueeze(0).expand(n, E))
        mask = torch.empty((n, L), dtype=torch.uint8, device=dev)
        pos = torch.empty((n, L), dtype=torch.int64, device=dev)
        ctx.gato_positions(eng.as_u8(prompt_token_mask).contiguous(), L, mask, pos)  # columns [0, Lp+1); the rest is the history's
        ctx.slot_assemble_history(obs_token.float().contiguous(), None, act, steps32, Lp + 1, tokens, mask, pos)
        self.transformer.prefill(cache, s, tokens, mask, pos, history=(steps32, act, Q, Lp + 1))

    release = VIMAPolicy.release
    fork_slots = VIMAPolicy.fork_slots
    swap_out = VIMAPolicy.swap_out
    swap_in = VIMAPolicy.swap_in
    refresh_weights = VIMAPolicy.refresh_weights

    def step_slots(self, cache, obs_token: torch.Tensor, action_token: Optional[torch.Tensor]) -> torch.Tensor:
        """One environment step of every slot: obs_token (1,S,Q,E), action_token (1,S,E) (each slot's previous action; ignored for
        slots at their first step; None = all zeros) -> predicted action token (1,S,E).  For an active slot the row equals
        `forward(...)[-1:]` at B=1 over that episode's own history; an inactive slot's row is unspecified."""
        eng.ctx_for(obs_token)
        _, S, Q, E = obs_token.shape
        self._check_obs(Q)
        cache.check_step(S, Q, E, eng.prec())
        cache.reserve_step(Q)
        out = self._slot_step(cache, obs_token, action_token)
        cache.advance_host(Q)
        return out

    def _slot_step(self, cache, obs_token, action_token):
        """The device side of `step_slots` (static shapes, no host synchronisation; captured by GraphedSlotStep)."""
        ctx = eng.ctx_for(obs_token)
        _, S, Q, E = obs_token.shape
        dev = obs_token.device
        L = Q + 1
        obs = obs_token[0].float().contiguous()
        ones = torch.ones((S, Q), dtype=torch.uint8, device=dev)
        act = torch.zeros((S, E), dtype=torch.float32, device=dev) if action_token is None else action_token[0].float().contiguous()
        tokens = torch.empty((S * L, E), dtype=torch.float32, device=dev)
        step_mask = torch.empty((S, L), dtype=torch.uint8, device=dev)
        pos = torch.empty((S, L), dtype=torch.int64, device=dev)
        ctx.slot_step_begin(obs, ones, act, Lmax=cache.Lmax, len_=cache.len, n_valid=cache.n_valid, has_action=cache.has_action,
                            active=cache.active, tokens=tokens, step_mask=step_mask, pos=pos, q_pos=cache.q_pos, slot_mask=cache.mask)
        x = self.transformer(tokens.view(S, L, E), custom_mask=step_mask.view(torch.bool), position_ids=pos, batch_first=True, cache=cache)
        out = torch.empty((S, E), dtype=torch.float32, device=dev)
        ctx.slot_step_end(x.reshape(S * L, E), S, Q, E, step_mask, len_=cache.len, n_valid=cache.n_valid, has_action=cache.has_action,
                          active=cache.active, out=out)
        return out.view(1, S, E)

    def capture_step_slots(self, cache, obs_token: torch.Tensor, action_token: torch.Tensor, *, warmup: int = 2):
        """`step_slots` for this (S, Q) captured into one CUDA graph (vima_b200.graphs.GraphedSlotStep); the cache's slot state is
        left as it was.  Call the result like step_slots without the cache: g(obs_token, action_token)."""
        from ..graphs import GraphedSlotStep

        self._check_obs(1 if obs_token.dim() == 3 else obs_token.shape[2])
        return GraphedSlotStep(self, cache, obs_token, action_token, warmup=warmup)

    # Closed loop: VIMAPolicy's with this class's _slot_step (VIMA-GPT and VIMA-Flamingo inherit both methods; VIMA-GPT's obs_token
    # is (1,S,E)).
    _act_slots = VIMAPolicy._act_slots
    _act_step = VIMAPolicy._act_step

    def act_slots(self, cache, obs_token: torch.Tensor, *, sampler=None):
        """obs_token (1,S,Q,E) -> (actions, log_prob, entropy), as VIMAPolicy.act_slots with every obs token valid."""
        self._check_obs(1 if obs_token.dim() == 3 else obs_token.shape[2])
        return self._act_slots(cache, (obs_token,), sampler)

    def capture_act_slots(self, cache, obs_token: torch.Tensor, *, sampler=None, warmup: int = 2):
        """`act_slots` captured into one CUDA graph, as VIMAPolicy.capture_act_slots; call the result as g(obs_token)."""
        from ..graphs import GraphedSlotStep

        self._check_obs(1 if obs_token.dim() == 3 else obs_token.shape[2])
        return GraphedSlotStep(self, cache, obs_token, warmup=warmup, act=True, sampler=sampler)

    def forward_prompt_assembly(self, prompts):
        """(token_types, word_batch, image_batch{"rgb": {view: (n_img,3,64,128)}}) -> (Lp,B,E), (B,Lp) bool (:193-251)."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        raw_prompts_token_type, word_batch, image_batch = prompts
        ref = image_batch["rgb"][sorted(self._views)[0]]
        ctx = eng.ctx_for(ref)
        p = eng.prec()
        dev = ref.device
        nq = self._obj_xf_num_queries
        word_ids = word_batch.to(device=dev, dtype=torch.int64).contiguous()
        img_emb = self.prompt_obj_post_layer(self.obj_encoder(**image_batch))  # (n_img, nq, 768)
        D = img_emb.shape[-1]
        lens = []
        for raw in raw_prompts_token_type:
            n = 0
            for item in raw:
                if item == 0:
                    n += 1
                elif item == 1:
                    n += nq
                else:
                    raise ValueError(f"Invalid prompt token type {item}")
            lens.append(n)
        B, Lp = len(raw_prompts_token_type), max(lens)
        kind = np.zeros((B, Lp), dtype=np.int32)
        index = np.zeros((B, Lp), dtype=np.int32)
        wp = ip = 0
        for b, raw in enumerate(raw_prompts_token_type):
            pos = 0
            for item in raw:
                if item == 0:
                    kind[b, pos], index[b, pos] = 1, wp
                    wp += 1
                    pos += 1
                else:
                    kind[b, pos:pos + nq] = 2
                    index[b, pos:pos + nq] = ip * nq + np.arange(nq)
                    ip += 1
                    pos += nq
        tokens = torch.empty((B, Lp, D), dtype=torch.float32, device=dev)
        masks_u8 = torch.empty((B, Lp), dtype=torch.uint8, device=dev)
        all_valid = torch.ones(max(img_emb.shape[0] * nq, 1), dtype=torch.uint8, device=dev)
        ctx.gather_prompt(torch.from_numpy(kind).to(dev), torch.from_numpy(index).to(dev), word_ids,
                          self.prompt_embedding._embed_layer.weight.detach(), img_emb.reshape(-1, D).contiguous(), all_valid, B, Lp, D, tokens, masks_u8)
        prompt_masks = masks_u8.view(torch.bool)
        need_post = not isinstance(self.t5_prompt_encoder_post_layer, nn.Identity)
        out32, out16 = self.t5_prompt_encoder.encode(tokens, prompt_masks, want16=need_post)
        if need_post:
            pl = self.t5_prompt_encoder_post_layer
            pw = self._wc.get("t5post", (pl.weight,), lambda: eng.pack_linear(ctx, pl.weight, None, transposed=False, p=p))
            out32, _ = eng.gemm(ctx, out16, pw, p, want_f32=True)
        return out32.view(B, Lp, -1).transpose(0, 1), prompt_masks

    def forward_obs_token(self, obs):
        """obs {"rgb": {view: (T,B,3,64,128) u8}, "ee": (T,B)} -> (T,B,Q,E)  (:253-262)."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        rgbs, ee = obs["rgb"], obs["ee"]
        lead = tuple(ee.shape[:2])
        ctx = eng.ctx_for(ee)
        p = eng.prec()
        img_feats = self.obj_encoder(rgb=rgbs)  # (T,B,Q,E)
        Q, E = img_feats.shape[-2], img_feats.shape[-1]
        if isinstance(self.obs_fusion_layer, nn.Identity):
            raise NotImplementedError("embed_dim == obs feature dim never happens for VIMA-Gato (E + 2 != E)")
        rows = lead[0] * lead[1] * Q
        a = eng.to_operand(ctx, img_feats.reshape(rows, E), p, pad_cols=E + 2)
        ctx.fill_ee(ee.to(torch.int64).contiguous(), self.end_effector_encoder.weight.detach().float().contiguous(), lead[0] * lead[1], Q,
                    a.hi, a.lo, E, 0, dtype=p.dtype)
        fl = self.obs_fusion_layer
        pw = self._wc.get("fusion", (fl.weight, fl.bias), lambda: eng.pack_linear(ctx, fl.weight, fl.bias, transposed=False, p=p))
        out32, _ = eng.gemm(ctx, a, pw, p, want_f32=True)
        return out32.view(*lead, Q, self.embed_dim)

    def forward_action_token(self, action):
        return self.action_encoder(self._de_discretize_actions(action))

    def forward_action_decoder(self, predicted_action_tokens: torch.Tensor):
        return self.action_decoder(predicted_action_tokens)

    discretize_action = VIMAPolicy.discretize_action
    _de_discretize_actions = VIMAPolicy._de_discretize_actions
    _bin_tensor = VIMAPolicy._bin_tensor
    postprocess_actions = VIMAPolicy.postprocess_actions
