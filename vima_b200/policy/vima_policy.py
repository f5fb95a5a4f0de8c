"""VIMAPolicy: the drop-in policy class (reference: /root/reference/vima/policy/vima_policy.py:11-322).

Same constructor, sub-module names (state-dict prefixes) and five entry methods as the reference; every tensor op
between the inputs and the returned tensors runs in the sm_90a kernels of libvima_b200.so.  Host Python only builds
the prompt index map from `token_types` (lists of ints) and launches kernels; there are no per-token Python loops on
tensors and no host synchronisation after the first call's input checks.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch
import torch.nn as nn

from .. import engine as eng
from .. import nn as vnn
from ..utils import *  # noqa: F401,F403  (the reference re-exports vima.utils here)


def history_steps(cache, s: list, obs_token: torch.Tensor, obs_mask: Optional[torch.Tensor], action_token: torch.Tensor, steps) -> tuple:
    """admit_history's checks of a recorded history for the destination slots `s` (before any state is touched): obs_token
    (T,n,Q,E), obs_mask (T,n,Q) or None, action_token (T,n,E), steps n host ints in [0, T] -> (steps as a list of ints, T, Q)."""
    if isinstance(steps, torch.Tensor):
        if steps.device.type != "cpu":
            raise TypeError("admit_history: steps must be host ints (a device tensor would need a synchronising read)")
        steps = steps.tolist()
    k = [int(x) for x in steps]
    n, E = len(s), cache.E
    if obs_token.dim() != 4 or obs_token.shape[1] != n or obs_token.shape[3] != E or obs_token.shape[2] < 1:
        raise ValueError(f"admit_history: {n} slots need obs_token (T, {n}, Q, {E}), got {tuple(obs_token.shape)}")
    T, _, Q, _ = obs_token.shape
    if obs_mask is not None and tuple(obs_mask.shape) != (T, n, Q):
        raise ValueError(f"admit_history: obs_mask must be ({T}, {n}, {Q}), got {tuple(obs_mask.shape)}")
    if tuple(action_token.shape) != (T, n, E):
        raise ValueError(f"admit_history: action_token must be ({T}, {n}, {E}), got {tuple(action_token.shape)}")
    if len(k) != n or any(not 0 <= x <= T for x in k):
        raise ValueError(f"admit_history: steps must be {n} ints in [0, T={T}], got {k}")
    return k, T, Q


def history_cols(k: int, Q: int) -> int:
    """Cache columns of k completed environment steps at obs width Q: [o_0, a_0, ..., a_{k-2}, o_{k-1}]."""
    return k * (Q + 1) - 1 if k else 0


class VIMAPolicy(nn.Module):
    def __init__(self, *, embed_dim: int, xf_n_layers: int, sattn_n_heads: int, xattn_n_heads: int):
        super().__init__()
        self.embed_dim = embed_dim
        self.xattn_gpt = vnn.XAttnGPT(embed_dim, n_layer=xf_n_layers, n_head=sattn_n_heads, dropout=0.1, xattn_n_head=xattn_n_heads,
                                      xattn_ff_expanding=4, xattn_n_positions=256, use_geglu=True)
        self.obj_encoder = vnn.ObjEncoder(transformer_emb_dim=embed_dim, views=["front", "top"], vit_output_dim=768, vit_resolution=32,
                                          vit_patch_size=16, vit_width=768, vit_layers=4, vit_heads=24, bbox_mlp_hidden_dim=768,
                                          bbox_mlp_hidden_depth=2)
        self.end_effector_encoder = vnn.Embedding(num_embeddings=2, embedding_dim=2)
        self.obs_fusion_layer = vnn.Linear(self.obj_encoder.output_dim + 2, embed_dim)
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

    def refresh_weights(self) -> None:
        """Drop every packed weight (the next call repacks from the parameters as they are).  Call it after writing parameters
        through `.data` (`param.data.copy_(t)`), which no version counter sees; every other update route is detected on its own
        (INTEGRATION.md).  Graphs captured and decode caches opened before it refuse to run."""
        eng.refresh_weights(self)

    # --------------------------------------------------------------------------------------------------
    def forward(self, obs_token: torch.Tensor, obs_mask: torch.Tensor, action_token: Optional[torch.Tensor], prompt_token: torch.Tensor,
                prompt_token_mask: torch.Tensor):
        """obs_token (T,B,Q,E), obs_mask (T,B,Q) bool, action_token (T-1,B,E)|None, prompt_token (Lp,B,E),
        prompt_token_mask (B,Lp) bool -> predicted action tokens (T,B,E)   (vima_policy.py:116-159)."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        ctx = eng.ctx_for(obs_token)
        T, B, Q, E = obs_token.shape
        La = 0 if action_token is None else action_token.shape[0]
        L = T * Q + La
        dev = obs_token.device
        obs = obs_token.float().contiguous()
        act = None if action_token is None else action_token.float().contiguous()
        tokens = torch.empty((L, B, E), dtype=torch.float32, device=dev)
        masks_bl = torch.empty((B, L), dtype=torch.uint8, device=dev)
        pos_bl = torch.empty((B, L), dtype=torch.int64, device=dev)
        ctx.assemble_history(obs, eng.as_u8(obs_mask), act, tokens, masks_bl, pos_bl)
        pmask_u8 = eng.as_u8(prompt_token_mask)
        prompt_pos = torch.empty(pmask_u8.shape, dtype=torch.int64, device=dev)
        ctx.mask_cumsum(pmask_u8, prompt_pos)
        tokens_out = self.xattn_gpt(
            obs_action_tokens=tokens,
            prompt_tokens=prompt_token,
            prompt_mask=pmask_u8.view(torch.bool),
            obs_action_masks=masks_bl.view(torch.bool),
            obs_action_position_ids=pos_bl,
            prompt_position_ids=prompt_pos,
        )
        return tokens_out[Q - 1 :: Q + 1]

    # --------------------------------------------------------------------------------------------------
    # Incremental decode (SURVEY.md 8(f)1; not in the reference, which re-runs the whole history each step).
    def start_decode(self, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor, *, max_tokens: Optional[int] = None):
        """Open a K/V cache for a batch of episodes: prompt_token (Lp,B,E), prompt_token_mask (B,Lp); room for `max_tokens`
        history tokens per episode (default: the decoder's n_positions).  Feed it to `forward_step` once per environment step."""
        Lp, B, E = prompt_token.shape
        ctx = eng.ctx_for(prompt_token)
        Lmax = self.xattn_gpt.n_positions if max_tokens is None else int(max_tokens)
        if not 0 < Lmax <= self.xattn_gpt.n_positions:
            raise ValueError(f"max_tokens={Lmax} outside (0, n_positions={self.xattn_gpt.n_positions}]")
        cache = vnn.DecodeCache(B=B, Lmax=Lmax, E=E, n_layer=self.xattn_gpt.n_layer, device=prompt_token.device, split=eng.prec().split,
                                precision=eng.prec().name, weights=eng.WeightState([self.xattn_gpt]))
        pmask_u8 = eng.as_u8(prompt_token_mask)
        cache.prompt = (prompt_token, pmask_u8, self._prompt_positions(ctx, pmask_u8))
        return cache

    def _prompt_positions(self, ctx, pmask_u8: torch.Tensor) -> torch.Tensor:
        """Prompt position ids of the cached paths: cumsum(mask) - 1, as `forward` computes them (vima_policy.py:147)."""
        pos = torch.empty(pmask_u8.shape, dtype=torch.int64, device=pmask_u8.device)
        ctx.mask_cumsum(pmask_u8, pos)
        return pos

    def forward_step(self, cache, obs_token: torch.Tensor, obs_mask: torch.Tensor, prev_action_token: Optional[torch.Tensor]):
        """One environment step through the cache: obs_token (1,B,Q,E), obs_mask (1,B,Q), prev_action_token (1,B,E) (None at
        the first step) -> predicted action token (1,B,E); equals `forward(...)[-1:]` over the whole history.  Q may differ
        from step to step: scripts/example.py:139-171 re-pads every earlier step to the running maximum, but padded slots are
        masked keys with weight exactly 0 that do not advance position ids, so earlier steps can stay at the width they were
        appended with.  The prediction is read at the LAST slot passed (a padded one if the caller padded), as the reference does."""
        ctx = eng.ctx_for(obs_token)
        _, B, Q, E = obs_token.shape
        if (prev_action_token is None) != (cache.L == 0):
            raise ValueError("forward_step: exactly one action token per previous step is required")
        dev = obs_token.device
        # every refusal happens before the cache is touched (a failed step must leave n_valid / L consistent)
        from ..nn.xattn_gpt import check_cache_append

        check_cache_append(cache, B, Q + (0 if prev_action_token is None else 1), E, eng.prec())
        new = obs_token[0].float().transpose(0, 1)  # (Q,B,E)
        m_new = eng.as_u8(obs_mask[0])
        if prev_action_token is not None:
            new = torch.cat([prev_action_token.float(), new], dim=0)
            m_new = torch.cat([torch.ones((B, 1), dtype=torch.uint8, device=dev), m_new], dim=1)
        new, m_new = new.contiguous(), m_new.contiguous()
        pos = torch.empty(m_new.shape, dtype=torch.int64, device=dev)
        ctx.mask_cumsum(m_new, pos)
        pos += cache.n_valid[:, None]
        prompt_token, pmask_u8, prompt_pos = cache.prompt
        out = self.xattn_gpt(obs_action_tokens=new, prompt_tokens=prompt_token, prompt_mask=pmask_u8.view(torch.bool),
                             obs_action_masks=m_new.view(torch.bool), obs_action_position_ids=pos, prompt_position_ids=prompt_pos,
                             cache=cache)
        cache.n_valid += m_new.sum(dim=1)  # only after the decoder accepted the step
        return out[-1:]

    # --------------------------------------------------------------------------------------------------
    # Slot decode (DESIGN.md 7 (f)1): each row of the batch is a slot holding one episode at a time, so episodes start and finish
    # independently (a vectorised environment resets each of its environments on its own).
    def open_slots(self, n_slots: int, *, max_tokens: Optional[int] = None, max_prompt_tokens: int = 256,
                   kv_pool_tokens: Optional[int] = None, prompt_pool_tokens: Optional[int] = None):
        """Allocate a SlotDecodeCache of `n_slots` slots (all inactive) with room for `max_tokens` history tokens (default: the
        decoder's n_positions) and `max_prompt_tokens` prompt tokens per episode, in the current precision mode.  The slots' history
        K/V live in a shared pool of 64-token pages holding `kv_pool_tokens` tokens (default: n_slots * max_tokens, rounded up to
        whole pages per slot, so every slot can reach max_tokens at once); a smaller pool refuses a step it cannot cover.  Their
        projected prompt K/V live in a second pool of 64-token pages holding `prompt_pool_tokens` tokens (default: n_slots *
        max_prompt_tokens, rounded up the same way); a smaller pool refuses an admission it cannot cover, and forked slots share
        their source's prompt pages."""
        dev = self.xattn_gpt.positions_embed.weight.device
        eng.ctx_for(self.xattn_gpt.positions_embed.weight)
        Lmax = self.xattn_gpt.n_positions if max_tokens is None else int(max_tokens)
        if not 1 < Lmax <= self.xattn_gpt.n_positions:
            raise ValueError(f"max_tokens={Lmax} outside (1, n_positions={self.xattn_gpt.n_positions}]")
        if not 0 < max_prompt_tokens <= self.xattn_gpt.xattn_n_positions:
            raise ValueError(f"max_prompt_tokens={max_prompt_tokens} outside (0, {self.xattn_gpt.xattn_n_positions}]")
        if n_slots < 1:
            raise ValueError("n_slots must be >= 1")
        p = eng.prec()
        return vnn.SlotDecodeCache(S=int(n_slots), Lmax=Lmax, Lp_cap=int(max_prompt_tokens), E=self.embed_dim, n_layer=self.xattn_gpt.n_layer,
                                   device=dev, split=p.split, precision=p.name, weights=eng.WeightState([self.xattn_gpt]),
                                   kv_pool_tokens=kv_pool_tokens, prompt_pool_tokens=prompt_pool_tokens)

    def admit(self, cache, slots, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor) -> None:
        """Start a new episode in each of `slots` (replacing whatever they held): prompt_token (Lp,n,E), prompt_token_mask (n,Lp),
        Lp <= the cache's max_prompt_tokens.  Runs the prompt key/value GEMMs of the n prompts only, on the current stream."""
        s = cache.slot_index(slots)
        Lp, n, E = prompt_token.shape
        if n != len(s) or E != cache.E or tuple(prompt_token_mask.shape) != (n, Lp):
            raise ValueError(f"admit: {len(s)} slots need prompt_token (Lp, {len(s)}, {cache.E}) and a ({len(s)}, Lp) mask, got "
                             f"{tuple(prompt_token.shape)} / {tuple(prompt_token_mask.shape)}")
        if Lp > cache.Lp_cap:
            raise ValueError(f"admit: prompt of {Lp} tokens exceeds the cache's max_prompt_tokens={cache.Lp_cap}")
        cache.check_precision(eng.prec())
        if not s:
            return
        ctx = eng.ctx_for(prompt_token)
        pmask_u8 = eng.as_u8(prompt_token_mask)
        self.xattn_gpt.admit_prompts(cache, s, prompt_token, pmask_u8, self._prompt_positions(ctx, pmask_u8))

    def release(self, cache, slots) -> None:
        """Mark `slots` inactive (their episodes ended) and return their K/V pages to the pool; they keep computing on whatever is
        passed (at column 0, over the zero page) but never advance."""
        s = cache.slot_index(slots)
        if s:
            cache.active.index_fill_(0, cache.device_ints(s), 0)
            cache.free_slots(s)
        for b in s:
            cache.active_host[b] = False

    def fork_slots(self, cache, src, dst) -> None:
        """Copy episodes between slots: after the call slot dst[i] holds slot src[i]'s episode exactly as it stands (its history,
        prompt, fed-back action and state), so the two continue from the same point; a source may repeat, a live destination's
        episode is replaced.  The history K/V pages are shared by reference and copied only when a sharer next writes into a
        partly filled one, so a fork takes no page and the pool never refuses it.  Group sampling: admit once, then
        `fork_slots(cache, [s] * (k - 1), others)` and `act_slots(..., sampler=...)`.  Refuses (ValueError, nothing touched) an
        inactive or out-of-range source, repeated destinations, a slot that is both, and a cache of another precision mode or of
        changed weights.  Queued on the current stream, no host synchronisation."""
        s, d = cache.check_fork(src, dst)
        cache.check_precision(eng.prec())
        cache.fork(s, d)

    def swap_out(self, cache, slots) -> list:
        """Park the episodes of `slots` in pinned host memory and release the slots: -> one vima_b200.SwappedEpisode per slot, holding
        the episode's history K/V pages, prompt K/V pages, fed-back action and state, so `swap_in` can resume it later exactly where
        it stands.  The slots' pages go back to the pools (a page still shared with a fork stays with the fork), so a driver whose
        overcommitted pool cannot cover the next step can preempt episodes instead of dropping them; `cache.kv_pages_freed_by(slots)`
        says how many pages a choice of slots frees.  Refuses (ValueError, nothing touched) an inactive, out-of-range or repeated
        slot and a cache of another precision mode or of changed weights.  Queued on the current stream, no host synchronisation:
        the episodes' host buffers are filled once the stream reaches the copies."""
        s = cache.check_swap_out(slots)
        cache.check_precision(eng.prec())
        return cache.swap_out(s)

    def swap_in(self, cache, slots, episodes) -> None:
        """Resume `episodes` (SwappedEpisode, from `swap_out` of this cache or of another cache of the same policy, precision mode,
        max_tokens and max_prompt_tokens) in `slots`: slot slots[i] continues episodes[i] bit for bit as if it had never left.  A live
        destination's episode is replaced; an episode can be swapped in again, into several slots or caches (each takes private
        pages).  Refuses (ValueError, nothing touched) out-of-range or repeated slots, a count that does not match, an episode of
        another precision mode, shape or policy or of weights changed since its swap-out, a cache of changed weights, and pools that
        cannot cover the episodes' pages (counting those the destinations give back).  Queued on the current stream, no host
        synchronisation."""
        s, eps = cache.check_swap_in(slots, episodes)
        cache.check_precision(eng.prec())
        cache.swap_in(s, eps)

    def admit_history(self, cache, slots, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor, obs_token: torch.Tensor,
                      obs_mask: torch.Tensor, action_token: torch.Tensor, steps) -> None:
        """Start each of `slots` (replacing whatever it held) mid-way through an episode whose history was recorded: prompt_token
        (Lp,n,E) / prompt_token_mask (n,Lp) as in `admit`, obs_token (T,n,Q,E), obs_mask (T,n,Q), action_token (T,n,E) (the embedding
        of the action taken after each observation), steps n host ints: episode j has completed steps[j] <= T environment steps.
        Rows t >= steps[j] are never read (they may hold anything), so episodes of different lengths share one call, padded to the
        longest.  Afterwards slot slots[j] holds episode j as if it had been admitted and stepped steps[j] times at width Q (a history
        stepped at other widths is re-padded to Q: padded obs tokens are masked keys that do not advance position ids); its next
        step feeds [a_{k-1}, o_k] and act_slots feeds back action_token[steps[j] - 1, j].  One batched prefill pass over the decoder
        (forward's arithmetic over n x the longest history), so the resumed K/V match the stepped ones within the bars of
        forward_step, not bit for bit.  Uses: resuming preempted episodes by recomputation instead of swapping, carrying running
        episodes across a weight update (open a new cache and admit their histories), starting from a recorded trajectory.  Refuses
        (ValueError, nothing touched) bad or repeated slots, shapes or steps, histories past max_tokens, prompts past
        max_prompt_tokens, pools that cannot cover the pages (counting those the destinations give back), and a cache of another
        precision mode or of changed weights; steps on the device raise TypeError.  Queued on the current stream, no host
        synchronisation."""
        self._admit_history(cache, slots, prompt_token, prompt_token_mask, obs_token, obs_mask, action_token, steps)

    def _admit_history(self, cache, slots, prompt_token, prompt_token_mask, obs_token, obs_mask, action_token, steps) -> None:
        """admit_history of the cross-attention policies (obs_mask None: every obs token valid)."""
        s = cache.slot_index(slots)
        k, T, Q = history_steps(cache, s, obs_token, obs_mask, action_token, steps)
        Lp, n, E = prompt_token.shape
        if not cache.Lp_cap:
            raise ValueError("admit_history: this SlotDecodeCache was opened for a decoder-only policy")
        if n != len(s) or E != cache.E or tuple(prompt_token_mask.shape) != (n, Lp):
            raise ValueError(f"admit_history: {len(s)} slots need prompt_token (Lp, {len(s)}, {cache.E}) and a ({len(s)}, Lp) mask, got "
                             f"{tuple(prompt_token.shape)} / {tuple(prompt_token_mask.shape)}")
        if Lp > cache.Lp_cap:
            raise ValueError(f"admit_history: prompt of {Lp} tokens exceeds the cache's max_prompt_tokens={cache.Lp_cap}")
        lens = [history_cols(x, Q) for x in k]
        cache.check_precision(eng.prec())
        cache.check_admit_history(s, lens, Lp)
        if not s:
            return
        ctx = eng.ctx_for(prompt_token)
        dev = prompt_token.device
        cache.reserve_history(s, lens, [x > 0 for x in k], Lp)
        steps32 = cache.device_ints(k).to(torch.int32)
        obs = obs_token.float().contiguous()
        act = action_token.float().contiguous()
        L = max(lens)
        tokens = torch.empty((L, n, E), dtype=torch.float32, device=dev)
        mask = torch.empty((n, L), dtype=torch.uint8, device=dev)
        pos = torch.empty((n, L), dtype=torch.int64, device=dev)
        ctx.slot_assemble_history(obs, None if obs_mask is None else eng.as_u8(obs_mask), act, steps32, 0, tokens, mask, pos)
        pmask_u8 = eng.as_u8(prompt_token_mask)
        self.xattn_gpt.prefill_history(cache, s, tokens, mask, pos, prompt_token, pmask_u8, self._prompt_positions(ctx, pmask_u8), steps32,
                                       act, Q)

    def step_slots(self, cache, obs_token: torch.Tensor, obs_mask: torch.Tensor, action_token: Optional[torch.Tensor]) -> torch.Tensor:
        """One environment step of every slot: obs_token (1,S,Q,E), obs_mask (1,S,Q), action_token (1,S,E) (the previous action of
        each slot; ignored for slots at their first step; None = all zeros) -> predicted action token (1,S,E).  For an active slot
        the row equals `forward(...)[-1:]` at B=1 over that episode's own history; an inactive slot's row is unspecified."""
        _, S, Q, E = obs_token.shape
        cache.check_step(S, Q, E, eng.prec())  # every refusal happens before any state is touched
        cache.reserve_step(Q)
        out = self._slot_step(cache, obs_token, obs_mask, action_token)
        cache.advance_host(Q)
        return out

    def _slot_step(self, cache, obs_token, obs_mask, action_token):
        """The device side of `step_slots`: static shapes for a fixed (S, Q), no host synchronisation (captured by GraphedSlotStep)."""
        ctx = eng.ctx_for(obs_token)
        _, S, Q, E = obs_token.shape
        dev = obs_token.device
        L = Q + 1
        obs = obs_token[0].float().contiguous()
        m = eng.as_u8(obs_mask[0])
        act = torch.zeros((S, E), dtype=torch.float32, device=dev) if action_token is None else action_token[0].float().contiguous()
        tokens = torch.empty((S * L, E), dtype=torch.float32, device=dev)
        step_mask = torch.empty((S, L), dtype=torch.uint8, device=dev)
        pos = torch.empty((S, L), dtype=torch.int64, device=dev)
        ctx.slot_step_begin(obs, m, act, Lmax=cache.Lmax, len_=cache.len, n_valid=cache.n_valid, has_action=cache.has_action,
                            active=cache.active, tokens=tokens, step_mask=step_mask, pos=pos, q_pos=cache.q_pos, slot_mask=cache.mask)
        x = self.xattn_gpt(obs_action_tokens=tokens.view(S, L, E), obs_action_position_ids=pos, prompt_tokens=None,
                           obs_action_masks=step_mask.view(torch.bool), batch_first=True, cache=cache)
        out = torch.empty((S, E), dtype=torch.float32, device=dev)
        ctx.slot_step_end(x.reshape(S * L, E), S, Q, E, step_mask, len_=cache.len, n_valid=cache.n_valid, has_action=cache.has_action,
                          active=cache.active, out=out)
        return out.view(1, S, E)

    def capture_step_slots(self, cache, obs_token: torch.Tensor, obs_mask: torch.Tensor, action_token: torch.Tensor, *, warmup: int = 2):
        """`step_slots` for this (S, Q) captured into one CUDA graph (vima_b200.graphs.GraphedSlotStep); the cache's slot state is
        left as it was.  Call the result like step_slots without the cache: g(obs_token, obs_mask, action_token)."""
        from ..graphs import GraphedSlotStep

        return GraphedSlotStep(self, cache, obs_token, obs_mask, action_token, warmup=warmup)

    # Closed loop (DESIGN.md 7 (f)5): step_slots, the action heads, the choice of action and its embedding, all on the device; the
    # embedding goes to cache.action_token, the action input of the slot's next step.
    def act_slots(self, cache, obs_token: torch.Tensor, obs_mask: torch.Tensor, *, sampler=None):
        """One environment step of every slot that also acts: obs_token (1,S,Q,E), obs_mask (1,S,Q) -> (actions, log_prob, entropy),
        dicts keyed like `forward_action_decoder(...)[k].mode()` with int64 / fp32 / fp32 tensors (1,S,n_k).  The action is each
        head's mode when `sampler` is None, else a draw from `sampler` (vima_b200.ActionSampler; all heads of all keys are one
        MultiCategorical in key order, one draw per call).  The step's action input is the embedding of each slot's previous action,
        which the call itself left in cache.action_token."""
        return self._act_slots(cache, (obs_token, obs_mask), sampler)

    def _act_slots(self, cache, inputs, sampler):
        """act_slots of all four policies: `inputs` are those of the policy's _slot_step before the action token."""
        obs_token = inputs[0]
        S, E = obs_token.shape[1], obs_token.shape[-1]
        Q = obs_token.shape[2] if obs_token.dim() == 4 else 1
        cache.check_step(S, Q, E, eng.prec())
        cache.reserve_step(Q)
        if "_act_grouped" not in self.__dict__:  # head buffers of its own, apart from forward_action_decoder's (one shape resident)
            self._act_grouped = vnn.action._GroupedMLPs()
        out = self._act_step(cache, *inputs, sampler=sampler, grouped=self._act_grouped)
        cache.advance_host(Q)
        return out

    def _act_step(self, cache, *inputs, sampler=None, grouped=None):
        """The device side of act_slots (static shapes, no host synchronisation; captured by GraphedSlotStep)."""
        S, E = cache.S, cache.E
        x = self._slot_step(cache, *inputs, cache.action_token.view(1, S, E))
        dec = self.action_decoder
        eng.uses(dec)  # fp32 parameters read by the kernels directly
        keys = list(dec._decoders.keys())
        logits, dims, spans = vnn.ActionDecoder.head_logits([dec._decoders[k] for k in keys], x.view(S, E), grouped)
        acts, lp, ent = vnn.action.sample_heads(logits, dims, sampler=sampler, log_prob=True, entropy=True)
        out = tuple({k: t[:, a:b].view(1, S, b - a) for k, (a, b) in zip(keys, spans)} for t in (acts, lp, ent))
        cache.action_token.copy_(self.forward_action_token(out[0]).view(S, E))
        return out

    def capture_act_slots(self, cache, obs_token: torch.Tensor, obs_mask: torch.Tensor, *, sampler=None, warmup: int = 2):
        """`act_slots` for this (S, Q) captured into one CUDA graph (vima_b200.graphs.GraphedSlotStep); the cache's slot state, its
        fed-back action tokens and the sampler's counter are left as they were.  Call the result as g(obs_token, obs_mask)."""
        from ..graphs import GraphedSlotStep

        return GraphedSlotStep(self, cache, obs_token, obs_mask, warmup=warmup, act=True, sampler=sampler)

    # --------------------------------------------------------------------------------------------------
    def forward_prompt_assembly(self, prompts):
        """(token_types, word_batch, image_batch) -> prompt tokens (Lp,B,E), masks (B,Lp) bool  (vima_policy.py:161-240)."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        raw_prompts_token_type, word_batch, image_batch = prompts
        ref = image_batch["cropped_img"][sorted(self._views)[0]]
        ctx = eng.ctx_for(ref)
        p = eng.prec()
        dev = ref.device
        word_ids = word_batch.to(device=dev, dtype=torch.int64).contiguous()
        img_feats = self.obj_encoder(**image_batch)                       # (n_img, Q, E) fp32
        n_img, n_max_objs = img_feats.shape[0], img_feats.shape[-2]
        img_emb = self.prompt_obj_post_layer(img_feats)                   # (n_img, Q, 768) fp32
        D = img_emb.shape[-1]
        obj_mask = torch.cat([image_batch["mask"][v].reshape(n_img, -1) for v in sorted(self._views)], dim=-1)

        # host: index map from the token-type lists (ints only)
        lens = []
        for raw in raw_prompts_token_type:
            n = 0
            for item in raw:
                if item == 0:
                    n += 1
                elif item == 1:
                    n += n_max_objs
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
                    kind[b, pos : pos + n_max_objs] = 2
                    index[b, pos : pos + n_max_objs] = ip * n_max_objs + np.arange(n_max_objs)
                    ip += 1
                    pos += n_max_objs
        kind_d = torch.from_numpy(kind).to(dev)
        index_d = torch.from_numpy(index).to(dev)
        tokens = torch.empty((B, Lp, D), dtype=torch.float32, device=dev)
        masks_u8 = torch.empty((B, Lp), dtype=torch.uint8, device=dev)
        ctx.gather_prompt(kind_d, index_d, word_ids, self.prompt_embedding._embed_layer.weight.detach(), img_emb.reshape(-1, D).contiguous(),
                          eng.as_u8(obj_mask.reshape(-1)), B, Lp, D, tokens, masks_u8)
        prompt_masks = masks_u8.view(torch.bool)
        if self.t5_prompt_encoder is None:
            return tokens.transpose(0, 1), prompt_masks
        need_post = not isinstance(self.t5_prompt_encoder_post_layer, nn.Identity)
        out32, out16 = self.t5_prompt_encoder.encode(tokens, prompt_masks, want16=need_post)
        if need_post:
            pl = self.t5_prompt_encoder_post_layer
            pw = self._wc.get("t5post", (pl.weight,), lambda: eng.pack_linear(ctx, pl.weight, None, transposed=False, p=p))
            out32, _ = eng.gemm(ctx, out16, pw, p, want_f32=True)
        prompt_tokens = out32.view(B, Lp, -1).transpose(0, 1)
        return prompt_tokens, prompt_masks

    # --------------------------------------------------------------------------------------------------
    def forward_obs_token(self, obs):
        """obs {"ee": (T,B) i64, "objects": {cropped_img,bbox,mask}x{front,top}} -> (T,B,Q,E), (T,B,Q) bool  (:242-259)."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        objects, ee = obs["objects"], obs["ee"]
        lead = tuple(ee.shape[:2])
        ctx = eng.ctx_for(ee)
        p = eng.prec()
        img_feats = self.obj_encoder(cropped_img=objects["cropped_img"], bbox=objects["bbox"], mask=objects["mask"])  # (T,B,Q,E)
        Q, E = img_feats.shape[-2], img_feats.shape[-1]
        rows = lead[0] * lead[1] * Q
        a = eng.to_operand(ctx, img_feats.reshape(rows, E), p, pad_cols=E + 2)   # [rows, E+8]: zero padded
        ctx.fill_ee(ee.to(torch.int64).contiguous(), self.end_effector_encoder.weight.detach().float().contiguous(), lead[0] * lead[1], Q,
                    a.hi, a.lo, E, 0, dtype=p.dtype)
        fl = self.obs_fusion_layer
        pw = self._wc.get("fusion", (fl.weight, fl.bias), lambda: eng.pack_linear(ctx, fl.weight, fl.bias, transposed=False, p=p))
        out32, _ = eng.gemm(ctx, a, pw, p, want_f32=True)
        obs_feats = out32.view(*lead, Q, self.embed_dim)
        obj_mask = torch.cat([objects["mask"][v].reshape(*lead, -1) for v in sorted(self._views)], dim=-1)
        return obs_feats, obj_mask

    # --------------------------------------------------------------------------------------------------
    def forward_action_token(self, action):
        return self.action_encoder(self._de_discretize_actions(action))

    def forward_action_decoder(self, predicted_action_tokens: torch.Tensor):
        return self.action_decoder(predicted_action_tokens)

    def discretize_action(self, action):
        """Training-side helper (vima_policy.py:267-299); not on the inference path."""
        device = action["pose0_position"].device
        bx = torch.linspace(0, 1, self._n_discrete_x_bins, device=device)
        by = torch.linspace(0, 1, self._n_discrete_y_bins, device=device)
        br = torch.linspace(0, 1, self._n_discrete_rot_bins, device=device)
        for k in ("pose0_position", "pose1_position"):
            action[k][..., 0] = torch.bucketize(action[k][..., 0].contiguous(), bx)
            action[k][..., 1] = torch.bucketize(action[k][..., 1].contiguous(), by)
        for k in ("pose0_rotation", "pose1_rotation"):
            action[k] = torch.bucketize(action[k].contiguous(), br)
        return {k: v.long() for k, v in action.items()}

    def postprocess_actions(self, actions, action_bounds_low: torch.Tensor, action_bounds_high: torch.Tensor):
        """The environment-facing step after the heads, scripts/example.py:199-232, in one kernel per action key: int64 bin
        indices -> de-discretised, scaled to the action bounds and clamped positions; rotations mapped to [-1, 1].
        Bounds: float32 (..., 2) broadcast over the leading dims of the position indices, or one row per episode."""
        out = {}
        for k, v in actions.items():
            ctx = eng.ctx_for(v)
            width = v.shape[-1]
            idx = v.to(torch.int64).contiguous()
            n = idx.numel() // width
            if k.endswith("position"):
                bins = self._bin_tensor(True, width, v.device)
                lo = action_bounds_low.to(device=v.device, dtype=torch.float32).reshape(-1, width).contiguous()
                hi = action_bounds_high.to(device=v.device, dtype=torch.float32).reshape(-1, width).contiguous()
                if lo.shape != hi.shape or lo.shape[0] not in (1, n):
                    raise ValueError(f"action bounds must hold 1 or {n} rows of {width} values, got {tuple(lo.shape)} / {tuple(hi.shape)}")
                stride = 0 if lo.shape[0] == 1 else width
            else:
                bins = self._bin_tensor(False, width, v.device)
                key = ("rot_bounds", width, str(v.device))
                if key not in self._bins:
                    self._bins[key] = (torch.full((1, width), -1.0, device=v.device), torch.full((1, width), 1.0, device=v.device))
                lo, hi = self._bins[key]
                stride = 0
            o = torch.empty(idx.shape, dtype=torch.float32, device=v.device)
            ctx.action_postprocess(idx.view(-1, width), n, width, bins, lo, hi, stride, o)
            out[k] = o
        return out

    def _bin_tensor(self, is_position: bool, width: int, device):
        key = (is_position, width, str(device))
        if key not in self._bins:
            b = [float(self._n_discrete_x_bins), float(self._n_discrete_y_bins)] if is_position else [float(self._n_discrete_rot_bins)] * width
            self._bins[key] = torch.tensor(b, dtype=torch.float32).to(device)
        return self._bins[key]

    def _de_discretize_actions(self, actions):
        """int64 indices -> float / bins  (vima_policy.py:301-322)."""
        out = {}
        for k, v in actions.items():
            ctx = eng.ctx_for(v)
            width = v.shape[-1]
            bins = self._bin_tensor(k.endswith("position"), width, v.device)
            idx = v.to(torch.int64).contiguous()
            o = torch.empty(idx.shape, dtype=torch.float32, device=v.device)
            ctx.action_scale(idx.view(-1, width), idx.numel() // width, width, bins, o)
            out[k] = o
        return out
