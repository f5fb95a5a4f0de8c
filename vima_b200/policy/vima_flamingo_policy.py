"""VIMAFlamingoPolicy: the XAttnGPT decoder over Perceiver-resampled image tokens
(reference: /root/reference/vima/policy/vima_flamingo_policy.py:10-291).

The decoder, prompt encoder and heads are those of VIMAPolicy; an observation is two 64x128 views -> shared Gato ViT ->
16 patch tokens -> Perceiver resampler -> 4 tokens.  `forward` follows the reference exactly: every history token valid,
DEFAULT position ids (no cumsum of masks), the prompt mask on the cross-attention keys.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from .. import engine as eng
from .. import nn as vnn
from ..utils import *  # noqa: F401,F403
from .vima_gato_policy import VIMAGatoPolicy
from .vima_policy import VIMAPolicy


class VIMAFlamingoPolicy(VIMAGatoPolicy):
    def __init__(self, *, embed_dim: int, dt_n_layers: int, dt_n_heads: int, xattn_n_heads: int):
        nn.Module.__init__(self)
        self.embed_dim = embed_dim
        self.xattn_gpt = vnn.XAttnGPT(embed_dim, n_layer=dt_n_layers, n_head=dt_n_heads, dropout=0.1, xattn_n_head=xattn_n_heads,
                                      xattn_ff_expanding=4, xattn_n_positions=256, use_geglu=True)
        self.obj_encoder = vnn.MultiViewRGBPerceiverEncoder(
            emb_dim=embed_dim, views=["front", "top"], img_size=(64, 128), vit_patch_size=32, vit_width=768, vit_layers=4, vit_heads=24,
            perceiver_num_queries=4, perceiver_num_blocks=4, perceiver_num_self_attends_per_block=4, perceiver_num_self_attention_heads=8,
            perceiver_num_cross_attention_heads=8, perceiver_attention_probs_dropout_prob=0.1)
        self._obj_xf_num_queries = 4
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

    def forward(self, obs_token: torch.Tensor, action_token: Optional[torch.Tensor], prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor):
        """obs_token (T,B,4,E), action_token (T-1,B,E)|None, prompt_token (Lp,B,E), prompt_token_mask (B,Lp) -> (T,B,E)
        (vima_flamingo_policy.py:129-163)."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        ctx = eng.ctx_for(obs_token)
        T, B, Q, E = obs_token.shape
        assert Q == self._obj_xf_num_queries
        La = 0 if action_token is None else action_token.shape[0]
        L = T * Q + La
        dev = obs_token.device
        tokens = torch.empty((L, B, E), dtype=torch.float32, device=dev)
        ones = torch.ones((T, B, Q), dtype=torch.uint8, device=dev)
        scratch_m = torch.empty((B, L), dtype=torch.uint8, device=dev)
        scratch_p = torch.empty((B, L), dtype=torch.int64, device=dev)
        ctx.assemble_history(obs_token.float().contiguous(), ones, None if action_token is None else action_token.float().contiguous(), tokens,
                             scratch_m, scratch_p)
        out = self.xattn_gpt(obs_action_tokens=tokens, prompt_tokens=prompt_token, prompt_mask=prompt_token_mask)
        return out[Q - 1 :: Q + 1]

    # --------------------------------------------------------------------------------------------------
    # Cached and slot decode: VIMAPolicy's (the same XAttnGPT decoder) with the two differences of `forward` above: every obs token
    # is valid, and the prompt position ids are the default arange.  Every decode method is defined here, so none of VIMA-Gato's
    # decoder-only versions is inherited.
    def _prompt_positions(self, ctx, pmask_u8: torch.Tensor) -> torch.Tensor:
        n, Lp = pmask_u8.shape
        return self.xattn_gpt.xattn_position_ids[None, :Lp].expand(n, Lp).contiguous()

    def _ones(self, obs_token: torch.Tensor) -> torch.Tensor:
        return torch.ones(obs_token.shape[:3], dtype=torch.bool, device=obs_token.device)

    def start_decode(self, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor, *, max_tokens: Optional[int] = None):
        """prompt_token (Lp,B,E), prompt_token_mask (B,Lp); room for `max_tokens` history tokens (default: n_positions)."""
        return VIMAPolicy.start_decode(self, prompt_token, prompt_token_mask, max_tokens=max_tokens)

    def forward_step(self, cache, obs_token: torch.Tensor, prev_action_token: Optional[torch.Tensor]):
        """obs_token (1,B,Q,E), prev_action_token (1,B,E) (None at the first step) -> (1,B,E); equals `forward(...)[-1:]`."""
        eng.ctx_for(obs_token)
        self._check_obs(obs_token.shape[2])
        return VIMAPolicy.forward_step(self, cache, obs_token, self._ones(obs_token), prev_action_token)

    def open_slots(self, n_slots: int, *, max_tokens: Optional[int] = None, max_prompt_tokens: int = 256,
                   kv_pool_tokens: Optional[int] = None, prompt_pool_tokens: Optional[int] = None):
        return VIMAPolicy.open_slots(self, n_slots, max_tokens=max_tokens, max_prompt_tokens=max_prompt_tokens, kv_pool_tokens=kv_pool_tokens,
                                     prompt_pool_tokens=prompt_pool_tokens)

    def admit(self, cache, slots, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor) -> None:
        eng.ctx_for(prompt_token)
        return VIMAPolicy.admit(self, cache, slots, prompt_token, prompt_token_mask)

    def admit_history(self, cache, slots, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor, obs_token: torch.Tensor,
                      action_token: torch.Tensor, steps) -> None:
        """VIMAPolicy.admit_history with every obs token valid: obs_token (T,n,Q,E), action_token (T,n,E), steps n host ints."""
        eng.ctx_for(prompt_token)
        if obs_token.dim() == 4:
            self._check_obs(obs_token.shape[2])
        return VIMAPolicy._admit_history(self, cache, slots, prompt_token, prompt_token_mask, obs_token, None, action_token, steps)

    release = VIMAPolicy.release
    fork_slots = VIMAPolicy.fork_slots
    swap_out = VIMAPolicy.swap_out
    swap_in = VIMAPolicy.swap_in

    def step_slots(self, cache, obs_token: torch.Tensor, action_token: Optional[torch.Tensor]) -> torch.Tensor:
        """obs_token (1,S,Q,E), action_token (1,S,E) | None -> (1,S,E), as VIMAPolicy.step_slots with every obs token valid."""
        # the checks and host bookkeeping shared with VIMA-Gato; the device step is this class's _slot_step
        return VIMAGatoPolicy.step_slots(self, cache, obs_token, action_token)

    def _slot_step(self, cache, obs_token, action_token):
        return VIMAPolicy._slot_step(self, cache, obs_token, self._ones(obs_token), action_token)

    def capture_step_slots(self, cache, obs_token: torch.Tensor, action_token: torch.Tensor, *, warmup: int = 2):
        """`step_slots` captured into one CUDA graph; call the result as g(obs_token, action_token)."""
        from ..graphs import GraphedSlotStep

        self._check_obs(obs_token.shape[2])
        return GraphedSlotStep(self, cache, obs_token, action_token, warmup=warmup)

    # forward_prompt_assembly (:165-228) and forward_obs_token (:230-240) are the inherited token-per-query versions with
    # `_obj_xf_num_queries == 4`: the object encoder returns (n, 4, E).
