"""VIMAGPTPolicy: the decoder-only baseline with ONE token per observation and per prompt image
(reference: /root/reference/vima/policy/vima_gpt_policy.py:10-316).

Same causal sequence as VIMA-Gato, [encoded prompt | separator | o0 a0 o1 a1 ...], through `HFGPT`; the image encoder is
the CLS-token rectangular ViT applied to both views with the two features concatenated (2E wide).  Constructor,
sub-module names (state-dict keys) and methods follow the reference; the arithmetic runs on the same sm_90a kernels.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from .. import engine as eng
from .. import nn as vnn
from ..utils import *  # noqa: F401,F403
from .vima_gato_policy import VIMAGatoPolicy


class VIMAGPTPolicy(VIMAGatoPolicy):
    def __init__(self, *, embed_dim: int, vocab_size=40478, n_positions=512, n_layer=12, n_head=12, dropout: float = 0.1):
        nn.Module.__init__(self)
        self.embed_dim = embed_dim
        self.transformer = vnn.HFGPT(n_embd=embed_dim, use_geglu=True, vocab_size=vocab_size, n_positions=n_positions, n_layer=n_layer,
                                     n_head=n_head, dropout=dropout)
        self.prompt_sep_token = nn.Parameter(torch.zeros(embed_dim))
        self.obj_encoder = vnn.MultiViewRGBEncoder(img_size=(64, 128), emb_dim=embed_dim, views=["front", "top"], vit_patch_size=32,
                                                   vit_width=768, vit_layers=4, vit_heads=24)
        self._obj_xf_num_queries = 1
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
        """obs_token (T,B,E), action_token (T-1,B,E)|None, prompt_token (Lp,B,E), prompt_token_mask (B,Lp) -> (T,B,E)
        (vima_gpt_policy.py:119-176): the Gato layout with one token per observation."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        return VIMAGatoPolicy.forward(self, obs_token.unsqueeze(2), action_token, prompt_token, prompt_token_mask)

    # Cached and slot decode: VIMA-Gato's with one token per observation.  start_decode, open_slots, admit, release and
    # capture_step_slots are the inherited ones (capture takes obs_token (1,S,E)).
    def forward_step(self, cache, obs_token: torch.Tensor, prev_action_token: Optional[torch.Tensor]):
        """obs_token (1,B,E), prev_action_token (1,B,E) (None at the first step) -> (1,B,E)."""
        return VIMAGatoPolicy.forward_step(self, cache, obs_token.unsqueeze(2), prev_action_token)

    def admit_history(self, cache, slots, prompt_token: torch.Tensor, prompt_token_mask: torch.Tensor, obs_token: torch.Tensor,
                      action_token: torch.Tensor, steps) -> None:
        """obs_token (T,n,E), action_token (T,n,E), steps n host ints: VIMAGatoPolicy.admit_history with one token per observation."""
        return VIMAGatoPolicy.admit_history(self, cache, slots, prompt_token, prompt_token_mask, obs_token.unsqueeze(2), action_token, steps)

    def step_slots(self, cache, obs_token: torch.Tensor, action_token: Optional[torch.Tensor]) -> torch.Tensor:
        """obs_token (1,S,E), action_token (1,S,E) | None -> (1,S,E)."""
        return VIMAGatoPolicy.step_slots(self, cache, obs_token.unsqueeze(2), action_token)

    def _slot_step(self, cache, obs_token, action_token):
        """obs_token (1,S,E) from a captured graph's inputs, or (1,S,1,E) from step_slots."""
        return VIMAGatoPolicy._slot_step(self, cache, obs_token.unsqueeze(2) if obs_token.dim() == 3 else obs_token, action_token)

    # forward_prompt_assembly (vima_gpt_policy.py:178-238) is the inherited one with `_obj_xf_num_queries == 1`: the image
    # encoder returns (n_img, 2E), the post-MLP (n_img, 768), one prompt slot per image.

    def forward_obs_token(self, obs):
        """obs {"rgb": {view: (T,B,3,64,128) u8}, "ee": (T,B)} -> (T,B,E)  (vima_gpt_policy.py:240-251)."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        rgbs, ee = obs["rgb"], obs["ee"]
        lead = tuple(ee.shape[:2])
        ctx = eng.ctx_for(ee)
        p = eng.prec()
        if isinstance(self.obs_fusion_layer, nn.Identity):
            raise NotImplementedError("2E + 2 == E never happens")
        F2 = self.obj_encoder.output_dim
        a = self.obj_encoder.encode16(rgbs, pad_cols=2)  # [T*B, 2E + 2] operands; the ee columns are filled next
        ctx.fill_ee(ee.to(torch.int64).contiguous(), self.end_effector_encoder.weight.detach().float().contiguous(), lead[0] * lead[1], 1,
                    a.hi, a.lo, F2, 0, dtype=p.dtype)
        fl = self.obs_fusion_layer
        pw = self._wc.get("fusion", (fl.weight, fl.bias), lambda: eng.pack_linear(ctx, fl.weight, fl.bias, transposed=False, p=p))
        out32, _ = eng.gemm(ctx, a, pw, p, want_f32=True)
        return out32.view(*lead, self.embed_dim)
