#!/usr/bin/env python
"""Mint tests/golden/long_history.npz from the UNMODIFIED reference (run in the build container only).

    python tests/golden/make_long_history_golden.py

Two fixtures for decoder histories past 768 keys, with the decoders built at n_positions = 1024 through the reference's public
constructors:

  (a) gato.*  `VIMAGatoPolicy(**GATO_CFGS["gato_tiny"], n_positions=1024)`, B = 2 with ragged prompts (135 and fewer tokens) and
      T = 45 steps: L = Lp + 17 T = 900 decoder tokens (900 mod 128 = 4, so the last query tile holds 4 rows).
      forward_prompt_assembly -> forward_obs_token -> forward_action_token -> forward -> raw logits -> .mode().
  (b) policy.*  The reference `VIMAPolicy` of the 2M model with its XAttnGPT rebuilt at n_positions=1024, B = 2, 16 object slots
      per view (Q = 32) with ragged object masks, T = 28 steps: L = 33 T - 1 = 923 decoder tokens.  Same chain.

Weights come from `oracle.detgen`, inputs from `oracle.synth` / `detgen`, stored strided like make_golden.py.  The cases are
defined here rather than in `synth.CASES`, which other tests and bench.py read.
"""
from __future__ import annotations

import dataclasses
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests.golden.make_golden import pack  # noqa: E402

N_POSITIONS = 1024
GATO_L = 900
POLICY_L = 923


def gato_case():
    """gato_tiny, B = 2, T = 45; prompt 0: 119 words + 1 image (Lp = 135), prompt 1 ragged (fewer words)."""
    from oracle import synth

    return dataclasses.replace(synth.GATO_CASES["gato_small"], name="long_gato", B=2, T=45, n_words=119, n_imgs=1, ragged=True, seed=60)


def policy_case():
    """2M model, B = 2, T = 28, 16 object slots per view with ragged masks; prompt 0: 8 words + 1 image (Lp = 40)."""
    from oracle import synth

    return dataclasses.replace(synth.CASES["cfg3_small"], name="long_hist", model="2M", B=2, T=28, n_slots=16, n_words=8, n_imgs=1,
                               ragged=True, seed=61)


def build_reference_gato(ref_vima):
    import torch

    from oracle import detgen, synth

    case = gato_case()
    torch.manual_seed(0)
    policy = ref_vima.VIMAGatoPolicy(**synth.GATO_CFGS[case.model], n_positions=N_POSITIONS)
    detgen.fill_module_(policy)
    return policy.eval(), case


def build_reference_policy(ref_vima):
    import torch

    from oracle import detgen, synth

    case = policy_case()
    cfg = synth.MODEL_CFGS[case.model]
    torch.manual_seed(0)
    policy = ref_vima.VIMAPolicy(**cfg)
    rnn = sys.modules["vima.nn"]
    policy.xattn_gpt = rnn.XAttnGPT(cfg["embed_dim"], n_positions=N_POSITIONS, n_layer=cfg["xf_n_layers"], n_head=cfg["sattn_n_heads"],
                                    dropout=0.1, xattn_n_head=cfg["xattn_n_heads"], xattn_ff_expanding=4, xattn_n_positions=256,
                                    use_geglu=True)
    detgen.fill_module_(policy)
    return policy.eval(), case


def raw_logits(policy, predicted):
    import torch

    return torch.cat([mlp(predicted[-1:]) for k in policy.action_decoder._decoders for mlp in policy.action_decoder._decoders[k].mlps],
                     dim=-1)


def run_gato(ref_vima, out):
    import torch

    from oracle import synth

    policy, case = build_reference_gato(ref_vima)
    DataDict = sys.modules["vima.utils"].DataDict
    with torch.no_grad():
        token_types, word_batch, image_batch = synth.make_gato_prompt(case)
        prompt_tokens, prompt_masks = policy.forward_prompt_assembly((token_types, word_batch, DataDict(image_batch)))
        pack(out, "gato.prompt_tokens", prompt_tokens)
        pack(out, "gato.prompt_masks", prompt_masks)
        obs = synth.make_gato_obs(case)
        obs_tokens = policy.forward_obs_token(DataDict({"ee": obs["ee"], "rgb": DataDict(obs["rgb"])}))
        pack(out, "gato.obs_tokens", obs_tokens)
        action_tokens = policy.forward_action_token(synth.make_actions(case, case.T))
        pack(out, "gato.action_tokens", action_tokens)
        T, B, Q, _ = obs_tokens.shape
        L = prompt_tokens.shape[0] + 1 + T * Q + T - 1
        assert L == GATO_L and 768 < L <= N_POSITIONS and 1 <= L % 128 <= 8, L
        predicted = policy.forward(obs_token=obs_tokens, action_token=action_tokens, prompt_token=prompt_tokens,
                                   prompt_token_mask=prompt_masks)
        pack(out, "gato.predicted", predicted)
        dists = policy.forward_action_decoder(predicted[-1:])
        pack(out, "gato.logits_raw", raw_logits(policy, predicted))
        for k, v in dists.items():
            m = v.mode()
            assert m.dtype == torch.int64
            pack(out, f"gato.mode.{k}", m)


def run_policy(ref_vima, out):
    import torch

    from oracle import synth

    policy, case = build_reference_policy(ref_vima)
    DataDict = sys.modules["vima.utils"].DataDict
    with torch.no_grad():
        token_types, word_batch, image_batch = synth.make_prompt(case)
        prompt_tokens, prompt_masks = policy.forward_prompt_assembly((token_types, word_batch, DataDict(image_batch)))
        pack(out, "policy.prompt_tokens", prompt_tokens)
        pack(out, "policy.prompt_masks", prompt_masks)
        obs = synth.make_obs(case)
        obs_tokens, obs_masks = policy.forward_obs_token(DataDict({"ee": obs["ee"], "objects": DataDict(obs["objects"])}))
        pack(out, "policy.obs_tokens", obs_tokens)
        pack(out, "policy.obs_masks", obs_masks)
        action_tokens = policy.forward_action_token(synth.make_actions(case, case.T))
        pack(out, "policy.action_tokens", action_tokens)
        T, B, Q, _ = obs_tokens.shape
        assert T * Q + T - 1 == POLICY_L and 768 < POLICY_L <= N_POSITIONS and not bool(obs_masks.all())
        predicted = policy.forward(obs_token=obs_tokens, obs_mask=obs_masks, action_token=action_tokens, prompt_token=prompt_tokens,
                                   prompt_token_mask=prompt_masks)
        pack(out, "policy.predicted", predicted)
        dists = policy.forward_action_decoder(predicted[-1:])
        pack(out, "policy.logits_raw", raw_logits(policy, predicted))
        for k, v in dists.items():
            m = v.mode()
            assert m.dtype == torch.int64
            pack(out, f"policy.mode.{k}", m)


def main():
    from oracle.ref_shim import load_reference

    ref_vima = load_reference()
    import torch

    torch.set_num_threads(os.cpu_count())
    t0 = time.time()
    out = {}
    run_gato(ref_vima, out)
    run_policy(ref_vima, out)
    path = os.path.join(HERE, "long_history.npz")
    np.savez_compressed(path, **out)
    print(f"long_history: {len(out)} arrays -> {path} ({os.path.getsize(path)/1e3:.0f} kB) in {time.time()-t0:.1f}s")


if __name__ == "__main__":
    main()
