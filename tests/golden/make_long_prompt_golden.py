#!/usr/bin/env python
"""Mint tests/golden/long_prompt.npz from the UNMODIFIED reference (run in the build container only).

    python tests/golden/make_long_prompt_golden.py

Two fixtures for prompts past the resident-K/V attention kernel's 384 keys:

  (a) policy.*  The reference `VIMAPolicy` of the 2M model with its XAttnGPT rebuilt at xattn_n_positions=512 (as bench.py builds
      workload cfg3x), B = 2: one prompt of exactly 512 tokens (480 words + one image of 32 object tokens), one ragged prompt of
      483 tokens.  forward_prompt_assembly -> forward_obs_token -> forward_action_token -> forward -> forward_action_decoder -> .mode().
  (b) t5.*      The reference `T5PromptEncoder` alone at Lp = 1000 (past 512, not a multiple of 64), B = 2: one full row and one
      ragged row.

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

XATTN_N_POSITIONS = 512
T5_LP, T5_B = 1000, 2


def policy_case():
    """2M model, B = 2, T = 2; prompt 0: 480 words + 1 image (Lp = 512), prompt 1: 451 words + 1 image (483 tokens)."""
    from oracle import synth

    return dataclasses.replace(synth.CASES["cfg3_small"], name="long512", model="2M", B=2, T=2, n_words=480, n_imgs=1, seed=50)


def t5_inputs():
    """(x (B, Lp, 768) fp32, mask (B, Lp) bool): row 0 all valid; row 1 valid up to 700 with ~25 % holes (token 0 valid)."""
    import torch

    from oracle import detgen

    x = detgen.uniform("long_prompt.t5.x", (T5_B, T5_LP, 768))
    mask = torch.ones(T5_B, T5_LP, dtype=torch.bool)
    mask[1] = detgen.randint("long_prompt.t5.mask", (T5_LP,), 0, 4) > 0
    mask[1, 700:] = False
    mask[1, 0] = True
    return x, mask


def build_reference_policy(ref_vima):
    import torch

    from oracle import detgen, synth

    case = policy_case()
    cfg = synth.MODEL_CFGS[case.model]
    torch.manual_seed(0)
    policy = ref_vima.VIMAPolicy(**cfg)
    rnn = sys.modules["vima.nn"]
    policy.xattn_gpt = rnn.XAttnGPT(cfg["embed_dim"], n_layer=cfg["xf_n_layers"], n_head=cfg["sattn_n_heads"], dropout=0.1,
                                    xattn_n_head=cfg["xattn_n_heads"], xattn_ff_expanding=4, xattn_n_positions=XATTN_N_POSITIONS,
                                    use_geglu=True)
    detgen.fill_module_(policy)
    return policy.eval(), case


def run_policy(ref_vima, out):
    import torch

    from oracle import synth

    policy, case = build_reference_policy(ref_vima)
    DataDict = sys.modules["vima.utils"].DataDict
    with torch.no_grad():
        token_types, word_batch, image_batch = synth.make_prompt(case)
        prompt_tokens, prompt_masks = policy.forward_prompt_assembly((token_types, word_batch, DataDict(image_batch)))
        assert prompt_tokens.shape[0] == XATTN_N_POSITIONS and 384 < int(prompt_masks[1].sum()) < XATTN_N_POSITIONS
        pack(out, "policy.prompt_tokens", prompt_tokens)
        pack(out, "policy.prompt_masks", prompt_masks)
        obs = synth.make_obs(case)
        obs_tokens, obs_masks = policy.forward_obs_token(DataDict({"ee": obs["ee"], "objects": DataDict(obs["objects"])}))
        pack(out, "policy.obs_tokens", obs_tokens)
        pack(out, "policy.obs_masks", obs_masks)
        action_tokens = policy.forward_action_token(synth.make_actions(case, case.T))
        pack(out, "policy.action_tokens", action_tokens)
        predicted = policy.forward(obs_token=obs_tokens, obs_mask=obs_masks, action_token=action_tokens, prompt_token=prompt_tokens,
                                   prompt_token_mask=prompt_masks)
        pack(out, "policy.predicted", predicted)
        dists = policy.forward_action_decoder(predicted[-1:])
        raw_logits = torch.cat([mlp(predicted[-1:]) for k in policy.action_decoder._decoders for mlp in policy.action_decoder._decoders[k].mlps],
                               dim=-1)
        pack(out, "policy.logits_raw", raw_logits)
        for k, v in dists.items():
            m = v.mode()
            assert m.dtype == torch.int64
            pack(out, f"policy.mode.{k}", m)


def run_t5(out):
    import torch

    from oracle import detgen

    enc = sys.modules["vima.nn"].T5PromptEncoder()
    detgen.fill_module_(enc)
    enc.eval()
    x, mask = t5_inputs()
    with torch.no_grad():
        y = enc(x, attention_mask=mask, batch_first=True)
    pack(out, "t5.mask", mask)
    pack(out, "t5.out", y)


def main():
    from oracle.ref_shim import load_reference

    ref_vima = load_reference()
    import torch

    torch.set_num_threads(os.cpu_count())
    t0 = time.time()
    out = {}
    run_policy(ref_vima, out)
    run_t5(out)
    path = os.path.join(HERE, "long_prompt.npz")
    np.savez_compressed(path, **out)
    print(f"long_prompt: {len(out)} arrays -> {path} ({os.path.getsize(path)/1e3:.0f} kB) in {time.time()-t0:.1f}s")


if __name__ == "__main__":
    main()
