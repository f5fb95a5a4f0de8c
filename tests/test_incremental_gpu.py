"""GPU: step-by-step decode through the K/V cache (VIMAPolicy.start_decode / forward_step, SURVEY.md 8(f)1) against the
reference-shaped full re-forward of the growing history (vima_policy.py:116-159 semantics) and against the CPU oracle."""
import pytest
import torch

from oracle import synth, vima_oracle as O
from tests.policy_runner import build_policy, to_dev
from tests.test_oracle_golden import oracle_state_dict
from tests.util import rel_l2

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode,tol", [("f16x3", 1e-3), ("f16f8", 1e-3)])
@pytest.mark.parametrize("case_name", ["cfg2_small", "ragged_4M", "cfg3_small"])  # cfg3_small: 200M shapes (11 layers, L=263, Lp=256)
def test_cached_steps_match_full_history(case_name, mode, tol):
    import vima_b200
    from vima_b200.utils import DataDict

    case = synth.CASES[case_name]
    cfg = synth.MODEL_CFGS[case.model]
    vima_b200.set_precision(mode)
    try:
        pol = build_policy(case.model)
        sd = oracle_state_dict(case.model)
        with torch.no_grad():
            tt, wb, ib = synth.make_prompt(case)
            p_tok, p_msk = pol.forward_prompt_assembly((tt, wb.cuda(), DataDict(to_dev(ib, "cuda"))))
            obs_tok, obs_msk = pol.forward_obs_token(DataDict(to_dev(synth.make_obs(case), "cuda")))  # (T,B,Q,E), (T,B,Q)
            T, B, Q, E = obs_tok.shape
            act_tok = pol.forward_action_token(to_dev(synth.make_actions(case, T), "cuda")) if T > 1 else None  # (T-1,B,E)
            cache = pol.start_decode(p_tok, p_msk, max_tokens=T * (Q + 1) - 1)
            for t in range(T):
                prev = None if t == 0 else act_tok[t - 1:t]
                step = pol.forward_step(cache, obs_tok[t:t + 1], obs_msk[t:t + 1], prev)
                full = pol.forward(obs_token=obs_tok[:t + 1], obs_mask=obs_msk[:t + 1], action_token=None if t == 0 else act_tok[:t],
                                   prompt_token=p_tok, prompt_token_mask=p_msk)[-1:]
                assert step.shape == (1, B, E)
                # same GEMM / LayerNorm kernels and per-row arithmetic; the attention of these rows runs on the wgmma kernel in the
                # cached step and -- when the full history leaves <= 8 rows past its last 128-row tile (t = 3: L = 131) -- on the
                # fp32 SIMT tail kernel in the re-forward: two roundings of the same product.  f16x3 keeps that at the 1e-6 level;
                # in f16f8 the e4m3 cross-term views of the following GEMMs re-quantise the difference (measured 1.4e-5)
                d = rel_l2(full.cpu(), step.cpu())
                assert d < (2e-6 if mode == "f16x3" else 5e-5), (t, d)
            assert cache.L == T * Q + T - 1
            # and the last step against the CPU oracle's full forward on the same tokens
            ref = O.policy_forward(sd, obs_tok.cpu(), obs_msk.cpu(), None if act_tok is None else act_tok.cpu(), p_tok.cpu(), p_msk.cpu(),
                                   n_head=cfg["sattn_n_heads"], xattn_n_head=cfg["xattn_n_heads"])[-1:]
            assert rel_l2(ref, step.cpu()) < tol
            with pytest.raises(ValueError):
                pol.forward_step(cache, obs_tok[:1], obs_msk[:1], None)  # cache is full / action token missing
    finally:
        vima_b200.set_precision("f16x3")


def test_growing_object_count_matches_repadded_history():
    """scripts/example.py:139-171 pads every cached step to the running maximum object count and re-runs the whole history;
    the cache appends each step's own slots instead.  Both give the same predicted token at every step."""
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = build_policy("4M")
    E, B, Lp = pol.embed_dim, 3, 12
    g = torch.Generator(device="cuda").manual_seed(21)
    p_tok = torch.randn(Lp, B, E, device="cuda", generator=g)
    p_msk = torch.ones(B, Lp, dtype=torch.bool, device="cuda")
    p_msk[1, 9:] = False
    slots = [2, 5, 1, 4, 5]
    obs = [torch.randn(1, B, q, E, device="cuda", generator=g) for q in slots]
    msk = [torch.rand(1, B, q, device="cuda", generator=g) > 0.3 for q in slots]
    for m in msk:
        m[..., 0] = True
    act = [torch.randn(1, B, E, device="cuda", generator=g) for _ in slots[:-1]]
    with torch.no_grad():
        cache = pol.start_decode(p_tok, p_msk)
        used = 0
        for t, q in enumerate(slots):
            qmax = max(slots[: t + 1])
            pad_o = [torch.cat([o, torch.zeros(1, B, qmax - o.shape[2], E, device="cuda")], 2) for o in obs[: t + 1]]
            pad_m = [torch.cat([m, torch.zeros(1, B, qmax - m.shape[2], dtype=torch.bool, device="cuda")], 2) for m in msk[: t + 1]]
            # the new step arrives padded to the running maximum (the prediction is read at its LAST slot, padded or not);
            # earlier steps stay in the cache at the width they had when they were appended
            step = pol.forward_step(cache, pad_o[t], pad_m[t], None if t == 0 else act[t - 1])
            used += qmax + (t > 0)
            full = pol.forward(obs_token=torch.cat(pad_o, 0), obs_mask=torch.cat(pad_m, 0), action_token=None if t == 0 else torch.cat(act[:t], 0),
                               prompt_token=p_tok, prompt_token_mask=p_msk)[-1:]
            d = rel_l2(full.cpu(), step.cpu())
            assert d < 2e-6, (t, d)
        assert cache.L == used
