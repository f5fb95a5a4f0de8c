"""Decoder histories past 512 keys: the streaming wgmma attention kernel (attention_tc.cu) with no key-length cap, and the policies
built at n_positions = 1024.

CPU:
  * the oracle's Gato and VIMAPolicy chains against tests/golden/long_history.npz (minted from the unmodified reference by
    tests/golden/make_long_history_golden.py): gato_tiny at n_positions = 1024 with L = 900 decoder tokens, and the 2M VIMAPolicy with
    its XAttnGPT at n_positions = 1024 with L = 923.
GPU:
  * the kernel against one fp64 statement of the reference attention at Lk = 513 .. 4096: causal self-attention and non-causal
    cross-attention, lockstep decode (kv_batch_rows / mask_ld / q_pos0) and slot decode (per-batch q_pos), with padded keys and a
    batch element whose first 600 keys are padded (the kernel's re-run of a tile whose rows have seen only padded keys);
  * keys past each slot's own length are never read: NaN there leaves the output bit-identical;
  * both policies against the fixture in f16x3, bf16x3 and f16f8;
  * forward_step, staggered step_slots and graph replay at Lmax = 1024 with histories past 768 tokens;
  * vnn.XAttnGPT cross-attending over a 1000-token prompt;
  * single-pass f16 past the resident mma.sync kernel's capacity is refused with the limit in the message.
"""
import math

import numpy as np
import pytest
import torch

from oracle import detgen, synth, vima_oracle as O
from tests.golden.make_long_history_golden import GATO_L, N_POSITIONS, POLICY_L, gato_case, policy_case
from tests.util import argmax_safe_mask, assert_close, golden_pick, load_golden, rel_l2

GOLDEN = "long_history"
ORACLE_TOL = 2e-5  # fp32 CPU vs fp32 CPU: summation-order noise only (as tests/test_oracle_golden.py)
POLICY_TOL = 1e-3  # north_star tolerance
BARS = {"f16x3": 2e-6, "bf16x3": 2e-5, "f16f8": 5e-5}  # cached step vs full re-forward: test_incremental_gpu.py's bars
DIMS = [n for d in O.ACTION_DIMS.values() for n in d]
STAGES = ("prompt_tokens", "obs_tokens", "action_tokens", "predicted", "logits_raw")


# ------------------------------------------------------------------------------------------------------------------------------
# oracle against the fixture (CPU)
# ------------------------------------------------------------------------------------------------------------------------------
def gato_state_dict():
    from oracle.state_dict_spec import gato_state_dict_spec

    spec = gato_state_dict_spec(**synth.GATO_CFGS[gato_case().model], n_positions=N_POSITIONS)
    return {k: w for k, w in ((k, detgen.weight_for(k, s)) for k, s in spec.items()) if w is not None}


def policy_state_dict():
    """The 2M VIMAPolicy with its XAttnGPT at n_positions = 1024, as detgen fills it."""
    from oracle.state_dict_spec import state_dict_spec, xattn_gpt_spec

    cfg = synth.MODEL_CFGS[policy_case().model]
    spec = {k: s for k, s in state_dict_spec(**cfg).items() if not k.startswith("xattn_gpt.")}
    spec.update(xattn_gpt_spec("xattn_gpt.", cfg["embed_dim"], cfg["xf_n_layers"], n_positions=N_POSITIONS))
    return {k: w for k, w in ((k, detgen.weight_for(k, s)) for k, s in spec.items()) if w is not None}


def test_oracle_gato_matches_long_history_golden():
    case = gato_case()
    cfg = synth.GATO_CFGS[case.model]
    sd = gato_state_dict()
    g = load_golden(GOLDEN)
    with torch.no_grad():
        pt, pm = O.gato_forward_prompt_assembly(sd, synth.make_gato_prompt(case))
        ot = O.gato_forward_obs_token(sd, synth.make_gato_obs(case))
        at = O.forward_action_token(sd, synth.make_actions(case, case.T))
        assert pt.shape[0] + 1 + case.T * (ot.shape[2] + 1) - 1 == GATO_L
        pred = O.gato_policy_forward(sd, ot, at, pt, pm, n_head=cfg["n_head"])
        logits = O.action_decoder_logits(sd, pred[-1:])
        modes = O.action_modes(logits)
    e, a = golden_pick(g, "gato.prompt_masks", pm)
    assert np.array_equal(e, a)
    for key, val in zip(STAGES, (pt, ot, at, pred, logits)):
        e, a = golden_pick(g, "gato." + key, val)
        assert_close("gato." + key, e, a, ORACLE_TOL)
    for k, v in modes.items():
        e, a = golden_pick(g, f"gato.mode.{k}", v)
        assert np.array_equal(e, a), k


def test_oracle_policy_matches_long_history_golden():
    case = policy_case()
    cfg = synth.MODEL_CFGS[case.model]
    sd = policy_state_dict()
    g = load_golden(GOLDEN)
    with torch.no_grad():
        pt, pm, _ = O.forward_prompt_assembly(sd, synth.make_prompt(case))
        ot, om = O.forward_obs_token(sd, synth.make_obs(case))
        at = O.forward_action_token(sd, synth.make_actions(case, case.T))
        tokens, _, _ = O.assemble_history(ot, om, at)
        assert tokens.shape[0] == POLICY_L
        pred = O.policy_forward(sd, ot, om, at, pt, pm, n_head=cfg["sattn_n_heads"], xattn_n_head=cfg["xattn_n_heads"])
        logits = O.action_decoder_logits(sd, pred[-1:])
        modes = O.action_modes(logits)
    for key, t in (("prompt_masks", pm), ("obs_masks", om)):
        e, a = golden_pick(g, "policy." + key, t)
        assert np.array_equal(e, a), key
    for key, val in zip(STAGES, (pt, ot, at, pred, logits)):
        e, a = golden_pick(g, "policy." + key, val)
        assert_close("policy." + key, e, a, ORACLE_TOL)
    for k, v in modes.items():
        e, a = golden_pick(g, f"policy.mode.{k}", v)
        assert np.array_equal(e, a), k


# ------------------------------------------------------------------------------------------------------------------------------
# the kernel against fp64 (GPU)
# ------------------------------------------------------------------------------------------------------------------------------
LKS = (513, 777, 1024, 2047, 4096)
FORMATS = ["f16-hilo", "f16-hi8", "bf16-hilo"]  # split operands: (hi, lo) out, fp16 hi + e4m3 views (f16f8), bf16 (hi, lo)
LAYOUTS = ["self", "cross", "cross33", "lockstep33", "slots33"]
D, H = 32, 2


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    return _C.Context.get(torch.device("cuda", 0))


def _ops(ctx, x, dt):
    """fp32 [rows, cols] -> (hi, lo) 16-bit operands with 8 NaN pad columns the kernel must not read."""
    from tests.test_kernel_variants_gpu import NAN16

    rows, cols = x.shape
    hi = torch.empty(rows, cols + 8, dtype=torch.int16, device="cuda")
    lo = torch.empty_like(hi)
    ctx.split(x, hi, lo, cols=cols, pad_cols=cols + 8, dtype=dt)
    hi[:, cols:] = NAN16[dt]
    lo[:, cols:] = NAN16[dt]
    return hi, lo


def _ref(Q, K, V, scale, causal, key_mask, q0):
    """fp64, one batch element: Q (Lq, E), K / V (Lk, E), query row i at key position q0 + i; -> (Lq, E)."""
    from tests.test_kernel_variants_gpu import ref_attention

    def heads(x):
        return x.reshape(x.shape[0], H, D).permute(1, 0, 2).double()[None]

    o = ref_attention(heads(Q), heads(K), heads(V), 1 / math.sqrt(D), causal, key_mask[None], q0)
    return o[0].permute(1, 0, 2).reshape(Q.shape[0], H * D)


def run_layout(ctx, fmt, layout, Lk, seed, junk=None):
    """One call of `layout` at capacity Lk (B = 3).  -> (outputs dict, fp64 reference closure, meta).  `junk` fills every K / V row
    and mask column past each batch element's own key count (slots33 only) instead of finite noise."""
    from tests.test_kernel_variants_gpu import DT, sentinel

    dtname, out = fmt.split("-")
    dt, _ = DT[dtname]
    want_lo, want8 = out == "hilo", out == "hi8"
    B, E = 3, H * D
    causal = layout in ("self", "lockstep33", "slots33")
    Lq = Lk if layout in ("self", "cross") else 33
    cap = Lk + 40 if layout in ("lockstep33", "slots33") else Lk  # K / V / mask rows per batch element
    g = torch.Generator(device="cuda").manual_seed(seed)
    Qm = torch.randn(B * Lq, E, device="cuda", generator=g)
    KV = torch.randn(B * cap, 2 * E, device="cuda", generator=g)
    key_mask = torch.rand(B, cap, device="cuda", generator=g) > 0.1  # ~10 % padded keys
    key_mask[:, 0] = True
    key_mask[1, :600] = False  # rows of element 1 before key 600 see only padded keys up to their diagonal
    if layout == "slots33":
        q_pos = [Lk - Lq, (Lk - Lq) // 2, min(590, Lk - Lq)]
        if junk is not None:
            for b, p0 in enumerate(q_pos):
                KV[b * cap + p0 + Lq:(b + 1) * cap] = junk
                key_mask[b, p0 + Lq:] = torch.rand(cap - p0 - Lq, device="cuda", generator=g) > 0.5
    else:
        q_pos = [Lk - Lq if causal else 0] * B
    kh, kl = _ops(ctx, KV, dt)
    qh, ql = _ops(ctx, Qm, dt)
    rows = B * Lq
    outs = {"hi": sentinel((rows + 3, E + 8), "i16"), "lo": sentinel((rows + 3, E + 8), "i16") if want_lo else None,
            "o8": (sentinel((rows + 3, E + 16), "u8"), sentinel((rows + 3, E + 16), "u8")) if want8 else None}
    args = dict(q=(qh, ql, E + 8, 0), k=(kh, kl, 2 * E + 8, 0), v=(kh, kl, 2 * E + 8, E), o=(outs["hi"], outs["lo"], E + 8, 0), B=B, H=H,
                Lq=Lq, Lk=Lk, D=D, scale=1 / math.sqrt(D), causal=causal, key_mask=key_mask.to(torch.uint8), dtype=dt, o8=outs["o8"])
    if layout == "lockstep33":
        args.update(kv_batch_rows=cap, mask_ld=cap, q_pos0=Lk - Lq)
    elif layout == "slots33":
        args.update(kv_batch_rows=cap, mask_ld=cap, q_pos=torch.tensor(q_pos, dtype=torch.int32, device="cuda"))

    def ref():
        res = []
        for b in range(B):
            n = q_pos[b] + Lq if layout == "slots33" else Lk  # this element's keys
            kv = KV[b * cap:b * cap + n]
            res.append(_ref(Qm[b * Lq:(b + 1) * Lq], kv[:, :E], kv[:, E:], 1 / math.sqrt(D), causal, key_mask[b, :n], q_pos[b]))
        return torch.cat(res, 0)

    return outs, ref, args, (dt, True, want_lo, want8, rows, E)


def attn_bar(dt, Lk):
    """test_kernel_variants_gpu.py's attention bar up to 1024 keys, then growing as sqrt(Lk): every 64-key chunk may rescale a row's
    fp32 accumulator by its new running maximum, so the rounding error of a row's output walks with the number of chunks."""
    from tests.test_kernel_variants_gpu import ATTN_TOL

    return ATTN_TOL[(dt, True)] * max(1.0, math.sqrt(Lk / 1024))


@pytest.mark.gpu
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_attention_past_512_keys_against_fp64(ctx, fmt, layout):
    """Split operands at Lk = 513 .. 4096 keys against fp64 (bars: attn_bar)."""
    from tests.test_long_prompt_gpu import check_outputs

    errs = {}
    for Lk in LKS:
        tol = attn_bar(1 if fmt.startswith("bf16") else 0, Lk)
        outs, ref, args, meta = run_layout(ctx, fmt, layout, Lk, seed=Lk + len(layout))
        ctx.attention(**args)
        torch.cuda.synchronize()
        errs[Lk] = check_outputs(outs, ref(), meta, tol, f"{fmt} {layout} Lk={Lk}")
    print(f"attention {fmt} {layout}: rel-L2 by Lk", {k: f"{v:.2e}" for k, v in errs.items()})


@pytest.mark.gpu
@pytest.mark.parametrize("Lk", [777, 2047])
def test_keys_past_each_slot_are_not_read(ctx, Lk):
    """Per-batch q_pos at a capacity past 512: NaN in every K / V row and random mask bits in every column past each element's own
    key count leave every output bit-identical to the plain call."""
    res = []
    for junk in (None, 0.5, float("nan")):
        outs, _, args, _ = run_layout(ctx, "f16-hilo", "slots33", Lk, seed=3, junk=junk)
        ctx.attention(**args)
        torch.cuda.synchronize()
        res.append((outs["hi"], outs["lo"]))
    for hi, lo in res[1:]:
        assert torch.equal(res[0][0], hi) and torch.equal(res[0][1], lo)


# ------------------------------------------------------------------------------------------------------------------------------
# policies against the fixture (GPU)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def _precision_reset():
    yield
    if torch.cuda.is_available():
        import vima_b200

        vima_b200.set_precision("f16x3")


_POLICIES = {}


def gato_policy(n_positions=N_POSITIONS):
    import vima_b200

    key = ("gato", n_positions)
    if key not in _POLICIES:
        pol = vima_b200.VIMAGatoPolicy(**synth.GATO_CFGS["gato_tiny"], n_positions=n_positions)
        detgen.fill_module_(pol)
        _POLICIES[key] = pol.cuda().eval()
    return _POLICIES[key]


def vima_policy():
    import vima_b200
    from vima_b200 import nn as vnn

    if "vima" not in _POLICIES:
        cfg = synth.MODEL_CFGS[policy_case().model]
        pol = vima_b200.VIMAPolicy(**cfg)
        pol.xattn_gpt = vnn.XAttnGPT(cfg["embed_dim"], n_positions=N_POSITIONS, n_layer=cfg["xf_n_layers"], n_head=cfg["sattn_n_heads"],
                                     dropout=0.1, xattn_n_head=cfg["xattn_n_heads"], xattn_ff_expanding=4, xattn_n_positions=256,
                                     use_geglu=True)
        detgen.fill_module_(pol)
        _POLICIES["vima"] = pol.cuda().eval()
    return _POLICIES["vima"]


def check_golden(prefix, r, masks):
    g = load_golden(GOLDEN)
    for key in masks:
        e, a = golden_pick(g, f"{prefix}.{key}", r[key])
        assert np.array_equal(e, a), key
    errs = {}
    for key in STAGES:
        e, a = golden_pick(g, f"{prefix}.{key}", r[key])
        assert np.isfinite(a).all(), key
        errs[key] = rel_l2(e, a)
    assert max(errs.values()) <= POLICY_TOL, errs
    # action indices: exact wherever the reference's top-2 logit gap exceeds the fp tolerance (ties are not defined)
    raw = g[f"{prefix}.logits_raw"]
    got = torch.cat([r["modes"][k] for k in O.ACTION_DIMS], dim=-1).cpu().numpy()
    exp = np.concatenate([g[f"{prefix}.mode.{k}"] for k in O.ACTION_DIMS], axis=-1)
    safe = argmax_safe_mask(raw, DIMS, margin=4 * POLICY_TOL * np.abs(raw).max())
    assert np.array_equal(got[safe], exp[safe]), f"{prefix}: action indices differ outside numerical ties"
    return errs, float(safe.mean())


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["f16x3", "bf16x3", "f16f8"])
def test_gato_1024_positions_matches_reference_golden(mode):
    import vima_b200
    from vima_b200.utils import DataDict
    from tests.policy_runner import to_dev

    pol = gato_policy()
    case = gato_case()
    vima_b200.set_precision(mode)
    with torch.no_grad():
        tt, wb, ib = synth.make_gato_prompt(case)
        pt, pm = pol.forward_prompt_assembly((tt, wb.cuda(), DataDict(to_dev(ib, "cuda"))))
        ot = pol.forward_obs_token(DataDict(to_dev(synth.make_gato_obs(case), "cuda")))
        at = pol.forward_action_token(to_dev(synth.make_actions(case, case.T), "cuda"))
        pred = pol.forward(obs_token=ot, action_token=at, prompt_token=pt, prompt_token_mask=pm)
        dists = pol.forward_action_decoder(pred[-1:])
        logits = torch.cat([dists[k].raw_logits for k in dists], dim=-1)
        modes = {k: dists[k].mode() for k in dists}
    r = dict(prompt_masks=pm, prompt_tokens=pt, obs_tokens=ot, action_tokens=at, predicted=pred, logits_raw=logits, modes=modes)
    errs, safe = check_golden("gato", r, ("prompt_masks",))
    print(mode, {k: f"{v:.1e}" for k, v in errs.items()}, f"modes checked {safe:.0%}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["f16x3", "bf16x3", "f16f8"])
def test_vima_policy_1024_positions_matches_reference_golden(mode):
    import vima_b200
    from tests.policy_runner import run_policy_case

    pol = vima_policy()
    vima_b200.set_precision(mode)
    r = run_policy_case(pol, policy_case())
    errs, safe = check_golden("policy", r, ("prompt_masks", "obs_masks"))
    print(mode, {k: f"{v:.1e}" for k, v in errs.items()}, f"modes checked {safe:.0%}")


# ------------------------------------------------------------------------------------------------------------------------------
# decode at Lmax = 1024 (GPU)
# ------------------------------------------------------------------------------------------------------------------------------
def _rand_prompt(g, Lp, E):
    tok = torch.randn(Lp, 1, E, device="cuda", generator=g)
    msk = torch.rand(1, Lp, device="cuda", generator=g) > 0.25
    msk[:, 0] = True
    return tok, msk


def _pad_cat(prompts):
    """[(tok (Lp_j,1,E), msk (1,Lp_j))] -> one admission batch padded to the longest prompt."""
    Lp = max(t.shape[0] for t, _ in prompts)
    E = prompts[0][0].shape[-1]
    toks = [torch.cat([t, torch.zeros(Lp - t.shape[0], 1, E, device="cuda")], 0) for t, _ in prompts]
    msks = [torch.cat([m, torch.zeros(1, Lp - m.shape[1], dtype=torch.bool, device="cuda")], 1) for _, m in prompts]
    return torch.cat(toks, 1), torch.cat(msks, 0)


def _gato_oracle(ot, at, pt, pm):
    c = lambda t: None if t is None else t.cpu()  # noqa: E731
    return O.gato_policy_forward(gato_state_dict(), c(ot), c(at), c(pt), c(pm), n_head=synth.GATO_CFGS["gato_tiny"]["n_head"])


def _vima_oracle(ot, om, at, pt, pm):
    cfg = synth.MODEL_CFGS[policy_case().model]
    c = lambda t: None if t is None else t.cpu()  # noqa: E731
    return O.policy_forward(policy_state_dict(), c(ot), c(om), c(at), c(pt), c(pm), n_head=cfg["sattn_n_heads"],
                            xattn_n_head=cfg["xattn_n_heads"])


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
def test_gato_cached_steps_past_768_tokens(mode):
    """forward_step at every step of two episodes (prompts of 100 and 61 valid-or-padded tokens) up to L = 865 against the full
    re-forward, and the CPU oracle at the end."""
    import vima_b200

    vima_b200.set_precision(mode)
    pol = gato_policy()
    E, Q, B, Lp, T = pol.embed_dim, pol._obj_xf_num_queries, 2, 100, 45
    g = torch.Generator(device="cuda").manual_seed(101)
    pt = torch.randn(Lp, B, E, device="cuda", generator=g)
    pm = torch.rand(B, Lp, device="cuda", generator=g) > 0.2
    pm[:, 0] = True
    pm[1, 61:] = False
    ot = torch.randn(T, B, Q, E, device="cuda", generator=g)
    at = torch.randn(T - 1, B, E, device="cuda", generator=g)
    with torch.no_grad():
        cache = pol.start_decode(pt, pm)
        assert cache.Lmax == N_POSITIONS
        for t in range(T):
            step = pol.forward_step(cache, ot[t:t + 1], None if t == 0 else at[t - 1:t])
            full = pol.forward(ot[:t + 1], None if t == 0 else at[:t], pt, pm)[-1:]
            d = rel_l2(full.cpu(), step.cpu())
            assert d < BARS[mode], (t, d)
        assert cache.L == Lp + 1 + T * (Q + 1) - 1 > 768
        assert rel_l2(_gato_oracle(ot, at, pt, pm)[-1:], step.cpu()) < POLICY_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
def test_vima_cached_steps_past_768_tokens(mode):
    """VIMAPolicy forward_step over 28 steps of 32 object tokens with ragged masks (L = 923) against the full re-forward, and the
    CPU oracle at the end."""
    import vima_b200

    vima_b200.set_precision(mode)
    pol = vima_policy()
    E, Q, B, Lp, T = pol.embed_dim, 32, 2, 40, 28
    g = torch.Generator(device="cuda").manual_seed(102)
    pt = torch.randn(Lp, B, E, device="cuda", generator=g)
    pm = torch.rand(B, Lp, device="cuda", generator=g) > 0.2
    pm[:, 0] = True
    ot = torch.randn(T, B, Q, E, device="cuda", generator=g)
    om = torch.rand(T, B, Q, device="cuda", generator=g) > 0.2
    om[..., 0] = True
    at = torch.randn(T - 1, B, E, device="cuda", generator=g)
    with torch.no_grad():
        cache = pol.start_decode(pt, pm)
        for t in range(T):
            a = None if t == 0 else at[t - 1:t]
            step = pol.forward_step(cache, ot[t:t + 1], om[t:t + 1], a)
            full = pol.forward(obs_token=ot[:t + 1], obs_mask=om[:t + 1], action_token=None if t == 0 else at[:t], prompt_token=pt,
                               prompt_token_mask=pm)[-1:]
            d = rel_l2(full.cpu(), step.cpu())
            assert d < BARS[mode], (t, d)
        assert cache.L == POLICY_L
        assert rel_l2(_vima_oracle(ot, om, at, pt, pm)[-1:], step.cpu()) < POLICY_TOL


# tick -> {slot: prompt length} admitted / [slots] released before the tick's step; slot 0 reaches 60 + 17 * 46 = 842 tokens
GATO_ADMITS = {0: {0: 60, 1: 23}, 5: {2: 41}, 20: {1: 30}}
GATO_RELEASES = {18: [1], 40: [2]}
GATO_TICKS = 46


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
def test_gato_staggered_slots_past_768_tokens(mode):
    """Four slots of Lmax = 1024 over 46 ticks (ragged prompts, admissions at ticks 0 / 5 / 20, releases at 18 / 40, slot 3 never
    admitted): every active slot's row equals forward(...)[-1:] at B=1 over its own history, and the oracle at the last tick."""
    import vima_b200

    vima_b200.set_precision(mode)
    pol = gato_policy()
    E, Q, S = pol.embed_dim, pol._obj_xf_num_queries, 4
    g = torch.Generator(device="cuda").manual_seed(103)
    eps = {}
    with torch.no_grad():
        cache = pol.open_slots(S)
        assert cache.Lmax == N_POSITIONS
        for t in range(GATO_TICKS):
            for b in GATO_RELEASES.get(t, []):
                pol.release(cache, [b])
                del eps[b]
            if t in GATO_ADMITS:
                slots = sorted(GATO_ADMITS[t])
                prompts = [_rand_prompt(g, GATO_ADMITS[t][b], E) for b in slots]
                ptok, pmsk = _pad_cat(prompts)
                for j, b in enumerate(slots):
                    eps[b] = dict(prompt=(ptok[:, j:j + 1], pmsk[j:j + 1]), obs=[], act=[])
                pol.admit(cache, slots, ptok, pmsk)
            obs = torch.randn(1, S, Q, E, device="cuda", generator=g)
            act = torch.randn(1, S, E, device="cuda", generator=g)
            for b, ep in eps.items():
                if ep["obs"]:
                    ep["act"].append(act[:, b:b + 1])
                ep["obs"].append(obs[:, b:b + 1])
            out = pol.step_slots(cache, obs, act)
            for b, ep in eps.items():
                ho, ha = torch.cat(ep["obs"], 0), (torch.cat(ep["act"], 0) if ep["act"] else None)
                full = pol.forward(ho, ha, *ep["prompt"])[-1:]
                d = rel_l2(full.cpu(), out[:, b:b + 1].cpu())
                assert d < BARS[mode], (t, b, d)
                if t == GATO_TICKS - 1:
                    assert rel_l2(_gato_oracle(ho, ha, *ep["prompt"])[-1:], out[:, b:b + 1].cpu()) < POLICY_TOL, b
        torch.cuda.synchronize()
        assert cache.active_host == [True, True, False, False]
        assert max(cache.len_host) > 768 and cache.len.tolist() == cache.len_host


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
def test_vima_staggered_slots_past_768_tokens(mode):
    """VIMAPolicy: three slots of Lmax = 1024 over 28 ticks of 32 object tokens (ragged masks), slot 1 admitted at tick 3 and
    slot 2 released at tick 20: rows equal forward(...)[-1:] at B=1 over each episode's history, and the oracle at the end."""
    import vima_b200

    vima_b200.set_precision(mode)
    pol = vima_policy()
    E, Q, S, ticks = pol.embed_dim, 32, 3, 28
    admits, releases = {0: {0: 40, 2: 17}, 3: {1: 25}}, {20: [2]}
    g = torch.Generator(device="cuda").manual_seed(104)
    eps = {}
    with torch.no_grad():
        cache = pol.open_slots(S, max_prompt_tokens=64)
        assert cache.Lmax == N_POSITIONS
        for t in range(ticks):
            for b in releases.get(t, []):
                pol.release(cache, [b])
                del eps[b]
            if t in admits:
                slots = sorted(admits[t])
                prompts = [_rand_prompt(g, admits[t][b], E) for b in slots]
                ptok, pmsk = _pad_cat(prompts)
                for j, b in enumerate(slots):
                    eps[b] = dict(prompt=prompts[j], obs=[], mask=[], act=[])
                pol.admit(cache, slots, ptok, pmsk)
            obs = torch.randn(1, S, Q, E, device="cuda", generator=g)
            msk = torch.rand(1, S, Q, device="cuda", generator=g) > 0.2
            msk[..., 0] = True
            act = torch.randn(1, S, E, device="cuda", generator=g)
            for b, ep in eps.items():
                if ep["obs"]:
                    ep["act"].append(act[:, b:b + 1])
                ep["obs"].append(obs[:, b:b + 1])
                ep["mask"].append(msk[:, b:b + 1])
            out = pol.step_slots(cache, obs, msk, act)
            for b, ep in eps.items():
                po, pm = torch.cat(ep["obs"], 0), torch.cat(ep["mask"], 0)
                pa = torch.cat(ep["act"], 0) if ep["act"] else None
                full = pol.forward(obs_token=po, obs_mask=pm, action_token=pa, prompt_token=ep["prompt"][0],
                                   prompt_token_mask=ep["prompt"][1])[-1:]
                d = rel_l2(full.cpu(), out[:, b:b + 1].cpu())
                assert d < BARS[mode], (t, b, d)
                if t == ticks - 1:
                    assert rel_l2(_vima_oracle(po, pm, pa, *ep["prompt"])[-1:], out[:, b:b + 1].cpu()) < POLICY_TOL, b
        torch.cuda.synchronize()
        assert cache.active_host == [True, True, False]
        assert cache.len_host[0] == POLICY_L


@pytest.mark.gpu
def test_gato_graph_replay_past_768_tokens_equals_eager():
    """capture_step_slots at Lmax = 1024 with prompts of ~700 tokens, so the replayed steps run past 768 keys: replays equal eager
    step_slots bit for bit across admissions and a release."""
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = gato_policy()
    E, Q, S, ticks = pol.embed_dim, pol._obj_xf_num_queries, 3, 8
    g = torch.Generator(device="cuda").manual_seed(105)
    prompts = {k: _rand_prompt(g, 700 - 9 * k, E) for k in range(4)}
    schedule = {0: ("admit", [0, 1], [0, 1]), 2: ("admit", [2], [2]), 5: ("release", [1], None), 6: ("admit", [1], [3])}
    obs = torch.randn(ticks, S, Q, E, device="cuda", generator=g)
    act = torch.randn(ticks, S, E, device="cuda", generator=g)

    def run(step, cache):
        outs = []
        for t in range(ticks):
            if t in schedule:
                kind, slots, pk = schedule[t]
                if kind == "admit":
                    pol.admit(cache, slots, *_pad_cat([prompts[k] for k in pk]))
                else:
                    pol.release(cache, slots)
            active = [b for b in range(S) if cache.active_host[b]]
            outs.append(step(cache, obs[t:t + 1], act[t:t + 1])[:, active].clone())
        torch.cuda.synchronize()
        return outs, max(cache.len_host)

    with torch.no_grad():
        eager, longest = run(pol.step_slots, pol.open_slots(S))
        assert longest > 768
        cache = pol.open_slots(S)
        pol.admit(cache, [2], *prompts[3])
        gs = pol.capture_step_slots(cache, obs[:1], act[:1])
        pol.release(cache, [2])
        graphed, _ = run(lambda c, o, a: gs(o, a), cache)
    for t, (w, x) in enumerate(zip(eager, graphed)):
        assert torch.equal(w, x), t
    assert gs.replays == ticks


# ------------------------------------------------------------------------------------------------------------------------------
# module and refusal (GPU)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_xattn_gpt_1000_prompt_tokens():
    """vnn.XAttnGPT built with xattn_n_positions = 1024 cross-attends over a 1000-token prompt (row 1 padded past 700) against the
    oracle's restatement of xattn_gpt.py:73-139."""
    import vima_b200
    from vima_b200 import nn as vnn

    vima_b200.set_precision("f16x3")
    E, nl, Hh, B, L, Lp = 256, 2, 8, 2, 67, 1000
    mod = vnn.XAttnGPT(E, n_layer=nl, n_head=Hh, dropout=0.1, xattn_n_head=Hh, xattn_ff_expanding=4, xattn_n_positions=1024, use_geglu=True)
    detgen.fill_module_(mod)
    sd = {"xattn_gpt." + k: v.detach().clone() for k, v in mod.state_dict().items()}
    mod = mod.cuda().eval()
    g = torch.Generator().manual_seed(19)
    tok = torch.randn(L, B, E, generator=g)
    ptk = torch.randn(Lp, B, E, generator=g)
    pmask = torch.rand(B, Lp, generator=g) > 0.1
    pmask[:, 0] = True
    pmask[1, 700:] = False
    omask = torch.rand(B, L, generator=g) > 0.15
    omask[:, 0] = True
    oa_pos = torch.cumsum(omask, dim=1) - 1
    p_pos = torch.cumsum(pmask, dim=1) - 1
    with torch.no_grad():
        ref = O.xattn_gpt_forward(sd, "xattn_gpt.", obs_action_tokens=tok, obs_action_position_ids=oa_pos, prompt_tokens=ptk, prompt_mask=pmask,
                                  prompt_position_ids=p_pos, obs_action_masks=omask, n_layer=nl, n_head=Hh, xattn_n_head=Hh)
        got = mod(obs_action_tokens=tok.cuda(), obs_action_position_ids=oa_pos.cuda(), prompt_tokens=ptk.cuda(), prompt_mask=pmask.cuda(),
                  prompt_position_ids=p_pos.cuda(), obs_action_masks=omask.cuda())
    assert rel_l2(ref, got.cpu()) < POLICY_TOL, rel_l2(ref, got.cpu())


@pytest.mark.gpu
def test_single_pass_f16_past_the_resident_kernel_is_refused():
    """Single-pass f16 runs on the resident-K/V mma.sync kernel, which holds 1536 keys at head_dim 32: a Gato forward of 1596 tokens
    (n_positions = 2048) raises the capacity error instead of running on, and the context keeps working."""
    import vima_b200

    pol = gato_policy(2048)
    E, Q, B, Lp, T = pol.embed_dim, pol._obj_xf_num_queries, 1, 100, 88
    g = torch.Generator(device="cuda").manual_seed(106)
    pt = torch.randn(Lp, B, E, device="cuda", generator=g)
    pm = torch.ones(B, Lp, dtype=torch.bool, device="cuda")
    ot = torch.randn(T, B, Q, E, device="cuda", generator=g)
    at = torch.randn(T - 1, B, E, device="cuda", generator=g)
    assert Lp + 1 + T * (Q + 1) - 1 == 1596
    vima_b200.set_precision("f16")
    with torch.no_grad():
        with pytest.raises(RuntimeError, match=r"resident-K/V kernel takes Lk <= 1536"):
            pol.forward(ot, at, pt, pm)
        torch.cuda.synchronize()
        out = pol.forward(ot[:40], at[:39], pt, pm)  # 780 tokens fit
        torch.cuda.synchronize()
    assert torch.isfinite(out).all()
