"""Prompts past the resident-K/V attention kernel's 384 keys: the T5 encoder on the K/V-streaming wgmma kernel (attention_tc.cu,
attention_bias_tc_kernel).

CPU:
  * the oracle's T5 encoder and VIMAPolicy chain against tests/golden/long_prompt.npz (minted from the unmodified reference by
    tests/golden/make_long_prompt_golden.py): a 512-position policy with a 512-token and a ragged 483-token prompt, and T5 alone at
    Lp = 1000.
  (What ptxas makes of the kernel is checked in tests/test_wgmma_ptxas_cpu.py.)
GPU:
  * the kernel against one fp64 statement of T5 attention in every operand and output format, at every chunk boundary up to 2048 keys,
    with attn_bias=tc and with the default options; the defaults leave every shape the resident kernel takes on that kernel, bit for bit;
  * vnn.T5PromptEncoder at Lp = 512 and 1000 against the golden and the oracle, and the 512-position VIMAPolicy chain against the golden.
"""

import numpy as np
import pytest
import torch

from oracle import detgen, synth, vima_oracle as O
from tests.golden.make_long_prompt_golden import XATTN_N_POSITIONS, policy_case, t5_inputs
from tests.util import assert_close, golden_pick, load_golden, rel_l2

GOLDEN = "long_prompt"
ORACLE_TOL = 2e-5  # fp32 CPU vs fp32 CPU: summation-order noise only (as tests/test_oracle_golden.py)
POLICY_TOL = 1e-3  # north_star tolerance
# vnn.T5PromptEncoder (12 layers of t5-base, detgen weights) against fp32 at Lp = 512 / 1000, rel-L2.  Measured worst on an H100 80GB
# HBM3: f16x3 9.8e-6, f16f8 2.0e-5 (both against the fixture at Lp = 1000).
T5_TOL = {"f16x3": 3e-5, "f16f8": 6e-5}


# ------------------------------------------------------------------------------------------------------------------------------
# oracle and fixtures (CPU)
# ------------------------------------------------------------------------------------------------------------------------------
def t5_state_dict():
    """The standalone T5PromptEncoder's encoder weights as detgen fills them (keys 't5.encoder.*')."""
    from oracle.state_dict_spec import t5_spec

    return {k: detgen.weight_for(k, s) for k, s in t5_spec("t5.").items() if k.startswith("t5.encoder.block.") or "final_layer_norm" in k}


def policy_state_dict():
    """The 2M VIMAPolicy with its XAttnGPT at xattn_n_positions=512, as detgen fills it."""
    from oracle.state_dict_spec import state_dict_spec, xattn_gpt_spec

    cfg = synth.MODEL_CFGS[policy_case().model]
    spec = {k: s for k, s in state_dict_spec(**cfg).items() if not k.startswith("xattn_gpt.")}
    spec.update(xattn_gpt_spec("xattn_gpt.", cfg["embed_dim"], cfg["xf_n_layers"], xattn_n_positions=XATTN_N_POSITIONS))
    sd = {}
    for k, s in spec.items():
        w = detgen.weight_for(k, s)
        if w is not None:
            sd[k] = w
    return sd


def oracle_t5(x, mask):
    with torch.no_grad():
        return O.t5_encoder_forward(t5_state_dict(), "t5.encoder.", x, mask)


def test_oracle_t5_matches_long_prompt_golden():
    g = load_golden(GOLDEN)
    x, mask = t5_inputs()
    e, a = golden_pick(g, "t5.mask", mask)
    assert np.array_equal(e, a)
    e, a = golden_pick(g, "t5.out", oracle_t5(x, mask))
    assert_close("t5.out", e, a, ORACLE_TOL)


def test_oracle_policy_matches_long_prompt_golden():
    g = load_golden(GOLDEN)
    case = policy_case()
    cfg = synth.MODEL_CFGS[case.model]
    sd = policy_state_dict()
    with torch.no_grad():
        prompt_tokens, prompt_masks, _ = O.forward_prompt_assembly(sd, synth.make_prompt(case))
        assert prompt_tokens.shape[0] == XATTN_N_POSITIONS and 384 < int(prompt_masks[1].sum()) < XATTN_N_POSITIONS
        obs_tokens, obs_masks = O.forward_obs_token(sd, synth.make_obs(case))
        action_tokens = O.forward_action_token(sd, synth.make_actions(case, case.T))
        predicted = O.policy_forward(sd, obs_tokens, obs_masks, action_tokens, prompt_tokens, prompt_masks, n_head=cfg["sattn_n_heads"],
                                     xattn_n_head=cfg["xattn_n_heads"])
        logits = O.action_decoder_logits(sd, predicted[-1:])
        modes = O.action_modes(logits)
    for key, t in (("prompt_masks", prompt_masks), ("obs_masks", obs_masks)):
        e, a = golden_pick(g, "policy." + key, t)
        assert np.array_equal(e, a), key
    for key, t in (("prompt_tokens", prompt_tokens), ("obs_tokens", obs_tokens), ("action_tokens", action_tokens), ("predicted", predicted),
                   ("logits_raw", logits)):
        e, a = golden_pick(g, "policy." + key, t)
        assert_close(key, e, a, ORACLE_TOL)
    for k, v in modes.items():
        e, a = golden_pick(g, f"policy.mode.{k}", v)
        assert np.array_equal(e, a), k


# ------------------------------------------------------------------------------------------------------------------------------
# the kernel against fp64 (GPU)
# ------------------------------------------------------------------------------------------------------------------------------
FORMATS = ["f16-x3-hilo", "f16-x3-hi8", "f16-x3-hilo8", "f16-single-hilo", "f16-single-hi8", "f16-single-hilo8", "bf16-x3-hilo",
           "bf16-single-hilo"]
LK_TC = (1, 63, 64, 65, 200, 384, 385, 512, 513, 1000, 2048)
LK_AUTO = (385, 512, 1000, 2048)


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    return _C.Context.get(torch.device("cuda", 0))


@pytest.fixture
def options(ctx):
    def set_(attn="tc", attn_bias="auto"):
        ctx.set_option("attn", attn)
        ctx.set_option("attn_bias", attn_bias)

    yield set_
    set_()


def run_t5_attention(ctx, fmt, L, seed):
    """One T5-shaped call (B = 2, H = 2, D = 64, scale 1, relative bias, key mask; batch element 1 has every key padded) with NaN in
    every operand column in [cols, ld) and sentinels around every output.  -> (outputs dict, fp64 reference [B*L, E], args)."""
    from tests.test_kernel_variants_gpu import DT, NAN16, sentinel

    dtname, mode, out = fmt.split("-")
    dt, tdt = DT[dtname]
    split = mode == "x3"
    want_lo, want8 = out in ("hilo", "hilo8"), out in ("hi8", "hilo8")
    B, H, D = 2, 2, 64
    E = H * D
    g = torch.Generator(device="cuda").manual_seed(seed)
    Qm = torch.randn(B * L, E, device="cuda", generator=g) * 0.35
    KV = torch.randn(B * L, 2 * E, device="cuda", generator=g)
    rel_bias = torch.randn(H, 2 * L - 1, device="cuda", generator=g)

    def ops(x):
        rows, cols = x.shape
        hi = torch.empty(rows, cols + 8, dtype=torch.int16, device="cuda")
        lo = torch.empty_like(hi) if split else None
        ctx.split(x, hi, lo, cols=cols, pad_cols=cols + 8, dtype=dt)
        for t in (hi, lo):
            if t is not None:
                t[:, cols:] = NAN16[dt]
        return hi, lo

    qh, ql = ops(Qm)
    kh, kl = ops(KV)
    key_mask = torch.rand(B, L, device="cuda", generator=g) > 0.2
    key_mask[0, 0] = True
    key_mask[1] = False
    outs = {"hi": sentinel((B * L + 3, E + 8), "i16"), "lo": sentinel((B * L + 3, E + 8), "i16") if want_lo else None,
            "o8": (sentinel((B * L + 3, E + 16), "u8"), sentinel((B * L + 3, E + 16), "u8")) if want8 else None}
    args = dict(q=(qh, ql, E + 8, 0), k=(kh, kl, 2 * E + 8, 0), v=(kh, kl, 2 * E + 8, E), o=(outs["hi"], outs["lo"], E + 8, 0), B=B, H=H,
                Lq=L, Lk=L, D=D, scale=1.0, causal=False, key_mask=key_mask.to(torch.uint8), rel_bias=rel_bias, dtype=dt, o8=outs["o8"])

    def ref():
        Q, K, V = Qm, KV[:, :E], KV[:, E:]
        if not split:
            Q, K, V = (t.to(tdt).float() for t in (Q, K, V))

        def heads(x):
            return x.reshape(B, L, H, D).permute(0, 2, 1, 3).double()

        ii = torch.arange(L, device="cuda")[:, None]
        jj = torch.arange(L, device="cuda")[None, :]
        s = torch.matmul(heads(Q), heads(K).transpose(-1, -2)) + rel_bias[:, jj - ii + L - 1].double()[None]
        s = s + (1.0 - key_mask[:, None, None, :].double()) * torch.finfo(torch.float32).min
        return torch.matmul(torch.softmax(s, -1), heads(V)).permute(0, 2, 1, 3).reshape(B * L, E)

    return outs, ref, args, (dt, split, want_lo, want8, B * L, E)


def check_outputs(outs, ref, meta, tol, what):
    """-> worst rel-L2 of the (hi, lo) and hi + lo8 reconstructions; asserts the bars, the sentinels and the e4m3 hi view."""
    from tests.test_kernel_variants_gpu import assert_canary, assert_hi8, f16view, rel

    dt, split, want_lo, want8, R, E = meta
    worst = 0.0
    h = f16view(outs["hi"][:R, :E], dt).double()
    assert_canary(outs["hi"], R, E, what)
    if want_lo:
        assert_canary(outs["lo"], R, E, what)
        got = h + f16view(outs["lo"][:R, :E], dt).double()
        e = rel(got, ref)
        worst = max(worst, e)
        assert torch.isfinite(got).all() and e < tol, (what, e)
    if want8:
        lo8, hi8 = outs["o8"]
        assert_canary(lo8, R, E, what); assert_canary(hi8, R, E, what)
        rec = h + lo8[:R, :E].view(torch.float8_e4m3fn).double() / 1024.0
        e = rel(rec, ref)
        worst = max(worst, e)
        assert torch.isfinite(rec).all() and e < tol + 2e-5, (what, e)
        assert_hi8(hi8[:R, :E], rec, what)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("attn_bias", ["tc", "auto"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_attention_bias_against_fp64(ctx, options, fmt, attn_bias):
    """T5 attention (scores unscaled, + bias[h][j - i + L - 1], + finfo.min for a padded key) against fp64, at every 64-key chunk
    boundary up to 2048 keys.  attn_bias=tc runs the streaming kernel at every length; the defaults run it past the resident kernel's
    capacity (384 keys split, 768 single-pass) and the resident kernel below."""
    from tests.test_kernel_variants_gpu import ATTN_TOL

    options(attn_bias=attn_bias)
    dt, split = (1 if fmt.startswith("bf16") else 0), "-x3-" in fmt
    tol = ATTN_TOL[(dt, split)]
    worst = 0.0
    for L in (LK_TC if attn_bias == "tc" else LK_AUTO):
        outs, ref, args, meta = run_t5_attention(ctx, fmt, L, seed=L)
        ctx.attention(**args)
        torch.cuda.synchronize()
        worst = max(worst, check_outputs(outs, ref(), meta, tol, f"{attn_bias} {fmt} L={L}"))
    print(f"attention_bias {attn_bias} {fmt}: worst rel-L2 {worst:.2e} (bar {tol:.0e})")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_default_options_keep_the_resident_kernel(ctx, options, fmt):
    """Under the default options every length the resident-K/V kernel takes stays on it: outputs equal attn=mma bit for bit."""
    lengths = (200, 384) if "-x3-" in fmt else (200, 384, 768)
    for L in lengths:
        res = []
        for attn in ("tc", "mma"):
            options(attn=attn)
            outs, _, args, _ = run_t5_attention(ctx, fmt, L, seed=7 * L)
            ctx.attention(**args)
            torch.cuda.synchronize()
            res.append([t for t in (outs["hi"], outs["lo"]) + (outs["o8"] or ()) if t is not None])
        for a, b in zip(*res):
            assert torch.equal(a, b), (fmt, L)


@pytest.mark.gpu
def test_refusals_are_unchanged(ctx, options):
    """attn=mma keeps the resident kernel and its refusal past 384 split keys, with attn_bias=tc too; without a relative bias, head_dim
    64 past 384 split keys is refused as before under every attn_bias setting.  Nothing is written."""
    from tests.test_kernel_variants_gpu import S16

    for attn, attn_bias, bias in (("mma", "auto", True), ("mma", "tc", True), ("tc", "auto", False), ("tc", "tc", False)):
        options(attn=attn, attn_bias=attn_bias)
        outs, _, args, _ = run_t5_attention(ctx, "f16-x3-hilo", 385, seed=1)
        if not bias:
            args["rel_bias"] = None
        with pytest.raises(RuntimeError, match=r"resident-K/V kernel takes Lk <= 384"):
            ctx.attention(**args)
        torch.cuda.synchronize()
        assert (outs["hi"] == S16).all(), (attn, attn_bias, bias)
    options()
    with pytest.raises(RuntimeError, match="unknown option"):
        ctx.set_option("attn_bias", "mma")


# ------------------------------------------------------------------------------------------------------------------------------
# module and policy (GPU)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def t5_module():
    from vima_b200 import nn as vnn

    enc = vnn.T5PromptEncoder()
    detgen.fill_module_(enc)
    return enc.cuda().eval()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
def test_t5_prompt_encoder_long_prompts(t5_module, mode):
    """vnn.T5PromptEncoder at Lp = 512 (row 1 ragged at 450) and Lp = 1000 (the fixture's input) against the oracle, and at 1000
    against the reference-minted fixture."""
    import vima_b200

    x, mask = t5_inputs()
    x512, mask512 = x[:, :512].contiguous(), mask[:, :512].clone()
    mask512[1, 450:] = False
    g = load_golden(GOLDEN)
    errs = {}
    vima_b200.set_precision(mode)
    try:
        for name, xi, mi in (("512", x512, mask512), ("1000", x, mask)):
            with torch.no_grad():
                got = t5_module(xi.cuda(), attention_mask=mi.cuda(), batch_first=True).cpu()
            assert torch.isfinite(got).all(), name
            errs[f"oracle {name}"] = rel_l2(oracle_t5(xi, mi).numpy(), got.numpy())
            if name == "1000":
                e, a = golden_pick(g, "t5.out", got)
                errs["golden 1000"] = rel_l2(e, a)
    finally:
        vima_b200.set_precision("f16x3")
    print(mode, {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) <= T5_TOL[mode], errs


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
def test_policy_512_prompt_matches_reference_golden(mode):
    """The 512-position VIMAPolicy encodes its own 512- and 483-token prompts through T5 and runs the whole chain: every stage within
    1e-3 rel-L2 of the reference-minted fixture, masks bit-exact, action indices exact."""
    import vima_b200
    from tests.policy_runner import run_policy_case
    from vima_b200 import nn as vnn

    case = policy_case()
    cfg = synth.MODEL_CFGS[case.model]
    pol = vima_b200.VIMAPolicy(**cfg)
    pol.xattn_gpt = vnn.XAttnGPT(cfg["embed_dim"], n_layer=cfg["xf_n_layers"], n_head=cfg["sattn_n_heads"], dropout=0.1,
                                 xattn_n_head=cfg["xattn_n_heads"], xattn_ff_expanding=4, xattn_n_positions=XATTN_N_POSITIONS, use_geglu=True)
    detgen.fill_module_(pol)
    pol = pol.cuda().eval()
    vima_b200.set_precision(mode)
    try:
        r = run_policy_case(pol, case)
    finally:
        vima_b200.set_precision("f16x3")
    g = load_golden(GOLDEN)
    for key in ("prompt_masks", "obs_masks"):
        e, a = golden_pick(g, "policy." + key, r[key])
        assert np.array_equal(e, a), key
    errs = {}
    for key in ("prompt_tokens", "obs_tokens", "action_tokens", "predicted", "logits_raw"):
        e, a = golden_pick(g, "policy." + key, r[key])
        assert np.isfinite(a).all(), key
        errs[key] = rel_l2(e, a)
    print(mode, {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) <= POLICY_TOL, errs
    for k in O.ACTION_DIMS:
        e, a = golden_pick(g, f"policy.mode.{k}", r["modes"][k])
        assert np.array_equal(e, a), f"action indices differ for {k}"
