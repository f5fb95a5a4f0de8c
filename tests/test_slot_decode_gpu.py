"""GPU: slot decode (VIMAPolicy.open_slots / admit / release / step_slots, DESIGN.md 7 (f)1): every row of the batch holds one
episode at its own history length.  The kernels against per-batch calls and torch statements, staggered episodes against the
full re-forward of each episode's own history at B=1 and the CPU oracle, lockstep slots against forward_step, graph replay against
eager steps, and the refusals."""
import math

import pytest
import torch

from oracle import synth, vima_oracle as O
from tests.policy_runner import build_policy
from tests.test_oracle_golden import oracle_state_dict
from tests.util import rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    return _C.Context.get(torch.device("cuda", 0))


def _split(ctx, x, dt, split):
    rows, cols = x.shape
    hi = torch.empty(rows, cols, dtype=torch.int16, device="cuda")
    lo = torch.empty_like(hi) if split else None
    ctx.split(x.contiguous(), hi, lo, cols=cols, pad_cols=cols, dtype=dt)
    return hi, lo


def _merge(hi, lo, tdt):
    a = hi.view(tdt).float()
    return a if lo is None else a + lo.view(tdt).float()


def _ref_attention(q, k, v, scale, q0, key_mask):
    """fp64, one batch element: q (H,Lq,D) at positions q0.., k / v (H,Lk,D); the reference's soft causal mask and key mask."""
    s = torch.matmul(q, k.transpose(-1, -2)) * scale
    Lq, Lk = s.shape[-2:]
    vis = (torch.arange(Lk, device=s.device)[None, :] <= torch.arange(Lq, device=s.device)[:, None] + q0).to(s.dtype)
    s = s * vis + -1e4 * (1 - vis)
    s = s + (1.0 - key_mask[None, None, :].to(s.dtype)) * torch.finfo(torch.float32).min
    return torch.matmul(torch.softmax(s, -1), v)


# (kernel option, operand format, split, Lq, Lmax): the wgmma kernel in f16x3 / bf16x3, the mma.sync kernel in single-pass f16 and
# forced with split operands, and the wgmma body + SIMT tail split (133 = 128 + 5 rows)
@pytest.mark.parametrize("impl,fmt,split,Lq,Lmax", [("tc", "f16", True, 33, 263), ("tc", "bf16", True, 33, 263), ("tc", "f16", False, 33, 263),
                                                     ("mma", "f16", True, 33, 263), ("tc", "f16", True, 133, 400)])
def test_attention_q_pos_equals_per_batch_calls(ctx, impl, fmt, split, Lq, Lmax):
    dt, tdt = {"f16": (0, torch.float16), "bf16": (1, torch.bfloat16)}[fmt]
    B, H, D = 5, 4, 32
    E = H * D
    g = torch.Generator(device="cuda").manual_seed(Lq + Lmax + dt)
    q_pos = [0, Lmax - Lq, 64, 97, 1]
    cache = torch.randn(B, Lmax, 2 * E, device="cuda", generator=g)
    for b, p0 in enumerate(q_pos):
        cache[b, p0 + Lq:] = 1e4  # past each element's keys: never read as valid keys
    key_mask = torch.rand(B, Lmax, device="cuda", generator=g) > 0.2
    key_mask[:, 0] = True
    qm = torch.randn(B * Lq, E, device="cuda", generator=g)
    ch, cl = _split(ctx, cache.reshape(B * Lmax, 2 * E), dt, split)
    qh, ql = _split(ctx, qm, dt, split)
    mask_u8 = key_mask.to(torch.uint8)
    qp = torch.tensor(q_pos, dtype=torch.int32, device="cuda")
    ctx.set_option("attn", impl)
    try:
        o_hi = torch.zeros(B * Lq, E, dtype=torch.int16, device="cuda"); o_lo = torch.zeros_like(o_hi)
        ctx.attention(q=(qh, ql, E, 0), k=(ch, cl, 2 * E, 0), v=(ch, cl, 2 * E, E), o=(o_hi, o_lo, E, 0), B=B, H=H, Lq=Lq, Lk=Lmax, D=D,
                      scale=1 / math.sqrt(D), causal=True, key_mask=mask_u8, dtype=dt, kv_batch_rows=Lmax, mask_ld=Lmax, q_pos=qp)
        s_hi = torch.zeros_like(o_hi); s_lo = torch.zeros_like(o_hi)
        sl = lambda t, r0, n: None if t is None else t[r0:r0 + n]
        for b, p0 in enumerate(q_pos):
            ctx.attention(q=(sl(qh, b * Lq, Lq), sl(ql, b * Lq, Lq), E, 0), k=(sl(ch, b * Lmax, Lmax), sl(cl, b * Lmax, Lmax), 2 * E, 0),
                          v=(sl(ch, b * Lmax, Lmax), sl(cl, b * Lmax, Lmax), 2 * E, E), o=(s_hi[b * Lq:(b + 1) * Lq], s_lo[b * Lq:(b + 1) * Lq], E, 0),
                          B=1, H=H, Lq=Lq, Lk=p0 + Lq, D=D, scale=1 / math.sqrt(D), causal=True, key_mask=mask_u8[b:b + 1], dtype=dt,
                          kv_batch_rows=Lmax, mask_ld=Lmax, q_pos0=p0)
        torch.cuda.synchronize()
    finally:
        ctx.set_option("attn", "tc")
    assert torch.equal(o_hi, s_hi) and torch.equal(o_lo, s_lo)
    # and the fp64 statement (test_kernels_gpu.py's bars; bf16 pairs carry 16 significand bits instead of 22)
    ck = _merge(ch, cl, tdt).view(B, Lmax, 2 * E).double() if split else cache.to(tdt).double()
    qq = _merge(qh, ql, tdt).double() if split else qm.to(tdt).double()
    got = _merge(o_hi, o_lo, tdt)
    hd = lambda x: x.reshape(-1, H, D).permute(1, 0, 2)
    for b, p0 in enumerate(q_pos):
        n = p0 + Lq
        ref = _ref_attention(hd(qq[b * Lq:(b + 1) * Lq]), hd(ck[b, :n, :E]), hd(ck[b, :n, E:]), 1 / math.sqrt(D), p0, key_mask[b, :n])
        ref = ref.permute(1, 0, 2).reshape(Lq, E)
        tol = (1e-5 if fmt == "f16" else 3e-5) if split else 2e-3
        d = ((got[b * Lq:(b + 1) * Lq].double() - ref).norm() / ref.norm()).item()
        assert d < tol, (b, d)


def test_slot_kv_append_and_step_kernels(ctx):
    S, Q, E, Lmax = 6, 7, 64, 40
    L = Q + 1
    g = torch.Generator(device="cuda").manual_seed(4)
    ri = lambda *s: torch.randint(-30000, 30000, s, dtype=torch.int16, device="cuda", generator=g)
    # ---- kv append: columns [E, 3E) of the step rows -> rows b*Lmax + q_pos[b] + r
    qkv_hi, qkv_lo = ri(S * L, 3 * E), ri(S * L, 3 * E)
    kv_hi, kv_lo = ri(S * Lmax, 2 * E), ri(S * Lmax, 2 * E)
    q_pos = torch.tensor([0, Lmax - L, 5, 13, 1, 20], dtype=torch.int32, device="cuda")
    want_hi, want_lo = kv_hi.clone(), kv_lo.clone()
    for b in range(S):
        r0 = b * Lmax + int(q_pos[b])
        want_hi[r0:r0 + L] = qkv_hi[b * L:(b + 1) * L, E:]
        want_lo[r0:r0 + L] = qkv_lo[b * L:(b + 1) * L, E:]
    ctx.slot_kv_append(qkv_hi, qkv_lo, 3 * E, E, 2 * E, S, L, q_pos, kv_hi, kv_lo, 2 * E, Lmax)
    torch.cuda.synchronize()
    assert torch.equal(kv_hi, want_hi) and torch.equal(kv_lo, want_lo)

    # ---- step begin
    obs = torch.randn(S, Q, E, device="cuda", generator=g)
    obs_mask = torch.rand(S, Q, device="cuda", generator=g) > 0.3
    action = torch.randn(S, E, device="cuda", generator=g)
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")
    len_, n_valid = i32([0, 9, 17, 3, 30, 0]), i32([0, 6, 11, 2, 21, 0])
    has_action, active = i32([0, 1, 1, 1, 1, 0]), i32([1, 1, 1, 0, 1, 0])
    tokens = torch.empty(S * L, E, device="cuda")
    step_mask = torch.empty(S, L, dtype=torch.uint8, device="cuda")
    pos = torch.empty(S, L, dtype=torch.int64, device="cuda")
    qp = torch.full((S,), -7, dtype=torch.int32, device="cuda")
    slot_mask = ri(S, Lmax).to(torch.uint8) & 1
    want_slot_mask = slot_mask.clone()
    ctx.slot_step_begin(obs, obs_mask.to(torch.uint8), action, Lmax=Lmax, len_=len_, n_valid=n_valid, has_action=has_action, active=active,
                        tokens=tokens, step_mask=step_mask, pos=pos, q_pos=qp, slot_mask=slot_mask)
    torch.cuda.synchronize()
    want_tok = torch.zeros(S, L, E, device="cuda")
    want_m = torch.zeros(S, L, dtype=torch.uint8, device="cuda")
    for b in range(S):
        if has_action[b]:
            want_tok[b, 0], want_tok[b, 1:] = action[b], obs[b]
            want_m[b, 0], want_m[b, 1:] = 1, obs_mask[b]
        else:
            want_tok[b, :Q] = obs[b]
            want_m[b, :Q] = obs_mask[b]
    want_pos = torch.where(active[:, None] != 0, n_valid[:, None].long() + want_m.long().cumsum(1) - 1, torch.zeros_like(pos))
    want_qp = torch.where(active != 0, len_, torch.zeros_like(len_))
    for b in range(S):
        want_slot_mask[b, int(want_qp[b]):int(want_qp[b]) + L] = want_m[b]
    assert torch.equal(tokens.view(S, L, E), want_tok)
    assert torch.equal(step_mask, want_m) and torch.equal(pos, want_pos) and torch.equal(qp, want_qp)
    assert torch.equal(slot_mask, want_slot_mask)

    # ---- step end: row Q-1+has_action of each slot, then the active slots advance
    x = torch.randn(S * L, E + 4, device="cuda", generator=g)
    out = torch.empty(S, E, device="cuda")
    want_out = torch.stack([x[b * L + Q - 1 + int(has_action[b]), :E] for b in range(S)])
    act_b = active != 0
    want_len = torch.where(act_b, len_ + Q + has_action, len_)
    want_nv = torch.where(act_b, n_valid + step_mask.int().sum(1).int(), n_valid)
    want_ha = torch.where(act_b, torch.ones_like(has_action), has_action)
    ctx.slot_step_end(x, S, Q, E, step_mask, len_=len_, n_valid=n_valid, has_action=has_action, active=active, out=out)
    torch.cuda.synchronize()
    assert torch.equal(out, want_out)
    assert torch.equal(len_, want_len) and torch.equal(n_valid, want_nv) and torch.equal(has_action, want_ha)


def _rand_prompt(g, Lp, E):
    tok = torch.randn(Lp, 1, E, device="cuda", generator=g)
    msk = torch.rand(1, Lp, device="cuda", generator=g) > 0.25
    msk[:, 0] = True
    return tok, msk


@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
def test_staggered_episodes_match_own_history(mode):
    """Five slots over ten ticks: admissions at different ticks with different prompt lengths (below max_prompt_tokens), one slot
    released and re-admitted, one released for good, one never admitted; the obs width of the call grows between ticks (each
    episode's history is re-padded to its widest step, as scripts/example.py does).  Every active slot's row equals
    forward(...)[-1:] at B=1 over its own history; at each episode's end also the CPU oracle."""
    import vima_b200

    vima_b200.set_precision(mode)
    try:
        pol = build_policy("4M")
        cfg = synth.MODEL_CFGS["4M"]
        sd = oracle_state_dict("4M")
        E, S, Lp_cap = pol.embed_dim, 5, 12
        g = torch.Generator(device="cuda").manual_seed(31)
        widths = [2, 2, 3, 3, 4, 4, 5, 5, 6, 6]
        # tick -> (admit {slot: prompt length}, release [slots]) applied before the tick's step
        admits = {0: {0: 12, 2: 7}, 1: {1: 9}, 3: {4: 5}, 7: {0: 10}}
        releases = {4: [2], 6: [0]}
        ends = {(2, 3), (0, 5), (0, 9), (1, 9), (4, 9)}  # (slot, last tick) of each episode: compared with the oracle too
        eps = {}  # slot -> dict(prompt, obs list, mask list, actions list)
        with torch.no_grad():
            cache = pol.open_slots(S, max_tokens=64, max_prompt_tokens=Lp_cap)
            for t, Q in enumerate(widths):
                for b in releases.get(t, []):
                    pol.release(cache, [b])
                    del eps[b]
                if t in admits:
                    slots = sorted(admits[t])
                    Lp = max(admits[t].values())
                    toks, msks = [], []
                    for b in slots:  # one admission call of prompts padded to the longest; each episode keeps its own length
                        tok, msk = _rand_prompt(g, admits[t][b], E)
                        eps[b] = dict(prompt=(tok, msk), obs=[], mask=[], act=[])
                        pad = Lp - tok.shape[0]
                        toks.append(torch.cat([tok, torch.zeros(pad, 1, E, device="cuda")], 0))
                        msks.append(torch.cat([msk, torch.zeros(1, pad, dtype=torch.bool, device="cuda")], 1))
                    pol.admit(cache, slots, torch.cat(toks, 1), torch.cat(msks, 0))
                obs = torch.randn(1, S, Q, E, device="cuda", generator=g)
                msk = torch.rand(1, S, Q, device="cuda", generator=g) > 0.3
                msk[..., 0] = True
                act = torch.randn(1, S, E, device="cuda", generator=g)
                for b, ep in eps.items():
                    if ep["obs"]:
                        ep["act"].append(act[:, b:b + 1])
                    ep["obs"].append(obs[:, b:b + 1])
                    ep["mask"].append(msk[:, b:b + 1])
                out = pol.step_slots(cache, obs, msk, act)
                assert out.shape == (1, S, E)
                for b, ep in eps.items():
                    qmax = max(o.shape[2] for o in ep["obs"])
                    po = torch.cat([torch.cat([o, torch.zeros(1, 1, qmax - o.shape[2], E, device="cuda")], 2) for o in ep["obs"]], 0)
                    pm = torch.cat([torch.cat([m, torch.zeros(1, 1, qmax - m.shape[2], dtype=torch.bool, device="cuda")], 2) for m in ep["mask"]], 0)
                    pa = torch.cat(ep["act"], 0) if ep["act"] else None
                    ptok, pmsk = ep["prompt"]
                    full = pol.forward(obs_token=po, obs_mask=pm, action_token=pa, prompt_token=ptok, prompt_token_mask=pmsk)[-1:]
                    d = rel_l2(full.cpu(), out[:, b:b + 1].cpu())
                    assert d < (2e-6 if mode == "f16x3" else 5e-5), (t, b, d)
                    if (b, t) in ends:
                        ref = O.policy_forward(sd, po.cpu(), pm.cpu(), None if pa is None else pa.cpu(), ptok.cpu(), pmsk.cpu(),
                                               n_head=cfg["sattn_n_heads"], xattn_n_head=cfg["xattn_n_heads"])[-1:]
                        assert rel_l2(ref, out[:, b:b + 1].cpu()) < 1e-3, (t, b)
            torch.cuda.synchronize()
            assert cache.active_host == [True, True, False, False, True]
            assert cache.len.tolist() == cache.len_host
            assert cache.active.tolist() == [1, 1, 0, 0, 1]
    finally:
        vima_b200.set_precision("f16x3")


@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
def test_lockstep_slots_equal_forward_step(mode):
    """All slots admitted together with full-length prompts: step_slots returns forward_step's rows bit for bit at every step
    (every kernel works per row; the first step's extra dummy row is causally hidden, and a hidden key contributes exactly 0 with
    a rescale of exactly 1)."""
    import vima_b200

    vima_b200.set_precision(mode)
    try:
        pol = build_policy("4M")
        E, B, Lp, Q, T = pol.embed_dim, 4, 12, 5, 5
        g = torch.Generator(device="cuda").manual_seed(8)
        p_tok = torch.randn(Lp, B, E, device="cuda", generator=g)
        p_msk = torch.rand(B, Lp, device="cuda", generator=g) > 0.2
        p_msk[:, 0] = True
        obs = torch.randn(T, B, Q, E, device="cuda", generator=g)
        msk = torch.rand(T, B, Q, device="cuda", generator=g) > 0.3
        msk[..., 0] = True
        act = torch.randn(T, B, E, device="cuda", generator=g)
        Lmax = T * (Q + 1)
        with torch.no_grad():
            dc = pol.start_decode(p_tok, p_msk, max_tokens=Lmax)
            sc = pol.open_slots(B, max_tokens=Lmax, max_prompt_tokens=Lp)
            pol.admit(sc, list(range(B)), p_tok, p_msk)
            for t in range(T):
                a = None if t == 0 else act[t - 1:t]
                want = pol.forward_step(dc, obs[t:t + 1], msk[t:t + 1], a)
                got = pol.step_slots(sc, obs[t:t + 1], msk[t:t + 1], act[t:t + 1] if a is None else a)
                assert torch.equal(want, got), (t, rel_l2(want.cpu(), got.cpu()))
            assert sc.len_host == [dc.L] * B
    finally:
        vima_b200.set_precision("f16x3")


def test_graph_replay_equals_eager_schedule():
    """A step captured once and replayed across a schedule with admissions and releases between replays equals the eager schedule
    bit for bit; capturing leaves the slot state as it was."""
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = build_policy("4M")
    E, S, Lp, Q, ticks = pol.embed_dim, 4, 10, 4, 7
    g = torch.Generator(device="cuda").manual_seed(12)
    prompts = {k: _rand_prompt(g, Lp, E) for k in range(4)}
    schedule = {0: ("admit", [0, 1], [0, 1]), 2: ("admit", [2], [2]), 3: ("release", [0], None), 4: ("admit", [0], [3])}
    obs = torch.randn(ticks, S, Q, E, device="cuda", generator=g)
    msk = torch.rand(ticks, S, Q, device="cuda", generator=g) > 0.3
    msk[..., 0] = True
    act = torch.randn(ticks, S, E, device="cuda", generator=g)

    def run(step, cache):
        outs = []
        for t in range(ticks):
            if t in schedule:
                kind, slots, pk = schedule[t]
                if kind == "admit":
                    pol.admit(cache, slots, torch.cat([prompts[k][0] for k in pk], 1), torch.cat([prompts[k][1] for k in pk], 0))
                else:
                    pol.release(cache, slots)
            active = [b for b in range(S) if cache.active_host[b]]  # an inactive slot's row is unspecified
            outs.append(step(cache, obs[t:t + 1], msk[t:t + 1], act[t:t + 1])[:, active].clone())
        torch.cuda.synchronize()
        return outs

    with torch.no_grad():
        eager = run(pol.step_slots, pol.open_slots(S, max_tokens=64, max_prompt_tokens=Lp))
        cache = pol.open_slots(S, max_tokens=64, max_prompt_tokens=Lp)
        pol.admit(cache, [3], prompts[3][0], prompts[3][1])  # capture with one slot already holding an episode
        before = cache.state()
        gs = pol.capture_step_slots(cache, obs[:1], msk[:1], act[:1])
        torch.cuda.synchronize()
        after = cache.state()
        assert all(torch.equal(x, y) for x, y in zip(before[0], after[0])) and before[1] == after[1]
        assert gs.kernels_per_replay > 20
        pol.release(cache, [3])
        graphed = run(lambda c, o, m, a: gs(o, m, a), cache)
    for t, (w, x) in enumerate(zip(eager, graphed)):
        assert torch.equal(w, x), t
    assert gs.replays == ticks


def test_refusals_leave_state_unchanged():
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = build_policy("4M")
    E, S, Lp, Q = pol.embed_dim, 3, 8, 5
    g = torch.Generator(device="cuda").manual_seed(2)
    ptok, pmsk = _rand_prompt(g, Lp, E)
    obs = torch.randn(1, S, Q, E, device="cuda", generator=g)
    msk = torch.ones(1, S, Q, dtype=torch.bool, device="cuda")
    act = torch.randn(1, S, E, device="cuda", generator=g)

    def same(a, b):
        return all(torch.equal(x, y) for x, y in zip(a[0], b[0])) and a[1] == b[1]

    with torch.no_grad():
        cache = pol.open_slots(S, max_tokens=2 * (Q + 1), max_prompt_tokens=Lp)
        pol.admit(cache, [1], ptok, pmsk)
        pol.step_slots(cache, obs, msk, act)  # slot 1 at len Q = 5 of 12
        torch.cuda.synchronize()
        st = cache.state()
        pm = cache.prompt_mask.clone()
        vima_b200.set_precision("f16f8")
        try:
            with pytest.raises(ValueError):
                pol.step_slots(cache, obs, msk, act)  # opened in f16x3
            with pytest.raises(ValueError):
                pol.admit(cache, [0], ptok, pmsk)
        finally:
            vima_b200.set_precision("f16x3")
        assert same(st, cache.state()) and torch.equal(pm, cache.prompt_mask)
        long_tok, long_msk = _rand_prompt(g, Lp + 1, E)
        with pytest.raises(ValueError):
            pol.admit(cache, [0], long_tok, long_msk)  # longer than max_prompt_tokens
        with pytest.raises(ValueError):
            pol.admit(cache, [3], ptok, pmsk)  # no such slot
        assert same(st, cache.state()) and torch.equal(pm, cache.prompt_mask)
        pol.step_slots(cache, obs, msk, act)  # slot 1 at len 5 + Q+1 = 11 of 12
        torch.cuda.synchronize()
        st = cache.state()
        with pytest.raises(ValueError):
            pol.step_slots(cache, obs, msk, act)  # capacity
        assert same(st, cache.state())
        # the deferred position-id error of a masked first obs token, as forward_step reports it
        pol.release(cache, [1])
        pol.admit(cache, [0], ptok, pmsk)
        bad = msk.clone()
        bad[0, 0, 0] = False
        with pytest.raises(IndexError):
            pol.step_slots(cache, obs[:, :, :1], bad[:, :, :1], act)
            pol.xattn_gpt.check_errors()
