"""GPU: slot episodes admitted mid-way from their recorded history (admit_history).  The two kernels against torch statements of the
layout and state; for all four policies in f16x3 and f16f8, a staggered schedule that releases episodes mid-run and re-admits them
from their recorded tokens (into other slots, several lengths in one call, one at steps = 0) stays within forward's bars at B = 1 and
the oracle's at episode ends; the bit-exact properties (steps = 0 equals admit, untouched slots, page placement on NaN pools, NaN in
ignored rows, forks and swaps of a resumed slot); episodes carried across a weight update into a new cache; Gato resumed past 768
tokens; graph replays across an admission; no host synchronisation; refusals touch nothing."""
import pytest
import torch

from oracle import synth, vima_oracle as O
from tests.test_baseline_decode_gpu import BARS, _oracle, _oracle_sd
from tests.test_kv_pages_gpu import NAN_BITS, _policy
from tests.test_kv_swap_gpu import _same, _snapshot
from tests.util import rel_l2

pytestmark = pytest.mark.gpu

KINDS = ["vima", "gato", "gpt", "flamingo"]
LP, T_EP = 12, 9  # prompt tokens, recorded steps per episode


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    return _C.Context.get(torch.device("cuda", 0))


@pytest.fixture(autouse=True)
def _precision_reset():
    yield
    import vima_b200

    vima_b200.set_precision("f16x3")


# ------------------------------------------------------------------------------------------------- kernels
def _ref_layout(obs, om, act, steps, P, L, pre_mask):
    """torch statement of vima_slot_assemble_history: tokens (L,n,E), mask / pos (n,L) with columns [0, P) of mask given."""
    T, n, Q, E = obs.shape
    tok = torch.zeros(L, n, E, device="cuda")
    mask = torch.zeros(n, L, dtype=torch.uint8, device="cuda")
    pos = torch.zeros(n, L, dtype=torch.int64, device="cuda")
    mask[:, :P] = pre_mask
    for j, k in enumerate(steps):
        cols, ms = [], []
        for t in range(k):
            cols += [obs[t, j, q] for q in range(Q)]
            ms += [int(om[t, j, q]) if om is not None else 1 for q in range(Q)]
            if t < k - 1:
                cols.append(act[t, j])
                ms.append(1)
        if cols:
            tok[P:P + len(cols), j] = torch.stack(cols)
            m = torch.tensor(ms, dtype=torch.int64, device="cuda")
            mask[j, P:P + len(cols)] = m.to(torch.uint8)
            pos[j, P:P + len(cols)] = int(pre_mask[j].sum()) + torch.cumsum(m, 0) - 1
    return tok, mask, pos


@pytest.mark.parametrize("P", [0, 13])
@pytest.mark.parametrize("masked", [True, False])
def test_history_kernels_equal_torch(ctx, P, masked):
    g = torch.Generator(device="cuda").manual_seed(P + masked)
    T, n, Q, E, S, Lmax = 5, 5, 3, 24, 7, 80
    steps = [2, 0, 5, 1, 3]
    obs = torch.randn(T, n, Q, E, device="cuda", generator=g)
    act = torch.randn(T, n, E, device="cuda", generator=g)
    om = (torch.rand(T, n, Q, device="cuda", generator=g) > 0.3).to(torch.uint8) if masked else None
    for j, k in enumerate(steps):  # rows never read
        obs[k:, j] = float("nan")
        act[k:, j] = float("nan")
        if om is not None:
            om[k:, j] = 7
    lens = [P + (k * (Q + 1) - 1 if k else 0) for k in steps]
    L = max(lens) + 3  # and padding past the longest
    pre = (torch.rand(n, P, device="cuda", generator=g) > 0.4).to(torch.uint8)
    tok = torch.full((L, n, E), float("nan"), device="cuda")
    mask = torch.full((n, L), 9, dtype=torch.uint8, device="cuda")
    pos = torch.full((n, L), -7, dtype=torch.int64, device="cuda")
    mask[:, :P] = pre
    tok[:P] = 1.5
    st = torch.tensor(steps, dtype=torch.int32, device="cuda")
    ctx.slot_assemble_history(obs, om, act, st, P, tok, mask, pos)
    wt, wm, wp = _ref_layout(obs, om, act, steps, P, L, pre)
    assert torch.equal(tok[P:], wt[P:]) and (tok[:P] == 1.5).all()
    assert torch.equal(mask, wm) and torch.equal(pos[:, P:], wp[:, P:]) and (pos[:, :P] == -7).all()
    # the state kernel: slots in arbitrary order, one out of range (skipped), untouched slots keep their rows
    slots = [4, 0, 6, 9, 2]
    smask = torch.full((S, Lmax), 5, dtype=torch.uint8, device="cuda")
    state = [torch.full((S,), -3, dtype=torch.int32, device="cuda") for _ in range(4)]
    atok = torch.full((S, E), 0.25, device="cuda")
    ctx.slot_admit_history(torch.tensor(slots, dtype=torch.int32, device="cuda"), st, Q, P, mask, act, Lmax, smask, len_=state[0],
                           n_valid=state[1], has_action=state[2], active=state[3], action_token=atok)
    for j, (b, k, ln) in enumerate(zip(slots, steps, lens)):
        if b >= S:
            continue
        want = torch.zeros(Lmax, dtype=torch.uint8, device="cuda")
        want[:ln] = wm[j, :ln]
        assert torch.equal(smask[b], want), j
        assert [int(t[b]) for t in state] == [ln, int(wm[j, :ln].sum()), int(k > 0), 1], j
        assert torch.equal(atok[b], act[k - 1, j] if k else torch.full((E,), 0.25, device="cuda")), j
    for b in (1, 3, 5):
        assert (smask[b] == 5).all() and all(int(t[b]) == -3 for t in state) and (atok[b] == 0.25).all()


def test_history_kernel_refusals(ctx):
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    obs, act = torch.zeros(1, 1, 2, 8, device="cuda"), torch.zeros(1, 1, 8, device="cuda")
    tok, m, p = torch.zeros(4, 1, 8, device="cuda"), torch.zeros(1, 4, dtype=torch.uint8, device="cuda"), torch.zeros(1, 4, dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match="slot_assemble_history"):
        ctx.slot_assemble_history(obs, None, act, st, 5, tok, m, p)  # P > L
    with pytest.raises(RuntimeError, match="slot_admit_history"):  # L > Lmax
        ctx.slot_admit_history(st, st, 2, 0, m, act, 3, torch.zeros(1, 3, dtype=torch.uint8, device="cuda"), len_=st, n_valid=st,
                               has_action=st, active=st, action_token=torch.zeros(1, 8, device="cuda"))


# ------------------------------------------------------------------------------------------------- policies
def _Q(kind, pol):
    return 4 if kind == "vima" else pol._obj_xf_num_queries


def _episodes(kind, pol, names, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    E, Q = pol.embed_dim, _Q(kind, pol)
    out = {}
    for nm in names:
        pm = torch.rand(1, LP, device="cuda", generator=g) > 0.25
        pm[:, 0] = True
        obs = torch.randn((T_EP, E) if kind == "gpt" else (T_EP, Q, E), device="cuda", generator=g)
        msk = torch.rand(T_EP, Q, device="cuda", generator=g) > 0.25 if kind == "vima" else torch.ones(T_EP, Q, dtype=torch.bool, device="cuda")
        msk[:, 0] = True
        out[nm] = dict(pt=torch.randn(LP, 1, E, device="cuda", generator=g), pm=pm, obs=obs, msk=msk,
                       act=torch.randn(T_EP, E, device="cuda", generator=g))
    return out


def _lmax(kind, pol, T=T_EP):
    return (LP + 1 if kind in ("gato", "gpt") else 0) + T * (_Q(kind, pol) + 1)


def _open(kind, pol, S, kv_pool_tokens=None, nan=False, Lmax=None):
    from vima_b200 import engine as eng

    Lmax = Lmax or _lmax(kind, pol)
    if kind in ("gato", "gpt"):
        c = pol.open_slots(S, max_tokens=Lmax, kv_pool_tokens=kv_pool_tokens)
    else:
        c = pol.open_slots(S, max_tokens=Lmax, max_prompt_tokens=LP, kv_pool_tokens=kv_pool_tokens)
    if nan:
        v = NAN_BITS[eng.prec().dtype]
        for t in c.kv_hi + c.kv_lo + (c.prompt_kv_hi + c.prompt_kv_lo if c.Lp_cap else []):
            if t is not None:
                t[64:] = v
    return c


def _admit(pol, cache, slots, eps):
    pol.admit(cache, slots, torch.cat([e["pt"] for e in eps], 1), torch.cat([e["pm"] for e in eps], 0))


def _admit_history(kind, pol, cache, slots, eps, steps, nan=False):
    """admit_history of episodes eps at steps, every recorded row passed (T = T_EP); rows t >= steps[j] zero, or NaN (mask True)."""
    obs = torch.stack([e["obs"] for e in eps], 1).clone()
    msk = torch.stack([e["msk"] for e in eps], 1).clone()
    act = torch.stack([e["act"] for e in eps], 1).clone()
    for j, k in enumerate(steps):
        obs[k:, j] = float("nan") if nan else 0.0
        act[k:, j] = float("nan") if nan else 0.0
        msk[k:, j] = nan
    pt, pm = torch.cat([e["pt"] for e in eps], 1), torch.cat([e["pm"] for e in eps], 0)
    if kind == "vima":
        pol.admit_history(cache, slots, pt, pm, obs, msk, act, steps)
    else:
        pol.admit_history(cache, slots, pt, pm, obs, act, steps)


def _step(kind, pol, cache, cur, steps):
    """step_slots with slot b fed episode cur[b] (a dict, or None) at its step steps[id(cur[b])]: -> (1, S, E)."""
    S, E = cache.S, pol.embed_dim
    Q = _Q(kind, pol)
    obs = torch.zeros((1, S, E) if kind == "gpt" else (1, S, Q, E), device="cuda")
    msk = torch.ones(1, S, Q, dtype=torch.bool, device="cuda")
    act = torch.zeros(1, S, E, device="cuda")
    for b, e in enumerate(cur):
        if e is not None:
            k = steps[id(e)]
            obs[0, b], msk[0, b] = e["obs"][k], e["msk"][k]
            if k:
                act[0, b] = e["act"][k - 1]
    out = pol.step_slots(cache, obs, msk, act) if kind == "vima" else pol.step_slots(cache, obs, act)
    for e in cur:
        if e is not None:
            steps[id(e)] += 1
    return out


def _forward_last(kind, pol, e, k):
    """forward(...)[-1:] at B = 1 over episode e's first k+1 observations and k actions."""
    a = e["act"][:k].unsqueeze(1) if k else None
    if kind == "vima":
        return pol.forward(e["obs"][:k + 1].unsqueeze(1), e["msk"][:k + 1].unsqueeze(1), a, e["pt"], e["pm"])[-1:]
    return pol.forward(e["obs"][:k + 1].unsqueeze(1), a, e["pt"], e["pm"])[-1:]


def _oracle_last(kind, e, k):
    a = e["act"][:k].unsqueeze(1).cpu() if k else None
    if kind == "vima":
        from tests.test_oracle_golden import oracle_state_dict

        cfg = synth.MODEL_CFGS["4M"]
        return O.policy_forward(oracle_state_dict("4M"), e["obs"][:k + 1].unsqueeze(1).cpu(), e["msk"][:k + 1].unsqueeze(1).cpu(), a,
                                e["pt"].cpu(), e["pm"].cpu(), n_head=cfg["sattn_n_heads"], xattn_n_head=cfg["xattn_n_heads"])[-1:]
    return _oracle(kind, _oracle_sd(kind), e["obs"][:k + 1].unsqueeze(1), a, e["pt"], e["pm"])[-1:]


@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
@pytest.mark.parametrize("kind", KINDS)
def test_resumed_episodes_match_own_history(kind, mode):
    """Five slots: e0, e1, e2 admitted at tick 0, e3 at tick 1; e1 released at tick 2, e0 and e3 at tick 3; at tick 4 one call
    re-admits e0 (3 steps) into slot 3, e1 (2 steps) into slot 0, e3 (2 steps) into slot 1 and starts e4 (0 steps) in slot 4.
    Every active slot's row at every tick is within BARS of forward(...)[-1:] at B = 1 over its own history; the last tick's rows
    are also within 1e-3 of the oracle."""
    import vima_b200

    vima_b200.set_precision(mode)
    pol = _policy(kind)
    ep = _episodes(kind, pol, ["e0", "e1", "e2", "e3", "e4"], 41)
    e0, e1, e2, e3, e4 = (ep[k] for k in ("e0", "e1", "e2", "e3", "e4"))
    steps = {id(e): 0 for e in ep.values()}
    ticks = 8
    with torch.no_grad():
        c = _open(kind, pol, 5)
        cur = [None] * 5
        for t in range(ticks):
            if t == 0:
                _admit(pol, c, [0, 1, 2], [e0, e1, e2])
                cur[:3] = [e0, e1, e2]
            if t == 1:
                _admit(pol, c, [3], [e3])
                cur[3] = e3
            if t == 2:
                pol.release(c, [1])
                cur[1] = None
            if t == 3:
                pol.release(c, [0, 3])
                cur[0] = cur[3] = None
            if t == 4:
                assert [steps[id(e)] for e in (e0, e1, e3, e4)] == [3, 2, 2, 0]
                _admit_history(kind, pol, c, [3, 0, 1, 4], [e0, e1, e3, e4], [3, 2, 2, 0])
                cur = [e1, e3, e2, e0, e4]
            before = {id(e): steps[id(e)] for e in cur if e is not None}
            out = _step(kind, pol, c, cur, steps)
            for b, e in enumerate(cur):
                if e is None:
                    continue
                k = before[id(e)]
                d = rel_l2(_forward_last(kind, pol, e, k).cpu(), out[:, b:b + 1].cpu())
                assert d < BARS[mode], (t, b, k, d)
                if t == ticks - 1:
                    assert rel_l2(_oracle_last(kind, e, k), out[:, b:b + 1].cpu()) < 1e-3, (t, b)
        torch.cuda.synchronize()
        assert c.len.tolist() == c.len_host and c.active.tolist() == [1] * 5


def _gather_rows(pool, table, b, cols):
    """Rows of cache columns [0, cols) of slot b through a page table."""
    idx = [int(table[b, j // 64]) * 64 + j % 64 for j in range(cols)]
    return pool[torch.tensor(idx, dtype=torch.int64, device="cuda")]


@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
@pytest.mark.parametrize("kind", KINDS)
def test_zero_steps_equals_admit(kind, mode):
    """admit_history with steps = 0 for every episode leaves the cache as admit does (state, mask rows, prompt / prefix K/V rows
    through the table, host mirrors), and the following steps are bit-identical."""
    import vima_b200

    vima_b200.set_precision(mode)
    pol = _policy(kind)
    ep = _episodes(kind, pol, ["a", "b"], 43)
    eps = [ep["a"], ep["b"]]
    with torch.no_grad():
        A, B = _open(kind, pol, 3, nan=True), _open(kind, pol, 3, nan=True)
        _admit(pol, A, [2, 0], eps)
        _admit_history(kind, pol, B, [2, 0], eps, [0, 0], nan=True)
        torch.cuda.synchronize()
        sa, sb = _snapshot(A), _snapshot(B)
        assert sa[1] == sb[1] and len(sa[0]) == len(sb[0])
        assert all(torch.equal(x, y) for i, (x, y) in enumerate(zip(sa[0], sb[0])) if i != 6)  # 6: the mask, compared up to len below
        for b in (0, 2):
            n = A.len_host[b]
            assert torch.equal(A.mask[b, :n], B.mask[b, :n])
            for pa, pb in zip(A.kv_hi + A.kv_lo, B.kv_hi + B.kv_lo):
                if pa is not None:
                    assert torch.equal(_gather_rows(pa, A.page_table, b, n), _gather_rows(pb, B.page_table, b, n))
            if A.Lp_cap:
                for pa, pb in zip(A.prompt_kv_hi + A.prompt_kv_lo, B.prompt_kv_hi + B.prompt_kv_lo):
                    if pa is not None:
                        assert torch.equal(_gather_rows(pa, A.prompt_page_table, b, 64), _gather_rows(pb, B.prompt_page_table, b, 64))
        outs = []
        for c in (A, B):
            steps = {id(e): 0 for e in eps}
            outs.append([_step(kind, pol, c, [eps[1], None, eps[0]], steps).clone() for _ in range(3)])
        torch.cuda.synchronize()
    for x, y in zip(*outs):
        assert torch.equal(x[:, [0, 2]], y[:, [0, 2]])


@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
@pytest.mark.parametrize("kind", KINDS)
def test_bit_exact_properties(kind, mode):
    """Reference R: slots 0 and 1 run e0 / e1 from tick 0; at tick 2 admit_history puts e2 (4 steps) into slot 2 and e3 (1 step)
    into slot 3 on the default pool (ignored rows zero), then three ticks.  Bit for bit:
      - a run without the admission gives slots 0 and 1 the same rows (slots outside the call are untouched);
      - the smallest pool with a shuffled free list, NaN-filled, and NaN in the ignored rows gives every slot the same rows;
      - forking slot 2 into slot 4 and swapping slot 3 out and back into slot 5 right after the admission: slots 4 and 5 continue
        as slots 2 and 3 do."""
    import vima_b200

    vima_b200.set_precision(mode)
    pol = _policy(kind)
    ep = _episodes(kind, pol, ["e0", "e1", "e2", "e3"], 47)
    e0, e1, e2, e3 = (ep[k] for k in ("e0", "e1", "e2", "e3"))

    def run(cache, admit=True, nan=False, branch=False, shuffle=False):
        if shuffle:
            import random

            random.Random(3).shuffle(cache.pages.free)
        steps = {id(e): 0 for e in ep.values()}
        steps[id(e2)], steps[id(e3)] = 4, 1
        cur = [e0, e1, None, None, None, None]
        _admit(pol, cache, [0, 1], [e0, e1])
        outs, peak = [], 0
        for t in range(5):
            if t == 2 and admit:
                _admit_history(kind, pol, cache, [2, 3], [e2, e3], [4, 1], nan=nan)
                cur[2:4] = [e2, e3]
                if branch:
                    pol.fork_slots(cache, [2], [4])
                    pol.swap_in(cache, [5], pol.swap_out(cache, [3]))
                    cur[3:6] = [None, e2, e3]
                    steps[id(e2)] = steps[id(e3)] = None  # per-slot counters below
            if branch and t >= 2:
                out = _step_branch(kind, pol, cache, cur, t)
            else:
                out = _step(kind, pol, cache, cur, steps)
            peak = max(peak, cache.kv_pages_total - cache.kv_pages_free)
            outs.append(out.clone())
        torch.cuda.synchronize()
        return outs, peak

    with torch.no_grad():
        R, peak = run(_open(kind, pol, 6))
        N, _ = run(_open(kind, pol, 6), admit=False)
        small = _open(kind, pol, 6, kv_pool_tokens=peak * 64, nan=True)
        Z, _ = run(small, nan=True, shuffle=True)
        F, _ = run(_open(kind, pol, 6, nan=True), branch=True)
    for t in range(5):
        assert torch.equal(R[t][:, :2], N[t][:, :2]), t
        live = 4 if t >= 2 else 2  # an inactive slot's row is unspecified
        assert torch.equal(R[t][:, :live], Z[t][:, :live]), t
        if t >= 2:
            assert torch.equal(R[t][:, :3], F[t][:, :3]) and torch.equal(R[t][:, 2], F[t][:, 4]) and torch.equal(R[t][:, 3], F[t][:, 5]), t


def _step_branch(kind, pol, cache, cur, t):
    """_step where slots 2 / 4 hold e2 and slot 5 e3, all at the step they reach at tick t (e2 resumed at 4 steps, e3 at 1)."""
    steps = {}
    for b, e in enumerate(cur):
        if e is not None:
            steps[id(e)] = {2: t - 2 + 4, 4: t - 2 + 4, 5: t - 2 + 1}.get(b, t)
    # _step advances per episode, but e2 sits in two slots at the same step: feed per slot
    S, E = cache.S, pol.embed_dim
    Q = _Q(kind, pol)
    obs = torch.zeros((1, S, E) if kind == "gpt" else (1, S, Q, E), device="cuda")
    msk = torch.ones(1, S, Q, dtype=torch.bool, device="cuda")
    act = torch.zeros(1, S, E, device="cuda")
    for b, e in enumerate(cur):
        if e is not None:
            k = steps[id(e)]
            obs[0, b], msk[0, b] = e["obs"][k], e["msk"][k]
            if k:
                act[0, b] = e["act"][k - 1]
    return pol.step_slots(cache, obs, msk, act) if kind == "vima" else pol.step_slots(cache, obs, act)


@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
@pytest.mark.parametrize("kind", KINDS)
def test_episodes_survive_a_weight_update(kind, mode):
    """Run two episodes three ticks, perturb the weights with load_state_dict: the old cache refuses to step, a new cache takes both
    episodes by admit_history, and its next steps are within BARS of forward(...)[-1:] under the new weights."""
    import vima_b200

    vima_b200.set_precision(mode)
    pol = _policy(kind)
    ep = _episodes(kind, pol, ["a", "b"], 53)
    eps = [ep["a"], ep["b"]]
    orig = {k: v.clone() for k, v in pol.state_dict().items()}
    try:
        with torch.no_grad():
            old = _open(kind, pol, 2)
            _admit(pol, old, [0, 1], eps)
            steps = {id(e): 0 for e in eps}
            for _ in range(3):
                _step(kind, pol, old, eps, steps)
            g = torch.Generator(device="cuda").manual_seed(5)
            sd = {k: (v + 0.01 * torch.randn(v.shape, device=v.device, generator=g) * v.abs().mean() if v.is_floating_point() and v.dim() == 2
                      else v) for k, v in orig.items()}
            pol.load_state_dict(sd)
            with pytest.raises(ValueError, match="weights"):
                _step(kind, pol, old, eps, dict(steps))
            new = _open(kind, pol, 3)
            _admit_history(kind, pol, new, [2, 0], eps, [3, 3])
            cur = [eps[1], None, eps[0]]
            for _ in range(3):
                k = steps[id(eps[0])]
                out = _step(kind, pol, new, cur, steps)
                for b, e in ((0, eps[1]), (2, eps[0])):
                    d = rel_l2(_forward_last(kind, pol, e, k).cpu(), out[:, b:b + 1].cpu())
                    assert d < BARS[mode], (b, k, d)
    finally:
        pol.load_state_dict(orig)


@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
def test_gato_resumed_past_768_tokens(mode):
    """gato_tiny at n_positions = 1024: two episodes of 40 and 45 recorded steps (prompt 20 tokens: 700 and 785 columns) resumed in
    one call, then two steps each, within test_long_history_gpu's bars of forward(...)[-1:]."""
    import vima_b200
    from tests.test_long_history_gpu import BARS as LBARS, gato_policy

    vima_b200.set_precision(mode)
    pol = gato_policy(1024)
    E, Q, Lp, T = pol.embed_dim, pol._obj_xf_num_queries, 20, 47
    g = torch.Generator(device="cuda").manual_seed(768)
    eps = []
    for _ in range(2):
        pm = torch.ones(1, Lp, dtype=torch.bool, device="cuda")
        pm[:, 15:] = False
        eps.append(dict(pt=torch.randn(Lp, 1, E, device="cuda", generator=g), pm=pm, obs=torch.randn(T, Q, E, device="cuda", generator=g),
                        msk=torch.ones(T, Q, dtype=torch.bool, device="cuda"), act=torch.randn(T, E, device="cuda", generator=g)))
    with torch.no_grad():
        c = pol.open_slots(2, max_tokens=1024)
        obs = torch.stack([e["obs"] for e in eps], 1)
        act = torch.stack([e["act"] for e in eps], 1)
        pol.admit_history(c, [1, 0], torch.cat([e["pt"] for e in eps], 1), torch.cat([e["pm"] for e in eps], 0), obs, act, [40, 45])
        assert c.len_host == [Lp + 1 + 45 * (Q + 1) - 1, Lp + 1 + 40 * (Q + 1) - 1] and c.len_host[0] > 768
        steps = {id(eps[0]): 40, id(eps[1]): 45}
        cur = [eps[1], eps[0]]
        for _ in range(2):
            ks = [steps[id(e)] for e in cur]
            out = _step("gato", pol, c, cur, steps)
            for b, (e, k) in enumerate(zip(cur, ks)):
                d = rel_l2(_forward_last("gato", pol, e, k).cpu(), out[:, b:b + 1].cpu())
                assert d < LBARS[mode], (b, k, d)


@pytest.mark.parametrize("kind", ["vima", "gato", "gpt", "flamingo"])
def test_graph_captured_before_admission_equals_eager(kind):
    """A capture_act_slots graph captured before an admit_history, replayed after it, equals eager act_slots (greedy)."""
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    ep = _episodes(kind, pol, ["a", "b", "c"], 59)
    E, Q, S = pol.embed_dim, _Q(kind, pol), 3
    runs = []
    with torch.no_grad():
        for graph in (False, True):
            c = _open(kind, pol, S)
            _admit(pol, c, [0], [ep["a"]])
            g = None
            if graph:
                obs = torch.zeros((1, S, E) if kind == "gpt" else (1, S, Q, E), device="cuda")
                args = (obs, torch.ones(1, S, Q, dtype=torch.bool, device="cuda")) if kind == "vima" else (obs,)
                g = pol.capture_act_slots(c, *args)
            _admit_history(kind, pol, c, [2, 1], [ep["b"], ep["c"]], [3, 1])
            cur, ks = [ep["a"], ep["c"], ep["b"]], [0, 1, 3]
            outs = []
            for t in range(3):
                obs = torch.stack([e["obs"][k + t] for e, k in zip(cur, ks)]).unsqueeze(0)
                msk = torch.stack([e["msk"][k + t] for e, k in zip(cur, ks)]).unsqueeze(0)
                args = (obs, msk) if kind == "vima" else (obs,)
                r = g(*args) if graph else pol.act_slots(c, *args)
                outs.append([d[k].clone() for d in r for k in sorted(d)] + [c.action_token.clone()])
            torch.cuda.synchronize()
            runs.append(outs)
    for x, y in zip(*runs):
        assert all(torch.equal(a, b) for a, b in zip(x, y))


@pytest.mark.parametrize("kind", ["vima", "gato"])
def test_admit_history_does_not_synchronise(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    ep = _episodes(kind, pol, ["a", "b"], 61)
    with torch.no_grad():
        c = _open(kind, pol, 4)
        _admit_history(kind, pol, c, [0, 1], [ep["a"], ep["b"]], [2, 0])  # first call: weights packed, guards armed
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            _admit_history(kind, pol, c, [3, 1, 2], [ep["b"], ep["a"], ep["a"]], [5, 1, 0])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        assert c.len.tolist() == c.len_host and c.active.tolist() == [int(a) for a in c.active_host] == [1, 1, 1, 1]
        assert c.has_action.tolist() == [int(a) for a in c.has_action_host] == [1, 1, 0, 1]
        want = torch.zeros_like(c.page_table)
        for b, own in enumerate(c.pages.owned):
            want[b, :len(own)] = torch.tensor(own, dtype=torch.int32)
        assert torch.equal(want, c.page_table)


@pytest.mark.parametrize("kind", KINDS)
def test_admit_history_refusals(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    ep = _episodes(kind, pol, ["a", "b"], 67)
    eps = [ep["a"], ep["b"]]
    Q, E = _Q(kind, pol), pol.embed_dim
    dec = kind in ("gato", "gpt")
    with torch.no_grad():
        c = _open(kind, pol, 3, kv_pool_tokens=2 * 64)  # one page left after slot 0's
        _admit(pol, c, [0], [ep["a"]])
        steps = {id(ep["a"]): 0}
        _step(kind, pol, c, [ep["a"], None, None], steps)
        torch.cuda.synchronize()
        st = _snapshot(c)

        def call(slots=(1, 2), k=(1, 1), n=2, **kw):
            a = dict(pt=torch.cat([e["pt"] for e in eps[:n]], 1), pm=torch.cat([e["pm"] for e in eps[:n]], 0),
                     obs=torch.stack([e["obs"] for e in eps[:n]], 1), msk=torch.stack([e["msk"] for e in eps[:n]], 1),
                     act=torch.stack([e["act"] for e in eps[:n]], 1))
            a.update(kw)
            if kind == "vima":
                pol.admit_history(c, list(slots), a["pt"], a["pm"], a["obs"], a["msk"], a["act"], k)
            else:
                pol.admit_history(c, list(slots), a["pt"], a["pm"], a["obs"], a["act"], k)

        bad = [dict(slots=(1, 1)), dict(slots=(1, 3)), dict(slots=(-1, 2)), dict(slots=(1,)), dict(k=(1,)), dict(k=(T_EP + 1, 0)),
               dict(k=(-1, 0)), dict(act=torch.zeros(T_EP, 2, E + 4, device="cuda")), dict(pm=torch.ones(2, LP + 1, dtype=torch.bool, device="cuda")),
               dict()]  # the last: two histories need two pages, one is free
        if kind == "vima":
            bad.append(dict(msk=torch.ones(T_EP, 2, Q + 1, dtype=torch.bool, device="cuda")))
        elif kind != "gpt":
            bad.append(dict(obs=torch.zeros(T_EP, 2, Q + 1, E, device="cuda")))
        if not dec:
            bad.append(dict(pt=torch.zeros(LP + 64, 2, E, device="cuda"), pm=torch.ones(2, LP + 64, dtype=torch.bool, device="cuda")))
        for kw in bad:
            with pytest.raises(ValueError):
                call(**kw)
        with pytest.raises(TypeError, match="host ints"):
            call(k=torch.ones(2, dtype=torch.int32, device="cuda"))
        # a history longer than max_tokens, in a cache whose pool is big enough
        short = _open(kind, pol, 2, Lmax=_lmax(kind, pol, 3))
        with pytest.raises(ValueError, match="max_tokens"):
            (pol.admit_history(short, [0], ep["a"]["pt"], ep["a"]["pm"], ep["a"]["obs"][:, None], ep["a"]["msk"][:, None], ep["a"]["act"][:, None], [4])
             if kind == "vima" else
             pol.admit_history(short, [0], ep["a"]["pt"], ep["a"]["pm"], ep["a"]["obs"][:, None], ep["a"]["act"][:, None], [4]))
        vima_b200.set_precision("f16f8")
        try:
            with pytest.raises(ValueError, match="precision"):
                call()
        finally:
            vima_b200.set_precision("f16x3")
        torch.cuda.synchronize()
        assert _same(st, _snapshot(c))
        pol.load_state_dict(pol.state_dict())  # same values, new version: the cache's K/V belong to the old weights
        with pytest.raises(ValueError, match="weights"):
            call()
        torch.cuda.synchronize()
        assert _same(st, _snapshot(c))
