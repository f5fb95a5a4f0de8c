"""GPU: seeded sampling on the action heads (vima_head_sample, MultiCategorical.sample / log_prob / entropy, ActionSampler) and the
closed-loop slot step of the four policies (act_slots, capture_act_slots).

Every draw is checked against an fp64 inverse-CDF choice made with the numpy restatement of the kernel's Philox uniform
(tests/test_philox_cpu.py); frequencies against fp64 probabilities; log-probabilities and entropies against
torch.distributions.Categorical in fp64; greedy acting against head_select and the hand-closed loop bit for bit."""
import math

import numpy as np
import pytest
import torch

from tests.policy_runner import build_policy
from tests.test_philox_cpu import head_uniforms

pytestmark = pytest.mark.gpu

VIMA_DIMS = [50, 100, 50, 50, 50, 50, 50, 100, 50, 50, 50, 50]  # the 12 sub-heads of VIMA's four action keys, in key order
ODD_DIMS = [1, 33, 64, 100, 7, 50, 130, 1500]  # one-wide, lane-crossing and multi-round (> 1024 columns) heads
BOUNDARY = 1e-6  # a draw whose u lies this close to a cumulative-probability boundary may go either way in fp32


def logit_rows(dims, n_rows, seed):
    """[n_rows, sum(dims)] fp32: row r is kind r % len(kinds) in every head -- ties, +-1e4, -inf columns, all -inf, and
    policy-like logits (a few dominant columns over a flat tail)."""
    g = torch.Generator().manual_seed(seed)

    def ties(w, gap):
        x = torch.randn(w, generator=g)
        x[1::gap] = 2.0
        return x

    def some_neg_inf(w):
        x = torch.randn(w, generator=g)
        x[torch.arange(w) % 3 == 0] = -math.inf
        if w == 1:
            x[0] = 0.5
        return x

    def policy_like(w):
        x = 0.3 * torch.randn(w, generator=g)
        x[torch.randint(0, w, (3,), generator=g)] += torch.tensor([4.0, 3.0, 2.5])
        return x

    def one_finite(w):
        x = torch.full((w,), -math.inf)
        x[int(torch.randint(0, w, (1,), generator=g))] = 1.0
        return x

    kinds = [
        lambda w: torch.randn(w, generator=g),
        lambda w: 3.0 * torch.randn(w, generator=g),
        lambda w: ties(w, 5),
        lambda w: ties(w, 32),
        lambda w: torch.full((w,), 0.25),
        some_neg_inf,
        one_finite,
        lambda w: 1e4 + torch.randn(w, generator=g),
        lambda w: -1e4 + torch.randn(w, generator=g),
        lambda w: torch.sign(torch.randn(w, generator=g)) * 1e4 + torch.randn(w, generator=g),
        lambda w: 1e4 + ties(w, 7),
        policy_like,
        policy_like,
        policy_like,
        lambda w: torch.full((w,), -math.inf),
    ]
    rows = [torch.cat([kinds[r % len(kinds)](w) for w in dims]).float() for r in range(n_rows)]
    return torch.stack(rows)


def _off(dims):
    return torch.tensor(np.concatenate([[0], np.cumsum(dims)]), dtype=torch.int32, device="cuda")


def expected_draws(x, dims, u):
    """fp64 inverse-CDF choice per (row, head) for uniforms u [rows, heads], and a mask of draws within BOUNDARY of a boundary."""
    x = x.double().numpy()
    want = np.zeros(u.shape, dtype=np.int64)
    near = np.zeros(u.shape, dtype=bool)
    o = 0
    for h, w in enumerate(dims):
        xs = x[:, o:o + w]
        o += w
        mx = xs.max(axis=1, keepdims=True)
        with np.errstate(invalid="ignore", divide="ignore"):
            p = np.exp(xs - mx)
            p[~np.isfinite(xs)] = 0.0
            cdf = np.cumsum(p, axis=1) / p.sum(axis=1, keepdims=True)
        uh = u[:, h:h + 1]
        want[:, h] = np.minimum((cdf <= uh).sum(axis=1), w - 1)
        near[:, h] = (np.abs(cdf - uh) <= BOUNDARY).any(axis=1)
    return want, near


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    return _C.Context.get(torch.device("cuda:0"))


@pytest.mark.parametrize("dims,n_rows", [(VIMA_DIMS, 4500), (ODD_DIMS, 600)])
def test_draws_are_fp64_inverse_cdf_choices(dims, n_rows):
    """Every draw equals the fp64 inverse-CDF choice with the restated Philox uniform, over consecutive draws whose index crosses
    the counter's 32-bit word boundary; draws within 1e-6 of a boundary are excluded (fewer than 0.01 % on the VIMA heads; the
    1500-column head has more boundaries, so there the bar is 0.1 %).  No draw is ever an
    out-of-head index or a -inf column; a head of all -inf logits gives 0."""
    from vima_b200.nn.action import ActionSampler, sample_heads

    x = logit_rows(dims, n_rows, seed=3)
    xd = x.cuda()
    seed = 0x9E3779B97F4A7C15
    s = ActionSampler(seed, "cuda")
    first = (1 << 32) - 3
    s.counter.fill_(first)
    n_draws, excluded, total = 6, 0, 0
    for k in range(n_draws):
        got = sample_heads(xd, dims, sampler=s)[0].cpu().numpy()
        u = head_uniforms(n_rows, len(dims), seed, first + k)
        want, near = expected_draws(x, dims, u)
        o = 0
        for h, w in enumerate(dims):
            xs = x[:, o:o + w]
            o += w
            g = got[:, h]
            assert ((g >= 0) & (g < w)).all(), (k, h)
            dead = torch.isinf(xs).all(dim=1).numpy() & (xs[:, 0] < 0).numpy()
            assert (g[dead] == 0).all()
            picked = xs[torch.arange(n_rows), torch.from_numpy(g)]
            assert not torch.isinf(picked[torch.from_numpy(~dead)]).any(), (k, h)
            ok = ~near[:, h] & ~dead
            bad = np.nonzero(g[ok] != want[ok, h])[0]
            assert bad.size == 0, (k, h, bad[:5], g[ok][bad[:5]], want[ok, h][bad[:5]])
            excluded += int((near[:, h] & ~dead).sum())
            total += int((~dead).sum())
    assert s.draws == first + n_draws
    print(f"{excluded} of {total} draws within {BOUNDARY} of a boundary ({100.0 * excluded / total:.4f} %)")
    assert excluded < (1e-4 if dims is VIMA_DIMS else 1e-3) * total


def test_frequencies_chi_square():
    """2^20 draws per head from one row of policy-like logits, repeated: the column counts fit the fp64 probabilities (chi-square over
    the columns expected >= 5 times, the rest pooled, p > 1e-4 for each head).  Deterministic given the seed."""
    from scipy.stats import chi2

    from vima_b200.nn.action import ActionSampler, sample_heads

    x = logit_rows(VIMA_DIMS, 12, seed=9)[11:12]  # a policy-like row
    rows, n_draws = 1 << 16, 16
    xd = x.cuda().expand(rows, -1).contiguous()
    s = ActionSampler(1234, "cuda")
    counts = [torch.zeros(w, dtype=torch.int64, device="cuda") for w in VIMA_DIMS]
    for _ in range(n_draws):
        a = sample_heads(xd, VIMA_DIMS, sampler=s)[0]
        for h, w in enumerate(VIMA_DIMS):
            counts[h] += torch.bincount(a[:, h], minlength=w)
    N = rows * n_draws
    o = 0
    for h, w in enumerate(VIMA_DIMS):
        p = torch.softmax(x[0, o:o + w].double(), 0).numpy()
        o += w
        c = counts[h].cpu().numpy()
        assert c.sum() == N
        e = p * N
        big = e >= 5
        obs = np.append(c[big], c[~big].sum())
        exp = np.append(e[big], e[~big].sum())
        if exp[-1] < 5:  # too rare to stand alone: pooled into the last column that does
            obs, exp = np.append(obs[:-2], obs[-2:].sum()), np.append(exp[:-2], exp[-2:].sum())
        stat = ((obs - exp) ** 2 / exp).sum()
        pval = chi2.sf(stat, len(obs) - 1)
        assert pval > 1e-4, (h, stat, len(obs), pval)


@pytest.mark.parametrize("dims", [VIMA_DIMS, ODD_DIMS])
def test_log_prob_and_entropy_match_torch_fp64(dims):
    """log_prob of sampled, greedy and random given actions and the entropy equal torch.distributions.Categorical in fp64 on the same
    fp32 logits within 1e-6 absolute (plus the fp32 rounding of the value itself, which at |log p| ~ 1e4 is ~1e-3).  NaN for a head of
    all -inf logits and for a given action outside the head."""
    from vima_b200.nn.action import ActionSampler, MultiCategorical

    x = logit_rows(dims, 300, seed=5)
    mc = MultiCategorical(x.cuda(), dims)
    g = torch.Generator().manual_seed(2)
    given = torch.stack([torch.randint(0, w, (x.shape[0],), generator=g) for w in dims], 1)
    acts = {"sampled": mc.sample(ActionSampler(7, "cuda")).cpu(), "mode": mc.mode().cpu(), "given": given}
    ent = mc.entropy().cpu()
    o = 0
    for h, w in enumerate(dims):
        xs = x[:, o:o + w].double()
        o += w
        dead = torch.isinf(xs).all(dim=1) & (xs[:, 0] < 0)
        ref = torch.distributions.Categorical(logits=xs[~dead], validate_args=False)
        tol = lambda r: 1e-6 + 2.0 ** -23 * r.abs()  # noqa: E731
        re = ref.entropy()
        assert (ent[~dead, h].double() - re).abs().le(tol(re)).all(), h
        assert ent[dead, h].isnan().all()
        for name, a in acts.items():
            lp = mc.log_prob(a.cuda()).cpu()[:, h].double()
            rl = ref.log_prob(a[~dead, h])
            fin = torch.isfinite(rl)
            assert torch.equal(torch.isinf(lp[~dead]), ~fin), (name, h)  # a -inf column given: -inf, as torch
            assert (lp[~dead][fin] - rl[fin]).abs().le(tol(rl[fin])).all(), (name, h)
            assert lp[dead].isnan().all(), (name, h)
    bad = given.clone()
    bad[0, 0], bad[1, 1], bad[2, 2] = -1, dims[1], 10 ** 9
    lp = mc.log_prob(bad.cuda()).cpu()
    assert lp[0, 0].isnan() and lp[1, 1].isnan() and lp[2, 2].isnan()
    assert torch.isfinite(lp[0, 1:]).any()


def test_greedy_is_head_select_bit_for_bit(ctx):
    """The kernel's greedy mode and vima_head_select give the same modes and the same normalised logits, bit for bit; greedy and
    scoring launches leave the draw counter alone and every sampling launch advances it by exactly one."""
    from vima_b200.nn.action import ActionSampler

    for dims in (VIMA_DIMS, ODD_DIMS):
        x = logit_rows(dims, 333, seed=11).cuda()
        B, n = x.shape[0], len(dims)
        off = _off(dims)
        norm0 = torch.full_like(x, 7.0)
        modes0 = torch.full((B, n), -5, dtype=torch.int64, device="cuda")
        ctx.head_select(x, B, n, off, norm0, modes0)
        norm1 = torch.full_like(x, 9.0)
        modes1 = torch.full((B, n), -6, dtype=torch.int64, device="cuda")
        s = ActionSampler(1, "cuda")
        ctx.head_sample(x, B, n, off, greedy=True, seed=s.seed, counter=s.counter, actions_out=modes1, logits_norm=norm1)
        ctx.head_sample(x, B, n, off, actions_in=modes1, seed=s.seed, counter=s.counter,
                        log_prob=torch.empty((B, n), device="cuda"))
        assert s.draws == 0
        assert torch.equal(modes0, modes1)
        assert torch.equal(norm0.view(torch.int32), norm1.view(torch.int32))
        for k in range(3):
            ctx.head_sample(x, B, n, off, seed=s.seed, counter=s.counter, actions_out=modes1)
            assert s.draws == k + 1


def test_rounding_fallback_takes_the_last_positive_column():
    """When rounding leaves u * sum at or past every running sum, the draw is the head's last column with p > 0, also when an earlier
    1024-column round left a positive column in a higher lane.  The head: 1500 columns, p > 0 only at 1023 (weight 1, lane 31 of round
    0) and at 1024 and 1056 (weight ~0.9 * 2^-24 each, lanes 0 and 1 of round 1): the total rounds to 1 + 2^-23, every running sum
    to 1, and at u >= 1 - 2^-23 (the draws below, found with the restated Philox) u * total rounds to 1, which no running sum
    exceeds."""
    from vima_b200.nn.action import ActionSampler, sample_heads

    x = torch.full((1, 1500), -math.inf)
    x[0, 1023] = 0.0
    x[0, [1024, 1056]] = math.log(0.9 * 2.0 ** -24)
    seed = 2024
    for draw in (4684430, 5231646):
        assert head_uniforms(1, 1, seed, draw)[0, 0] >= 1 - 2.0 ** -23
        s = ActionSampler(seed, "cuda")
        s.counter.fill_(draw)
        assert sample_heads(x.cuda(), [1500], sampler=s)[0].item() == 1056, draw
    s.counter.fill_(0)  # an ordinary u lands on the column holding almost all the mass
    assert head_uniforms(1, 1, seed, 0)[0, 0] < 0.99
    assert sample_heads(x.cuda(), [1500], sampler=s)[0].item() == 1023


def test_sampling_no_rows_advances_the_counter():
    """A sampling call over an empty batch draws nothing and still counts: the counter advances by one; greedy and scoring calls over
    no rows leave it alone."""
    from vima_b200.nn.action import ActionSampler, sample_heads

    s = ActionSampler(3, "cuda")
    x = torch.empty(0, 4, sum(VIMA_DIMS), device="cuda")
    a = sample_heads(x, VIMA_DIMS, sampler=s, log_prob=True, entropy=True)
    assert [t.shape for t in a] == [(0, 4, len(VIMA_DIMS))] * 3
    assert s.draws == 1
    sample_heads(x, VIMA_DIMS, entropy=True)
    sample_heads(x, VIMA_DIMS, actions=torch.empty(0, 4, len(VIMA_DIMS), dtype=torch.int64, device="cuda"), log_prob=True)
    assert s.draws == 1


def test_counter_streams():
    """The same seed gives the same sequence; another seed or the next draw another; rows and heads of one launch draw from
    different streams (identical rows do not all draw alike)."""
    from vima_b200.nn.action import ActionSampler, sample_heads

    x = torch.zeros(2048, sum(VIMA_DIMS), device="cuda")  # uniform heads: the draw is floor(u * w) up to rounding
    a, b, c = ActionSampler(42, "cuda"), ActionSampler(42, "cuda"), ActionSampler(43, "cuda")
    seq = lambda s: torch.stack([sample_heads(x, VIMA_DIMS, sampler=s)[0] for _ in range(4)])  # noqa: E731
    sa, sb, sc = seq(a), seq(b), seq(c)
    assert torch.equal(sa, sb)
    assert not torch.equal(sa, sc)
    assert not torch.equal(sa[0], sa[1])
    assert len(torch.unique(sa[0][:, 1])) > 90  # rows of one launch: different streams
    assert not torch.equal(sa[0][:, 2], sa[0][:, 3])  # heads of one launch: different streams
    assert a.draws == b.draws == c.draws == 4


# ------------------------------------------------------------------------------------------------------------------------------
# policy level


def _pol(kind):
    import vima_b200
    from oracle import detgen, synth

    if kind == "vima":
        return build_policy("4M")
    cls = {"gato": vima_b200.VIMAGatoPolicy, "gpt": vima_b200.VIMAGPTPolicy, "flamingo": vima_b200.VIMAFlamingoPolicy}[kind]
    pol = cls(**(synth.FLAMINGO_CFGS["flamingo_tiny"] if kind == "flamingo" else synth.GATO_CFGS["gato_tiny"]))
    detgen.fill_module_(pol)
    return pol.cuda().eval()


class _Sim:
    """A staggered schedule for one policy kind: ragged prompts, admissions and releases mid-run, one admission over a live
    episode.  `inputs(t)` are the step inputs before the action token."""

    S, TICKS, LMAX = 4, 7, 64
    SCHEDULE = {0: [("admit", [0, 1], [6, 9])], 2: [("admit", [2], [4])], 3: [("release", [0], None)],
                4: [("admit", [0], [8]), ("admit", [1], [5])]}  # tick 4 re-admits slot 1 while its episode is live

    def __init__(self, kind, pol, seed):
        self.kind, self.pol = kind, pol
        E = pol.embed_dim
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.Q = 1 if kind == "gpt" else (5 if kind == "vima" else pol._obj_xf_num_queries)
        shape = (self.TICKS, self.S, E) if kind == "gpt" else (self.TICKS, self.S, self.Q, E)
        self.obs = torch.randn(*shape, device="cuda", generator=g)
        self.msk = torch.rand(self.TICKS, self.S, self.Q, device="cuda", generator=g) > 0.3
        self.msk[..., 0] = True
        self.prompts = {}
        for t, evs in self.SCHEDULE.items():
            for kind_, slots, lens in evs:
                if kind_ == "admit":
                    Lp = max(lens)
                    tok = torch.randn(Lp, len(slots), E, device="cuda", generator=g)
                    m = torch.arange(Lp, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None]
                    self.prompts[(t, tuple(slots))] = (tok, m)

    def open(self):
        if self.kind in ("vima", "flamingo"):
            return self.pol.open_slots(self.S, max_tokens=self.LMAX, max_prompt_tokens=12)
        return self.pol.open_slots(self.S, max_tokens=2 * self.LMAX)

    def events(self, t, cache):
        for kind_, slots, _ in self.SCHEDULE.get(t, []):
            if kind_ == "admit":
                self.pol.admit(cache, slots, *self.prompts[(t, tuple(slots))])
            else:
                self.pol.release(cache, slots)

    def inputs(self, t):
        return (self.obs[t:t + 1], self.msk[t:t + 1]) if self.kind == "vima" else (self.obs[t:t + 1],)


def _hand_step(pol, cache, inputs, token, sampler=None):
    """step_slots -> forward_action_decoder -> mode() (or one MultiCategorical over all sub-heads sampled) -> forward_action_token."""
    from vima_b200.nn.action import MultiCategorical

    S = cache.S
    x = pol.step_slots(cache, *inputs, token)
    dists = pol.forward_action_decoder(x)
    keys = list(dists.keys())
    if sampler is None:
        acts = {k: dists[k].mode() for k in keys}
        return acts, None, None, pol.forward_action_token(acts)
    dims = [n for k in keys for n in dists[k]._action_dims]
    mc = MultiCategorical(torch.cat([dists[k].raw_logits for k in keys], -1), dims)
    a = mc.sample(sampler)
    lp, ent = mc.log_prob(a), mc.entropy()
    out, o = [{}, {}, {}], 0
    for k in keys:
        n = len(dists[k]._action_dims)
        for d, t in zip(out, (a, lp, ent)):
            d[k] = t[..., o:o + n]
        o += n
    return out[0], out[1], out[2], pol.forward_action_token(out[0]).view(1, S, -1)


@pytest.mark.parametrize("kind", ["vima", "gato", "gpt", "flamingo"])
def test_greedy_act_slots_equal_hand_closed_loop(kind):
    """Greedy act_slots over the staggered schedule equals step_slots + heads + mode() + forward_action_token bit for bit, in the
    actions and in the fed-back tokens of every active slot."""
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _pol(kind)
    sim = _Sim(kind, pol, seed=21)
    with torch.no_grad():
        ca, cb = sim.open(), sim.open()
        assert torch.equal(ca.action_token, torch.zeros_like(ca.action_token))
        tok = torch.zeros(1, sim.S, pol.embed_dim, device="cuda")
        for t in range(sim.TICKS):
            sim.events(t, ca)
            sim.events(t, cb)
            active = [b for b in range(sim.S) if ca.active_host[b]]
            acts, lp, ent = pol.act_slots(ca, *sim.inputs(t))
            want, _, _, tok = _hand_step(pol, cb, sim.inputs(t), tok)
            assert set(acts) == set(want)
            for k in acts:
                assert acts[k].shape == lp[k].shape == ent[k].shape == (1, sim.S, want[k].shape[-1])
                assert torch.equal(acts[k][:, active], want[k][:, active]), (t, k)
                assert torch.isfinite(lp[k][:, active]).all() and (ent[k][:, active] >= 0).all()
            assert torch.equal(ca.action_token[active], tok[0, active]), t
        assert ca.len_host == cb.len_host and ca.len.tolist() == ca.len_host


@pytest.mark.parametrize("kind", ["vima", "gpt"])
def test_sampled_act_slots_equal_multicategorical(kind):
    """Sampled act_slots returns exactly what MultiCategorical.sample / log_prob / entropy give on that step's raw logits (all
    sub-heads of all keys as one MultiCategorical) at the same counter, and feeds back the embedding of that action."""
    import vima_b200

    vima_b200.set_precision("f16f8")
    try:
        pol = _pol(kind)
        sim = _Sim(kind, pol, seed=22)
        sa, sb = vima_b200.ActionSampler(77, "cuda"), vima_b200.ActionSampler(77, "cuda")
        with torch.no_grad():
            ca, cb = sim.open(), sim.open()
            tok = torch.zeros(1, sim.S, pol.embed_dim, device="cuda")
            for t in range(sim.TICKS):
                sim.events(t, ca)
                sim.events(t, cb)
                active = [b for b in range(sim.S) if ca.active_host[b]]
                got = pol.act_slots(ca, *sim.inputs(t), sampler=sa)
                *want, tok = _hand_step(pol, cb, sim.inputs(t), tok, sampler=sb)
                for g, w in zip(got, want):
                    for k in g:
                        assert torch.equal(g[k][:, active], w[k][:, active]), (t, k)
                assert torch.equal(ca.action_token[active], tok[0, active]), t
            assert sa.draws == sb.draws == sim.TICKS
    finally:
        vima_b200.set_precision("f16x3")


def test_capture_act_slots_replays_equal_eager():
    """capture_act_slots leaves the slot state, the fed-back tokens and the sampler as they were; its replays equal eager act_slots
    from the same seed bit for bit over the schedule, with an eager forward_action_decoder at another batch size between replays
    (the graph's heads run on buffers of its own).  Replays refuse after a weight update of the action heads or embedding."""
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _pol("vima")
    sim = _Sim("vima", pol, seed=23)
    sim.TICKS, sim.LMAX = 12, 128
    g = torch.Generator(device="cuda").manual_seed(3)
    sim.obs = torch.randn(sim.TICKS, sim.S, sim.Q, pol.embed_dim, device="cuda", generator=g)
    sim.msk = torch.ones(sim.TICKS, sim.S, sim.Q, dtype=torch.bool, device="cuda")
    with torch.no_grad():
        se, sg = vima_b200.ActionSampler(5, "cuda"), vima_b200.ActionSampler(5, "cuda")
        ce, cg = sim.open(), sim.open()
        p_tok, p_msk = sim.prompts[(0, (0, 1))]
        pol.admit(cg, [3], p_tok[:, :1], p_msk[:1])  # capture with one slot already holding an episode
        cg.action_token.normal_()
        before, tok0 = cg.state(), cg.action_token.clone()
        gs = pol.capture_act_slots(cg, *sim.inputs(0), sampler=sg)
        torch.cuda.synchronize()
        after = cg.state()
        assert all(torch.equal(x, y) for x, y in zip(before[0], after[0])) and before[1] == after[1]
        assert torch.equal(cg.action_token, tok0) and sg.draws == 0
        pol.release(cg, [3])
        cg.action_token.zero_()
        for t in range(sim.TICKS):
            sim.events(t, ce)
            sim.events(t, cg)
            active = [b for b in range(sim.S) if ce.active_host[b]]
            want = pol.act_slots(ce, *sim.inputs(t), sampler=se)
            pol.forward_action_decoder(torch.randn(3, 5, pol.embed_dim, device="cuda"))
            got = gs(*sim.inputs(t))
            for w_, g_ in zip(want, got):
                for k in w_:
                    assert torch.equal(w_[k][:, active], g_[k][:, active]), (t, k)
            assert torch.equal(ce.action_token[active], cg.action_token[active]), t
        assert gs.replays == sim.TICKS and sg.draws == se.draws == sim.TICKS
        for p in (next(iter(pol.action_decoder.parameters())), next(iter(pol.action_encoder.parameters()))):
            p.mul_(1.0)  # an in-place write: the graph's recorded version no longer matches
            with pytest.raises(RuntimeError, match="weights changed"):
                gs(*sim.inputs(0))
            gs = pol.capture_act_slots(cg, *sim.inputs(0), sampler=sg)


def test_captured_closed_loop_owns_its_head_buffers():
    """The graph of capture_act_slots keeps the head buffers its warm-up allocated and its kernels address: after every other
    reference is gone and the allocator has released its cache, fresh tensors never land on them, and a replay leaves those tensors
    alone."""
    import gc

    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _pol("vima")
    sim = _Sim("vima", pol, seed=24)
    with torch.no_grad():
        cache = sim.open()
        sim.events(0, cache)
        gs = pol.capture_act_slots(cache, *sim.inputs(0), sampler=vima_b200.ActionSampler(9, "cuda"))
        bufs = [t for st in gs.grouped._bufs.values() for t in [st["x"]] + [h for h, _ in st["h"]]]
        assert bufs
        spans = [(t.data_ptr(), t.data_ptr() + t.numel() * t.element_size()) for t in bufs]
        del bufs
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        junk = []
        for stream in (torch.cuda.current_stream(), side):
            with torch.cuda.stream(stream):
                junk += [torch.full(((hi - lo) // 4,), 7.0, device="cuda") for lo, hi in spans]
        torch.cuda.current_stream().wait_stream(side)
        for j in junk:
            a, b = j.data_ptr(), j.data_ptr() + j.numel() * 4
            assert all(b <= lo or a >= hi for lo, hi in spans)
        gs(*sim.inputs(0))
        torch.cuda.synchronize()
        assert all(bool((j == 7.0).all()) for j in junk)


def test_teacher_forcing_log_prob():
    """forward over all T steps -> forward_action_decoder -> log_prob(expert indices) equals torch's fp64 log_softmax of the same raw
    logits within 1e-6."""
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = build_policy("4M")
    E, B, Lp, Q, T = pol.embed_dim, 3, 10, 4, 5
    g = torch.Generator(device="cuda").manual_seed(4)
    p_tok = torch.randn(Lp, B, E, device="cuda", generator=g)
    p_msk = torch.ones(B, Lp, dtype=torch.bool, device="cuda")
    obs = torch.randn(T, B, Q, E, device="cuda", generator=g)
    msk = torch.ones(T, B, Q, dtype=torch.bool, device="cuda")
    act = torch.randn(T - 1, B, E, device="cuda", generator=g)
    with torch.no_grad():
        x = pol.forward(obs_token=obs, obs_mask=msk, action_token=act, prompt_token=p_tok, prompt_token_mask=p_msk)
        dists = pol.forward_action_decoder(x)
    assert x.shape[:2] == (T, B)
    for k, d in dists.items():
        dims = list(d._action_dims)
        expert = torch.stack([torch.randint(0, w, (T, B), device="cuda", generator=g) for w in dims], -1)
        lp = d.log_prob(expert).double()
        raw = d.raw_logits.double()
        o = 0
        for h, w in enumerate(dims):
            ref = torch.log_softmax(raw[..., o:o + w], -1).gather(-1, expert[..., h:h + 1])[..., 0]
            o += w
            assert (lp[..., h] - ref).abs().max().item() < 1e-6, (k, h)
