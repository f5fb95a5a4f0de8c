"""GPU: the paged prompt K/V of the slot cache's cross-attention.  Paged non-causal attention with a per-batch key count (kv_len)
equals the contiguous call at Lk = kv_len[b] bit for bit (wgmma, mma.sync and SIMT tail kernels; NaN in every pool row the call must
not read, including the pages its table lists past the key count); the cross-attention policies' staggered schedules on the default
prompt pool, on the smallest pool with a shuffled free list, and per prompt length on a cache whose max_prompt_tokens is that length,
bit for bit, and against forward(...)[-1:] at B=1; forks share prompt pages; graph replays across admissions and forks; no host
synchronisation in the page side of admission, release and fork; refusals."""
import random

import pytest
import torch

from tests.test_kv_pages_gpu import NAN_BITS, _policy, _split
from tests.util import rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    c = _C.Context.get(torch.device("cuda", 0))
    yield c
    c.set_option("attn", "tc")


# ------------------------------------------------------------------------------------------------- kernels
# (kernel option, operand format, split, Lq): the wgmma kernel, the mma.sync kernel (f16 / bf16, split and single-pass), and the
# wgmma body + SIMT tail split (133 = 128 + 5 rows)
KCASES = [("tc", "f16", True, 33), ("tc", "bf16", True, 33), ("mma", "f16", True, 33), ("mma", "bf16", True, 33), ("mma", "f16", False, 33),
          ("mma", "bf16", False, 33), ("tc", "f16", True, 133)]


@pytest.mark.parametrize("impl,fmt,split,Lq", KCASES)
def test_kv_len_paged_equals_contiguous_per_element(ctx, impl, fmt, split, Lq):
    dt = {"f16": 0, "bf16": 1}[fmt]
    cap, H, D = 256, 4, 32
    E = H * D
    kv_len = [1, 63, 64, 65, cap, 150]
    B = len(kv_len)
    seed = KCASES.index((impl, fmt, split, Lq))
    g = torch.Generator(device="cuda").manual_seed(seed)
    rng = random.Random(seed)
    page_ld = cap // 64
    owned = [-(-n // 64) for n in kv_len]
    n_pages = 1 + sum(owned) + 2  # the zero page, every element's pages, two NaN pages
    perm = list(range(1, n_pages))
    rng.shuffle(perm)
    nan_pages = perm[-2:]
    table = torch.zeros(B, page_ld, dtype=torch.int32)
    it = iter(perm)
    for b in range(B):
        for k in range(page_ld):  # entries past the element's key count name a NaN page: such chunks must never be read
            table[b, k] = next(it) if k < owned[b] else nan_pages[k % 2]
    table = table.cuda()
    nan = NAN_BITS[dt]
    pool_hi = torch.full((n_pages * 64, 2 * E), nan, dtype=torch.int16, device="cuda")
    pool_lo = torch.full_like(pool_hi, nan) if split else None
    pools = [t for t in (pool_hi, pool_lo) if t is not None]
    for b in range(B):  # the element's pages: its keys, then zeros to the end of the last page (as the slot cache keeps them)
        j = torch.arange(owned[b] * 64, device="cuda")
        rows = table[b, j // 64].long() * 64 + j % 64
        kh, kl = _split(ctx, torch.randn(rows.numel(), 2 * E, device="cuda", generator=g), dt, split)
        for t, v in zip(pools, (kh, kl)):
            v[kv_len[b]:] = 0
            t[rows] = v
    for t in pools:
        t[:64] = 0
    qh, ql = _split(ctx, torch.randn(B * Lq, E, device="cuda", generator=g), dt, split)
    mask = (torch.rand(B, cap, device="cuda", generator=g) > 0.3).to(torch.uint8)  # holes
    mask[:, 0] = 1
    mask[3, 10:60] = 0
    kl_dev = torch.tensor(kv_len, dtype=torch.int32, device="cuda")

    def out(n):
        o_hi = torch.full((n * Lq, E), 0x1234, dtype=torch.int16, device="cuda")
        return o_hi, (torch.full_like(o_hi, 0x1234) if split else None)

    ctx.set_option("attn", impl)
    try:
        ph, pl = out(B)
        ctx.attention(q=(qh, ql, E, 0), k=(pool_hi, pool_lo, 2 * E, 0), v=(pool_hi, pool_lo, 2 * E, E), o=(ph, pl, E, 0), B=B, H=H, Lq=Lq,
                      Lk=cap, D=D, scale=D ** -0.5, causal=False, key_mask=mask, dtype=dt, kv_pages=table, kv_pool_pages=n_pages,
                      kv_len=kl_dev)
        for b in range(B):
            n = kv_len[b]
            j = torch.arange(n, device="cuda")
            crow = table[b, j // 64].long() * 64 + j % 64
            ch, cl = out(1)
            kh = pool_hi[crow].contiguous()
            kl = pool_lo[crow].contiguous() if split else None
            qs = slice(b * Lq, (b + 1) * Lq)
            ctx.attention(q=(qh[qs], None if ql is None else ql[qs], E, 0), k=(kh, kl, 2 * E, 0), v=(kh, kl, 2 * E, E), o=(ch, cl, E, 0), B=1,
                          H=H, Lq=Lq, Lk=n, D=D, scale=D ** -0.5, causal=False, key_mask=mask[b:b + 1, :n].contiguous(), dtype=dt)
            assert torch.equal(ph[qs], ch), (b, n)
            if split:
                assert torch.equal(pl[qs], cl), (b, n)
    finally:
        ctx.set_option("attn", "tc")
    tdt = torch.float16 if dt == 0 else torch.bfloat16
    assert torch.isfinite(ph.view(tdt)).all()


def test_kv_len_refusals(ctx):
    B, H, D, E, Lq = 2, 4, 32, 128, 9
    z = torch.zeros(B * 128, 3 * E, dtype=torch.int16, device="cuda")
    o = torch.zeros(B * Lq, E, dtype=torch.int16, device="cuda")
    qp = torch.zeros(B, dtype=torch.int32, device="cuda")
    kl = torch.full((B,), 5, dtype=torch.int32, device="cuda")
    table = torch.ones(B, 2, dtype=torch.int32, device="cuda")
    bias = torch.zeros(H, 2 * 128 - 1, device="cuda")
    kw = dict(q=(z, z, 3 * E, 0), k=(z, z, 3 * E, E), v=(z, z, 3 * E, 2 * E), o=(o, o, E, 0), B=B, H=H, Lq=Lq, D=D, scale=0.1)
    with pytest.raises(RuntimeError, match="kv_len"):
        ctx.attention(Lk=128, causal=True, kv_len=kl, **kw)
    with pytest.raises(RuntimeError, match="kv_len|q_pos"):
        ctx.attention(Lk=128, causal=True, q_pos=qp, kv_len=kl, **kw)
    with pytest.raises(RuntimeError, match="kv_len|bias"):
        ctx.attention(Lk=128, causal=False, rel_bias=bias, kv_len=kl, **kw)
    with pytest.raises(RuntimeError, match="paged"):
        ctx.attention(Lk=129, causal=False, kv_pages=table, kv_pool_pages=2, kv_len=kl, **kw)  # Lk past kv_page_ld*64
    with pytest.raises(RuntimeError, match="paged"):
        ctx.attention(Lk=128, causal=True, kv_pages=table, kv_pool_pages=2, **kw)  # causal paged still needs q_pos


# ------------------------------------------------------------------------------------------------- policies
def _prompt(g, n, E):
    m = torch.rand(1, n, device="cuda", generator=g) > 0.25
    m[:, 0] = True
    return torch.randn(n, 1, E, device="cuda", generator=g), m


def _nan_pools(c, dt):
    """Every pool row outside the zero page starts as NaN: a page read without being written, or a prompt page's tail left
    unzeroed, shows in the outputs."""
    for t in c.kv_hi + c.kv_lo + c.prompt_kv_hi + c.prompt_kv_lo:
        if t is not None:
            t[64:] = NAN_BITS[dt]


class _Stagger:
    """Five slots over eight ticks, one prompt length per admission call: prompts of 40, 150, 65 and 64 tokens, a release, a
    re-admission over a live slot (tick 4) and one into a released slot (tick 6)."""

    S, T = 5, 8
    ADMITS = {0: ([0, 1], 40), 1: ([2], 150), 2: ([3], 65), 4: ([1], 64), 5: ([4], 150), 6: ([0], 65)}
    RELEASES = {3: [2], 5: [0]}

    def __init__(self, kind, pol):
        self.kind, self.pol = kind, pol
        E = pol.embed_dim
        self.Q = 4 if kind == "vima" else pol._obj_xf_num_queries
        g = torch.Generator(device="cuda").manual_seed(5)
        self.prompts = {t: _prompt(g, n, E) for t, (_, n) in self.ADMITS.items()}
        self.obs = torch.randn(self.T, self.S, self.Q, E, device="cuda", generator=g)
        self.msk = torch.rand(self.T, self.S, self.Q, device="cuda", generator=g) > 0.2
        self.msk[..., 0] = True
        self.act = torch.randn(self.T, self.S, E, device="cuda", generator=g)
        self.Lmax = self.T * (self.Q + 1)

    def open(self, Lp_cap=150, prompt_pool_tokens=None):
        from vima_b200 import engine as eng

        c = self.pol.open_slots(self.S, max_tokens=self.Lmax, max_prompt_tokens=Lp_cap, prompt_pool_tokens=prompt_pool_tokens)
        _nan_pools(c, eng.prec().dtype)
        return c

    def step(self, cache, t):
        o, a = self.obs[t:t + 1], self.act[t:t + 1]
        return self.pol.step_slots(cache, o, self.msk[t:t + 1], a) if self.kind == "vima" else self.pol.step_slots(cache, o, a)

    def forward(self, po, pm, pa, ptok, pmsk):
        if self.kind == "vima":
            return self.pol.forward(obs_token=po, obs_mask=pm, action_token=pa, prompt_token=ptok, prompt_token_mask=pmsk)[-1:]
        return self.pol.forward(po, pa, ptok, pmsk)[-1:]

    def run(self, cache, only_len=None, peak=None, own_history=False, bar=None):
        """-> per tick {slot: (prompt length, output row)} of the active slots.  only_len: admit only the calls of that prompt length
        (the other slots stay idle)."""
        outs, eps = [], {}
        for t in range(self.T):
            for b in self.RELEASES.get(t, []):
                if b in eps:
                    self.pol.release(cache, [b])
                    del eps[b]
            if t in self.ADMITS and (only_len is None or self.ADMITS[t][1] == only_len):
                slots, n = self.ADMITS[t]
                tok, m = self.prompts[t]
                self.pol.admit(cache, slots, tok.expand(-1, len(slots), -1).contiguous(), m.expand(len(slots), -1).contiguous())
                for b in slots:
                    eps[b] = dict(n=n, prompt=(tok, m), t0=t)
            out = self.step(cache, t)
            if peak is not None:
                peak.append(cache.prompt_pages_total - cache.prompt_pages_free)
            outs.append({b: (ep["n"], out[:, b:b + 1].clone()) for b, ep in eps.items()})
            if own_history:
                for b, ep in eps.items():
                    t0 = ep["t0"]
                    po, pm = self.obs[t0:t + 1, b:b + 1], self.msk[t0:t + 1, b:b + 1]
                    pa = self.act[t0 + 1:t + 1, b:b + 1] if t > t0 else None
                    full = self.forward(po, pm, pa, *ep["prompt"])
                    d = rel_l2(full.cpu(), out[:, b:b + 1].cpu())
                    assert d < bar, (self.kind, t, b, d)
        torch.cuda.synchronize()
        return outs


@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
@pytest.mark.parametrize("kind", ["vima", "flamingo"])
def test_prompt_pages_exact_across_caps(kind, mode):
    import vima_b200

    vima_b200.set_precision(mode)
    try:
        pol = _policy(kind)
        sched = _Stagger(kind, pol)
        with torch.no_grad():
            peak = []
            ref = sched.run(sched.open(), peak=peak, own_history=True, bar=2e-6 if mode == "f16x3" else 5e-5)
            # (b) the smallest prompt pool the schedule fits, pages recycled in scrambled order
            small = sched.open(prompt_pool_tokens=max(peak) * 64)
            assert small.prompt_pages_total == max(peak) < 5 * 3
            random.Random(1).shuffle(small.prompt_pages.free)
            got = sched.run(small)
            assert len(got) == len(ref)
            for a, b in zip(ref, got):
                assert a.keys() == b.keys() and all(torch.equal(a[s][1], b[s][1]) for s in a)
            # (c) per prompt length n: the slots holding an n-token prompt equal a cache whose max_prompt_tokens is n
            for n in sorted({n for _, n in sched.ADMITS.values()}):
                own = sched.run(sched.open(Lp_cap=n), only_len=n)
                hits = 0
                for a, b in zip(ref, own):
                    for s, (ln, row) in a.items():
                        if ln == n and s in b:
                            assert torch.equal(row, b[s][1]), (n, s)
                            hits += 1
                assert hits > 0
    finally:
        vima_b200.set_precision("f16x3")


class _Group:
    """Group sampling: one episode (a 150-token prompt) in slot 0 runs two ticks, then forks into slots 1..3; every slot then gets
    inputs of its own.  The replay admits all four slots at tick 0 with the same prompt and feeds them slot 0's inputs until the
    fork."""

    S, T, FORK = 4, 6, 2

    def __init__(self, pol):
        self.pol = pol
        E = pol.embed_dim
        g = torch.Generator(device="cuda").manual_seed(8)
        self.tok, self.m = _prompt(g, 150, E)
        self.obs = torch.randn(self.T, self.S, 4, E, device="cuda", generator=g)
        self.msk = torch.rand(self.T, self.S, 4, device="cuda", generator=g) > 0.2
        self.msk[..., 0] = True
        self.act = torch.randn(self.T, self.S, E, device="cuda", generator=g)

    def open(self, prompt_pool_tokens=None):
        from vima_b200 import engine as eng

        c = self.pol.open_slots(self.S, max_tokens=self.T * 5, max_prompt_tokens=150, prompt_pool_tokens=prompt_pool_tokens)
        _nan_pools(c, eng.prec().dtype)
        return c

    def admit(self, c, slots):
        self.pol.admit(c, slots, self.tok.expand(-1, len(slots), -1).contiguous(), self.m.expand(len(slots), -1).contiguous())

    def step(self, c, t, rows):
        return self.pol.step_slots(c, self.obs[t:t + 1, rows], self.msk[t:t + 1, rows], self.act[t:t + 1, rows])

    def run_fork(self, c, used=None):
        outs = []
        self.admit(c, [0])
        for t in range(self.T):
            if t == self.FORK:
                self.pol.fork_slots(c, [0] * (self.S - 1), list(range(1, self.S)))
                if used is not None:
                    used.append(c.prompt_pages_total - c.prompt_pages_free)
            outs.append(self.step(c, t, list(range(self.S))).clone())
        torch.cuda.synchronize()
        return outs

    def run_replay(self, c):
        self.admit(c, list(range(self.S)))
        outs = [self.step(c, t, [0] * self.S if t < self.FORK else list(range(self.S))).clone() for t in range(self.T)]
        torch.cuda.synchronize()
        return outs


def test_fork_shares_prompt_pages():
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy("vima")
    grp = _Group(pol)
    with torch.no_grad():
        used = []
        x = grp.run_fork(grp.open(), used)
        assert used == [3]  # one prompt's pages for all four slots
        y = grp.run_replay(grp.open())
        for t, (a, b) in enumerate(zip(x, y)):
            rows = [0] if t < grp.FORK else list(range(grp.S))
            assert torch.equal(a[:, rows], b[:, rows]), t
        x1 = grp.run_fork(grp.open(prompt_pool_tokens=3 * 64))  # fits the fork, not the replay
        for t, (a, b) in enumerate(zip(x, x1)):
            rows = [0] if t < grp.FORK else list(range(grp.S))
            assert torch.equal(a[:, rows], b[:, rows]), t
        with pytest.raises(ValueError, match="prompt pages"):
            grp.run_replay(grp.open(prompt_pool_tokens=3 * 64))


def test_graph_replays_across_admissions_and_forks_equal_eager():
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy("vima")
    sched = _Stagger("vima", pol)
    events = {1: ("admit", [1], 150), 2: ("fork", [1], [2]), 3: ("admit", [0], 65), 4: ("fork", [0], [1]), 5: ("admit", [3, 4], 64),
              6: ("release", [2])}
    g = torch.Generator(device="cuda").manual_seed(12)
    prompts = {t: _prompt(g, e[2], pol.embed_dim) for t, e in events.items() if e[0] == "admit"}

    def apply(c, t):
        if t == 0:
            tok, m = _prompt(torch.Generator(device="cuda").manual_seed(13), 40, pol.embed_dim)
            pol.admit(c, [0], tok, m)
        e = events.get(t)
        if e is None:
            return
        if e[0] == "admit":
            tok, m = prompts[t]
            pol.admit(c, e[1], tok.expand(-1, len(e[1]), -1).contiguous(), m.expand(len(e[1]), -1).contiguous())
        elif e[0] == "fork":
            pol.fork_slots(c, e[1], e[2])
        else:
            pol.release(c, e[1])

    def inputs(t):
        return sched.obs[t:t + 1], sched.msk[t:t + 1], sched.act[t:t + 1]

    with torch.no_grad():
        c = sched.open()
        ref = []
        for t in range(sched.T):
            apply(c, t)
            ref.append(([b for b in range(sched.S) if c.active_host[b]], pol.step_slots(c, *inputs(t)).clone()))
        c = sched.open()
        apply(c, 0)
        first = pol.step_slots(c, *inputs(0)).clone()
        table, plen = c.prompt_page_table.clone(), c.prompt_len.clone()
        gr = pol.capture_step_slots(c, *inputs(1))
        torch.cuda.synchronize()
        assert torch.equal(table, c.prompt_page_table) and torch.equal(plen, c.prompt_len)
        got = [([0], first)]
        for t in range(1, sched.T):
            apply(c, t)
            got.append(([b for b in range(sched.S) if c.active_host[b]], gr(*inputs(t)).clone()))
        torch.cuda.synchronize()
    for (a0, o0), (a1, o1) in zip(ref, got):
        assert a0 == a1 and torch.equal(o0[:, a0], o1[:, a1])


def test_prompt_page_side_does_not_synchronise():
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy("vima")
    grp = _Group(pol)
    with torch.no_grad():
        c = grp.open()
        grp.admit(c, [0])
        grp.step(c, 0, [0, 1, 2, 3])  # first-call host checks
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            c.check_prefix([1, 2], 0, 65)
            c.free_slots([1, 2], prompt_cols=65)  # admission's page side, a partial last page zeroed
            pol.fork_slots(c, [0], [3])
            pol.release(c, [1])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        want = torch.zeros_like(c.prompt_page_table)
        for b, own in enumerate(c.prompt_pages.owned):
            want[b, :len(own)] = torch.tensor(own, dtype=torch.int32)
        assert torch.equal(want, c.prompt_page_table)
        assert (c.prompt_kv_hi[0][c.prompt_pages.owned[2][1] * 64:][:64] == 0).all()  # the zeroed tail page
        assert c.prompt_len[3].item() == 150 and c.prompt_pages.owned[3] == c.prompt_pages.owned[0]


@pytest.mark.parametrize("kind", ["vima", "flamingo"])
def test_prompt_pool_refusals(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    E = pol.embed_dim
    g = torch.Generator(device="cuda").manual_seed(3)
    with pytest.raises(ValueError, match="prompt_pool_tokens"):
        pol.open_slots(3, max_tokens=64, max_prompt_tokens=150, prompt_pool_tokens=3 * 3 * 64 + 1)
    with pytest.raises(ValueError, match="prompt_pool_tokens"):
        pol.open_slots(3, max_tokens=64, max_prompt_tokens=150, prompt_pool_tokens=0)
    with torch.no_grad():
        c = pol.open_slots(3, max_tokens=64, max_prompt_tokens=150, prompt_pool_tokens=3 * 64)
        tok, m = _prompt(g, 65, E)
        pol.admit(c, [0], tok, m)  # two of three pages
        torch.cuda.synchronize()
        snap = lambda: (c.state(), c.prompt_pages.state(), c.prompt_page_table.clone(), c.prompt_len.clone(), c.prompt_mask.clone(),  # noqa: E731
                        c.pages.state(), c.page_table.clone())
        before = snap()
        tok2, m2 = _prompt(g, 100, E)
        with pytest.raises(ValueError, match="prompt pages"):
            pol.admit(c, [1], tok2, m2)
        torch.cuda.synchronize()
        after = snap()
        assert all(torch.equal(a, b) for a, b in zip(before[0][0], after[0][0])) and before[0][1] == after[0][1]
        assert before[1] == after[1] and before[5] == after[5]
        assert all(torch.equal(before[i], after[i]) for i in (2, 3, 4, 6))
        pol.admit(c, [0], tok2, m2)  # over the live slot: its two pages come back first
        assert c.prompt_pages_free == 1
