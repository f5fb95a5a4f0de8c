"""GPU: the paged slot K/V cache.  Paged attention equals the same call on a contiguous copy of the K/V bit for bit (wgmma,
mma.sync and SIMT tail kernels; NaN in every row the call must not read); the paged append / scatter kernels against a torch
statement of the row mapping; every policy's staggered slot schedule on a pool just big enough for it (free list shuffled, so
pages recycle in scrambled order) against the default pool, bit for bit, eager, sampled and graphed; refusals; and no host
synchronisation in page reservation, release and re-admission."""
import random

import pytest
import torch

from tests.policy_runner import build_policy

pytestmark = pytest.mark.gpu

NAN_BITS = {0: 0x7E00, 1: 0x7FC0}  # a quiet NaN in fp16 / bf16


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    c = _C.Context.get(torch.device("cuda", 0))
    yield c
    c.set_option("attn", "tc")


def _split(ctx, x, dt, split):
    rows, cols = x.shape
    hi = torch.empty(rows, cols, dtype=torch.int16, device="cuda")
    lo = torch.empty_like(hi) if split else None
    ctx.split(x.contiguous(), hi, lo, cols=cols, pad_cols=cols, dtype=dt)
    return hi, lo


CASES = [(impl, fmt, split) for impl, fmt, split in [("tc", "f16", True), ("tc", "bf16", True), ("tc", "f16", False), ("mma", "f16", True),
                                                      ("mma", "bf16", True), ("mma", "bf16", False)]]


@pytest.mark.parametrize("cap", [63, 65, 127, 129, 511, 513, 1023, 1024])
@pytest.mark.parametrize("Lq", [17, 33, 133])
@pytest.mark.parametrize("impl,fmt,split", CASES)
def test_paged_attention_equals_contiguous_copy(ctx, impl, fmt, split, Lq, cap):
    if Lq > cap or (impl == "mma" and split and cap > 513):  # the resident-K/V kernel's shared memory (split operands)
        pytest.skip("shape outside the kernel's range")
    dt = {"f16": 0, "bf16": 1}[fmt]
    B, H, D = 4, 4, 32
    E = H * D
    seed = cap * 1000 + Lq * 10 + CASES.index((impl, fmt, split))
    g = torch.Generator(device="cuda").manual_seed(seed)
    rng = random.Random(seed)
    page_ld = -(-cap // 64)
    q_pos = [0, cap - Lq, rng.randint(0, cap - Lq), rng.randint(0, cap - Lq)]
    keys = [p + Lq for p in q_pos]
    owned = [-(-k // 64) for k in keys]
    n_pages = 1 + sum(owned) + 3  # the zero page, every element's pages and three pages nobody owns
    perm = list(range(1, n_pages))
    rng.shuffle(perm)
    table = torch.zeros(B, page_ld, dtype=torch.int32)
    it = iter(perm)
    for b in range(B):
        for k in range(owned[b]):
            table[b, k] = next(it)
    table = table.cuda()
    nan = NAN_BITS[dt]
    pool_hi = torch.full((n_pages * 64, 2 * E), nan, dtype=torch.int16, device="cuda")
    pool_lo = torch.full_like(pool_hi, nan) if split else None
    pool_hi[:64] = 0
    if split:
        pool_lo[:64] = 0
    rows = torch.cat([table[b, torch.arange(keys[b], device="cuda") // 64].long() * 64 + torch.arange(keys[b], device="cuda") % 64
                      for b in range(B)])
    kh, kl = _split(ctx, torch.randn(rows.numel(), 2 * E, device="cuda", generator=g), dt, split)
    pool_hi[rows] = kh
    if split:
        pool_lo[rows] = kl
    # the contiguous copy [B*cap, 2E]: each element's columns gathered through its table (zero page past its pages, NaN past its
    # keys inside its last page)
    j = torch.arange(cap, device="cuda")
    crow = torch.cat([table[b, j // 64].long() * 64 + j % 64 for b in range(B)])
    cont_hi = pool_hi[crow].contiguous()
    cont_lo = pool_lo[crow].contiguous() if split else None
    qh, ql = _split(ctx, torch.randn(B * Lq, E, device="cuda", generator=g), dt, split)
    mask = (torch.rand(B, cap, device="cuda", generator=g) > 0.2).to(torch.uint8)
    mask[:, 0] = 1
    qp = torch.tensor(q_pos, dtype=torch.int32, device="cuda")

    def run(k_hi, k_lo, **kw):
        o_hi = torch.full((B * Lq, E), 0x1234, dtype=torch.int16, device="cuda")
        o_lo = torch.full_like(o_hi, 0x1234) if split else None
        ctx.attention(q=(qh, ql, E, 0), k=(k_hi, k_lo, 2 * E, 0), v=(k_hi, k_lo, 2 * E, E), o=(o_hi, o_lo, E, 0), B=B, H=H, Lq=Lq, Lk=cap,
                      D=D, scale=D ** -0.5, causal=True, key_mask=mask, dtype=dt, mask_ld=cap, q_pos=qp, **kw)
        return o_hi, o_lo

    ctx.set_option("attn", impl)
    try:
        ph, pl = run(pool_hi, pool_lo, kv_pages=table, kv_pool_pages=n_pages)
        ch, cl = run(cont_hi, cont_lo, kv_batch_rows=cap)
    finally:
        ctx.set_option("attn", "tc")
    tdt = torch.float16 if dt == 0 else torch.bfloat16
    assert torch.isfinite(ph.view(tdt)).all()
    assert torch.equal(ph, ch)
    if split:
        assert torch.equal(pl, cl)


def test_paged_attention_refusals(ctx):
    B, H, D, E, Lq = 2, 4, 32, 128, 9
    z = torch.zeros(B * 128, 3 * E, dtype=torch.int16, device="cuda")
    o = torch.zeros(B * Lq, E, dtype=torch.int16, device="cuda")
    qp = torch.zeros(B, dtype=torch.int32, device="cuda")
    table = torch.ones(B, 2, dtype=torch.int32, device="cuda")
    kw = dict(q=(z, z, 3 * E, 0), k=(z, z, 3 * E, E), v=(z, z, 3 * E, 2 * E), o=(o, o, E, 0), B=B, H=H, Lq=Lq, D=D, scale=0.1, causal=True)
    with pytest.raises(RuntimeError, match="paged"):
        ctx.attention(Lk=128, kv_pages=table, kv_pool_pages=2, **kw)  # no q_pos
    with pytest.raises(RuntimeError, match="paged"):
        ctx.attention(Lk=129, q_pos=qp, kv_pages=table, kv_pool_pages=2, **kw)  # Lk past kv_page_ld*64
    with pytest.raises(RuntimeError, match="paged"):
        ctx.attention(Lk=128, q_pos=qp, kv_pages=table, kv_pool_pages=1 << 25, **kw)  # pool rows past 2^31


@pytest.mark.parametrize("split", [True, False])
def test_paged_append_and_scatter_kernels(ctx, split):
    S, L, E, page_ld, n_pages = 5, 9, 64, 4, 11
    g = torch.Generator(device="cuda").manual_seed(7)
    ri = lambda *s: torch.randint(-30000, 30000, s, dtype=torch.int16, device="cuda", generator=g)  # noqa: E731
    table = torch.tensor([[3, 7, 0, 0], [5, 1, 9, 0], [0, 0, 0, 0], [2, -1, 10, 4], [8, 6, n_pages + 4, 0]], dtype=torch.int32)
    q_pos = [0, 60, 5, 120, 90]
    qkv_hi, qkv_lo = ri(S * L, 3 * E), (ri(S * L, 3 * E) if split else None)
    kv_hi, kv_lo = ri(n_pages * 64, 2 * E), (ri(n_pages * 64, 2 * E) if split else None)
    want_hi, want_lo = kv_hi.clone(), (kv_lo.clone() if split else None)
    for b in range(S):
        for r in range(L):
            col = q_pos[b] + r
            pg = int(table[b, col // 64])
            if 0 < pg < n_pages:  # page 0 and entries outside the pool are skipped
                want_hi[pg * 64 + col % 64] = qkv_hi[b * L + r, E:]
                if split:
                    want_lo[pg * 64 + col % 64] = qkv_lo[b * L + r, E:]
    ctx.slot_kv_append_paged(qkv_hi, qkv_lo, 3 * E, E, 2 * E, S, L, torch.tensor(q_pos, dtype=torch.int32, device="cuda"), kv_hi, kv_lo,
                             2 * E, table.cuda(), n_pages)
    assert torch.equal(kv_hi, want_hi) and (not split or torch.equal(kv_lo, want_lo))
    # prefill scatter: rows (j, r) -> column r of slot slots[j]
    slots, Lq = [4, 1, 3], 130
    qkv_hi, qkv_lo = ri(len(slots) * Lq, 3 * E), (ri(len(slots) * Lq, 3 * E) if split else None)
    want_hi, want_lo = kv_hi.clone(), (kv_lo.clone() if split else None)
    for j, b in enumerate(slots):
        for r in range(Lq):
            pg = int(table[b, r // 64])
            if 0 < pg < n_pages:
                want_hi[pg * 64 + r % 64] = qkv_hi[j * Lq + r, E:]
                if split:
                    want_lo[pg * 64 + r % 64] = qkv_lo[j * Lq + r, E:]
    ctx.slot_kv_scatter_paged(qkv_hi, qkv_lo, 3 * E, E, 2 * E, len(slots), Lq, torch.tensor(slots, dtype=torch.int32, device="cuda"), kv_hi,
                              kv_lo, 2 * E, table.cuda(), n_pages)
    assert torch.equal(kv_hi, want_hi) and (not split or torch.equal(kv_lo, want_lo))
    assert torch.equal(kv_hi[:64], want_hi[:64])


# ------------------------------------------------------------------------------------------------- policies
def _policy(kind):
    if kind == "vima":
        return build_policy("4M")
    from tests.test_baseline_decode_gpu import _policy as bp

    return bp(kind)


class _Schedule:
    """Five slots over 14 ticks: admissions (ragged prompts) at different ticks, a release and re-admission, an admission over a
    live slot, one slot never admitted.  Steps alternate between step_slots and act_slots with a sampler; page boundaries are
    crossed by every episode."""

    S, TICKS = 5, 14
    ADMITS = {0: [0, 2], 1: [1], 4: [4], 6: [2], 9: [0]}  # tick 9 re-admits slot 0 while it is live
    RELEASES = {5: [2], 11: [1]}

    def __init__(self, kind, pol):
        self.kind, self.pol = kind, pol
        E = pol.embed_dim
        self.Q = 6 if kind == "vima" else pol._obj_xf_num_queries
        self.decoder_only = kind in ("gato", "gpt")
        g = torch.Generator(device="cuda").manual_seed(11)
        self.Lp = 40
        self.prompts = {(t, b): (torch.randn(self.Lp, 1, E, device="cuda", generator=g),
                                 torch.rand(1, self.Lp, device="cuda", generator=g) > 0.2) for t, bs in self.ADMITS.items() for b in bs}
        for _, m in self.prompts.values():
            m[:, 0] = True
        shape = (self.TICKS, self.S, E) if kind == "gpt" else (self.TICKS, self.S, self.Q, E)
        self.obs = torch.randn(*shape, device="cuda", generator=g)
        self.msk = torch.rand(self.TICKS, self.S, self.Q, device="cuda", generator=g) > 0.2
        self.msk[..., 0] = True
        self.act = torch.randn(self.TICKS, self.S, E, device="cuda", generator=g)
        self.Lmax = (self.Lp + 1 if self.decoder_only else 0) + self.TICKS * (self.Q + 1)

    def open(self, kv_pool_tokens=None):
        if self.kind in ("vima", "flamingo"):
            return self.pol.open_slots(self.S, max_tokens=self.Lmax, max_prompt_tokens=self.Lp, kv_pool_tokens=kv_pool_tokens)
        return self.pol.open_slots(self.S, max_tokens=self.Lmax, kv_pool_tokens=kv_pool_tokens)

    def events(self, t, cache):
        for b in self.RELEASES.get(t, []):
            self.pol.release(cache, [b])
        if t in self.ADMITS:
            bs = self.ADMITS[t]
            self.pol.admit(cache, bs, torch.cat([self.prompts[(t, b)][0] for b in bs], 1), torch.cat([self.prompts[(t, b)][1] for b in bs], 0))

    def inputs(self, t):
        o = self.obs[t:t + 1]
        return (o, self.msk[t:t + 1]) if self.kind == "vima" else (o,)

    def step(self, t, cache, sampler, graph=None):
        if graph is not None:
            return graph(*self.inputs(t))
        if t % 2:
            return self.pol.act_slots(cache, *self.inputs(t), sampler=sampler)
        return self.pol.step_slots(cache, *self.inputs(t), self.act[t:t + 1])

    def run(self, cache, sampler, graph=None, peak=None):
        outs = []
        for t in range(self.TICKS):
            self.events(t, cache)
            active = [b for b in range(self.S) if cache.active_host[b]]
            r = self.step(t, cache, sampler, graph)
            if peak is not None:
                peak.append(cache.kv_pages_total - cache.kv_pages_free)
            flat = [r] if isinstance(r, torch.Tensor) else [d[k] for d in r for k in sorted(d)]
            outs.append([x[:, active].clone() for x in flat])
        torch.cuda.synchronize()
        return outs


def _small_pool(cache_default, peak):
    """The smallest pool the schedule fits, in tokens: its peak page count, from the host allocator over the default-pool run."""
    assert max(peak) < cache_default.kv_pages_total, (max(peak), cache_default.kv_pages_total)
    return max(peak) * 64


@pytest.mark.parametrize("mode", ["f16x3", "f16f8"])
@pytest.mark.parametrize("kind", ["vima", "gato", "gpt", "flamingo"])
def test_small_shuffled_pool_equals_default_pool(kind, mode):
    import vima_b200

    vima_b200.set_precision(mode)
    try:
        pol = _policy(kind)
        sched = _Schedule(kind, pol)
        with torch.no_grad():
            peak = []
            c0 = sched.open()
            ref = sched.run(c0, vima_b200.ActionSampler(3, "cuda"), peak=peak)
            c1 = sched.open(_small_pool(c0, peak))
            random.Random(1).shuffle(c1.pages.free)
            got = sched.run(c1, vima_b200.ActionSampler(3, "cuda"))
            assert max(peak) == c1.kv_pages_total
        for t, (a, b) in enumerate(zip(ref, got)):
            assert len(a) == len(b)
            for x, y in zip(a, b):
                assert torch.equal(x, y), (kind, mode, t)
    finally:
        vima_b200.set_precision("f16x3")


@pytest.mark.parametrize("kind", ["vima", "gato"])
def test_graph_on_recycled_pages_equals_eager(kind):
    """capture_act_slots on a small shuffled pool, replayed across page-boundary crossings and admissions onto recycled pages, equals
    the eager run on the default pool bit for bit; the capture leaves the page table and the free list as they were."""
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    sched = _Schedule(kind, pol)
    sched.step = lambda t, cache, sampler, graph=None: (graph(*sched.inputs(t)) if graph is not None else
                                                        pol.act_slots(cache, *sched.inputs(t), sampler=sampler))
    with torch.no_grad():
        peak = []
        c0 = sched.open()
        ref = sched.run(c0, vima_b200.ActionSampler(5, "cuda"), peak=peak)
        c1 = sched.open(_small_pool(c0, peak))
        random.Random(2).shuffle(c1.pages.free)
        s1 = vima_b200.ActionSampler(5, "cuda")
        sched.events(0, c1)
        before, table = c1.state(), c1.page_table.clone()
        gs = pol.capture_act_slots(c1, *sched.inputs(0), sampler=s1)
        torch.cuda.synchronize()
        after = c1.state()
        assert all(torch.equal(x, y) for x, y in zip(before[0], after[0])) and before[1] == after[1]
        assert torch.equal(table, c1.page_table)
        sched.ADMITS = dict(sched.ADMITS)
        del sched.ADMITS[0]  # tick 0's admissions happened before the capture
        got = sched.run(c1, s1, graph=gs)
        sched.ADMITS = _Schedule.ADMITS
    for t, (a, b) in enumerate(zip(ref, got)):
        for x, y in zip(a, b):
            assert torch.equal(x, y), t


@pytest.mark.parametrize("kind", ["vima", "gato"])
def test_pool_refusals_change_nothing(kind):
    """A pool of two slots' first steps: the third episode's first step (VIMAPolicy: admission takes no page) or its admission
    (VIMA-Gato: the prefix takes pages) raises ValueError and changes nothing; after a release it goes through and matches the
    default pool."""
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    sched = _Schedule(kind, pol)
    dec, Q = sched.decoder_only, sched.Q
    # decoder-only prompts of 64 tokens: prompt + separator end one column into a second page, and a slot's first two steps stay
    # in the pages its first step takes (Q <= 30)
    Lp = 64 if dec else sched.Lp
    pre = Lp + 1 if dec else 0
    first = -(-(pre + Q + 1) // 64)
    assert first == -(-(pre + 2 * Q + 2) // 64)
    g = torch.Generator(device="cuda").manual_seed(5)
    prompts = [(torch.randn(Lp, 1, pol.embed_dim, device="cuda", generator=g), torch.ones(1, Lp, dtype=torch.bool, device="cuda"))
               for _ in range(3)]
    step = lambda c, t: pol.step_slots(c, *sched.inputs(t), sched.act[t:t + 1])  # noqa: E731
    with torch.no_grad():
        ref, cache = sched.open(), sched.open(64 * 2 * first)
        a, b = [], []
        for c, out in ((ref, a), (cache, b)):
            pol.admit(c, [0, 2], torch.cat([prompts[0][0], prompts[2][0]], 1), torch.cat([prompts[0][1], prompts[2][1]], 0))
            out.append(step(c, 0))
            if not dec:
                pol.admit(c, [1], *prompts[1])
        assert torch.equal(a[0][:, [0, 2]], b[0][:, [0, 2]]) and cache.kv_pages_free == 0
        torch.cuda.synchronize()
        st, mask = cache.state(), cache.mask.clone()
        with pytest.raises(ValueError, match="K/V pages"):
            if dec:
                pol.admit(cache, [1], *prompts[1])  # the prefix finds no free page
            else:
                step(cache, 1)  # slot 1's first step finds no free page
        torch.cuda.synchronize()
        now = cache.state()
        assert all(torch.equal(x, y) for x, y in zip(st[0], now[0])) and st[1] == now[1] and torch.equal(mask, cache.mask)
        for c, out in ((ref, a), (cache, b)):
            pol.release(c, [2])
            if dec:
                pol.admit(c, [1], *prompts[1])
            out.append(step(c, 1))
        assert torch.equal(a[1][:, [0, 1]], b[1][:, [0, 1]])


def test_page_reservation_release_readmission_do_not_synchronise():
    """Between steps that cross page boundaries: each step's check and page reservation, a release, and the page side of a
    re-admission (check_prefix, then the slot's pages back to the pool and new ones for its prefix) run with CUDA sync debugging
    set to raise; the device table then equals the host allocator's."""
    import vima_b200
    from vima_b200 import engine as eng

    vima_b200.set_precision("f16x3")
    pol = _policy("gato")
    sched = _Schedule("gato", pol)
    Q, E = sched.Q, pol.embed_dim
    with torch.no_grad():
        cache = sched.open()
        sched.events(0, cache)
        sched.events(1, cache)
        pol.step_slots(cache, *sched.inputs(0), sched.act[:1])  # first-call host checks, kernel attributes
        torch.cuda.synchronize()
        for t in range(1, 8):  # Q + 1 = 17 columns a tick: page boundaries every few ticks
            torch.cuda.set_sync_debug_mode("error")
            try:
                if t == 3:
                    pol.release(cache, [2])
                if t == 5:
                    cache.check_prefix([0], sched.Lp + 1)
                    cache.free_slots([0], sched.Lp + 1)
                cache.check_step(cache.S, Q, E, eng.prec())
                cache.reserve_step(Q)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            if t == 5:  # the re-admission's prefill and state reset (their own page operations repeat the above)
                pol.admit(cache, [0], *sched.prompts[(0, 0)])
                cache.check_step(cache.S, Q, E, eng.prec())
                cache.reserve_step(Q)
            pol._slot_step(cache, *sched.inputs(t), sched.act[t:t + 1])
            cache.advance_host(Q)
        torch.cuda.synchronize()
        assert cache.len.tolist() == cache.len_host
        want = torch.zeros_like(cache.page_table)
        for b, own in enumerate(cache.pages.owned):
            want[b, :len(own)] = torch.tensor(own, dtype=torch.int32)
        assert torch.equal(want, cache.page_table)
        assert max(len(o) for o in cache.pages.owned) >= 2
