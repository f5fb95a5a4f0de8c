"""GPU: forked slots.  vima_kv_copy_blocks against a torch index copy (NaN in every row it must not write); for all four policies,
a schedule that forks slots (one of them live, one from an already forked slot, at a page boundary or inside a page) equals, bit for
bit, a schedule that admits every fork as an episode of its own and replays the shared prefix with the same inputs -- on pools
whose rows outside the zero page start as NaN, greedy and then sampled; the forked schedule fits a pool the replayed one does not;
graph replays with forks between them equal eager steps; forks and copy-on-write reservations do not synchronise; refusals."""
import pytest
import torch

from tests.test_kv_pages_gpu import NAN_BITS, _policy

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    return _C.Context.get(torch.device("cuda", 0))


# ------------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("block_rows", [64, 256, 77])
def test_copy_blocks_equals_index_copy(ctx, block_rows):
    g = torch.Generator(device="cuda").manual_seed(block_rows)
    rows, W = 12 * block_rows, 136  # 272-byte rows
    nan = torch.tensor(NAN_BITS[0], dtype=torch.int16)
    bufs = [torch.full((rows, W), int(nan), dtype=torch.int16, device="cuda") for _ in range(3)]
    src_blocks = [0, 3, 5, 3]
    dst_blocks = [1, 7, 9, 11]
    for b in bufs:  # data in the source blocks only: every other row is NaN and must stay so unless a copy writes it
        for s in set(src_blocks):
            b[s * block_rows:(s + 1) * block_rows] = torch.randint(-30000, 30000, (block_rows, W), dtype=torch.int16, device="cuda",
                                                                   generator=g)
    src = [s * block_rows for s in src_blocks] + [-1, rows - block_rows + 1, 2 * block_rows]
    dst = [d * block_rows for d in dst_blocks] + [4 * block_rows, 4 * block_rows, rows]  # the last three are skipped
    want = [b.clone() for b in bufs]
    for w in want:
        for s, d in zip(src[:4], dst[:4]):
            w[d:d + block_rows] = w[s:s + block_rows]
    ptrs = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device="cuda")
    dev = lambda v: torch.tensor(v, dtype=torch.int64, device="cuda")  # noqa: E731
    ctx.kv_copy_blocks(ptrs, W * 2, dev(src), dev(dst), block_rows, rows)
    for b, w in zip(bufs, want):
        assert torch.equal(b, w)
    assert (bufs[0][4 * block_rows:5 * block_rows] == nan).all()  # skipped blocks wrote nothing
    # a sub-range of the buffers: buf_rows bounds the blocks, not the allocation
    ctx.kv_copy_blocks(ptrs[:1], W * 2, dev([0]), dev([2 * block_rows]), block_rows, 2 * block_rows)
    assert torch.equal(bufs[0], want[0])


def test_copy_blocks_refusals(ctx):
    b = torch.zeros(64, 16, dtype=torch.int16, device="cuda")
    ptrs = torch.tensor([b.data_ptr()], dtype=torch.int64, device="cuda")
    z = torch.zeros(1, dtype=torch.int64, device="cuda")
    for kw in (dict(row_bytes=24), dict(row_bytes=0), dict(block_rows=0), dict(bufs=ptrs[:0]), dict(buf_rows=-1)):
        a = dict(bufs=ptrs, row_bytes=32, src_row0=z, dst_row0=z, block_rows=1, buf_rows=64)
        a.update(kw)
        with pytest.raises(RuntimeError, match="kv_copy_blocks"):
            ctx.kv_copy_blocks(**a)
    from ctypes import c_int64, c_void_p

    assert ctx.lib.vima_kv_copy_blocks(ctx.h, None, 1, c_int64(32), c_void_p(z.data_ptr()), c_void_p(z.data_ptr()), 1, 1, c_int64(64),
                                       c_void_p(ctx._s())) == 1


# ------------------------------------------------------------------------------------------------- policies
class _Fork:
    """Forked schedule X on S = 6 slots and its replay Y on 7.  X: tick 0 admits P0 into slot 0 and P5 into slot 5 and forks slot 0
    into slot 4 right after admission; tick t1 forks slot 0 into slots 1, 2 and the live slot 5; tick t1+2 forks the forked slot 1
    into slot 3; tick t1+3 releases slot 2 and admits P2 into it.  Y admits every branch at tick 0 with its ancestor's prompt and
    feeds it its ancestor's inputs up to the fork (P5's episode lives in slot 6, so after t1 every X slot is the same row in Y and
    draws the same samples).  Ticks before the second fork act greedily, later ones sample."""

    def __init__(self, kind, pol, t1):
        self.kind, self.pol, self.t1 = kind, pol, t1
        self.greedy_until = t1 + 2  # X's slot 1 samples in row 1 between the two forks, Y's replay of slot 3 in row 3
        self.dec = kind in ("gato", "gpt")
        self.Q = 4 if kind == "vima" else pol._obj_xf_num_queries
        self.Lp = 63 - self.Q if self.dec else 40  # decoder-only: [prompt | separator] + one step ends on a page boundary
        self.T = t1 + 5
        E = pol.embed_dim
        g = torch.Generator(device="cuda").manual_seed(100 + t1)
        self.prompts = {}
        for k in ("P0", "P5", "P2"):
            m = torch.rand(1, self.Lp, device="cuda", generator=g) > 0.2
            m[:, 0] = True
            self.prompts[k] = (torch.randn(self.Lp, 1, E, device="cuda", generator=g), m)
        shape = (self.T, 6, E) if kind == "gpt" else (self.T, 6, self.Q, E)
        self.obs = torch.randn(*shape, device="cuda", generator=g)
        self.msk = torch.rand(self.T, 6, self.Q, device="cuda", generator=g) > 0.2
        self.msk[..., 0] = True
        self.Lmax = (self.Lp + 1 if self.dec else 0) + self.T * (self.Q + 1)
        t2, t3 = t1 + 2, t1 + 3
        # Y: (slot, start tick, end tick or None, prompt, X row of its inputs as a function of the tick)
        self.branches = [(0, 0, None, "P0", lambda t: 0), (6, 0, t1, "P5", lambda t: 5), (4, 0, None, "P0", lambda t: 4),
                         (1, 0, None, "P0", lambda t: 0 if t < t1 else 1), (2, 0, t3, "P0", lambda t: 0 if t < t1 else 2),
                         (5, 0, None, "P0", lambda t: 0 if t < t1 else 5), (3, 0, None, "P0", lambda t: 0 if t < t1 else 1 if t < t2 else 3),
                         (2, t3, None, "P2", lambda t: 2)]
        self.ymap = lambda b, t: 6 if (b == 5 and t < t1) else b  # the Y row of X slot b at tick t

    def open(self, S, kv_pool_tokens=None):
        from vima_b200 import engine as eng

        if self.dec:
            c = self.pol.open_slots(S, max_tokens=self.Lmax, kv_pool_tokens=kv_pool_tokens)
        else:
            c = self.pol.open_slots(S, max_tokens=self.Lmax, max_prompt_tokens=self.Lp, kv_pool_tokens=kv_pool_tokens)
        nan = NAN_BITS[eng.prec().dtype]
        for t in c.kv_hi + c.kv_lo:  # a missing or misdirected page copy reads NaN
            if t is not None:
                t[64:] = nan
        return c

    def admit(self, cache, slots, key):
        p, m = self.prompts[key]
        self.pol.admit(cache, slots, p.expand(-1, len(slots), -1).contiguous(), m.expand(len(slots), -1).contiguous())

    def step_inputs(self, t, rows):
        o = self.obs[t:t + 1, rows]
        return (o, self.msk[t:t + 1, rows]) if self.kind == "vima" else (o,)

    def act(self, cache, t, rows, sampler, graph=None):
        if graph is not None:
            return graph(*self.step_inputs(t, rows))
        return self.pol.act_slots(cache, *self.step_inputs(t, rows), sampler=sampler if t >= self.greedy_until else None)

    def events_x(self, t, cache):
        pol = self.pol
        if t == 0:
            self.admit(cache, [0], "P0")
            self.admit(cache, [5], "P5")
            pol.fork_slots(cache, [0], [4])
        if t == self.t1:
            pol.fork_slots(cache, [0, 0, 0], [1, 2, 5])
        if t == self.t1 + 2:
            pol.fork_slots(cache, [1], [3])
        if t == self.t1 + 3:
            pol.release(cache, [2])
            self.admit(cache, [2], "P2")

    def run_x(self, cache, sampler, peak=None):
        outs = []
        for t in range(self.T):
            self.events_x(t, cache)
            r = self.act(cache, t, list(range(6)), sampler)
            if peak is not None:
                peak.append(cache.kv_pages_total - cache.kv_pages_free)
            active = [b for b in range(6) if cache.active_host[b]]
            outs.append((active, [d[k][:, active].clone() for d in r for k in sorted(d)]))
        torch.cuda.synchronize()
        return outs

    def run_y(self, cache, sampler, peak=None):
        outs = []
        for t in range(self.T):
            for y, t0, t_end, key, _ in self.branches:
                if t_end == t:
                    self.pol.release(cache, [y])
            for y, t0, t_end, key, _ in self.branches:
                if t0 == t:
                    self.admit(cache, [y], key)
            rows = [0] * 7
            for y, t0, t_end, key, row in self.branches:
                if t0 <= t and (t_end is None or t < t_end):
                    rows[y] = row(t)
            r = self.act(cache, t, rows, sampler)
            if peak is not None:
                peak.append(cache.kv_pages_total - cache.kv_pages_free)
            outs.append([d[k].clone() for d in r for k in sorted(d)])
        torch.cuda.synchronize()
        return outs

    def fork_ticks(self):
        """Fork ticks t1 with the column `len` of slot 0 at the fork: inside a page, and on a page boundary."""
        pre = self.Lp + 1 if self.dec else 0
        length = lambda n: pre + n * (self.Q + 1) - (1 if n else 0)  # noqa: E731
        boundary = next(n for n in range(1, 64) if length(n) % 64 == 0)
        return [(2, length(2)), (boundary, length(boundary))]


def _compare(sched, x, y):
    for t, ((active, xs), ys) in enumerate(zip(x, y)):
        rows = [sched.ymap(b, t) for b in active]
        for a, b in zip(xs, ys):
            assert torch.equal(a, b[:, rows]), (sched.kind, sched.t1, t)
        for a in xs[len(xs) // 3:]:  # log-probs and entropies
            assert torch.isfinite(a).all(), (sched.kind, sched.t1, t)


@pytest.mark.parametrize("where", ["inside", "boundary"])
@pytest.mark.parametrize("kind", ["vima", "gato", "gpt", "flamingo"])
def test_fork_equals_replay(kind, where):
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    t1, length = _Fork(kind, pol, 1).fork_ticks()[0 if where == "inside" else 1]
    assert (length % 64 != 0) == (where == "inside")
    sched = _Fork(kind, pol, t1)
    with torch.no_grad():
        px, py = [], []
        cx = sched.open(6)
        x = sched.run_x(cx, vima_b200.ActionSampler(9, "cuda"), peak=px)
        cy = sched.open(7)
        y = sched.run_y(cy, vima_b200.ActionSampler(9, "cuda"), peak=py)
    _compare(sched, x, y)
    assert max(px) < max(py)
    if sched.dec:  # the fork right after admission shared the prompt pages; the first step copied the separator's page only
        assert (sched.Lp + 1) % 64 != 0


@pytest.mark.parametrize("kind", ["gato", "vima"])
def test_forked_schedule_fits_a_pool_the_replay_does_not(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    sched = _Fork(kind, pol, 2)
    with torch.no_grad():
        px, py = [], []
        x0 = sched.run_x(sched.open(6), vima_b200.ActionSampler(4, "cuda"), peak=px)
        sched.run_y(sched.open(7), vima_b200.ActionSampler(4, "cuda"), peak=py)
        assert max(px) < max(py)
        small = max(px) * 64
        x1 = sched.run_x(sched.open(6, small), vima_b200.ActionSampler(4, "cuda"))
        with pytest.raises(ValueError, match="K/V pages"):
            sched.run_y(sched.open(7, small), vima_b200.ActionSampler(4, "cuda"))
    for (a0, o0), (a1, o1) in zip(x0, x1):
        assert a0 == a1 and all(torch.equal(p, q) for p, q in zip(o0, o1))


@pytest.mark.parametrize("kind", ["vima", "gato"])
def test_graph_replays_with_forks_equal_eager(kind):
    """capture_act_slots after tick 0 (its warm-up leaves the page table, counts and free list as they were), replayed through
    forks, a fork of a fork and a re-admission, equals eager act_slots bit for bit (all ticks sampled)."""
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    sched = _Fork(kind, pol, 2)
    sched.greedy_until = 0  # every tick samples
    all6 = list(range(6))
    with torch.no_grad():
        ref = sched.run_x(sched.open(6), vima_b200.ActionSampler(6, "cuda"))
        c = sched.open(6)
        s = vima_b200.ActionSampler(6, "cuda")
        sched.events_x(0, c)
        pol.act_slots(c, *sched.step_inputs(0, all6), sampler=s)  # tick 0, eager
        before, table = c.state(), c.page_table.clone()
        g = pol.capture_act_slots(c, *sched.step_inputs(1, all6), sampler=s)
        torch.cuda.synchronize()
        after = c.state()
        assert all(torch.equal(a, b) for a, b in zip(before[0], after[0])) and before[1] == after[1]
        assert torch.equal(table, c.page_table)
        got = []
        for t in range(1, sched.T):
            sched.events_x(t, c)  # forks at ticks 2 and 4, a release and re-admission at tick 5
            r = g(*sched.step_inputs(t, all6))
            active = [b for b in range(6) if c.active_host[b]]
            got.append((active, [d[k][:, active].clone() for d in r for k in sorted(d)]))
        torch.cuda.synchronize()
    for (a0, o0), (a1, o1) in zip(ref[1:], got):
        assert a0 == a1 and all(torch.equal(p, q) for p, q in zip(o0, o1))


def test_fork_and_copy_on_write_do_not_synchronise():
    import vima_b200
    from vima_b200 import engine as eng

    vima_b200.set_precision("f16x3")
    pol = _policy("gato")
    sched = _Fork("gato", pol, 2)
    with torch.no_grad():
        c = sched.open(6)
        sched.admit(c, [0], "P0")
        for t in range(2):  # first-call host checks; len = 64 + Q + 1 after two steps, inside the second page
            pol.act_slots(c, *sched.step_inputs(t, list(range(6))))
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            pol.fork_slots(c, [0, 0], [1, 2])
            assert c.len_host[0] % 64 != 0
            c.check_step(c.S, sched.Q, pol.embed_dim, eng.prec())
            c.reserve_step(sched.Q)  # two copies on write
        finally:
            torch.cuda.set_sync_debug_mode(0)
        pol._act_step(c, *sched.step_inputs(2, list(range(6))), grouped=pol._act_grouped)
        c.advance_host(sched.Q)
        torch.cuda.synchronize()
        assert c.len.tolist() == c.len_host
        want = torch.zeros_like(c.page_table)
        for b, own in enumerate(c.pages.owned):
            want[b, :len(own)] = torch.tensor(own, dtype=torch.int32)
        assert torch.equal(want, c.page_table)
        assert len({c.pages.owned[b][-1] for b in range(3)}) == 3


@pytest.mark.parametrize("kind", ["vima", "flamingo", "gato", "gpt"])
def test_fork_refusals(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    sched = _Fork(kind, pol, 2)
    with torch.no_grad():
        c = sched.open(6)
        sched.admit(c, [0, 1], "P0")
        torch.cuda.synchronize()
        st = c.state()
        for src, dst in (([2], [3]), ([6], [3]), ([0, 0], [3, 3]), ([0], [0]), ([0, 1], [1, 2]), ([0], [6]), ([0], [3, 4])):
            with pytest.raises(ValueError):
                pol.fork_slots(c, src, dst)
        vima_b200.set_precision("f16f8")
        try:
            with pytest.raises(ValueError, match="precision"):
                pol.fork_slots(c, [0], [3])
        finally:
            vima_b200.set_precision("f16x3")
        torch.cuda.synchronize()
        now = c.state()
        assert all(torch.equal(a, b) for a, b in zip(st[0], now[0])) and st[1] == now[1]
        pol.refresh_weights()
        with pytest.raises(ValueError, match="weights|changed|Open a new cache"):
            pol.fork_slots(c, [0], [3])
