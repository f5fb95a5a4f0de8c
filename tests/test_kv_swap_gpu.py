"""GPU: swapped slot episodes.  vima_kv_pack_blocks against a torch index gather and scatter (NaN in every row it must not write); for
all four policies in f16x3 and f16f8, a schedule that swaps episodes out mid-run (a forked source whose fork stays live, an
episode before its first step, prompts whose last page is partly filled) and back in later (into other slots, into a second cache
with another slot count and smaller pools, one episode into two slots) equals, bit for bit, every episode run without
interruption -- on pools whose rows outside the zero page start as NaN; sampled runs and graph replays with swap round trips
between ticks equal the runs without; swap_out / swap_in do not synchronise; refusals touch nothing."""
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
def test_pack_unpack_equals_index_gather_and_scatter(ctx, block_rows):
    g = torch.Generator(device="cuda").manual_seed(block_rows)
    rows, W, nb = 12 * block_rows, 136, 3  # 272-byte rows
    nan = int(torch.tensor(NAN_BITS[0], dtype=torch.int16))
    bufs = [torch.randint(-30000, 30000, (rows, W), dtype=torch.int16, device="cuda", generator=g) for _ in range(nb)]
    blocks = [5, 0, 11, 5, 7]  # block 5 twice
    row0 = [b * block_rows for b in blocks] + [-1, rows - block_rows + 1]  # the last two are skipped
    dev = lambda v: torch.tensor(v, dtype=torch.int64, device="cuda")  # noqa: E731
    ptrs = dev([b.data_ptr() for b in bufs])
    packed = torch.full((len(row0), nb, block_rows, W), nan, dtype=torch.int16, device="cuda")
    ctx.kv_pack_blocks(ptrs, W * 2, dev(row0), block_rows, rows, packed, False)
    for i, r in enumerate(row0[:5]):
        for z in range(nb):
            assert torch.equal(packed[i, z], bufs[z][r:r + block_rows])
    assert (packed[5:] == nan).all()  # skipped blocks wrote nothing
    # unpack into NaN buffers at other blocks: exactly those rows are written, with the packed rows
    dst = [1, 3, 9, 10, 4]
    out = [torch.full_like(b, nan) for b in bufs]
    src = torch.randint(-30000, 30000, packed.shape, dtype=torch.int16, device="cuda", generator=g)
    ctx.kv_pack_blocks(dev([b.data_ptr() for b in out]), W * 2, dev([d * block_rows for d in dst] + row0[5:]), block_rows, rows, src, True)
    for z in range(nb):
        want = torch.full_like(bufs[z], nan)
        for i, d in enumerate(dst):
            want[d * block_rows:(d + 1) * block_rows] = src[i, z]
        assert torch.equal(out[z], want)
    # a round trip restores the blocks; buf_rows bounds the blocks, not the allocation
    back = [torch.full_like(b, nan) for b in bufs]
    ctx.kv_pack_blocks(dev([b.data_ptr() for b in back]), W * 2, dev(row0), block_rows, rows, packed, True)
    for z in range(nb):
        idx = torch.cat([torch.arange(r, r + block_rows, device="cuda") for r in row0[:5]])
        assert torch.equal(back[z][idx], bufs[z][idx])
    ctx.kv_pack_blocks(ptrs[:1], W * 2, dev([2 * block_rows]), block_rows, 2 * block_rows, packed, False)
    assert torch.equal(packed[0, 0], bufs[0][5 * block_rows:6 * block_rows])


def test_pack_blocks_refusals(ctx):
    b = torch.zeros(64, 16, dtype=torch.int16, device="cuda")
    ptrs = torch.tensor([b.data_ptr()], dtype=torch.int64, device="cuda")
    z = torch.zeros(1, dtype=torch.int64, device="cuda")
    pk = torch.zeros(64, 32, dtype=torch.uint8, device="cuda")
    for kw in (dict(row_bytes=24), dict(row_bytes=0), dict(block_rows=0), dict(bufs=ptrs[:0]), dict(buf_rows=-1), dict(packed=pk.view(-1)[1:])):
        a = dict(bufs=ptrs, row_bytes=32, row0=z, block_rows=1, buf_rows=64, packed=pk, unpack=False)
        a.update(kw)
        with pytest.raises(RuntimeError, match="kv_pack_blocks"):
            ctx.kv_pack_blocks(**a)
    from ctypes import c_int64, c_void_p

    assert ctx.lib.vima_kv_pack_blocks(ctx.h, None, 1, c_int64(32), c_void_p(z.data_ptr()), 1, 1, c_int64(64), c_void_p(pk.data_ptr()), 0,
                                       c_void_p(ctx._s())) == 1
    assert ctx.lib.vima_kv_pack_blocks(ctx.h, c_void_p(ptrs.data_ptr()), 1, c_int64(32), c_void_p(z.data_ptr()), 1, 1, c_int64(64), None, 0,
                                       c_void_p(ctx._s())) == 1
    assert ctx.lib.vima_kv_pack_blocks(ctx.h, c_void_p(ptrs.data_ptr()), 1, c_int64(32), c_void_p(z.data_ptr()), 1, 1, c_int64(64),
                                       c_void_p(pk.data_ptr()), 2, c_void_p(ctx._s())) == 1


# ------------------------------------------------------------------------------------------------- policies
class _Swap:
    """Schedule X on cache A (S = 6) and cache B (S = 4, smaller pools); events at the start of a tick, before its act_slots:
      t0: admit e0 -> A0, e1 -> A1
      t1: fork A1 -> A2 (e2); admit e3 -> A3 and swap it out before its first step
      t2: swap out A0 (e0) and A1 (e1, whose fork e2 stays live in A2)
      t3: swap e0 into B3; swap e3 into A0 and A5 (e3, e3b)
      t4: swap e1 into A4 and into B0 (e1, e1b)
    Every episode's k-th step takes the inputs of (episode, k), inherited from the episode it was forked or copied from for the steps
    before the branch.  The reference Y runs every episode uninterrupted in a row of its own.  Prompts of 40 tokens (the last
    prompt page, or for the decoder-only policies the last page of [prompt | separator], partly filled)."""

    T = 7
    ROOT = {"e2": ("e1", 1), "e1b": ("e1", 2), "e3b": ("e3", 0)}  # branch: (parent, steps inherited)
    PROMPT = {"e0": "P0", "e1": "P1", "e2": "P1", "e1b": "P1", "e3": "P3", "e3b": "P3"}

    def __init__(self, kind, pol):
        self.kind, self.pol = kind, pol
        self.dec = kind in ("gato", "gpt")
        self.Q = 4 if kind == "vima" else pol._obj_xf_num_queries
        self.Lp = 40
        E = pol.embed_dim
        g = torch.Generator(device="cuda").manual_seed(5)
        self.prompts = {}
        for k in ("P0", "P1", "P3"):
            m = torch.rand(1, self.Lp, device="cuda", generator=g) > 0.2
            m[:, 0] = True
            self.prompts[k] = (torch.randn(self.Lp, 1, E, device="cuda", generator=g), m)
        self.inp = {}
        for name in ("e0", "e1", "e2", "e1b", "e3", "e3b"):
            for k in range(self.T):
                o = torch.randn(E, device="cuda", generator=g) if kind == "gpt" else torch.randn(self.Q, E, device="cuda", generator=g)
                m = torch.rand(self.Q, device="cuda", generator=g) > 0.2
                m[0] = True
                self.inp[(name, k)] = (o, m)
        self.Lmax = (self.Lp + 1 if self.dec else 0) + self.T * (self.Q + 1)

    def key(self, name, k):
        if name in self.ROOT and k < self.ROOT[name][1]:
            return self.key(self.ROOT[name][0], k)
        return (name, k)

    def open(self, S, kv_pool_tokens=None, prompt_pool_tokens=None, Lmax=None, Lp=None):
        from vima_b200 import engine as eng

        Lmax = Lmax or self.Lmax
        if self.dec:
            c = self.pol.open_slots(S, max_tokens=Lmax, kv_pool_tokens=kv_pool_tokens)
        else:
            c = self.pol.open_slots(S, max_tokens=Lmax, max_prompt_tokens=Lp or self.Lp, kv_pool_tokens=kv_pool_tokens,
                                    prompt_pool_tokens=prompt_pool_tokens)
        nan = NAN_BITS[eng.prec().dtype]
        for t in c.kv_hi + c.kv_lo + (c.prompt_kv_hi + c.prompt_kv_lo if c.Lp_cap else []):  # a page not restored reads NaN
            if t is not None:
                t[64:] = nan
        return c

    def admit(self, cache, slot, name):
        p, m = self.prompts[self.PROMPT[name]]
        self.pol.admit(cache, [slot], p, m)

    def act(self, cache, names, steps, sampler=None, graph=None):
        """One act_slots of `cache` whose slot b holds episode names[b] (None: idle) at its step steps[name]."""
        E, S = self.pol.embed_dim, cache.S
        obs = torch.zeros((1, S, E) if self.kind == "gpt" else (1, S, self.Q, E), device="cuda")
        msk = torch.ones(1, S, self.Q, dtype=torch.bool, device="cuda")
        for b, n in enumerate(names):
            if n is not None:
                o, m = self.inp[self.key(n, steps[n])]
                obs[0, b], msk[0, b] = o, m
        args = (obs, msk) if self.kind == "vima" else (obs,)
        r = graph(*args) if graph is not None else self.pol.act_slots(cache, *args, sampler=sampler)
        return [d[k].clone() for d in r for k in sorted(d)] + [cache.action_token.view(1, S, E).clone()]

    @staticmethod
    def record(out, outs, names, steps):
        for b, n in enumerate(names):
            if n is not None:
                outs[(n, steps[n])] = [t[:, b] for t in out]
                steps[n] += 1

    def run_x(self, pol, A, B):
        a, b = [None] * A.S, [None] * B.S
        steps, outs, ep = {}, {}, {}
        for t in range(self.T):
            if t == 0:
                for s, n in ((0, "e0"), (1, "e1")):
                    self.admit(A, s, n)
                    a[s], steps[n] = n, 0
            if t == 1:
                pol.fork_slots(A, [1], [2])
                a[2], steps["e2"] = "e2", steps["e1"]
                self.admit(A, 3, "e3")
                (ep["e3"],) = pol.swap_out(A, [3])
                steps["e3"] = 0
            if t == 2:
                ep["e0"], ep["e1"] = pol.swap_out(A, [0, 1])
                a[0] = a[1] = None
            if t == 3:
                pol.swap_in(B, [3], [ep["e0"]])
                b[3] = "e0"
                pol.swap_in(A, [0, 5], [ep["e3"], ep["e3"]])
                a[0], a[5], steps["e3b"] = "e3", "e3b", steps["e3"]
            if t == 4:
                pol.swap_in(A, [4], [ep["e1"]])
                pol.swap_in(B, [0], [ep["e1"]])
                a[4], b[0], steps["e1b"] = "e1", "e1b", steps["e1"]
            assert [n is not None for n in a] == A.active_host and [n is not None for n in b] == B.active_host
            self.record(self.act(A, a, steps), outs, a, steps)
            if any(b):
                self.record(self.act(B, b, steps), outs, b, steps)
        torch.cuda.synchronize()
        return outs

    def run_y(self, cache):
        names = ["e0", "e1", "e2", "e1b", "e3", "e3b"]
        steps, outs = {n: 0 for n in names}, {}
        for s, n in enumerate(names):
            self.admit(cache, s, n)
        for t in range(self.T):
            self.record(self.act(cache, names, steps), outs, names, steps)
        torch.cuda.synchronize()
        return outs


@pytest.mark.parametrize("prec", ["f16x3", "f16f8"])
@pytest.mark.parametrize("kind", ["vima", "gato", "gpt", "flamingo"])
def test_swapped_schedule_equals_uninterrupted_episodes(kind, prec):
    import vima_b200

    vima_b200.set_precision(prec)
    try:
        pol = _policy(kind)
        sched = _Swap(kind, pol)
        page_ld = -(-sched.Lmax // 64)
        with torch.no_grad():
            A = sched.open(6)
            B = sched.open(4, kv_pool_tokens=(2 * page_ld + 1) * 64, prompt_pool_tokens=2 * 64)
            assert B.kv_pages_total < 4 * page_ld
            x = sched.run_x(pol, A, B)
            y = sched.run_y(sched.open(6))
    finally:
        vima_b200.set_precision("f16x3")
    assert len(x) == 6 + 5 + 6 + 3 + 4 + 4  # steps of e0, e1, e2, e1b, e3, e3b
    for k, xs in x.items():
        for a, b in zip(xs, y[k]):
            assert torch.equal(a, b), (kind, prec, k)
        assert all(torch.isfinite(a.float()).all() for a in xs), (kind, prec, k)


def _round_trip_runs(kind, seed, graph):
    """A sampled act_slots run of four staggered episodes (S = 4, Lmax 6 steps) twice: without swaps, and with every active slot
    swapped out and back into the same slot between ticks (with `graph`: act_slots replayed from one graph captured at tick 1)."""
    import vima_b200

    pol = _policy(kind)
    sched = _Swap(kind, pol)
    names = ["e0", "e1", "e3", "e2"]
    runs = []
    for swap in (False, True):
        c = sched.open(4)
        s = vima_b200.ActionSampler(seed, "cuda")
        cur, steps, outs, g = [None] * 4, {}, {}, None
        for t in range(sched.T - 1):
            if t in (0, 1):
                for b in ((0, 1) if t == 0 else (2, 3)):
                    sched.admit(c, b, names[b])
                    cur[b], steps[names[b]] = names[b], 0
            if swap and t:
                act = [b for b in range(4) if cur[b]]
                pol.swap_in(c, act, pol.swap_out(c, act))
            if graph and t == 1:
                E = pol.embed_dim
                obs = torch.zeros((1, 4, E) if kind == "gpt" else (1, 4, sched.Q, E), device="cuda")
                args = (obs, torch.ones(1, 4, sched.Q, dtype=torch.bool, device="cuda")) if kind == "vima" else (obs,)
                g = pol.capture_act_slots(c, *args, sampler=s)
            sched.record(sched.act(c, cur, steps, sampler=s, graph=g), outs, cur, steps)
        torch.cuda.synchronize()
        runs.append(outs)
    return runs


@pytest.mark.parametrize("kind", ["vima", "gato", "flamingo"])
def test_sampled_round_trips_equal_the_run_without_swaps(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    with torch.no_grad():
        ref, got = _round_trip_runs(kind, 11, graph=False)
    assert ref.keys() == got.keys()
    for k in ref:
        assert all(torch.equal(a, b) for a, b in zip(ref[k], got[k])), (kind, k)


@pytest.mark.parametrize("kind", ["vima", "gato"])
def test_graph_replays_with_swaps_equal_eager(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    with torch.no_grad():
        ref, _ = _round_trip_runs(kind, 12, graph=False)
        _, got = _round_trip_runs(kind, 12, graph=True)
    assert ref.keys() == got.keys()
    for k in ref:
        assert all(torch.equal(a, b) for a, b in zip(ref[k], got[k])), (kind, k)


@pytest.mark.parametrize("kind", ["vima", "gato"])
def test_swap_out_and_in_do_not_synchronise(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    sched = _Swap(kind, pol)
    with torch.no_grad():
        c = sched.open(6)
        cur, steps = ["e0", "e1", None, None, None, None], {"e0": 0, "e1": 0}
        sched.admit(c, 0, "e0")
        sched.admit(c, 1, "e1")
        for _ in range(2):
            sched.record(sched.act(c, cur, steps), {}, cur, steps)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            eps = pol.swap_out(c, [0, 1])
            pol.swap_in(c, [3, 4, 5], [eps[0], eps[1], eps[1]])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        assert c.len.tolist() == c.len_host and c.active.tolist() == [int(a) for a in c.active_host] == [0, 0, 0, 1, 1, 1]
        want = torch.zeros_like(c.page_table)
        for b, own in enumerate(c.pages.owned):
            want[b, :len(own)] = torch.tensor(own, dtype=torch.int32)
        assert torch.equal(want, c.page_table)
        assert all(e.nbytes == e.kv.numel() + e.prompt.numel() + e.state.numel() and e.kv.is_pinned() for e in eps)


def _snapshot(c):
    dev, host = c.state()
    out = [t.clone() for t in dev] + [c.mask.clone()]
    host = [host, list(c.pages.free)]
    if c.Lp_cap:
        out += [c.prompt_page_table.clone(), c.prompt_len.clone(), c.prompt_mask.clone()]
        host.append(c.prompt_pages.state())
    return out, host


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a[0], b[0])) and a[1] == b[1]


def _twin(kind):
    """A second policy of the kind with the same weight values in other parameters."""
    import vima_b200
    from oracle import detgen, synth

    if kind == "vima":
        pol = vima_b200.VIMAPolicy(**synth.MODEL_CFGS["4M"])
    elif kind == "flamingo":
        pol = vima_b200.VIMAFlamingoPolicy(**synth.FLAMINGO_CFGS["flamingo_tiny"])
    else:
        pol = {"gato": vima_b200.VIMAGatoPolicy, "gpt": vima_b200.VIMAGPTPolicy}[kind](**synth.GATO_CFGS["gato_tiny"])
    detgen.fill_module_(pol)
    return pol.cuda().eval()


@pytest.mark.parametrize("kind", ["vima", "flamingo", "gato", "gpt"])
def test_swap_refusals(kind):
    import vima_b200

    vima_b200.set_precision("f16x3")
    pol = _policy(kind)
    sched = _Swap(kind, pol)
    with torch.no_grad():
        c = sched.open(4)
        sched.admit(c, 0, "e0")
        sched.admit(c, 1, "e1")
        cur, steps = ["e0", "e1", None, None], {"e0": 0, "e1": 0}
        for _ in range(2):
            sched.record(sched.act(c, cur, steps), {}, cur, steps)
        (ep,) = pol.swap_out(c, [1])
        torch.cuda.synchronize()
        st = _snapshot(c)
        for slots in ([1], [4], [-1], [0, 0]):
            with pytest.raises(ValueError):
                pol.swap_out(c, slots)
        for slots, eps in (([3, 2], [ep]), ([3], [ep, ep]), ([4], [ep]), ([2, 2], [ep, ep]), ([2], ["not an episode"])):
            with pytest.raises(ValueError):
                pol.swap_in(c, slots, eps)
        torch.cuda.synchronize()
        assert _same(st, _snapshot(c))
        # pools that hold the episode once
        small = sched.open(2, kv_pool_tokens=ep.kv_pages * 64, prompt_pool_tokens=max(ep.prompt_pages, 1) * 64)
        pol.swap_in(small, [0], [ep])
        torch.cuda.synchronize()
        st_small = _snapshot(small)
        with pytest.raises(ValueError, match="pages"):
            pol.swap_in(small, [1], [ep])
        pol.swap_in(small, [0], [ep])  # the destination gives its pages back first
        torch.cuda.synchronize()
        assert _same(st_small, _snapshot(small))
        # caches of another max_tokens, max_prompt_tokens or precision mode
        others = [sched.open(4, Lmax=sched.Lmax + 64)]
        if not sched.dec:
            others.append(sched.open(4, Lp=sched.Lp + 64))
        for o in others:
            with pytest.raises(ValueError, match="swap_in"):
                pol.swap_in(o, [0], [ep])
        vima_b200.set_precision("f16f8")
        try:
            with pytest.raises(ValueError, match="swap_in"):
                pol.swap_in(sched.open(4), [0], [ep])
            with pytest.raises(ValueError, match="precision"):
                pol.swap_out(c, [0])
        finally:
            vima_b200.set_precision("f16x3")
        # another policy of the same kind and weight values (other parameters)
        twin = _twin(kind)
        tc = twin.open_slots(4, max_tokens=sched.Lmax) if sched.dec else twin.open_slots(4, max_tokens=sched.Lmax, max_prompt_tokens=sched.Lp)
        with pytest.raises(ValueError, match="other weights"):
            twin.swap_in(tc, [0], [ep])
        del twin, tc
        # weights changed by load_state_dict after the swap-out: a cache opened before it and the episode in a new cache are refused
        before = sched.open(4)
        pol.load_state_dict(pol.state_dict())
        with pytest.raises(ValueError, match="weights"):
            pol.swap_in(before, [0], [ep])
        with pytest.raises(ValueError, match="other weights"):
            pol.swap_in(sched.open(4), [0], [ep])
        torch.cuda.synchronize()
        assert _same(st, _snapshot(c))
