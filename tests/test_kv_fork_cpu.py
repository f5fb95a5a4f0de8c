"""CPU: forked slots on the paged K/V cache's host side -- reference-counted pages shared by a fork, copy on write of the one
partly filled page a sharer writes into, page counting (kv_pages_needed / check_step / check_prefix) with shared pages, state
round trips, and seeded random admit / fork / step / release schedules against the allocator's invariants.  The cache runs on a
host-only stand-in (CPU state vectors, table pushes and page copies recorded instead of launched); plus the copy kernel's ptxas
report."""
import os
import random
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from vima_b200.nn.xattn_gpt import KVPagePool, SlotDecodeCache


class _HostCache(SlotDecodeCache):
    """SlotDecodeCache without a GPU: state vectors on the CPU, table pushes applied to a numpy table, page copies recorded."""

    def __init__(self, S, Lmax, kv_pool_tokens=None):
        page_ld = KVPagePool.pages_for(Lmax)
        n_use = S * page_ld if kv_pool_tokens is None else KVPagePool.pages_for(kv_pool_tokens)
        self.S, self.Lmax, self.E, self.Lp_cap = S, Lmax, 8, 0
        self.pages = KVPagePool(S, page_ld, n_use + 1)
        self.table = np.zeros((S, page_ld), np.int32)
        z = lambda: torch.zeros(S, dtype=torch.int32)  # noqa: E731
        self.len, self.n_valid, self.has_action, self.active = z(), z(), z(), z()
        self.action_token = torch.zeros(S, 8)
        self.mask = torch.zeros(S, Lmax, dtype=torch.uint8)
        self.len_host, self.has_action_host, self.active_host = [0] * S, [False] * S, [False] * S
        self.copies = []

    def device_ints(self, values):
        return torch.tensor(values, dtype=torch.int64)

    def _push_pages(self, upd):
        for i, pg in upd:
            self.table.reshape(-1)[i] = pg

    def _copy_pages(self, copies):
        self.copies += copies

    def check_precision(self, p):
        pass

    def admit(self, slots, prefix=0):
        if prefix:
            self.check_prefix(slots, prefix)
        self.free_slots(slots, prefix)
        for b in slots:
            self.len_host[b], self.has_action_host[b], self.active_host[b] = prefix, False, True
            self.len[b], self.active[b] = prefix, 1

    def release(self, slots):
        self.free_slots(slots)
        for b in slots:
            self.active_host[b] = False
            self.active[b] = 0

    def fork_(self, src, dst):
        s, d = self.check_fork(src, dst)
        self.fork(s, d)

    def step(self, Q):
        self.check_step(self.S, Q, self.E, None)
        self.reserve_step(Q)
        for b in range(self.S):  # what vima_slot_step_end does to the device state
            if self.active_host[b]:
                self.len[b] += Q + int(self.has_action_host[b])
                self.has_action[b] = 1
        self.advance_host(Q)

    def check_invariants(self):
        P = self.pages
        held = {}
        for own in P.owned:
            for pg in own:
                held[pg] = held.get(pg, 0) + 1
        assert 0 not in held and P.refs[0] == 0  # the zero page is never held
        assert all(P.refs[pg] == held.get(pg, 0) for pg in range(P.n_pages))  # counts = table rows holding the page
        assert len(P.free) + len(held) == self.kv_pages_total and not set(P.free) & set(held)
        assert sorted(P.free + list(held)) == list(range(1, P.n_pages))
        want = np.zeros_like(self.table)
        for b, own in enumerate(P.owned):
            want[b, :len(own)] = own
        assert np.array_equal(want, self.table)
        assert all(0 not in c for c in self.copies)  # page 0 is never copied from or to
        assert self.len.tolist() == self.len_host and self.active.tolist() == [int(a) for a in self.active_host]
        for b in range(self.S):  # a slot holds exactly the pages of its written columns, plus at most the step's lookahead
            if self.active_host[b]:
                assert len(P.owned[b]) >= P.pages_for(self.len_host[b])
            else:
                assert not P.owned[b]


def test_fork_shares_pages_and_takes_none():
    c = _HostCache(S=4, Lmax=320)
    c.admit([0], prefix=100)  # two pages
    free = c.kv_pages_free
    c.fork_([0, 0], [1, 3])
    assert c.kv_pages_free == free and c.pages.owned[1] == c.pages.owned[0] == c.pages.owned[3]
    assert [c.pages.refs[pg] for pg in c.pages.owned[0]] == [3, 3]
    assert c.len_host == [100, 100, 0, 100] and c.len.tolist() == [100, 100, 0, 100] and c.active.tolist() == [1, 1, 0, 1]
    assert not c.copies
    c.check_invariants()


def test_copy_on_write_only_inside_a_shared_page_and_last_sharer_keeps_it():
    c = _HostCache(S=4, Lmax=320)
    c.admit([2], prefix=100)  # len 100: column 100 lies inside the second page
    orig = list(c.pages.owned[2])
    c.fork_([2, 2], [0, 3])
    assert c.kv_pages_needed(5) == 2  # two copies; the step's columns [100, 106) stay inside the second page
    c.step(5)
    # slots visited in ascending order: 0 and 2 copy, 3 (the last sharer) keeps the original page
    assert [old for old, _ in c.copies] == [orig[1], orig[1]]
    assert c.pages.owned[3] == orig and c.pages.owned[0][1] != orig[1] and c.pages.owned[2][1] != orig[1]
    assert c.pages.owned[0][0] == c.pages.owned[2][0] == orig[0] and c.pages.refs[orig[0]] == 3  # full pages stay shared
    assert c.pages.refs[orig[1]] == 1
    c.check_invariants()
    n = len(c.copies)
    c.step(5)  # nothing is shared at column len any more
    assert len(c.copies) == n
    c.check_invariants()


def test_no_copy_at_a_page_boundary():
    c = _HostCache(S=3, Lmax=320)
    c.admit([0], prefix=128)  # len 128: the next step starts a page of its own
    c.fork_([0], [1])
    assert c.kv_pages_needed(10) == 2  # one new page each, no copy
    c.step(10)
    assert not c.copies and c.pages.owned[0][:2] == c.pages.owned[1][:2] and c.pages.owned[0][2] != c.pages.owned[1][2]
    c.check_invariants()


def test_fork_after_the_first_step_shares_only_written_pages():
    """A first step of Q = 64 reserves columns [0, 65) (two pages) but writes len = 64: the fork shares one page; the lookahead page
    stays the source's alone."""
    c = _HostCache(S=2, Lmax=320)
    c.admit([0])
    c.step(64)
    assert c.len_host[0] == 64 and len(c.pages.owned[0]) == 2
    c.fork_([0], [1])
    assert c.pages.owned[1] == c.pages.owned[0][:1] and c.pages.refs[c.pages.owned[0][1]] == 1
    assert c.kv_pages_needed(10) == 1  # slot 1 takes its own second page; no copy
    c.step(10)
    assert not c.copies
    c.check_invariants()


def test_release_frees_a_shared_page_only_with_its_last_holder():
    c = _HostCache(S=3, Lmax=256)
    c.admit([0], prefix=70)
    pages = list(c.pages.owned[0])
    c.fork_([0, 0], [1, 2])
    free = c.kv_pages_free
    c.release([0])
    assert c.kv_pages_free == free and [c.pages.refs[p] for p in pages] == [2, 2]
    c.release([2])
    assert c.kv_pages_free == free
    c.release([1])
    assert c.kv_pages_free == free + 2 and sorted(c.pages.free[-2:]) == sorted(pages)
    c.check_invariants()


def test_fork_over_a_live_destination_releases_it_first():
    c = _HostCache(S=3, Lmax=256)
    c.admit([0], prefix=70)
    c.admit([1], prefix=150)
    c.fork_([0], [1])
    assert c.pages.owned[1] == c.pages.owned[0] and c.kv_pages_free == c.kv_pages_total - 2 and c.len_host[1] == 70
    c.check_invariants()


def test_fork_refusals_touch_nothing():
    c = _HostCache(S=4, Lmax=256)
    c.admit([0, 1], prefix=70)
    st, table = c.pages.state(), c.table.copy()
    for src, dst in (([2], [3]), ([4], [3]), ([-1], [3]), ([0, 0], [3, 3]), ([0], [0]), ([0, 1], [1, 2]), ([0], [4]), ([0, 1], [2])):
        with pytest.raises(ValueError, match="fork|slots"):
            c.fork_(src, dst)
        assert c.pages.state() == st and np.array_equal(c.table, table) and c.active_host == [True, True, False, False]


def test_needed_and_check_step_count_copies():
    c = _HostCache(S=3, Lmax=256, kv_pool_tokens=4 * 64)
    c.admit([0], prefix=100)  # two pages
    c.fork_([0, 0], [1, 2])
    assert c.kv_pages_free == 2 and c.kv_pages_needed(20) == 2  # two copies, no new page (columns [100, 121))
    c.step(20)
    assert c.kv_pages_free == 0 and len(c.copies) == 2
    c.check_invariants()
    c2 = _HostCache(S=4, Lmax=256, kv_pool_tokens=4 * 64)
    c2.admit([0], prefix=100)
    c2.fork_([0, 0, 0], [1, 2, 3])
    assert c2.kv_pages_needed(20) == 3 and c2.kv_pages_free == 2
    st, table, lens = c2.pages.state(), c2.table.copy(), list(c2.len_host)
    with pytest.raises(ValueError, match="3 more K/V pages, 2 of 4"):
        c2.step(20)
    assert c2.pages.state() == st and np.array_equal(c2.table, table) and c2.len_host == lens and not c2.copies
    c2.release([3])
    c2.step(20)
    c2.check_invariants()


def test_check_prefix_counts_only_pages_given_back():
    c = _HostCache(S=4, Lmax=256, kv_pool_tokens=4 * 64)
    c.admit([0], prefix=100)  # two pages
    c.fork_([0], [1])
    c.admit([2], prefix=100)  # two more: the pool is full
    with pytest.raises(ValueError, match="needs 2 K/V pages, 0 are free"):
        c.admit([1], prefix=100)  # slot 1's pages are still slot 0's too
    c.admit([0, 1], prefix=60)  # together they give both pages back
    c.check_invariants()
    c.fork_([2], [3])
    with pytest.raises(ValueError, match="needs 4 K/V pages, 1 are free"):
        c.admit([2, 0], prefix=100)  # slot 0's page comes back, slot 2's stay with slot 3
    c.admit([2, 3], prefix=60)  # slots 2 and 3 together give the shared pages back
    c.check_invariants()
    c.check_invariants()


def test_state_restore_includes_counts():
    c = _HostCache(S=3, Lmax=256)
    c.admit([0], prefix=100)
    c.fork_([0], [1])
    st = c.pages.state()
    assert st[0] == c.pages.free and st[1] == c.pages.owned and st[2] == c.pages.refs
    c.step(5)
    c.release([1])
    assert c.pages.state() != st
    c.pages.restore(st)
    assert c.pages.state() == st and c.pages.refs[c.pages.owned[0][0]] == 2
    st[2][1] = 99  # the snapshot is a copy
    assert c.pages.state() != st


@pytest.mark.parametrize("seed", range(6))
def test_random_schedules_keep_the_invariants(seed):
    rng = random.Random(seed)
    S, Q = 6, rng.choice([3, 16, 31, 63, 64])
    c = _HostCache(S=S, Lmax=512, kv_pool_tokens=rng.choice([None, 40 * 64, 24 * 64]))
    rng.shuffle(c.pages.free)
    refused = 0
    for _ in range(120):
        op = rng.random()
        active = [b for b in range(S) if c.active_host[b]]
        try:
            if op < 0.2:
                c.admit(rng.sample(range(S), rng.randint(1, 2)), prefix=rng.choice([0, 0, 40, 64, 100]))
            elif op < 0.4 and active:
                dst = rng.sample(range(S), rng.randint(1, 3))
                src = [rng.choice(active) for _ in dst]
                if set(src) & set(dst):
                    with pytest.raises(ValueError):
                        c.fork_(src, dst)
                else:
                    c.fork_(src, dst)
            elif op < 0.5 and active:
                c.release(rng.sample(active, 1))
            else:
                if any(c.active_host[b] and c.len_host[b] + Q + 1 > c.Lmax for b in range(S)):
                    c.release([b for b in range(S) if c.active_host[b] and c.len_host[b] + Q + 1 > c.Lmax])
                st, table, lens = c.pages.state(), c.table.copy(), list(c.len_host)
                need, free, n_cow = c.kv_pages_needed(Q), c.kv_pages_free, len(c._cow_plan())
                n0 = len(c.copies)
                try:
                    c.step(Q)
                except ValueError:
                    assert need > free
                    assert c.pages.state() == st and np.array_equal(c.table, table) and c.len_host == lens
                    refused += 1
                else:
                    assert free - c.kv_pages_free == need  # new pages plus copies, exactly
                    assert len(c.copies) - n0 == n_cow
        except ValueError as e:
            assert "K/V pages" in str(e)
            refused += 1
        c.check_invariants()
    c.release(list(range(S)))
    assert sorted(c.pages.free) == list(range(1, c.pages.n_pages)) and not any(c.pages.refs)


def test_copy_kernel_ptxas():
    """slots.cu as vima_b200/build.py compiles it, plus -Xptxas -v: the block copy kernel has no spill."""
    from vima_b200 import build as vbuild

    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        pytest.skip("nvcc not found")
    tmp = tempfile.mkdtemp(prefix="vima_ptxas_copy_")
    try:
        r = subprocess.run([nvcc, *vbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(vbuild.CSRC, "slots.cu"), "-o",
                            os.path.join(tmp, "s.o")], capture_output=True, text=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    assert r.returncode == 0, r.stderr[-4000:]
    fns = re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    copy = [f for f in fns if "kv_copy_blocks_kernel" in f[0]]
    assert len(copy) == 1 and copy[0][1:] == ("0", "0"), fns
