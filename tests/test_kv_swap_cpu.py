"""CPU: swapped slot episodes on the paged K/V cache's host side -- swap-out gives back only the pages no other slot holds, swap-in
takes private pages and rebuilds the table row and host mirrors, refusals touch nothing, an episode can be swapped in more than
once, and seeded random admit / fork / step / release / swap-out / swap-in schedules keep the allocator's invariants.  The cache
runs on the host-only stand-in of test_kv_fork_cpu (the packed pages are recorded as the page numbers they came from); plus the
pack kernel's ptxas report."""
import os
import random
import re
import shutil
import subprocess
import tempfile

import pytest
import torch

from tests.test_kv_fork_cpu import _HostCache
from vima_b200.nn.xattn_gpt import SwappedEpisode


class _SwapCache(_HostCache):
    """_HostCache with the device side of swapping replaced: a swapped episode's `kv` holds the numbers of the pages it was packed
    from and `state` its device len; an unpack records (destination page, source page) pairs."""

    precision, weights = "host", None
    kv_hi = kv_lo = [None]  # one layer, no lo pool (swap_key)

    def __init__(self, S, Lmax, kv_pool_tokens=None):
        super().__init__(S, Lmax, kv_pool_tokens)
        self.unpacked = []

    def _swap_out_data(self, slots, kv, prompt):
        return [(torch.tensor(ps, dtype=torch.int64), torch.zeros(0, dtype=torch.uint8), self.len[b:b + 1].clone())
                for b, ps in zip(slots, kv)]

    def _swap_in_data(self, slots, episodes, kv, prompt):
        for b, ep, ps in zip(slots, episodes, kv):
            assert len(ps) == ep.kv_pages == ep.kv.numel()
            self.unpacked += list(zip(ps, ep.kv.tolist()))
            self.len[b], self.active[b], self.has_action[b] = int(ep.state[0]), 1, int(ep.has_action_host)

    def swap_out_(self, slots):
        return self.swap_out(self.check_swap_out(slots))

    def swap_in_(self, slots, eps):
        self.swap_in(*self.check_swap_in(slots, eps))

    def snapshot(self):
        return (self.pages.state(), self.table.tolist(), list(self.len_host), list(self.has_action_host), list(self.active_host),
                self.len.tolist(), self.active.tolist(), len(self.unpacked))


def test_swap_out_of_a_forked_slot_gives_back_only_its_own_pages():
    c = _SwapCache(S=4, Lmax=320)
    c.admit([0], prefix=130)  # three pages
    c.fork_([0], [1])
    shared = list(c.pages.owned[0])
    free = c.kv_pages_free
    assert c.kv_pages_freed_by([0]) == 0 and c.kv_pages_freed_by([0, 1]) == 3
    (ep,) = c.swap_out_([0])
    assert c.kv_pages_free == free and c.pages.owned[1] == shared and [c.pages.refs[p] for p in shared] == [1, 1, 1]
    assert ep.kv.tolist() == shared and ep.kv_pages == 3 and ep.len_host == 130
    assert not c.active_host[0] and c.active[0] == 0 and not c.pages.owned[0] and not c.table[0].any()
    c.check_invariants()
    # after a step inside the shared second page, slot 2 holds a private copy of it (and a lookahead page): those come back
    c.admit([2], prefix=100)
    c.fork_([2], [3])
    c.step(5)
    own2 = list(c.pages.owned[2])
    assert c.kv_pages_freed_by([2]) == len(own2) - 1  # the first page stays with slot 3
    free = c.kv_pages_free
    (ep2,) = c.swap_out_([2])
    assert c.kv_pages_free == free + len(own2) - 1 and ep2.kv.tolist() == own2[:c.pages.pages_for(105)]
    c.check_invariants()


def test_swap_in_takes_private_pages_and_rebuilds_the_table_row():
    c = _SwapCache(S=4, Lmax=320)
    c.admit([0], prefix=100)
    c.step(10)  # len 110, columns [0, 111) reserved: two pages
    (ep,) = c.swap_out_([0])
    assert ep.kv_pages == 2 and ep.len_host == 110 and ep.has_action_host
    c.admit([1], prefix=200)  # takes (some of) the pages slot 0 gave back
    free = c.kv_pages_free
    c.swap_in_([3], [ep])
    own = c.pages.owned[3]
    assert len(own) == 2 and c.kv_pages_free == free - 2 and all(c.pages.refs[p] == 1 for p in own)
    assert list(c.table[3, :2]) == own and not c.table[3, 2:].any()
    assert c.unpacked == list(zip(own, ep.kv.tolist()))
    assert c.len_host[3] == 110 and c.has_action_host[3] and c.active_host[3] and c.len[3] == 110
    c.check_invariants()
    c.step(10)  # the resumed slot takes its next page like any other
    c.check_invariants()


def test_swap_in_over_a_live_slot_replaces_it_and_counts_its_pages():
    c = _SwapCache(S=3, Lmax=256, kv_pool_tokens=4 * 64)
    c.admit([0], prefix=100)
    (ep,) = c.swap_out_([0])
    c.admit([1], prefix=190)  # three pages; one is left
    with pytest.raises(ValueError, match="need 2 K/V pages, 1 are free"):
        c.swap_in_([2], [ep])
    c.swap_in_([1], [ep])  # slot 1 gives its three pages back first
    assert c.len_host[1] == 100 and len(c.pages.owned[1]) == 2 and c.kv_pages_free == 2
    c.check_invariants()


def test_refusals_touch_nothing():
    c = _SwapCache(S=4, Lmax=256, kv_pool_tokens=6 * 64)
    c.admit([0, 1], prefix=70)
    eps = c.swap_out_([1])
    c.admit([1], prefix=70)
    other = _SwapCache(S=4, Lmax=320)
    other.admit([0], prefix=10)
    foreign = other.swap_out_([0])[0]  # another Lmax
    alien = SwappedEpisode(kv=eps[0].kv, prompt=eps[0].prompt, state=eps[0].state, kv_pages=2, prompt_pages=0, len_host=70,
                           has_action_host=False, key=eps[0].key, weights=object())  # K/V of some other weights
    snap = c.snapshot()
    for slots in ([2], [4], [-1], [0, 0]):
        with pytest.raises(ValueError, match="swap_out|slots"):
            c.swap_out_(slots)
        assert c.snapshot() == snap
    for slots, e in (([2, 3], eps), ([2], eps * 2), ([4], eps), ([2, 2], eps * 2), ([2], [foreign]), ([2], ["x"]), ([2], [alien]),
                     ([2, 3], eps * 2)):  # the last: 4 pages needed, 2 free
        with pytest.raises(ValueError, match="swap_in|slots"):
            c.swap_in_(slots, e)
        assert c.snapshot() == snap


def test_an_episode_can_be_swapped_in_twice():
    c = _SwapCache(S=4, Lmax=256)
    c.admit([0], prefix=100)
    c.step(3)
    (ep,) = c.swap_out_([0])
    c.swap_in_([1, 2], [ep, ep])
    assert not set(c.pages.owned[1]) & set(c.pages.owned[2]) and c.len_host[1] == c.len_host[2] == ep.len_host
    c.swap_in_([3], [ep])
    assert len({p for b in (1, 2, 3) for p in c.pages.owned[b]}) == 3 * ep.kv_pages
    c.check_invariants()


@pytest.mark.parametrize("seed", range(8))
def test_random_schedules_keep_the_invariants(seed):
    rng = random.Random(seed)
    S, Q = 6, rng.choice([3, 16, 31, 63, 64])
    c = _SwapCache(S=S, Lmax=512, kv_pool_tokens=rng.choice([None, 40 * 64, 16 * 64]))
    rng.shuffle(c.pages.free)
    parked = []
    counts = {"swap_out": 0, "swap_in": 0}
    for _ in range(160):
        op = rng.random()
        active = [b for b in range(S) if c.active_host[b]]
        snap = c.snapshot()
        try:
            if op < 0.15:
                c.admit(rng.sample(range(S), rng.randint(1, 2)), prefix=rng.choice([0, 0, 40, 64, 100]))
            elif op < 0.3 and active:
                dst = rng.sample(range(S), rng.randint(1, 2))
                src = [rng.choice(active) for _ in dst]
                if not set(src) & set(dst):
                    c.fork_(src, dst)
            elif op < 0.38 and active:
                c.release(rng.sample(active, 1))
            elif op < 0.55 and active:
                slots = rng.sample(active, rng.randint(1, min(2, len(active))))
                want = c.kv_pages_freed_by(slots)
                free = c.kv_pages_free
                eps = c.swap_out_(slots)
                assert c.kv_pages_free == free + want
                assert all(e.kv_pages == c.pages.pages_for(e.len_host) for e in eps)
                parked += eps
                counts["swap_out"] += 1
            elif op < 0.7 and parked:
                slots = rng.sample(range(S), rng.randint(1, 2))
                eps = [rng.choice(parked) for _ in slots]
                try:
                    c.swap_in_(slots, eps)
                except ValueError:
                    assert sum(e.kv_pages for e in eps) > c.kv_pages_free + c.pages.freed_by(slots)
                    assert c.snapshot() == snap
                    raise
                assert [c.len_host[b] for b in slots] == [e.len_host for e in eps]
                assert all(len(c.pages.owned[b]) == e.kv_pages for b, e in zip(slots, eps))
                counts["swap_in"] += 1
                if rng.random() < 0.5:
                    parked.remove(eps[0])  # others stay: an episode can be resumed again
            else:
                if any(c.active_host[b] and c.len_host[b] + Q + 1 > c.Lmax for b in range(S)):
                    c.release([b for b in range(S) if c.active_host[b] and c.len_host[b] + Q + 1 > c.Lmax])
                    snap = c.snapshot()
                c.step(Q)
        except ValueError as e:
            assert "pages" in str(e)
            assert c.snapshot() == snap
        c.check_invariants()
    assert counts["swap_out"] and counts["swap_in"]
    c.release(list(range(S)))
    assert sorted(c.pages.free) == list(range(1, c.pages.n_pages)) and not any(c.pages.refs)


def test_pack_kernel_ptxas():
    """slots.cu as vima_b200/build.py compiles it, plus -Xptxas -v: the block pack kernel has no spill."""
    from vima_b200 import build as vbuild

    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        pytest.skip("nvcc not found")
    tmp = tempfile.mkdtemp(prefix="vima_ptxas_pack_")
    try:
        r = subprocess.run([nvcc, *vbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(vbuild.CSRC, "slots.cu"), "-o",
                            os.path.join(tmp, "s.o")], capture_output=True, text=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    assert r.returncode == 0, r.stderr[-4000:]
    fns = re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    pack = [f for f in fns if "kv_pack_blocks_kernel" in f[0]]
    assert len(pack) == 1 and pack[0][1:] == ("0", "0"), fns
