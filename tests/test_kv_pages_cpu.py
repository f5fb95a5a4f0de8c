"""CPU: the paged slot K/V cache's host side -- the page allocator (KVPagePool), the step / admission page rules of
SlotDecodeCache (exercised on a host-only stand-in: no device state), the slot_decode_bench schedule's page counts, and the
vima_attn_desc v6 tail of the C ABI."""
import ctypes
import os
import random
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from vima_b200 import _C
from vima_b200.nn.xattn_gpt import KVPagePool, SlotDecodeCache

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _HostCache(SlotDecodeCache):
    """SlotDecodeCache's host bookkeeping without device tensors: the table pushes are recorded instead of copied."""

    def __init__(self, S, Lmax, kv_pool_tokens=None):
        page_ld = KVPagePool.pages_for(Lmax)
        n_use = S * page_ld if kv_pool_tokens is None else KVPagePool.pages_for(kv_pool_tokens)
        self.S, self.Lmax, self.E = S, Lmax, 8
        self.pages = KVPagePool(S, page_ld, n_use + 1)
        self.table = np.zeros((S, page_ld), np.int32)
        self.len_host, self.has_action_host, self.active_host = [0] * S, [False] * S, [False] * S

    def _push_pages(self, upd):
        for i, pg in upd:
            self.table.reshape(-1)[i] = pg

    def check_precision(self, p):
        pass

    def admit(self, slots, prefix=0):
        """What the policies' admit does on the host: check_prefix (decoder-only), then free / reserve the slots' pages."""
        if prefix:
            self.check_prefix(slots, prefix)
        self.free_slots(slots, prefix)
        for b in slots:
            self.len_host[b], self.has_action_host[b], self.active_host[b] = prefix, False, True

    def release(self, slots):
        self.free_slots(slots)
        for b in slots:
            self.active_host[b] = False

    def step(self, Q):
        self.check_step(self.S, Q, self.E, None)
        self.reserve_step(Q)
        self.advance_host(Q)

    def table_matches(self):
        want = np.zeros_like(self.table)
        for b, own in enumerate(self.pages.owned):
            want[b, :len(own)] = own
        return np.array_equal(want, self.table)


def test_step_pages_first_and_later_steps():
    c = _HostCache(S=2, Lmax=300)
    assert c.kv_pages_total == 2 * 5 and c.kv_pages_free == 10
    c.admit([0])
    assert c.kv_pages_needed(5) == 1  # first step: Q = 5 columns + the dummy at [0, 6)
    assert c.kv_pages_needed(63) == 1 and c.kv_pages_needed(64) == 2  # 64 columns fill one page, 65 take two
    c.step(5)
    assert c.len_host[0] == 5 and len(c.pages.owned[0]) == 1
    # later steps write action + Q obs = Q + 1 columns at [len, len + Q + 1)
    # (new pages: the slot owns one already)
    assert c.kv_pages_needed(58) == 0 and c.kv_pages_needed(59) == 1  # 5 + 58 + 1 = 64 fits one page, 5 + 59 + 1 crosses
    for _ in range(9):
        c.step(5)
    assert c.len_host[0] == 59 and len(c.pages.owned[0]) == 1  # the last step's columns [0, 53 + 6)
    c.step(5)
    assert c.len_host[0] == 65 and len(c.pages.owned[0]) == 2  # [0, 59 + 6) crosses into the second page
    assert c.table_matches()


def test_page_boundary_crossings():
    c = _HostCache(S=1, Lmax=640)
    c.admit([0])
    owned = []
    while c.len_host[0] + 8 <= 640:
        before = c.len_host[0]
        c.step(7)
        owned.append(len(c.pages.owned[0]))
        assert owned[-1] == -(-(before + 8) // 64)  # the step's columns [0, len + Q + 1)
    assert owned == sorted(owned) and owned[-1] == 10 and len(set(owned)) == 10
    assert c.table_matches()


def test_decoder_only_prefix_pages():
    c = _HostCache(S=3, Lmax=512)
    c.admit([0, 2], prefix=128)  # 127 prompt tokens + separator: exactly two pages
    assert [len(o) for o in c.pages.owned] == [2, 0, 2]
    c.admit([1], prefix=129)  # one more column: a third page
    assert len(c.pages.owned[1]) == 3
    assert c.kv_pages_needed(16) == 1 + 0 + 1  # 128 + 17 columns cross into a third page; 129 + 17 stay in three
    assert c.table_matches()


def test_refusals_leave_free_list_and_table_untouched():
    c = _HostCache(S=3, Lmax=256, kv_pool_tokens=4 * 64)
    c.admit([0, 1], prefix=100)  # two pages each: the pool is full
    assert c.kv_pages_free == 0
    st, table = c.pages.state(), c.table.copy()
    with pytest.raises(ValueError, match="2 more K/V pages, 0 of 4"):
        c.step(40)  # 100 + 41 columns: a third page for each
    with pytest.raises(ValueError, match="needs 2 K/V pages, 0 are free"):
        c.admit([2], prefix=100)
    assert c.pages.state() == st and np.array_equal(c.table, table) and c.len_host == [100, 100, 0]
    c.admit([1], prefix=100)  # re-admission over a live slot reuses its own pages
    assert c.pages.state()[0] == [] and sorted(c.pages.owned[1]) == sorted(st[1][1])
    c.release([1])
    assert c.kv_pages_free == 2 and c.table_matches()
    c.step(20)  # 100 + 21 columns: slot 0 keeps its two pages
    assert c.kv_pages_free == 2 and c.len_host[0] == 120
    c.admit([2], prefix=100)
    assert c.kv_pages_free == 0 and c.table_matches()
    st, table = c.pages.state(), c.table.copy()
    with pytest.raises(ValueError, match="2 more K/V pages, 0 of 4"):
        c.step(40)  # slots 0 and 2 both cross into a third page
    assert c.pages.state() == st and np.array_equal(c.table, table)
    c.release([2])
    c.step(40)  # the same step goes through once a slot gave its pages back
    assert len(c.pages.owned[0]) == 3 and c.table_matches()


def test_release_and_readmission_recycle_pages():
    rng = random.Random(5)
    c = _HostCache(S=4, Lmax=200)
    rng.shuffle(c.pages.free)
    seen = set()
    for ep in range(12):
        b = ep % 4
        c.admit([b])  # over a live slot when its previous episode was not released
        for _ in range(rng.randint(1, 20)):
            if max(c.len_host[x] for x in range(4) if c.active_host[x]) + 8 > 200:
                break
            c.step(7)
        seen |= set(c.pages.owned[b])
        if ep % 2:
            c.release([b])
        assert c.table_matches() and c.kv_pages_free + sum(map(len, c.pages.owned)) == c.kv_pages_total
    c.release([0, 1, 2, 3])
    assert sorted(c.pages.free) == list(range(1, c.pages.n_pages)) and not c.table.any()
    assert seen <= set(range(1, c.pages.n_pages))


def test_state_restore():
    c = _HostCache(S=2, Lmax=128)
    c.admit([0, 1])
    c.step(3)
    st = c.pages.state()
    c.step(60)
    c.release([1])
    assert c.pages.state() != st
    c.pages.restore(st)
    assert c.pages.state() == st
    st[0].append(99)  # the snapshot is a copy
    assert c.pages.state() != st


def test_pool_size_is_checked():
    with pytest.raises(ValueError):
        KVPagePool(1, 1, 1)  # the zero page alone
    c = _HostCache(S=2, Lmax=65)
    assert c.pages.page_ld == 2 and c.kv_pages_total == 4


@pytest.mark.parametrize("case,peak,mean_share", [("cfg3", 1091, 0.34), ("cfg5", 1639, 0.58), ("gato1024", 2473, 0.42)])
def test_slot_decode_bench_schedule_peak_pages(case, peak, mean_share):
    """The page counts of tools/slot_decode_bench.py's seeded schedules (seed 0, 1024 episodes, 256 slots) that DESIGN.md 7 quotes."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        from slot_decode_bench import pages_per_tick
    finally:
        sys.path.pop(0)
    Q, steps, prefix = {"cfg3": (32, 15, 0), "cfg5": (16, 15, 257), "gato1024": (16, 45, 257)}[case]
    lengths = np.random.default_rng(0).integers(1, steps + 1, size=1024).tolist()
    pt = pages_per_tick(lengths, 256, Q, prefix)
    full = 256 * -(-(prefix + steps * (Q + 1)) // 64)
    assert max(pt) == peak and round(sum(pt) / len(pt) / full, 2) == mean_share
    # the same schedule through the allocator: pages in use after each step's reservation
    c = _HostCache(S=256, Lmax=prefix + steps * (Q + 1), kv_pool_tokens=peak * 64)
    queue, remaining, used = list(lengths), [0] * 256, []
    while True:
        take = [b for b in range(256) if not remaining[b]][:len(queue)]
        for b in take:
            remaining[b] = queue.pop(0)
        if take:
            c.admit(take, prefix)
        idle = [b for b in range(256) if not remaining[b] and c.active_host[b]]
        if idle:
            c.release(idle)
        if not any(remaining):
            break
        c.step(Q)
        used.append(c.kv_pages_total - c.kv_pages_free)
        remaining = [max(r - 1, 0) for r in remaining]
    assert used == pt


def test_attn_desc_v6_layout_matches_header():
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = r"""
#include <stdio.h>
#include <stddef.h>
#include "vima_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu\n", offsetof(vima_attn_desc, q_pos), offsetof(vima_attn_desc, kv_pages),
         offsetof(vima_attn_desc, kv_page_ld), offsetof(vima_attn_desc, kv_pool_pages), (size_t)VIMA_ATTN_DESC_V5_SIZE,
         sizeof(vima_attn_desc));
  return VIMA_KV_PAGE_TOKENS == 64 ? 0 : 1;
}
"""
    tmp = tempfile.mkdtemp(prefix="vima_abi_")
    try:
        c_file, exe = os.path.join(tmp, "t.c"), os.path.join(tmp, "t")
        open(c_file, "w").write(src)
        r = subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), c_file, "-o", exe],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr  # the header compiles as C
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    q_pos, kv_pages, page_ld, pool_pages, v5, v6 = map(int, out)
    A = _C.AttnDesc
    assert (A.q_pos.offset, A.kv_pages.offset, A.kv_page_ld.offset, A.kv_pool_pages.offset) == (q_pos, kv_pages, page_ld, pool_pages)
    assert v5 == kv_pages and v6 == ctypes.sizeof(A) and _C.KV_PAGE_TOKENS == 64


def test_attn_desc_sizes_v4_to_v6_are_accepted():
    """load_desc takes any struct_size in [V4, sizeof]: the v4 and v5 sizes sit inside, with the v6 tail read as zero (unpaged)."""
    A = _C.AttnDesc
    v4, v5 = A.q_pos.offset, A.kv_pages.offset
    assert v4 < v5 < ctypes.sizeof(A)
    src = open(os.path.join(ROOT, "vima_b200", "csrc", "api.cu")).read()
    assert "load_desc(c, d_in, &d_local, VIMA_ATTN_DESC_V4_SIZE" in src
    import __graft_entry__

    __graft_entry__.build()
    lib = _C.load_library()
    assert lib.vima_sizeof_attn_desc() == ctypes.sizeof(A)
    for name in ("vima_slot_kv_append_paged", "vima_slot_kv_scatter_paged"):
        assert hasattr(lib, name) and name in _C.EXPORTS


def test_paged_attention_kernel_ptxas():
    """attention_tc_paged.cu as vima_b200/build.py compiles it, plus -Xptxas -v: the paged decoder kernel (f16 and bf16) has no
    wgmma serialisation warning and no spill, like the unpaged one (tests/test_wgmma_ptxas_cpu.py)."""
    import re

    from vima_b200 import build as vbuild

    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        pytest.skip("nvcc not found")
    tmp = tempfile.mkdtemp(prefix="vima_ptxas_paged_")
    try:
        r = subprocess.run([nvcc, *vbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(vbuild.CSRC, "attention_tc_paged.cu"), "-o",
                            os.path.join(tmp, "a.o")], capture_output=True, text=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    assert r.returncode == 0, r.stderr[-4000:]
    assert not re.search(r"C75[12]0|wgmma\.mma_async instructions are serialized", r.stderr)
    fns = re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    paged = [f for f in fns if "attention_tc_paged_kernel" in f[0]]
    assert len(paged) == 2 and all(f[1:] == ("0", "0") for f in paged), fns
