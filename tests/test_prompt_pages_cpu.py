"""CPU: the paged prompt K/V of the slot cache's cross-attention.  The v7 descriptor tail (kv_len) compiled from the header as C
against the ctypes mirror, and older descriptor sizes still accepted; the prompt page pool's host side -- admission, release and
fork through a host-only stand-in of SlotDecodeCache over seeded random schedules, against the allocator's invariants; and what
ptxas makes of every attention translation unit (no new spill, no wgmma serialisation, the unpaged kernels' register counts)."""
import ctypes
import os
import random
import re
import shutil
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

from vima_b200 import _C
from vima_b200.nn.xattn_gpt import KVPagePool, SlotDecodeCache

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------- C ABI
def test_attn_desc_v7_layout_matches_header():
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = r"""
#include <stdio.h>
#include <stddef.h>
#include "vima_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu\n", offsetof(vima_attn_desc, kv_pool_pages), offsetof(vima_attn_desc, kv_len),
         (size_t)VIMA_ATTN_DESC_V6_SIZE, (size_t)VIMA_ATTN_DESC_V7_SIZE, sizeof(vima_attn_desc));
  return 0;
}
"""
    tmp = tempfile.mkdtemp(prefix="vima_abi7_")
    try:
        c_file, exe = os.path.join(tmp, "t.c"), os.path.join(tmp, "t")
        open(c_file, "w").write(src)
        r = subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), c_file, "-o", exe],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    pool_pages, kv_len, v6, v7, size = map(int, out)
    A = _C.AttnDesc
    assert (A.kv_pool_pages.offset, A.kv_len.offset) == (pool_pages, kv_len)
    assert v6 == kv_len > pool_pages and v7 == size == ctypes.sizeof(A)


def test_attn_desc_sizes_v4_to_v7_are_accepted():
    """load_desc takes any struct_size in [V4, sizeof] and zeroes the rest: a v4, v5 or v6 caller's kv_len reads as NULL."""
    A = _C.AttnDesc
    v4, v5, v6 = A.q_pos.offset, A.kv_pages.offset, A.kv_len.offset
    assert v4 < v5 < v6 < ctypes.sizeof(A)
    src = open(os.path.join(ROOT, "vima_b200", "csrc", "api.cu")).read()
    assert "load_desc(c, d_in, &d_local, VIMA_ATTN_DESC_V4_SIZE" in src
    assert re.search(r"memset\(out, 0, sizeof\(D\)\);\s*memcpy\(out, in, sz\);", src)
    assert "p.kv_len = d->kv_len;" in src
    import __graft_entry__

    __graft_entry__.build()
    lib = _C.load_library()
    assert lib.vima_sizeof_attn_desc() == ctypes.sizeof(A)


# ------------------------------------------------------------------------------------------------- prompt page pool
class _HostCache(SlotDecodeCache):
    """SlotDecodeCache of a cross-attention model without a GPU: history and prompt pools' host mirrors, CPU state vectors, table
    pushes applied to numpy tables, prompt-page zeroing recorded."""

    def __init__(self, S, Lp_cap, prompt_pool_tokens=None, Lmax=128):
        page_ld, p_ld = KVPagePool.pages_for(Lmax), KVPagePool.pages_for(Lp_cap)
        n_prompt = S * p_ld if prompt_pool_tokens is None else KVPagePool.pages_for(prompt_pool_tokens)
        self.S, self.Lmax, self.E, self.Lp_cap = S, Lmax, 8, Lp_cap
        self.pages = KVPagePool(S, page_ld, S * page_ld + 1)
        self.prompt_pages = KVPagePool(S, p_ld, n_prompt + 1)
        self.page_table = np.zeros((S, page_ld), np.int32)
        self.prompt_page_table = np.zeros((S, p_ld), np.int32)
        z = lambda: torch.zeros(S, dtype=torch.int32)  # noqa: E731
        self.len, self.n_valid, self.has_action, self.active, self.prompt_len = z(), z(), z(), z(), z()
        self.action_token = torch.zeros(S, 8)
        self.mask = torch.zeros(S, Lmax, dtype=torch.uint8)
        self.prompt_mask = torch.zeros(S, Lp_cap, dtype=torch.uint8)
        self.len_host, self.has_action_host, self.active_host = [0] * S, [False] * S, [False] * S
        self.zeroed = []

    def device_ints(self, values):
        return torch.tensor(values, dtype=torch.int64)

    def _push_pages(self, upd, table=None):
        t = self.page_table if table is None else table
        for i, pg in upd:
            t.reshape(-1)[i] = pg

    def _zero_prompt_pages(self, pages):
        self.zeroed += pages

    def admit(self, slots, Lp):
        """The page side of XAttnGPT.admit_prompts and the state it sets."""
        self.check_prefix(slots, 0, Lp)
        self.free_slots(slots, prompt_cols=Lp)
        for b in slots:
            self.prompt_len[b], self.active[b], self.len[b] = Lp, 1, 0
            self.len_host[b], self.has_action_host[b], self.active_host[b] = 0, False, True

    def release(self, slots):
        self.free_slots(slots)
        for b in slots:
            self.active_host[b] = False
            self.active[b] = 0

    def fork_(self, src, dst):
        s, d = self.check_fork(src, dst)
        self.fork(s, d)

    def snapshot(self):
        P = self.prompt_pages
        return (P.state(), self.prompt_page_table.copy(), self.pages.state(), self.page_table.copy(), self.prompt_len.clone(),
                list(self.active_host), list(self.zeroed))

    def check_invariants(self):
        P = self.prompt_pages
        held = {}
        for own in P.owned:
            for pg in own:
                held[pg] = held.get(pg, 0) + 1
        assert 0 not in held and P.refs[0] == 0
        assert all(P.refs[pg] == held.get(pg, 0) for pg in range(P.n_pages))  # counts = holders
        assert all((P.refs[pg] == 0) == (pg in P.free) for pg in range(1, P.n_pages))  # free iff unreferenced
        assert sorted(P.free + list(held)) == list(range(1, P.n_pages)) and len(P.free) == self.prompt_pages_free
        want = np.zeros_like(self.prompt_page_table)
        for b, own in enumerate(P.owned):
            want[b, :len(own)] = own
        assert np.array_equal(want, self.prompt_page_table)  # table rows = owned lists; a freed slot's row is zero
        for b in range(self.S):
            if self.active_host[b]:
                assert len(P.owned[b]) == P.pages_for(int(self.prompt_len[b]))
            else:
                assert not P.owned[b]
        assert 0 not in self.zeroed


def test_prompt_pool_sizes_and_refusal_at_open():
    c = _HostCache(S=4, Lp_cap=150)
    assert c.prompt_pages_total == 4 * 3 and c.prompt_pages_free == 12
    assert _HostCache(S=4, Lp_cap=150, prompt_pool_tokens=65).prompt_pages_total == 2
    for bad in (0, 4 * 3 * 64 + 1):
        with pytest.raises(ValueError, match="prompt_pool_tokens"):
            SlotDecodeCache(S=4, Lmax=64, Lp_cap=150, E=8, n_layer=1, device="cpu", split=True, precision="f16x3", prompt_pool_tokens=bad)
    d = SlotDecodeCache(S=4, Lmax=64, Lp_cap=0, E=8, n_layer=1, device="cpu", split=True, precision="f16x3")
    assert d.prompt_pages_total == d.prompt_pages_free == 0 and d.prompt_page_table is None


def test_admission_takes_pages_and_zeroes_the_partial_last_page():
    c = _HostCache(S=4, Lp_cap=256)
    c.admit([0, 2], 65)  # two pages each; the second holds one row
    assert [len(c.prompt_pages.owned[b]) for b in range(4)] == [2, 0, 2, 0]
    assert c.zeroed == [c.prompt_pages.owned[0][1], c.prompt_pages.owned[2][1]]
    c.admit([1], 128)  # fills its pages: nothing to zero
    assert len(c.zeroed) == 2 and c.prompt_pages_free == 16 - 6
    c.admit([0], 40)  # re-admission over a live slot gives its two pages back first
    assert len(c.prompt_pages.owned[0]) == 1 and c.prompt_pages_free == 16 - 5
    c.release([1])
    assert c.prompt_pages_free == 16 - 3 and not c.prompt_page_table[1].any()
    c.check_invariants()


def test_fork_shares_prompt_pages_and_takes_none():
    c = _HostCache(S=5, Lp_cap=200)
    c.admit([0], 150)
    c.admit([3], 10)
    free, zeroed = c.prompt_pages_free, len(c.zeroed)
    c.fork_([0, 0, 0], [1, 2, 3])  # slot 3 is live: it lets go of its page first
    assert c.prompt_pages_free == free + 1 and len(c.zeroed) == zeroed
    assert c.prompt_pages.owned[1] == c.prompt_pages.owned[2] == c.prompt_pages.owned[3] == c.prompt_pages.owned[0]
    assert [c.prompt_pages.refs[pg] for pg in c.prompt_pages.owned[0]] == [4, 4, 4]
    assert c.prompt_pages_total - c.prompt_pages_free == 3  # one prompt's pages
    assert c.prompt_len.tolist() == [150, 150, 150, 150, 0]
    c.check_invariants()
    c.release([0, 1])
    assert c.prompt_pages_total - c.prompt_pages_free == 3
    c.release([2, 3])
    assert c.prompt_pages_free == c.prompt_pages_total
    c.check_invariants()


def test_admission_refusal_changes_nothing():
    c = _HostCache(S=4, Lp_cap=256, prompt_pool_tokens=5 * 64)
    c.admit([0], 256)  # four pages of five
    c.fork_([0], [1])
    st = c.snapshot()
    with pytest.raises(ValueError, match="prompt pages"):
        c.admit([2, 3], 40)  # two pages, one free
    with pytest.raises(ValueError, match="prompt pages"):
        c.admit([1], 129)  # slot 1's pages are still held by slot 0: nothing comes back
    after = c.snapshot()
    assert st[0] == after[0] and np.array_equal(st[1], after[1]) and st[2] == after[2] and np.array_equal(st[3], after[3])
    assert torch.equal(st[4], after[4]) and st[5:] == after[5:]
    c.admit([0, 1], 64)  # re-admitting both sharers gives all four pages back
    assert c.prompt_pages_free == 5 - 2
    c.check_invariants()


@pytest.mark.parametrize("seed", range(6))
def test_random_schedules_keep_the_invariants(seed):
    rng = random.Random(seed)
    S = 8
    Lp_cap = rng.choice([64, 150, 256])
    pool = rng.choice([None, 2 * KVPagePool.pages_for(Lp_cap) * 64, 11 * 64])
    c = _HostCache(S=S, Lp_cap=Lp_cap, prompt_pool_tokens=pool)
    rng.shuffle(c.prompt_pages.free)  # pages recycle in scrambled order
    refusals = 0
    for _ in range(300):
        op = rng.random()
        active = [b for b in range(S) if c.active_host[b]]
        if op < 0.4:
            slots = rng.sample(range(S), rng.randint(1, 3))
            Lp = rng.choice([1, 40, 63, 64, 65, 128, 150, Lp_cap])
            Lp = min(Lp, Lp_cap)
            need = len(slots) * KVPagePool.pages_for(Lp)
            can = need <= c.prompt_pages_free + c.prompt_pages.freed_by(slots)
            st = c.snapshot()
            if can:
                c.admit(slots, Lp)
            else:
                refusals += 1
                with pytest.raises(ValueError, match="prompt pages"):
                    c.admit(slots, Lp)
                after = c.snapshot()
                assert st[0] == after[0] and np.array_equal(st[1], after[1]) and torch.equal(st[4], after[4]) and st[5:] == after[5:]
        elif op < 0.75 and active:
            src = [rng.choice(active) for _ in range(rng.randint(1, 3))]
            others = [b for b in range(S) if b not in src]
            dst = rng.sample(others, min(len(src), len(others)))
            src = src[:len(dst)]
            free = c.prompt_pages_free
            gone = c.prompt_pages.freed_by(dst)
            c.fork_(src, dst)
            assert c.prompt_pages_free == free + gone  # a fork takes no page; live destinations give theirs back
            for a, b in zip(src, dst):
                assert c.prompt_pages.owned[b] == c.prompt_pages.owned[a] and int(c.prompt_len[b]) == int(c.prompt_len[a])
        elif active:
            c.release(rng.sample(active, rng.randint(1, len(active))))
        c.check_invariants()
    assert pool is None or refusals > 0 or seed % 2  # the small pools do refuse


# ------------------------------------------------------------------------------------------------- ptxas
ATTN_SOURCES = ["attention.cu", "attention_tc.cu", "attention_tc_paged.cu", "attention_tail.cu"]
# (registers, spill store bytes) of every attention instantiation as built by vima_b200/build.py with CUDA 12.9 before per-batch
# key counts existed; the mma.sync kernel's split head_dim-32 instantiations spilled already then
BEFORE = {
    "attention_bias_tc_kernelILi0ELb0EE": (115, 0), "attention_bias_tc_kernelILi0ELb1EE": (128, 0),
    "attention_bias_tc_kernelILi1ELb0EE": (115, 0), "attention_bias_tc_kernelILi1ELb1EE": (128, 0),
    "attention_kernelILi32ELi0ELb0EE": (127, 0), "attention_kernelILi32ELi0ELb1EE": (128, 44),
    "attention_kernelILi32ELi1ELb0EE": (127, 0), "attention_kernelILi32ELi1ELb1EE": (128, 44),
    "attention_kernelILi64ELi0ELb0EE": (170, 0), "attention_kernelILi64ELi0ELb1EE": (217, 0),
    "attention_kernelILi64ELi1ELb0EE": (170, 0), "attention_kernelILi64ELi1ELb1EE": (214, 0),
    "attention_tail_kernelILi0ELb0EE": (139, 0), "attention_tail_kernelILi0ELb1EE": (130, 0),
    "attention_tail_kernelILi1ELb0EE": (139, 0), "attention_tail_kernelILi1ELb1EE": (130, 0),
    "attention_tc_kernelILi0EE": (127, 0), "attention_tc_kernelILi1EE": (128, 0),
    "attention_tc_paged_kernelILi0EE": (128, 0), "attention_tc_paged_kernelILi1EE": (128, 0),
}
PAGED = ("attention_tc_paged_kernel", "attention_tail_kernelILi0ELb1EE", "attention_tail_kernelILi1ELb1EE")


def test_attention_ptxas_registers_and_spills():
    from vima_b200 import build as vbuild

    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        pytest.skip("nvcc not found")
    tmp = tempfile.mkdtemp(prefix="vima_ptxas_attn_")

    def one(src):
        return subprocess.run([nvcc, *vbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(vbuild.CSRC, src), "-o",
                               os.path.join(tmp, src + ".o")], capture_output=True, text=True)

    try:
        with ThreadPoolExecutor(max_workers=len(ATTN_SOURCES)) as ex:
            results = list(ex.map(one, ATTN_SOURCES))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    got = {}
    for src, r in zip(ATTN_SOURCES, results):
        assert r.returncode == 0, r.stderr[-4000:]
        assert not re.search(r"C75[12]0|wgmma\.mma_async instructions are serialized", r.stderr), src
        for m in re.finditer(r"Function properties for \S*?\d(attention_\w*?kernelI\w*?E)Ev\S*\n\s*\d+ bytes stack frame, (\d+) bytes spill "
                             r"stores, \d+ bytes spill loads\nptxas info\s*: Used (\d+) registers", r.stderr):
            got[m.group(1)] = (int(m.group(3)), int(m.group(2)))
    assert set(got) == set(BEFORE), sorted(got)
    for k, (regs, spill) in got.items():
        assert spill == BEFORE[k][1], (k, spill)  # no new spill (streaming and tail kernels: none at all)
        if not k.startswith(PAGED):
            assert regs == BEFORE[k][0], (k, regs)  # the unpaged kernels keep their register counts
