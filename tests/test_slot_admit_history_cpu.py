"""CPU: slot episodes admitted mid-way from a recorded history, on the paged K/V cache's host side -- each destination takes
ceil(len/64) private pages, pages it shares with a fork stay with the fork, the host mirrors follow the history, refusals leave
allocator, table and mirrors as they were, and seeded random admit / fork / step / release / swap / admit_history schedules keep
the allocator's invariants.  The cache runs on the host-only stand-in of test_kv_fork_cpu; plus the new kernels' ptxas report and
the policy-side argument checks that run before any device work."""
import os
import random
import re
import shutil
import subprocess
import tempfile

import pytest
import torch

from tests.test_kv_swap_cpu import _SwapCache
from vima_b200.policy.vima_policy import history_cols, history_steps


class _HistCache(_SwapCache):
    def admit_history_(self, slots, lens, has_action):
        """What admit_history does on the host, plus the device state its kernel writes."""
        self.check_admit_history(slots, lens)
        self.reserve_history(slots, lens, has_action)
        for b, c, a in zip(slots, lens, has_action):
            self.len[b], self.active[b], self.has_action[b] = c, 1, int(a)


def test_each_destination_takes_its_own_pages():
    c = _HistCache(S=4, Lmax=512)
    free = c.kv_pages_free
    c.admit_history_([2, 0, 3], [0, 130, 64], [False, True, True])
    assert [len(c.pages.owned[b]) for b in range(4)] == [3, 0, 0, 1]
    assert c.kv_pages_free == free - 4
    assert c.len_host == [130, 0, 0, 64] and c.has_action_host == [True, False, False, True]
    assert c.active_host == [True, False, True, True]
    assert all(c.pages.refs[p] == 1 for b in range(4) for p in c.pages.owned[b])
    c.check_invariants()
    c.step(5)  # columns [130, 136) inside slot 0's third page, [64, 70) a new page for slot 3, [0, 6) a first page for slot 2
    assert [len(c.pages.owned[b]) for b in range(4)] == [3, 0, 1, 2]
    c.check_invariants()


def test_pages_shared_with_a_fork_stay_with_the_fork():
    c = _HistCache(S=4, Lmax=320, kv_pool_tokens=5 * 64)
    c.admit([0], prefix=130)  # three pages
    c.fork_([0], [1])
    shared = list(c.pages.owned[0])
    assert c.kv_pages_free == 2
    # slot 0 gives back nothing (slot 1 holds its pages): three new pages do not fit, two do
    with pytest.raises(ValueError, match="need 3 K/V pages, 2 are free"):
        c.admit_history_([0], [129], [True])
    c.admit_history_([0], [128], [True])
    assert c.pages.owned[1] == shared and [c.pages.refs[p] for p in shared] == [1, 1, 1]
    assert not set(c.pages.owned[0]) & set(shared) and c.kv_pages_free == 0
    c.check_invariants()
    # over both sharers: their three pages come back
    c.admit_history_([1, 0], [190, 0], [True, False])
    assert len(c.pages.owned[1]) == 3 and c.pages.owned[0] == [] and c.kv_pages_free == 2
    c.check_invariants()


def test_refusals_touch_nothing():
    c = _HistCache(S=4, Lmax=256, kv_pool_tokens=6 * 64)
    c.admit([0, 1], prefix=70)
    c.step(3)
    snap = c.snapshot()
    for slots, lens in (([2, 2], [10, 10]), ([4], [10]), ([-1], [10]), ([2], [257]), ([2], [-1]), ([2, 3], [200, 200])):
        with pytest.raises(ValueError, match="slots|admit_history"):
            c.admit_history_(c.slot_index(slots), lens, [True] * len(lens))
        assert c.snapshot() == snap
    c.admit_history_([0, 1, 2], [64, 64, 256], [True, True, True])  # exactly the pool, counting slots 0 and 1's pages
    assert c.kv_pages_free == 0
    c.check_invariants()


def test_history_geometry_and_argument_checks():
    assert [history_cols(k, 4) for k in range(4)] == [0, 4, 9, 14]
    assert history_cols(3, 1) == 5

    class C:
        E = 8

    s = [0, 3]
    obs, msk, act = torch.zeros(5, 2, 4, 8), torch.ones(5, 2, 4, dtype=torch.bool), torch.zeros(5, 2, 8)
    assert history_steps(C, s, obs, msk, act, [0, 5]) == ([0, 5], 5, 4)
    assert history_steps(C, s, obs, None, act, torch.tensor([2, 1])) == ([2, 1], 5, 4)
    for args in ((obs, msk, act, [0, 6]), (obs, msk, act, [-1, 0]), (obs, msk, act, [1]), (obs[:, :1], msk, act, [1, 1]),
                 (obs, msk[:, :, :3], act, [1, 1]), (obs, msk, act[:4], [1, 1]), (obs[..., :4], msk, act, [1, 1])):
        with pytest.raises(ValueError, match="admit_history"):
            history_steps(C, s, *args)
    meta = torch.tensor([1, 1], device="meta")  # any non-host tensor: reading it would synchronise
    with pytest.raises(TypeError, match="host ints"):
        history_steps(C, s, obs, msk, act, meta)


@pytest.mark.parametrize("seed", range(8))
def test_random_schedules_keep_the_invariants(seed):
    rng = random.Random(100 + seed)
    S, Q = 6, rng.choice([3, 16, 31, 63, 64])
    c = _HistCache(S=S, Lmax=512, kv_pool_tokens=rng.choice([None, 40 * 64, 16 * 64]))
    rng.shuffle(c.pages.free)
    parked = []
    count = 0
    for _ in range(200):
        op = rng.random()
        active = [b for b in range(S) if c.active_host[b]]
        snap = c.snapshot()
        try:
            if op < 0.1:
                c.admit(rng.sample(range(S), rng.randint(1, 2)), prefix=rng.choice([0, 0, 40, 64, 100]))
            elif op < 0.22 and active:
                dst = rng.sample(range(S), rng.randint(1, 2))
                src = [rng.choice(active) for _ in dst]
                if not set(src) & set(dst):
                    c.fork_(src, dst)
            elif op < 0.3 and active:
                c.release(rng.sample(active, 1))
            elif op < 0.38 and active:
                parked += c.swap_out_(rng.sample(active, 1))
            elif op < 0.44 and parked:
                c.swap_in_(rng.sample(range(S), 1), [parked.pop()])
            elif op < 0.62:
                slots = rng.sample(range(S), rng.randint(1, 3))
                k = [rng.randint(0, 12) for _ in slots]
                prefix = rng.choice([0, 0, 41])
                lens = [prefix + history_cols(x, Q) for x in k]
                need = sum(c.pages.pages_for(x) for x in lens)
                room = c.kv_pages_free + c.pages.freed_by(slots)
                try:
                    c.admit_history_(slots, lens, [x > 0 for x in k])
                except ValueError:
                    assert need > room or max(lens) > c.Lmax
                    assert c.snapshot() == snap
                    raise
                assert c.kv_pages_free == room - need
                assert [len(c.pages.owned[b]) for b in slots] == [c.pages.pages_for(x) for x in lens]
                assert [c.len_host[b] for b in slots] == lens and all(c.pages.refs[p] == 1 for b in slots for p in c.pages.owned[b])
                count += 1
            else:
                full = [b for b in range(S) if c.active_host[b] and c.len_host[b] + Q + 1 > c.Lmax]
                if full:
                    c.release(full)
                    snap = c.snapshot()
                c.step(Q)
        except ValueError as e:
            assert "pages" in str(e) or "max_tokens" in str(e)
            assert c.snapshot() == snap
        c.check_invariants()
    assert count
    c.release(list(range(S)))
    assert sorted(c.pages.free) == list(range(1, c.pages.n_pages)) and not any(c.pages.refs)


def test_history_kernels_ptxas():
    """slots.cu as vima_b200/build.py compiles it, plus -Xptxas -v: the history assembly and admission kernels have no spill."""
    from vima_b200 import build as vbuild

    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        pytest.skip("nvcc not found")
    tmp = tempfile.mkdtemp(prefix="vima_ptxas_hist_")
    try:
        r = subprocess.run([nvcc, *vbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(vbuild.CSRC, "slots.cu"), "-o",
                            os.path.join(tmp, "s.o")], capture_output=True, text=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    assert r.returncode == 0, r.stderr[-4000:]
    fns = re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    hist = [f for f in fns if any(k in f[0] for k in ("slot_history_mask_kernel", "slot_history_tokens_kernel", "slot_admit_history_kernel"))]
    assert len(hist) == 3 and all(f[1:] == ("0", "0") for f in hist), fns
