"""XAttnGPT: cross-attention to the prompt alternating with causal self-attention over the obs/action history.

Module surface and state-dict keys of /root/reference/vima/nn/seq_modeling/xattn_gpt/{xattn_gpt.py:13-177,
components.py:14-263}; the arithmetic runs on the sm_90a kernels (wgmma GEMMs with fused bias / GELU / GEGLU /
residual epilogues, fused masked attention, warp-shuffle LayerNorm).  Per layer (reference order, xattn_gpt.py:123-132):

    XAttention (pre-LN, bias-free, components.py:158-228)        Block (GPT-1 post-LN, components.py:23-37)
      q  = Wq LN(x)            k,v = Wkv (prompt + pos)             qkv = c_attn(x)
      a  = Wo attn(q,k,v) + x          [+ row sums of a]            s   = c_proj(causal_attn(qkv)) + x   [+ row sums of s]
      h  = gelu(W1 LN2(a)) * (Wg a)    [ONE GEGLU GEMM over a:      h   = gelu(c_fc LN1(s)) * (Wg LN1(s))  [one GEGLU GEMM over s,
           LN2 folded into W1, the gate reads UN-normalised a]            LN1 folded into both halves]
      x' = W2 h + a                                                 x'' = LN2(c_proj h + LN1(s))   [LN1(s) rebuilt in the epilogue]

LayerNorm folding (DESIGN.md): W (gamma (x - mean) rstd + beta) = rstd ((W gamma) x - mean rowsum(W gamma)) + W beta, so the GEMM
runs on the un-normalised rows and its epilogue applies (mean, rstd); the producing GEMM's epilogue emits the row sums.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn as nn

from .. import _C
from .. import engine as eng
from .basic import Conv1D


class _SelfAttention(nn.Module):
    """Parameter holder for HF openai `Attention` + the reference's persistent causal `bias` buffer (components.py:40-49)."""

    def __init__(self, nx: int, n_positions: int):
        super().__init__()
        self.register_buffer("bias", torch.tril(torch.ones(n_positions, n_positions)).view(1, 1, n_positions, n_positions), persistent=True)
        self.c_attn = Conv1D(3 * nx, nx)
        self.c_proj = Conv1D(nx, nx)


class _MLP(nn.Module):
    def __init__(self, nx: int, geglu: bool):
        super().__init__()
        self.c_fc = Conv1D(4 * nx, nx)
        self.c_proj = Conv1D(nx, 4 * nx)
        self.gated_layer = nn.Linear(nx, 4 * nx, bias=False) if geglu else None


class Block(nn.Module):
    def __init__(self, nx: int, n_positions: int, n_head: int, geglu: bool, eps: float = 1e-5):
        super().__init__()
        self.n_head = n_head
        self.attn = _SelfAttention(nx, n_positions)
        self.ln_1 = nn.LayerNorm(nx, eps=eps)
        self.mlp = _MLP(nx, geglu)
        self.ln_2 = nn.LayerNorm(nx, eps=eps)


def pack_block(ctx, blk: "Block", p) -> dict:
    """Packed weights of one GPT block.  ln_1 is folded into c_fc || gated_layer (both read ln_1(s), components.py:31-36); without
    GEGLU (`afn != "geglu"`, components.py:92-94) into c_fc alone."""
    ln1 = (blk.ln_1.weight.detach(), blk.ln_1.bias.detach())
    d = {
        "c_attn": eng.pack_linear(ctx, blk.attn.c_attn.weight, blk.attn.c_attn.bias, transposed=True, p=p, f8=True),
        "c_proj": eng.pack_linear(ctx, blk.attn.c_proj.weight, blk.attn.c_proj.bias, transposed=True, p=p, f8=True),
        "mlp_proj": eng.pack_linear(ctx, blk.mlp.c_proj.weight, blk.mlp.c_proj.bias, transposed=True, p=p, f8=True),
    }
    if blk.mlp.gated_layer is not None:
        d["fc_glu"] = eng.pack_glu(ctx, blk.mlp.c_fc.weight, blk.mlp.c_fc.bias, blk.mlp.gated_layer.weight, val_transposed=True,
                                   gate_transposed=False, p=p, f8=True, ln=ln1, ln_gate=True)
    else:
        d["fc"] = eng.pack_linear(ctx, blk.mlp.c_fc.weight, blk.mlp.c_fc.bias, transposed=True, p=p, f8=True, ln=ln1)
    return d


class DecodeCache:
    """Per-layer K/V cache of one batch of episodes for step-by-step decode (SURVEY.md 8(f)1).

    The reference re-runs the whole history every environment step (scripts/example.py:139-171); with the cache a step
    only pushes its Q+1 new tokens through the stack: the prompt's key/value projections are computed once, and every
    causal block appends the new tokens' keys/values to `kv[i]` ([B*Lmax, 2E] (hi, lo) pairs) and attends over the
    cached prefix (`vima_attention` with kv_batch_rows / mask_ld / q_pos0)."""

    def __init__(self, *, B: int, Lmax: int, E: int, n_layer: int, device, split: bool, precision: str = "", weights=None):
        self.B, self.Lmax, self.E, self.L = B, Lmax, E, 0
        self.precision = precision  # the operand format the K/V rows are stored in; forward_step refuses any other mode
        self.weights = weights  # engine.WeightState of the decoder at open: the cached K/V were projected with these weights
        mk = lambda: torch.zeros((B * Lmax, 2 * E), dtype=torch.int16, device=device)
        self.kv_hi = [mk() for _ in range(n_layer)]
        self.kv_lo = [mk() if split else None for _ in range(n_layer)]
        self.mask = torch.zeros((B, Lmax), dtype=torch.uint8, device=device)
        self.n_valid = torch.zeros((B,), dtype=torch.int64, device=device)  # valid tokens so far -> next position id
        self.prompt_kv = None  # per-layer projected prompt keys/values (filled by the first step)

    def append_kv(self, i: int, qkv16, L0: int, Ln: int):
        E, B = self.E, self.B
        self.kv_hi[i].view(B, self.Lmax, 2 * E)[:, L0:L0 + Ln].copy_(qkv16.hi.view(B, Ln, -1)[:, :, E:3 * E])
        if self.kv_lo[i] is not None:
            self.kv_lo[i].view(B, self.Lmax, 2 * E)[:, L0:L0 + Ln].copy_(qkv16.lo.view(B, Ln, -1)[:, :, E:3 * E])


class KVPagePool:
    """Host allocator of a paged slot K/V cache (DESIGN.md 4 and 7 (f)1): pages 1 .. n_pages-1 of KV_PAGE_TOKENS cache columns each;
    page 0 is the zero page that no slot owns.  `owned[b]` lists the pages of slot b's columns [0, 64*len(owned[b])) in column order,
    so row b of the page table is owned[b] followed by zeros.  `free` is the free list (taken from its end).  `refs[p]` counts the
    slots holding page p: a fork shares pages by reference, a page goes back to the free list when its last holder lets it go, and
    a holder that is about to write into a shared page takes a private copy first (`cow`).  Pure Python: the cache pushes the table
    entries that each call returns, as (flat index b*page_ld + k, page) pairs."""

    def __init__(self, S: int, page_ld: int, n_pages: int):
        if n_pages < 2:
            raise ValueError(f"a page pool needs the zero page and at least one more, got {n_pages} pages")
        self.S, self.page_ld, self.n_pages = S, page_ld, n_pages
        self.free = list(range(n_pages - 1, 0, -1))
        self.owned = [[] for _ in range(S)]
        self.refs = [0] * n_pages  # refs[0] stays 0: the zero page is never counted

    @staticmethod
    def pages_for(cols: int) -> int:
        return -(-cols // _C.KV_PAGE_TOKENS)

    def needed(self, b: int, cols: int) -> int:
        """New pages slot b needs so that it owns columns [0, cols)."""
        return max(0, self.pages_for(cols) - len(self.owned[b]))

    def reserve(self, b: int, cols: int) -> list:
        """Give slot b pages up to column `cols` (the caller has checked `needed` against the free list)."""
        own = self.owned[b]
        upd = []
        for _ in range(self.needed(b, cols)):
            pg = self.free.pop()
            self.refs[pg] = 1
            upd.append((b * self.page_ld + len(own), pg))
            own.append(pg)
        return upd

    def release(self, b: int) -> list:
        """Let go of slot b's pages (each returns to the free list when no other slot holds it); its table row goes back to zeros."""
        own = self.owned[b]
        upd = [(b * self.page_ld + k, 0) for k in range(len(own))]
        for pg in reversed(own):
            self.refs[pg] -= 1
            if self.refs[pg] == 0:
                self.free.append(pg)
        self.owned[b] = []
        return upd

    def fork(self, s: int, d: int, n: int) -> list:
        """Slot d (holding no pages) takes slot s's first n pages by reference; nothing is allocated."""
        own = self.owned[s][:n]
        for pg in own:
            self.refs[pg] += 1
        self.owned[d] = list(own)
        return [(d * self.page_ld + k, pg) for k, pg in enumerate(own)]

    def cow_plan(self, cols: list) -> list:
        """Which of the (slot, column) pairs, visited in the given order, must copy a shared page before writing `column`: the
        column lies inside a page (col % 64 != 0; at a page boundary the write starts a page of its own) that some later visitor
        still holds.  So the last holder in visiting order keeps the page in place.  Changes nothing (`cow` does the copies)."""
        left, out = {}, []
        for b, col in cols:
            k = col // _C.KV_PAGE_TOKENS
            if col % _C.KV_PAGE_TOKENS == 0 or k >= len(self.owned[b]):
                continue
            pg = self.owned[b][k]
            r = left.get(pg, self.refs[pg])
            if r > 1:
                left[pg] = r - 1
                out.append(b)
        return out

    def cow(self, b: int, col: int) -> tuple:
        """Give slot b a private copy of the shared page holding column `col` (after cow_plan said so and a free page was checked):
        returns (table update, (old page, new page)) -- the caller copies the old page's rows into the new one."""
        k = col // _C.KV_PAGE_TOKENS
        old, new = self.owned[b][k], self.free.pop()
        self.refs[old] -= 1
        self.refs[new] = 1
        self.owned[b][k] = new
        return (b * self.page_ld + k, new), (old, new)

    def freed_by(self, slots: list) -> int:
        """Pages that would return to the free list if every slot of `slots` let go of its pages."""
        drop = {}
        for b in slots:
            for pg in self.owned[b]:
                drop[pg] = drop.get(pg, 0) + 1
        return sum(1 for pg, n in drop.items() if self.refs[pg] == n)

    def state(self) -> tuple:
        return list(self.free), [list(o) for o in self.owned], list(self.refs)

    def restore(self, st: tuple) -> None:
        self.free, self.owned, self.refs = list(st[0]), [list(o) for o in st[1]], list(st[2])


class SwappedEpisode:
    """One slot episode parked in pinned host memory by `swap_out` (DESIGN.md 7 (f)1), to be written back by `swap_in` into a slot
    of any cache of the same policy, precision mode and shapes, as often as wanted.  `kv` holds its history pages (the `kv_pages`
    whole pages of its columns [0, len)) and `prompt` its `prompt_pages` prompt pages (cross-attention policies), both packed
    [page][buffer][64 rows][row bytes] over every layer's hi and lo pool; `state` is its record of the per-slot device state (len,
    n_valid, has_action, fed-back action token, history mask, prompt length and mask); `len_host` / `has_action_host` are the
    host mirrors.  The three are views of the pinned buffer of one swap_out call."""

    def __init__(self, *, kv, prompt, state, kv_pages: int, prompt_pages: int, len_host: int, has_action_host: bool, key: tuple, weights):
        self.kv, self.prompt, self.state = kv, prompt, state
        self.kv_pages, self.prompt_pages = kv_pages, prompt_pages
        self.len_host, self.has_action_host = len_host, has_action_host
        self.key = key  # SlotDecodeCache.swap_key() of the source cache: swap_in refuses a cache of another
        self.weights = weights  # the source cache's engine.WeightState: its K/V rows were computed with these weights

    @property
    def nbytes(self) -> int:
        """Pinned host bytes of the episode (K/V pages, prompt pages and state)."""
        return self.kv.numel() + self.prompt.numel() + self.state.numel()


class SlotDecodeCache:
    """K/V cache of `S` slots, each holding one episode at its own history length (DESIGN.md 4 and 7 (f)1).

    Self-attention K/V per layer: `kv_hi[i]` / `kv_lo[i]`, a pool of `kv_pages_total + 1` pages of 64 rows [(P+1)*64, 2E] (page 0
    is the zero page); `page_table` int32 [S, ceil(Lmax/64)] on the device maps column j of slot b to row page_table[b, j//64]*64 +
    j%64 (0 = no page: reads see zeros, writes are skipped), and `pages` (KVPagePool) is its host mirror with the free list.  A slot
    takes pages on the host before each step (check_step / reserve_step, the step's columns [0, len + Q + 1)) and returns them on
    release or re-admission; `fork` gives a slot another's pages by reference and `reserve_step` copies a shared page before a
    sharer writes into it (copy on write).

    Projected prompt K/V per layer (cross-attention models, Lp_cap > 0): `prompt_kv_hi[i]` / `prompt_kv_lo[i]`, a second pool of
    `prompt_pages_total + 1` pages [(P_p+1)*64, 2E] with its own table `prompt_page_table` int32 [S, ceil(Lp_cap/64)] and host mirror
    `prompt_pages` (a second KVPagePool), `prompt_len` int32 [S] (the admitted prompt's length: the cross-attention's per-slot key
    count) and `prompt_mask` [S, Lp_cap] (a shorter prompt's tail columns are masked).  An admission takes ceil(Lp/64) pages per slot
    and writes them once; the rows of the last page past Lp are zero.  A fork shares the source's prompt pages by reference (prompt
    pages are never written after admission, so they need no copy on write); release and re-admission give them back.  The two
    pools have separate budgets: `kv_pages_*` count history pages only.

    Per-slot device state, int32 [S]: `len` (cache columns used), `n_valid` (next position id), `has_action`, `active`; `q_pos` is
    the step's scratch copy of `len`.  `action_token` fp32 [S, E] is the embedding of each slot's last action that `act_slots` feeds back to the next step (zero at open; a slot's first step ignores it).
    The host mirrors len / has_action / active (it knows them from admissions and the step width), so capacity and pages are
    checked and allocated without reading the device.  A decoder-only model (HFGPT) opens it with Lp_cap = 0: its prompt and
    separator are the first columns of the self-attention cache (HFGPT.prefill), and there is no prompt pool / prompt_mask.

    kv_pool_tokens: cache columns the pool holds across all slots (rounded up to pages); None = S*ceil(Lmax/64) pages, so that
    every slot can reach Lmax at once.  A smaller pool overcommits: a step or admission the free pages cannot cover raises
    ValueError before any state is touched (`kv_pages_needed` tells a driver how many the next step takes).  prompt_pool_tokens:
    the same for the prompt pool; None = S*ceil(Lp_cap/64) pages, so that every slot can hold a full-length prompt at once."""

    Lp_cap = 0  # prompt columns per slot; 0 = no prompt pool (also for host-side stand-ins that only set up the history pool)

    def __init__(self, *, S: int, Lmax: int, Lp_cap: int, E: int, n_layer: int, device, split: bool, precision: str, weights=None,
                 kv_pool_tokens: Optional[int] = None, prompt_pool_tokens: Optional[int] = None):
        self.S, self.Lmax, self.Lp_cap, self.E, self.precision = S, Lmax, Lp_cap, E, precision
        self.weights = weights  # engine.WeightState of the decoder at open; admit and step refuse once it has changed
        page_ld = KVPagePool.pages_for(Lmax)
        n_use = S * page_ld if kv_pool_tokens is None else KVPagePool.pages_for(int(kv_pool_tokens))
        if not 1 <= n_use <= S * page_ld:
            raise ValueError(f"kv_pool_tokens={kv_pool_tokens} must cover 1 .. {S * page_ld} pages of {_C.KV_PAGE_TOKENS} tokens "
                             f"({S} slots of max_tokens={Lmax})")
        if Lp_cap:
            p_ld = KVPagePool.pages_for(Lp_cap)
            n_prompt = S * p_ld if prompt_pool_tokens is None else KVPagePool.pages_for(int(prompt_pool_tokens))
            if not 1 <= n_prompt <= S * p_ld:
                raise ValueError(f"prompt_pool_tokens={prompt_pool_tokens} must cover 1 .. {S * p_ld} pages of {_C.KV_PAGE_TOKENS} "
                                 f"tokens ({S} slots of max_prompt_tokens={Lp_cap})")
        self.pages = KVPagePool(S, page_ld, n_use + 1)
        self.page_table = torch.zeros((S, page_ld), dtype=torch.int32, device=device)
        mk = lambda rows: torch.zeros((rows, 2 * E), dtype=torch.int16, device=device)
        rows = self.pages.n_pages * _C.KV_PAGE_TOKENS
        self.kv_hi = [mk(rows) for _ in range(n_layer)]
        self.kv_lo = [mk(rows) if split else None for _ in range(n_layer)]
        z = lambda: torch.zeros((S,), dtype=torch.int32, device=device)
        self.prompt_pages = self.prompt_page_table = self.prompt_kv_hi = self.prompt_kv_lo = self.prompt_len = self.prompt_mask = None
        if Lp_cap:
            self.prompt_pages = KVPagePool(S, p_ld, n_prompt + 1)
            self.prompt_page_table = torch.zeros((S, p_ld), dtype=torch.int32, device=device)
            rows = self.prompt_pages.n_pages * _C.KV_PAGE_TOKENS
            self.prompt_kv_hi = [mk(rows) for _ in range(n_layer)]
            self.prompt_kv_lo = [mk(rows) if split else None for _ in range(n_layer)]
            self.prompt_len = z()
            self.prompt_mask = torch.zeros((S, Lp_cap), dtype=torch.uint8, device=device)
        self.mask = torch.zeros((S, Lmax), dtype=torch.uint8, device=device)
        self.len, self.n_valid, self.has_action, self.active, self.q_pos = z(), z(), z(), z(), z()
        self.action_token = torch.zeros((S, E), dtype=torch.float32, device=device)
        self._copy_bufs = {}  # base addresses of the buffers vima_kv_copy_blocks copies rows in, on the device (copy_bufs)
        self.len_host = [0] * S
        self.has_action_host = [False] * S
        self.active_host = [False] * S

    @property
    def kv_pages_total(self) -> int:
        """Pages the slots can own (the pool without its zero page)."""
        return self.pages.n_pages - 1

    @property
    def kv_pages_free(self) -> int:
        return len(self.pages.free)

    @property
    def prompt_pages_total(self) -> int:
        """Pages of the prompt pool the slots can own (0 without cross-attention prompts)."""
        return self.prompt_pages.n_pages - 1 if self.Lp_cap else 0

    @property
    def prompt_pages_free(self) -> int:
        return len(self.prompt_pages.free) if self.Lp_cap else 0

    def _cow_plan(self) -> list:
        """Active slots whose next step writes into a page shared with another slot (a fork's), in ascending slot order."""
        return self.pages.cow_plan([(b, self.len_host[b]) for b in range(self.S) if self.active_host[b]])

    def kv_pages_needed(self, Q: int) -> int:
        """New pages the next step of Q obs tokens takes: every active slot must own its columns [0, len + Q + 1), and a slot whose
        column `len` lies inside a page it shares takes a private copy of that page first."""
        new = sum(self.pages.needed(b, self.len_host[b] + Q + 1) for b in range(self.S) if self.active_host[b])
        return new + len(self._cow_plan())

    def slot_index(self, slots) -> list:
        s = [int(x) for x in (slots.tolist() if isinstance(slots, torch.Tensor) else slots)]
        if len(set(s)) != len(s) or any(not 0 <= x < self.S for x in s):
            raise ValueError(f"slots must be distinct indices in [0, {self.S}), got {s}")
        return s

    def check_step(self, S: int, Q: int, E: int, p) -> None:
        """Everything that can refuse a step, BEFORE any state is touched."""
        if S != self.S or E != self.E:
            raise ValueError(f"SlotDecodeCache(S={self.S}, E={self.E}) does not match the step's {S} slots / width {E}")
        if Q < 1 or Q + 1 > self.Lmax:
            raise ValueError(f"a step of {Q} obs tokens does not fit SlotDecodeCache(Lmax={self.Lmax})")
        full = [b for b in range(self.S) if self.active_host[b] and self.len_host[b] + Q + 1 > self.Lmax]
        if full:
            raise ValueError(f"slots {full} cannot take {Q + 1} more tokens (Lmax={self.Lmax}, lengths {[self.len_host[b] for b in full]})")
        need = self.kv_pages_needed(Q)
        if need > self.kv_pages_free:
            raise ValueError(f"the step needs {need} more K/V pages, {self.kv_pages_free} of {self.kv_pages_total} are free: release "
                             "slots or open the cache with a larger kv_pool_tokens")
        self.check_precision(p)

    def reserve_step(self, Q: int) -> None:
        """Take the pages the next step needs (after check_step, so it cannot fail): first a private copy of each shared page a slot
        is about to write into (one vima_kv_copy_blocks over every layer's pool), then the new pages.  Asynchronous, no host
        synchronisation; the copies are queued on the current stream ahead of the step's kernels."""
        upd, copies = [], []
        for b in self._cow_plan():
            u, c = self.pages.cow(b, self.len_host[b])
            upd.append(u)
            copies.append(c)
        for b in range(self.S):
            if self.active_host[b]:
                upd += self.pages.reserve(b, self.len_host[b] + Q + 1)
        if copies:
            self._copy_pages(copies)
        self._push_pages(upd)

    def copy_bufs(self, which: str) -> torch.Tensor:
        """int64 device array of base addresses: "pool" = every layer's K/V pool, hi and lo (copy on write of a shared page),
        "prompt" = every layer's prompt pool, hi and lo (zeroing an admitted prompt's last page).  Built on first use."""
        if which not in self._copy_bufs:
            ts = self.kv_hi + self.kv_lo if which == "pool" else self.prompt_kv_hi + self.prompt_kv_lo
            self._copy_bufs[which] = self.device_ints([t.data_ptr() for t in ts if t is not None])
        return self._copy_bufs[which]

    def _copy_pages(self, copies: list) -> None:
        """(old page, new page) pairs: the old page's 64 rows -> the new page's, in every layer's hi and lo pool, one launch."""
        rows = self.device_ints([old * _C.KV_PAGE_TOKENS for old, _ in copies] + [new * _C.KV_PAGE_TOKENS for _, new in copies])
        rows = rows.view(2, len(copies))
        _C.Context.get(self.page_table.device).kv_copy_blocks(self.copy_bufs("pool"), self.kv_hi[0].stride(0) * 2, rows[0], rows[1],
                                                              _C.KV_PAGE_TOKENS, self.pages.n_pages * _C.KV_PAGE_TOKENS)

    def check_prefix(self, slots: list, cols: int, prompt_cols: int = 0) -> None:
        """Refuses (before any state is touched) an admission of `slots` whose first `cols` columns the pool cannot cover, or (with
        cross-attention prompts) whose prompts of `prompt_cols` tokens the prompt pool cannot cover, counting the pages the slots give
        back (a page still shared with a slot outside `slots` is not given back)."""
        need = len(slots) * self.pages.pages_for(cols)
        have = self.kv_pages_free + self.pages.freed_by(slots)
        if need > have:
            raise ValueError(f"admitting {len(slots)} prefixes of {cols} tokens needs {need} K/V pages, {have} are free: release "
                             "slots or open the cache with a larger kv_pool_tokens")
        if self.Lp_cap:
            need = len(slots) * self.prompt_pages.pages_for(prompt_cols)
            have = self.prompt_pages_free + self.prompt_pages.freed_by(slots)
            if need > have:
                raise ValueError(f"admitting {len(slots)} prompts of {prompt_cols} tokens needs {need} prompt pages, {have} are free: "
                                 "release slots or open the cache with a larger prompt_pool_tokens")

    def free_slots(self, slots: list, prefix_cols=0, prompt_cols: int = 0) -> None:
        """Return the pages of `slots` (released or re-admitted), history and prompt, and give each `prefix_cols` columns (an int, or
        one per slot) of new history pages and `prompt_cols` columns of new prompt pages (checked by check_prefix or
        check_admit_history), the rows of the last prompt page past `prompt_cols` zeroed.  Asynchronous, no host synchronisation."""
        cols = prefix_cols if isinstance(prefix_cols, list) else [prefix_cols] * len(slots)
        upd = []
        for b in slots:
            upd += self.pages.release(b)
        for b, c in zip(slots, cols):
            upd += self.pages.reserve(b, c)
        self._push_pages(upd)
        if self.Lp_cap:
            upd = []
            for b in slots:
                upd += self.prompt_pages.release(b)
            for b in slots:
                upd += self.prompt_pages.reserve(b, prompt_cols)
            self._push_pages(upd, self.prompt_page_table)
            if prompt_cols % _C.KV_PAGE_TOKENS:
                self._zero_prompt_pages([self.prompt_pages.owned[b][-1] for b in slots])

    def _zero_prompt_pages(self, pages: list) -> None:
        """Copy the zero page over `pages` in every layer's prompt pool (one launch).  The attention kernels read whole pages, so the
        rows of a prompt's last page past its length must hold no earlier tenant's values: a NaN there would reach the output as
        0 * NaN."""
        if not pages:
            return
        rows = self.device_ints([0] * len(pages) + [pg * _C.KV_PAGE_TOKENS for pg in pages]).view(2, len(pages))
        _C.Context.get(self.page_table.device).kv_copy_blocks(self.copy_bufs("prompt"), self.prompt_kv_hi[0].stride(0) * 2, rows[0], rows[1],
                                                              _C.KV_PAGE_TOKENS, self.prompt_pages.n_pages * _C.KV_PAGE_TOKENS)

    def check_fork(self, src, dst) -> tuple:
        """Everything that can refuse a fork, before any state is touched: -> (src, dst) as lists of ints."""
        s = [int(x) for x in (src.tolist() if isinstance(src, torch.Tensor) else src)]
        d = self.slot_index(dst)
        if len(s) != len(d):
            raise ValueError(f"fork: {len(s)} sources for {len(d)} destinations")
        bad = [x for x in s if not 0 <= x < self.S or not self.active_host[x]]
        if bad:
            raise ValueError(f"fork: sources {bad} are not active slots of [0, {self.S})")
        both = sorted(set(s) & set(d))
        if both:
            raise ValueError(f"fork: slots {both} are both a source and a destination")
        return s, d

    def fork(self, src: list, dst: list) -> None:
        """Slot dst[i] takes a copy of slot src[i]'s episode (after check_fork): its pages by reference (the pages of the columns
        [0, len) the source has written, and all its prompt pages; no page is taken and no K/V row is copied), its per-slot state,
        fed-back action, history mask, prompt mask and prompt length.  A live destination lets go of its pages first.  Asynchronous,
        no host synchronisation."""
        if not dst:
            return
        upd = []
        for b in dst:
            upd += self.pages.release(b)
        for a, b in zip(src, dst):
            upd += self.pages.fork(a, b, self.pages.pages_for(self.len_host[a]))
        self._push_pages(upd)
        n = len(dst)
        idx = self.device_ints(src + dst)
        si, di = idx[:n], idx[n:]
        rows = [self.len, self.n_valid, self.has_action, self.active, self.action_token, self.mask]
        if self.Lp_cap:
            upd = []
            for b in dst:
                upd += self.prompt_pages.release(b)
            for a, b in zip(src, dst):
                upd += self.prompt_pages.fork(a, b, len(self.prompt_pages.owned[a]))
            self._push_pages(upd, self.prompt_page_table)
            rows += [self.prompt_mask, self.prompt_len]
        for t in rows:
            t.index_copy_(0, di, t.index_select(0, si))
        for a, b in zip(src, dst):
            self.len_host[b], self.has_action_host[b], self.active_host[b] = self.len_host[a], self.has_action_host[a], True

    # ---- resumed episodes: a slot admitted mid-way from its recorded history (DESIGN.md 7 (f)1)
    def check_admit_history(self, slots: list, lens: list, prompt_cols: int = 0) -> None:
        """Everything on the cache's side that can refuse admitting slots[j] at lens[j] cache columns (prefix and history) with
        (cross-attention policies) a prompt of `prompt_cols` tokens, before any state is touched: a length past Lmax, and pools that
        cannot cover ceil(lens[j]/64) history pages each and ceil(prompt_cols/64) prompt pages each, counting the pages the
        destinations give back (a page still shared with a slot outside `slots` is not given back)."""
        over = [(b, c) for b, c in zip(slots, lens) if not 0 <= c <= self.Lmax]
        if over:
            raise ValueError(f"admit_history: (slot, history columns) {over} do not fit max_tokens={self.Lmax}")
        need = sum(self.pages.pages_for(c) for c in lens)
        have = self.kv_pages_free + self.pages.freed_by(slots)
        if need > have:
            raise ValueError(f"admit_history: {len(slots)} histories of {list(lens)} columns need {need} K/V pages, {have} are free: "
                             "release or swap out slots, or open the cache with a larger kv_pool_tokens")
        if self.Lp_cap:
            need = len(slots) * self.prompt_pages.pages_for(prompt_cols)
            have = self.prompt_pages_free + self.prompt_pages.freed_by(slots)
            if need > have:
                raise ValueError(f"admit_history: {len(slots)} prompts of {prompt_cols} tokens need {need} prompt pages, {have} are free: "
                                 "release or swap out slots, or open the cache with a larger prompt_pool_tokens")

    def reserve_history(self, slots: list, lens: list, has_action: list, prompt_cols: int = 0) -> None:
        """The page-taking step of a history admission (after check_admit_history, so it cannot fail): the destinations let go of
        their pages (a live episode is replaced; a page a fork still holds stays with it), slots[j] takes ceil(lens[j]/64) private
        history pages and ceil(prompt_cols/64) prompt pages, the table rows are pushed, and the host mirrors become len = lens[j],
        has_action[j], active.  The device rows and state are written by the prefill that follows.  Asynchronous, no host
        synchronisation."""
        self.free_slots(slots, list(lens), prompt_cols)
        for b, c, a in zip(slots, lens, has_action):
            self.len_host[b], self.has_action_host[b], self.active_host[b] = int(c), bool(a), True

    # ---- swapped episodes: a slot's episode to pinned host memory and back (DESIGN.md 7 (f)1)
    def swap_key(self) -> tuple:
        """What a swapped episode must share with the cache it is swapped into: (precision mode, Lmax, Lp_cap, E, layers, split)."""
        return (self.precision, self.Lmax, self.Lp_cap, self.E, len(self.kv_hi), self.kv_lo[0] is not None)

    def kv_pages_freed_by(self, slots) -> int:
        """History pages that swapping out or releasing `slots` would return to the free list (a page that a slot outside `slots`
        still holds, a fork's, stays)."""
        return self.pages.freed_by(self.slot_index(slots))

    def check_swap_out(self, slots) -> list:
        """Everything that can refuse a swap-out, before any state is touched: -> slots as a list of ints."""
        s = self.slot_index(slots)
        bad = [b for b in s if not self.active_host[b]]
        if bad:
            raise ValueError(f"swap_out: slots {bad} are not active")
        return s

    def swap_out(self, slots: list) -> list:
        """The episodes of `slots` (after check_swap_out) -> SwappedEpisode each: their history pages of columns [0, len), their prompt
        pages and state rows, packed on the device and copied to one pinned host buffer; then the slots are released (a page still
        shared with a fork stays with the fork).  Asynchronous, no host synchronisation: the host buffer is complete once the work
        queued on the current stream so far has run."""
        if not slots:
            return []
        kv = [self.pages.owned[b][:self.pages.pages_for(self.len_host[b])] for b in slots]
        pr = [list(self.prompt_pages.owned[b]) if self.Lp_cap else [] for b in slots]
        views = self._swap_out_data(slots, kv, pr)
        key = self.swap_key()
        eps = [SwappedEpisode(kv=k, prompt=p, state=st, kv_pages=len(kv[i]), prompt_pages=len(pr[i]), len_host=self.len_host[b],
                              has_action_host=self.has_action_host[b], key=key, weights=self.weights)
               for i, (b, (k, p, st)) in enumerate(zip(slots, views))]
        self.active.index_fill_(0, self.device_ints(slots), 0)  # what release does
        self.free_slots(slots)
        for b in slots:
            self.active_host[b] = False
        return eps

    def check_swap_in(self, slots, episodes) -> tuple:
        """Everything that can refuse a swap-in, before any state is touched: -> (slots, episodes) as lists.  The pools must cover
        the episodes' pages, counting the pages the destinations give back (as check_prefix does)."""
        s = self.slot_index(slots)
        eps = list(episodes)
        if len(eps) != len(s):
            raise ValueError(f"swap_in: {len(eps)} episodes for {len(s)} slots")
        key = self.swap_key()
        for i, ep in enumerate(eps):
            if not isinstance(ep, SwappedEpisode):
                raise ValueError(f"swap_in: episode {i} is a {type(ep).__name__}, not a SwappedEpisode")
            if ep.key != key:
                raise ValueError(f"swap_in: episode {i} comes from a cache of (precision, max_tokens, max_prompt_tokens, E, layers, split) = "
                                 f"{ep.key}; this cache is {key}")
            if (ep.weights is None) != (self.weights is None) or (ep.weights is not None and not ep.weights.matches(self.weights)):
                raise ValueError(f"swap_in: episode {i}'s K/V rows belong to other weights (another policy's, or weights changed since "
                                 "the swap-out or since this cache was opened)")
        need, have = sum(ep.kv_pages for ep in eps), self.kv_pages_free + self.pages.freed_by(s)
        if need > have:
            raise ValueError(f"swap_in: {len(eps)} episodes need {need} K/V pages, {have} are free: release or swap out slots, or open "
                             "the cache with a larger kv_pool_tokens")
        if self.Lp_cap:
            need, have = sum(ep.prompt_pages for ep in eps), self.prompt_pages_free + self.prompt_pages.freed_by(s)
            if need > have:
                raise ValueError(f"swap_in: {len(eps)} episodes need {need} prompt pages, {have} are free: release or swap out slots, "
                                 "or open the cache with a larger prompt_pool_tokens")
        return s, eps

    def swap_in(self, slots: list, episodes: list) -> None:
        """Slot slots[i] resumes episodes[i] (after check_swap_in) exactly where it was swapped out: the destination lets go of its
        pages (a live one is replaced), takes private pages for the episode's history and prompt pages, and gets their rows, its state
        rows and host mirrors back.  The episodes stay usable.  Asynchronous, no host synchronisation."""
        if not slots:
            return
        upd, kv = [], []
        for b in slots:
            upd += self.pages.release(b)
        for b, ep in zip(slots, episodes):
            upd += self.pages.reserve(b, ep.kv_pages * _C.KV_PAGE_TOKENS)
            kv.append(list(self.pages.owned[b]))
        self._push_pages(upd)
        pr = [[] for _ in slots]
        if self.Lp_cap:
            upd = []
            for b in slots:
                upd += self.prompt_pages.release(b)
            for i, (b, ep) in enumerate(zip(slots, episodes)):
                upd += self.prompt_pages.reserve(b, ep.prompt_pages * _C.KV_PAGE_TOKENS)
                pr[i] = list(self.prompt_pages.owned[b])
            self._push_pages(upd, self.prompt_page_table)
        self._swap_in_data(slots, episodes, kv, pr)
        for b, ep in zip(slots, episodes):
            self.len_host[b], self.has_action_host[b], self.active_host[b] = ep.len_host, ep.has_action_host, True

    def _state_layout(self) -> tuple:
        """([(device state tensor [S, ...], byte offset, bytes)], record bytes): one slot's state rows in a swapped episode's record,
        4-byte fields first; the record size is a multiple of 16."""
        rows = [self.len, self.n_valid, self.has_action] + ([self.prompt_len] if self.Lp_cap else [])
        rows += [self.action_token, self.mask] + ([self.prompt_mask] if self.Lp_cap else [])
        out, off = [], 0
        for t in rows:
            nb = t[0].numel() * t.element_size()
            out.append((t, off, nb))
            off += nb
        return out, -(-off // 16) * 16

    @staticmethod
    def _field(rec: torch.Tensor, t: torch.Tensor, off: int, nb: int) -> torch.Tensor:
        """Field (t, off, nb) of the records rec uint8 [n, record bytes], as a [n, ...] view of t's dtype."""
        return rec[:, off:off + nb].view(t.dtype).view((rec.shape[0],) + tuple(t.shape[1:]))

    def _page_bytes(self, which: str) -> int:
        """Packed bytes of one page of the "pool" (history) or "prompt" pool across every layer's hi and lo buffers."""
        ts = self.kv_hi + self.kv_lo if which == "pool" else self.prompt_kv_hi + self.prompt_kv_lo
        ts = [t for t in ts if t is not None]
        return len(ts) * _C.KV_PAGE_TOKENS * ts[0].stride(0) * ts[0].element_size()

    def _pack_pages(self, which: str, pages: list, packed: torch.Tensor, unpack: bool) -> None:
        """`pages` of the "pool" or "prompt" pool <-> packed (device uint8), one vima_kv_pack_blocks launch."""
        if not pages:
            return
        t0, n_pages = (self.kv_hi[0], self.pages.n_pages) if which == "pool" else (self.prompt_kv_hi[0], self.prompt_pages.n_pages)
        rows = self.device_ints([pg * _C.KV_PAGE_TOKENS for pg in pages])
        _C.Context.get(self.page_table.device).kv_pack_blocks(self.copy_bufs(which), t0.stride(0) * t0.element_size(), rows,
                                                              _C.KV_PAGE_TOKENS, n_pages * _C.KV_PAGE_TOKENS, packed, unpack)

    def _swap_out_data(self, slots: list, kv: list, prompt: list) -> list:
        """Device side of swap_out: the history pages kv[i] and prompt pages prompt[i] of slot slots[i] (one pack launch per pool) and
        its state rows (index_select) into one device staging buffer, copied to one pinned host buffer -> [(kv, prompt, state)] views
        of it per episode."""
        dev = self.page_table.device
        kb, pb = self._page_bytes("pool"), (self._page_bytes("prompt") if self.Lp_cap else 0)
        lay, rec = self._state_layout()
        n = len(slots)
        k_end = sum(map(len, kv)) * kb
        p_end = k_end + sum(map(len, prompt)) * pb
        stage = torch.empty(p_end + n * rec, dtype=torch.uint8, device=dev)
        self._pack_pages("pool", [pg for ps in kv for pg in ps], stage[:k_end], False)
        if self.Lp_cap:
            self._pack_pages("prompt", [pg for ps in prompt for pg in ps], stage[k_end:p_end], False)
        st = stage[p_end:].view(n, rec)
        idx = self.device_ints(slots)
        for t, off, nb in lay:
            self._field(st, t, off, nb).copy_(t.index_select(0, idx))
        host = torch.empty(stage.numel(), dtype=torch.uint8, pin_memory=True)
        host.copy_(stage, non_blocking=True)
        out, ko, po = [], 0, k_end
        for i in range(n):
            k, p = len(kv[i]) * kb, len(prompt[i]) * pb
            out.append((host[ko:ko + k], host[po:po + p], host[p_end + i * rec:p_end + (i + 1) * rec]))
            ko, po = ko + k, po + p
        return out

    def _swap_in_data(self, slots: list, episodes: list, kv: list, prompt: list) -> None:
        """Device side of swap_in: the episodes copied from pinned host memory into one device staging buffer, their history pages
        unpacked into kv[i] and prompt pages into prompt[i] (one unpack launch per pool), their state rows index_copy_'d into
        slots[i], which become active."""
        dev = self.page_table.device
        lay, rec = self._state_layout()
        n = len(slots)
        k_end = sum(ep.kv.numel() for ep in episodes)
        p_end = k_end + sum(ep.prompt.numel() for ep in episodes)
        stage = torch.empty(p_end + n * rec, dtype=torch.uint8, device=dev)
        ko, po = 0, k_end
        for i, ep in enumerate(episodes):
            for src, o in ((ep.kv, ko), (ep.prompt, po), (ep.state, p_end + i * rec)):
                if src.numel():
                    stage[o:o + src.numel()].copy_(src, non_blocking=True)
            ko, po = ko + ep.kv.numel(), po + ep.prompt.numel()
        self._pack_pages("pool", [pg for ps in kv for pg in ps], stage[:k_end], True)
        if self.Lp_cap:
            self._pack_pages("prompt", [pg for ps in prompt for pg in ps], stage[k_end:p_end], True)
        st = stage[p_end:].view(n, rec)
        idx = self.device_ints(slots)
        for t, off, nb in lay:
            t.index_copy_(0, idx, self._field(st, t, off, nb).contiguous())
        self.active.index_fill_(0, idx, 1)

    def _push_pages(self, upd: list, table: Optional[torch.Tensor] = None) -> None:
        """Page-table entries (flat index, page) -> the device table (default: the history pool's `page_table`): one copy from pinned
        host memory and one scatter, both queued on the current stream.  A later entry for the same index wins (a re-admitted slot's
        page 0 of its released row is given again): the scatter gets each index once, since its order among duplicates is
        undefined."""
        last = dict(upd)
        if not last:
            return
        d = self.device_ints(list(last) + list(last.values())).view(2, len(last))
        (self.page_table if table is None else table).view(-1).scatter_(0, d[0], d[1].to(torch.int32))

    def device_ints(self, values: list) -> torch.Tensor:
        """int64 [len(values)] on the cache's device, copied from pinned host memory without a host synchronisation."""
        h = torch.tensor(values, dtype=torch.int64).pin_memory()
        return h.to(self.page_table.device, non_blocking=True)

    def check_precision(self, p) -> None:
        """The mode and the weights the cache was opened with are still in force (its K/V rows were computed with them)."""
        if self.precision != p.name:
            raise ValueError(f"SlotDecodeCache was opened in precision mode {self.precision!r}; the current mode is {p.name!r}")
        check_cache_weights(self)

    def advance_host(self, Q: int) -> None:
        """Host mirror of what vima_slot_step_end does on the device."""
        for b in range(self.S):
            if self.active_host[b]:
                self.len_host[b] += Q + int(self.has_action_host[b])
                self.has_action_host[b] = True

    def state(self) -> tuple:
        """Copies of the per-slot state: device vectors and page table, host mirror and page allocator."""
        return (tuple(t.clone() for t in (self.len, self.n_valid, self.has_action, self.active, self.action_token, self.page_table)),
                (list(self.len_host), list(self.has_action_host), list(self.active_host), self.pages.state()))

    def restore(self, st: tuple) -> None:
        for dst, src in zip((self.len, self.n_valid, self.has_action, self.active, self.action_token, self.page_table), st[0]):
            dst.copy_(src)
        self.len_host, self.has_action_host, self.active_host = (list(x) for x in st[1][:3])
        self.pages.restore(st[1][3])


def check_cache_append(cache: "DecodeCache", B: int, L: int, E: int, p) -> None:
    """Everything that can refuse an append, BEFORE any cache state is touched (capacity, shapes, precision mode)."""
    if cache.B != B or cache.E != E:
        raise ValueError(f"DecodeCache(B={cache.B}, E={cache.E}) does not match the step's batch {B} / width {E}")
    if cache.L + L > cache.Lmax:
        raise ValueError(f"DecodeCache(B={cache.B}, Lmax={cache.Lmax}) cannot take {L} more tokens at length {cache.L}")
    if cache.precision and cache.precision != p.name:
        raise ValueError(f"DecodeCache was opened in precision mode {cache.precision!r}; the current mode is {p.name!r}")
    check_cache_weights(cache)


def check_cache_weights(cache) -> None:
    """A cache's K/V rows were projected with the weights in force when it was opened: refuse to mix them with new ones."""
    why = None if cache.weights is None else cache.weights.changed()
    if why is not None:
        raise ValueError(f"{type(cache).__name__}: {why} since the cache was opened; its K/V rows belong to the old weights. "
                         "Open a new cache.")


def run_block(ctx, p, W, blk: "Block", x32, x16, c16, *, B, L, E, H, omask, chain_ln=None, want16=False, out_f32=None, cache=None,
              layer=0, kv_scatter=None):
    """GPT-1 post-LN block (components.py:23-37 / gpt.py:223-249): returns (LN2 output fp32, operands of the NEXT consumer):
    with `chain_ln` the operands are chain_ln(LN2(...)) (next layer's query LayerNorm), with `want16` they are LN2(...) itself.
    With `cache` (DecodeCache or SlotDecodeCache) the L rows are the NEW tokens of each episode and attention runs over the cached
    prefix + themselves.  With `kv_scatter` = (slots int32 [B], cache) and no `cache`, attention is local and the keys / values of
    sequence j also go to column r of slot slots[j] of the cache (decoder-only prefill, HFGPT.prefill).

    ln_1 never runs as a kernel: c_proj's epilogue emits s = attn + x as fp32 + operands together with per-row partial sums, the
    GEGLU GEMM takes the un-normalised s with ln_1 folded into its weights (rstd / mean applied in its epilogue), and the MLP's
    c_proj normalises its residual ln_1(s) on the fly from the same (mean, rstd)."""
    M = B * L
    d = E // H
    dev = x32.device
    # operand formats: attention inputs keep the 16-bit (hi, lo) pair; everything that only feeds a GEMM carries e4m3
    # cross-term views in "f16f8" mode (out_f8=True is a no-op in the other modes)
    _, qkv16 = eng.gemm(ctx, x16, W["c_attn"], p, want16=True)
    o8 = None if c16.lo8 is None else (c16.lo8, c16.hi8)
    if cache is None:
        if kv_scatter is not None:
            sl, kc = kv_scatter
            if isinstance(kc, SlotDecodeCache):
                ctx.slot_kv_scatter_paged(qkv16.hi, qkv16.lo, qkv16.ld, E, 2 * E, B, L, sl, kc.kv_hi[layer], kc.kv_lo[layer], 2 * E,
                                          kc.page_table, kc.pages.n_pages)
            else:
                ctx.slot_kv_scatter(qkv16.hi, qkv16.lo, qkv16.ld, E, 2 * E, B, L, sl, kc.kv_hi[layer], kc.kv_lo[layer], 2 * E, kc.Lmax)
        ctx.attention(q=(qkv16.hi, qkv16.lo, qkv16.ld, 0), k=(qkv16.hi, qkv16.lo, qkv16.ld, E), v=(qkv16.hi, qkv16.lo, qkv16.ld, 2 * E),
                      o=(c16.hi, c16.lo, c16.ld, 0), B=B, H=H, Lq=L, Lk=L, D=d, scale=1.0 / math.sqrt(d), causal=True, key_mask=omask,
                      dtype=p.dtype, o8=o8)
    elif isinstance(cache, SlotDecodeCache):  # every slot at its own length: columns and causal positions from cache.q_pos, rows
        # through the page table
        khi, klo, pt, n_pages = cache.kv_hi[layer], cache.kv_lo[layer], cache.page_table, cache.pages.n_pages
        ctx.slot_kv_append_paged(qkv16.hi, qkv16.lo, qkv16.ld, E, 2 * E, B, L, cache.q_pos, khi, klo, 2 * E, pt, n_pages)
        ctx.attention(q=(qkv16.hi, qkv16.lo, qkv16.ld, 0), k=(khi, klo, 2 * E, 0), v=(khi, klo, 2 * E, E), o=(c16.hi, c16.lo, c16.ld, 0),
                      B=B, H=H, Lq=L, Lk=cache.Lmax, D=d, scale=1.0 / math.sqrt(d), causal=True, key_mask=cache.mask, dtype=p.dtype, o8=o8,
                      mask_ld=cache.Lmax, q_pos=cache.q_pos, kv_pages=pt, kv_pool_pages=n_pages)
    else:
        L0 = cache.L
        cache.append_kv(layer, qkv16, L0, L)
        khi, klo = cache.kv_hi[layer], cache.kv_lo[layer]
        ctx.attention(q=(qkv16.hi, qkv16.lo, qkv16.ld, 0), k=(khi, klo, 2 * E, 0), v=(khi, klo, 2 * E, E), o=(c16.hi, c16.lo, c16.ld, 0),
                      B=B, H=H, Lq=L, Lk=L0 + L, D=d, scale=1.0 / math.sqrt(d), causal=True, key_mask=cache.mask, dtype=p.dtype, o8=o8,
                      kv_batch_rows=cache.Lmax, mask_ld=cache.Lmax, q_pos0=L0)
    part = eng.stats_buffer(ctx, M, W["c_proj"], dev)
    s32, s16 = eng.gemm(ctx, c16, W["c_proj"], p, residual=x32, want_f32=True, want16=True, out_f8=True, stats_out=part)
    st = eng.row_stats_of(ctx, part, M, E, blk.ln_1.eps)
    if "fc_glu" in W:
        _, h16 = eng.gemm(ctx, s16, W["fc_glu"], p, act=_C.ACT_GELU, want16=True, out_f8=True, row_stats=st)
    else:  # afn = "gelu" (HF NewGELUActivation, the OpenAIGPTConfig default): act(c_fc(ln_1(s))), components.py:92-98
        _, h16 = eng.gemm(ctx, s16, W["fc"], p, act=_C.ACT_GELU_TANH, want16=True, out_f8=True, row_stats=st)
    t32, _ = eng.gemm(ctx, h16, W["mlp_proj"], p, residual=s32, res_ln=(st, blk.ln_1.weight.detach(), blk.ln_1.bias.detach()), want_f32=True)
    del h16, s32, s16
    w, b = blk.ln_2.weight.detach(), blk.ln_2.bias.detach()
    if chain_ln is not None:
        y32, _, nxt16 = eng.norm(ctx, t32, p, rows=M, cols=E, w=w, b=b, eps=blk.ln_2.eps, w2=chain_ln.weight.detach(), b2=chain_ln.bias.detach(),
                                 eps2=chain_ln.eps, want16=True, out_f32=out_f32, want_f32=out_f32 is None, out_f8=True)
    else:
        y32, _, nxt16 = eng.norm(ctx, t32, p, rows=M, cols=E, w=w, b=b, eps=blk.ln_2.eps, want16=want16, out_f32=out_f32, want_f32=out_f32 is None,
                                 out_f8=True)
    return y32, nxt16


class PosIdGuard:
    """Deferred report of out-of-range position ids (the reference's nn.Embedding raises IndexError on every call, xattn_gpt.py:
    103-114; ids of -1 arise when an episode's first history slot is masked).  The kernels set a persistent device flag; the
    first call of a module checks it synchronously, later calls copy it to pinned host memory asynchronously and the NEXT call
    (or `check()`) raises -- no host synchronisation on the steady-state path."""

    def __init__(self):
        self.flag = None      # int32[1] on the device
        self.host = None      # pinned int32[1]
        self.event = None
        self.checked_sync = False

    def device_flag(self, dev) -> torch.Tensor:
        if self.flag is None or self.flag.device != dev:
            self.flag = torch.zeros(1, dtype=torch.int32, device=dev)
            self.host = torch.zeros(1, dtype=torch.int32).pin_memory()
            self.event, self.checked_sync = None, False
        return self.flag

    def poll(self):
        """Raise if a PREVIOUS call saw a bad id (its flag copy has landed)."""
        if self.event is not None and not torch.cuda.is_current_stream_capturing() and self.event.query():
            self.event = None
            if int(self.host[0]) != 0:
                self.reset()
                raise IndexError("index out of range in self (a previous call passed a position id outside the embedding table)")

    def after_launch(self):
        if not self.checked_sync:
            self.checked_sync = True
            if int(self.flag.item()) != 0:
                self.reset()
                raise IndexError("index out of range in self (position id outside the embedding table)")
            return
        if torch.cuda.is_current_stream_capturing():
            return
        self.host.copy_(self.flag, non_blocking=True)
        self.event = torch.cuda.Event()
        self.event.record()

    def check(self):
        """Synchronous check (host sync)."""
        if self.flag is not None and int(self.flag.item()) != 0:
            self.reset()
            raise IndexError("index out of range in self (position id outside the embedding table)")

    def reset(self):
        if self.flag is not None:
            self.flag.zero_()
        self.event = None


class XAttention(nn.Module):
    def __init__(self, dim: int, *, num_heads: int, ff_expanding: int, kv_n_positions: int, use_geglu: bool):
        super().__init__()
        if dim % num_heads != 0:
            raise ValueError(f"dim ({dim}) must be divisible by num_heads ({num_heads}).")
        self.num_heads = num_heads
        self.dim = dim
        inner = int(dim * ff_expanding)
        self.layernorm = nn.LayerNorm(dim)
        self.query = nn.Linear(dim, dim, bias=False)
        self.key_value = nn.Linear(dim, 2 * dim, bias=False)
        self.attention_out = nn.Linear(dim, dim, bias=False)
        self.ln = nn.LayerNorm(dim)
        self.linear1 = nn.Linear(dim, inner, bias=False)
        self.linear2 = nn.Linear(inner, dim, bias=False)
        self.gated_layer = nn.Linear(dim, inner, bias=False) if use_geglu else None
        self.register_buffer("kv_position_ids", torch.arange(kv_n_positions))


class XAttnGPT(nn.Module):
    def __init__(
        self,
        embd_dim: int = 768,
        *,
        n_positions: int = 512,
        n_layer: int = 12,
        n_head: int = 12,
        dropout: float = 0.1,
        xattn_n_head: int = 8,
        xattn_ff_expanding: int = 4,
        xattn_detach_qk: bool = False,
        xattn_n_positions: int,
        use_geglu: bool = False,
    ):
        super().__init__()
        self.embd_dim, self.n_layer, self.n_head, self.xattn_n_head = embd_dim, n_layer, n_head, xattn_n_head
        self.n_positions, self.xattn_n_positions = n_positions, xattn_n_positions
        self.positions_embed = nn.Embedding(n_positions, embd_dim)
        self.xattn_positions_embed = nn.Embedding(xattn_n_positions, embd_dim)
        self.h = nn.ModuleList([Block(embd_dim, n_positions, n_head, use_geglu) for _ in range(n_layer)])
        self.xattns = nn.ModuleList(
            [XAttention(embd_dim, num_heads=xattn_n_head, ff_expanding=xattn_ff_expanding, kv_n_positions=xattn_n_positions, use_geglu=use_geglu)
             for _ in range(n_layer)]
        )
        self.register_buffer("position_ids", torch.arange(n_positions))
        self.register_buffer("xattn_position_ids", torch.arange(xattn_n_positions))
        for m in self.modules():
            if isinstance(m, (nn.Linear, nn.Embedding)):
                nn.init.normal_(m.weight, std=0.02)
        self._input_checked = False
        self._wc = eng.WeightCache(self)
        self._pos_guard = PosIdGuard()

    def check_errors(self):
        """Host-synchronising check of the deferred position-id error flag (see PosIdGuard)."""
        self._pos_guard.check()

    # ---------------------------------------------------------------------------------------------
    def _packed(self, ctx, p):
        def build():
            L = []
            for blk, xa in zip(self.h, self.xattns):
                d = {}
                d["wq"] = eng.pack_linear(ctx, xa.query.weight, None, transposed=False, p=p, f8=True)
                d["wkv"] = eng.pack_linear(ctx, xa.key_value.weight, None, transposed=False, p=p, f8=True)
                d["wo"] = eng.pack_linear(ctx, xa.attention_out.weight, None, transposed=False, p=p, f8=True)
                # linear1 reads ln(a), the gate reads a itself (components.py:218-221): one GEGLU GEMM over the un-normalised a with
                # `ln` folded into the value half only
                xln = (xa.ln.weight.detach(), xa.ln.bias.detach())
                if xa.gated_layer is not None:
                    d["w1g"] = eng.pack_glu(ctx, xa.linear1.weight, None, xa.gated_layer.weight, val_transposed=False, gate_transposed=False,
                                            p=p, f8=True, ln=xln, ln_gate=False)
                else:  # use_geglu=False (components.py:139-142,218-223): gelu(linear1(ln(a))), no gate
                    d["w1"] = eng.pack_linear(ctx, xa.linear1.weight, None, transposed=False, p=p, f8=True, ln=xln)
                d["w2"] = eng.pack_linear(ctx, xa.linear2.weight, None, transposed=False, p=p, f8=True)
                d.update(pack_block(ctx, blk, p))
                L.append(d)
            return L

        params = tuple(t for t in self.parameters())
        return self._wc.get("layers", params, build)

    def _check_input(self, obs_action_tokens, prompt_tokens, prompt_mask, batch_first, obs_action_masks):
        """xattn_gpt.py:141-177 (first call only; host syncs)."""
        assert obs_action_tokens.dim() == 3 and obs_action_tokens.dtype == torch.float32
        assert prompt_tokens.dim() == 3 and prompt_tokens.dtype == torch.float32
        if batch_first:
            B_oa, L_oa, E_oa = obs_action_tokens.shape
            B_p, L_p, E_p = prompt_tokens.shape
        else:
            L_oa, B_oa, E_oa = obs_action_tokens.shape
            L_p, B_p, E_p = prompt_tokens.shape
        assert B_oa == B_p and E_oa == E_p
        if prompt_mask is not None:
            assert prompt_mask.shape == (B_oa, L_p) or prompt_mask.shape == (B_oa, 1, L_p), \
                f"Expect `prompt_mask` to have shape of either ({B_oa, 1, L_p}) or ({B_oa, L_p}), but got {prompt_mask.shape}"
            assert torch.all(prompt_mask.sum(dim=-1) > 0), "each source token should attend to at least one target token"
            assert prompt_mask.dtype == torch.bool
        if obs_action_masks is not None:
            assert obs_action_masks.shape == (B_oa, L_oa)
            assert torch.all(obs_action_masks.sum(dim=-1) > 0)
            assert obs_action_masks.dtype == torch.bool

    def _prompt_operand(self, ctx, p, prompt_tokens, prompt_position_ids, batch_first, B, Lp, E, err) -> "eng.Opnd":
        """prompt + xattn_positions_embed[ids], the key_value GEMM's operand [B*Lp, E] (out-of-range ids set `err`)."""
        dev = prompt_tokens.device
        ptk = prompt_tokens if prompt_tokens.stride(-1) == 1 else prompt_tokens.contiguous()
        psb, psl = (ptk.stride(0), ptk.stride(1)) if batch_first else (ptk.stride(1), ptk.stride(0))
        if prompt_position_ids is None:
            prompt_position_ids = self.xattn_position_ids[None, :Lp].expand(B, Lp)
        pr_ids = prompt_position_ids.to(torch.int64).contiguous()
        Mp = B * Lp
        kv16 = eng.Opnd(Mp, E, dev, p.split, f8=p.f8)
        if p.f8:  # prompt + position embedding feeds only the key_value GEMM: fp32 once, then hi16 + e4m3 views
            kv32 = torch.empty((Mp, E), dtype=torch.float32, device=dev)
            ctx.add_pos_embed(ptk, psb, psl, pr_ids, self.xattn_positions_embed.weight.detach(), B, Lp, E, out_f32=kv32, hi=kv16.hi, lo=None,
                              dtype=p.dtype, err_flag=err)
            ctx.split_f8(kv32, kv16.lo8, kv16.hi8)
            del kv32
        else:
            ctx.add_pos_embed(ptk, psb, psl, pr_ids, self.xattn_positions_embed.weight.detach(), B, Lp, E, hi=kv16.hi, lo=kv16.lo,
                              dtype=p.dtype, err_flag=err)
        return kv16

    @torch.no_grad()
    def admit_prompts(self, cache: SlotDecodeCache, slots: list, prompt_tokens: torch.Tensor, prompt_mask_u8: torch.Tensor,
                      prompt_position_ids: torch.Tensor) -> None:
        """Projected prompt keys/values of every layer for the n new prompts only (prompt_tokens (Lp,n,E), mask / position ids (n,Lp)),
        written into ceil(Lp/64) fresh prompt pages of each of `slots` (the rows past Lp of the last page are zero); their prompt
        masks are padded to Lp_cap with masked columns, their prompt length is Lp and their state is reset to an empty history.  The
        caller has validated shapes, slots and the precision mode; a prompt pool that cannot cover the admission raises ValueError
        before any state is touched."""
        Lp, n, E = prompt_tokens.shape
        cache.check_prefix(slots, 0, Lp)
        ctx = eng.ctx_for(prompt_tokens)
        p = eng.prec()
        dev = prompt_tokens.device
        self._pos_guard.poll()
        err = self._pos_guard.device_flag(dev)  # a bad prompt position id is reported by the next step
        kv16 = self._prompt_operand(ctx, p, prompt_tokens.float(), prompt_position_ids, False, n, Lp, E, err)
        # the slots' history pages go back to the pool (their first step takes new ones); their prompt pages are replaced
        cache.free_slots(slots, prompt_cols=Lp)
        idx = cache.device_ints(slots)
        sl = idx.to(torch.int32)
        for i, W in enumerate(self._packed(ctx, p)):
            self._scatter_prompt_kv(ctx, cache, sl, eng.gemm(ctx, kv16, W["wkv"], p, want16=True)[1], i, n, Lp, E)
        self._set_prompt_rows(cache, idx, prompt_mask_u8, Lp)
        for t, v in ((cache.len, 0), (cache.n_valid, 0), (cache.has_action, 0), (cache.active, 1)):
            t.index_fill_(0, idx, v)
        for b in slots:
            cache.len_host[b], cache.has_action_host[b], cache.active_host[b] = 0, False, True

    @staticmethod
    def _scatter_prompt_kv(ctx, cache: SlotDecodeCache, sl: torch.Tensor, kv: "eng.Opnd", layer: int, n: int, Lp: int, E: int) -> None:
        """Layer `layer`'s projected prompt keys/values kv [n*Lp, 2E] -> the prompt pages of slots sl (int32 [n], device)."""
        ctx.slot_kv_scatter_paged(kv.hi, kv.lo, kv.ld, 0, 2 * E, n, Lp, sl, cache.prompt_kv_hi[layer], cache.prompt_kv_lo[layer], 2 * E,
                                  cache.prompt_page_table, cache.prompt_pages.n_pages)

    @staticmethod
    def _set_prompt_rows(cache: SlotDecodeCache, idx: torch.Tensor, prompt_mask_u8: torch.Tensor, Lp: int) -> None:
        """Prompt mask rows (padded to Lp_cap with masked columns) and prompt length of the admitted slots idx (int64, device)."""
        cache.prompt_mask.index_fill_(0, idx, 0)
        cache.prompt_mask[idx, :Lp] = prompt_mask_u8
        cache.prompt_len.index_fill_(0, idx, Lp)

    @torch.no_grad()
    def prefill_history(self, cache: SlotDecodeCache, slots: list, tokens: torch.Tensor, mask_u8: torch.Tensor, position_ids: torch.Tensor,
                        prompt_tokens: torch.Tensor, prompt_mask_u8: torch.Tensor, prompt_position_ids: torch.Tensor, steps: torch.Tensor,
                        actions: torch.Tensor, Q: int) -> None:
        """Slot episodes admitted mid-way (after cache.reserve_history gave slots[j] its pages): tokens (L,n,E) hold each episode's
        recorded history as vima_slot_assemble_history lays it out (mask / position ids (n,L), padding columns masked), prompt_tokens
        (Lp,n,E) / prompt mask / position ids (n,Lp) its prompt.  One pass of forward's arithmetic over the n*L rows: each layer's
        key_value GEMM of the prompts feeds the cross-attention and is scattered into the slots' prompt pages (as admit_prompts does),
        and each causal block's keys / values go to the slots' history pages (run_block kv_scatter; columns past a slot's pages land
        on the zero page and are skipped).  Then vima_slot_admit_history writes the mask rows, state and fed-back actions (steps int32
        [n] on the device, actions (T,n,E)).  With L = 0 (no history) only the prompt is projected, as admit_prompts does.  The caller
        has validated everything; no host synchronisation."""
        L, n, E = tokens.shape
        Lp = prompt_tokens.shape[0]
        ctx = eng.ctx_for(prompt_tokens)
        p = eng.prec()
        dev = prompt_tokens.device
        self._pos_guard.poll()
        err = self._pos_guard.device_flag(dev)  # a bad position id is reported by the next step
        kv16 = self._prompt_operand(ctx, p, prompt_tokens.float(), prompt_position_ids, False, n, Lp, E, err)
        idx = cache.device_ints(slots)
        sl = idx.to(torch.int32)

        def prompt_kv(i, W):
            kv = eng.gemm(ctx, kv16, W["wkv"], p, want16=True)[1]
            self._scatter_prompt_kv(ctx, cache, sl, kv, i, n, Lp, E)
            return kv.hi, kv.lo, kv.ld, {}

        if L == 0:
            for i, W in enumerate(self._packed(ctx, p)):
                prompt_kv(i, W)
        else:
            x32 = torch.empty((n * L, E), dtype=torch.float32, device=dev)
            ctx.add_pos_embed(tokens, tokens.stride(1), tokens.stride(0), position_ids, self.positions_embed.weight.detach(), n, L, E,
                              out_f32=x32, err_flag=err)
            self._layers(ctx, p, x32, B=n, L=L, E=E, Lp=Lp, omask=mask_u8, pmask=prompt_mask_u8, prompt_kv=prompt_kv,
                         kv_scatter=(sl, cache))
        self._set_prompt_rows(cache, idx, prompt_mask_u8, Lp)
        ctx.slot_admit_history(sl, steps, Q, 0, mask_u8, actions, cache.Lmax, cache.mask, len_=cache.len, n_valid=cache.n_valid,
                               has_action=cache.has_action, active=cache.active, action_token=cache.action_token)

    # ---------------------------------------------------------------------------------------------
    def forward(
        self,
        *,
        obs_action_tokens: torch.Tensor,
        obs_action_position_ids: Optional[torch.Tensor] = None,
        prompt_tokens: torch.Tensor,
        prompt_mask: Optional[torch.Tensor] = None,
        prompt_position_ids: Optional[torch.Tensor] = None,
        batch_first: bool = False,
        obs_action_masks: Optional[torch.Tensor] = None,
        cache=None,
    ):
        """Reference signature (xattn_gpt.py:89-99) plus `cache`: with a DecodeCache the obs/action arguments describe only the
        tokens appended this step (their position ids are absolute) and the return value holds only their rows.  With a
        SlotDecodeCache they are one step block per slot as vima_slot_step_begin lays it out (the slots' prompts are in the cache;
        `prompt_tokens` is not read)."""
        ctx = eng.ctx_for(obs_action_tokens)
        p = eng.prec()
        slots = isinstance(cache, SlotDecodeCache)
        if not self._input_checked and cache is None:
            self._check_input(obs_action_tokens, prompt_tokens, prompt_mask, batch_first, obs_action_masks)
        dev = obs_action_tokens.device
        if batch_first:
            B, L, E = obs_action_tokens.shape
        else:
            L, B, E = obs_action_tokens.shape
        if slots:
            Lp = cache.Lp_cap
        else:
            Lp = prompt_tokens.shape[1] if batch_first else prompt_tokens.shape[0]
        assert E == self.embd_dim
        assert Lp <= self.xattn_n_positions and L <= self.n_positions
        if cache is not None:
            if obs_action_position_ids is None or obs_action_masks is None:
                raise ValueError("cached decode needs absolute position ids and masks for the appended tokens")
            if slots:
                cache.check_step(B, L - 1, E, p)
            else:
                check_cache_append(cache, B, L, E, p)
        if obs_action_tokens.dtype != torch.float32 or (not slots and prompt_tokens.dtype != torch.float32):
            raise TypeError("XAttnGPT expects float32 tokens (xattn_gpt.py:150,152)")
        tok = obs_action_tokens if obs_action_tokens.stride(-1) == 1 else obs_action_tokens.contiguous()
        sb, sl = (tok.stride(0), tok.stride(1)) if batch_first else (tok.stride(1), tok.stride(0))
        if obs_action_position_ids is None:
            obs_action_position_ids = self.position_ids[None, :L].expand(B, L)
        oa_ids = obs_action_position_ids.to(torch.int64).contiguous()
        if prompt_mask is not None and prompt_mask.dim() == 3:
            prompt_mask = prompt_mask.squeeze(1)
        if slots:
            pmask = cache.prompt_mask
        else:
            pmask = None if prompt_mask is None else eng.as_u8(prompt_mask)
        omask = None if obs_action_masks is None else eng.as_u8(obs_action_masks)
        if cache is not None and not slots:  # (the slot step's mask columns are written by vima_slot_step_begin)
            cache.mask[:, cache.L:cache.L + L].copy_(omask)

        M, H, Hx = B * L, self.n_head, self.xattn_n_head
        d_s, d_x = E // H, E // Hx
        self._pos_guard.poll()
        err = self._pos_guard.device_flag(dev)
        # x = tokens + positions_embed[ids] (fp32 residual stream); kv = prompt + xattn_positions_embed[ids] (operands only)
        x32 = torch.empty((M, E), dtype=torch.float32, device=dev)
        ctx.add_pos_embed(tok, sb, sl, oa_ids, self.positions_embed.weight.detach(), B, L, E, out_f32=x32, err_flag=err)
        need_prompt = cache is None or (not slots and cache.prompt_kv is None)
        kv16 = self._prompt_operand(ctx, p, prompt_tokens, prompt_position_ids, batch_first, B, Lp, E, err) if need_prompt else None
        self._pos_guard.after_launch()  # first call: synchronous check; later: asynchronous copy, reported by the next call
        if cache is None:
            self._input_checked = True

        layers = self._packed(ctx, p)
        if cache is not None and need_prompt:
            cache.prompt_kv = [eng.gemm(ctx, kv16, W["wkv"], p, want16=True)[1] for W in layers]

        def prompt_kv(i, W):
            if slots:  # each slot's prompt through its page table, prompt_len[b] keys
                return cache.prompt_kv_hi[i], cache.prompt_kv_lo[i], 2 * E, dict(kv_pages=cache.prompt_page_table,
                                                                                 kv_pool_pages=cache.prompt_pages.n_pages, kv_len=cache.prompt_len)
            kvp16 = cache.prompt_kv[i] if cache is not None else eng.gemm(ctx, kv16, W["wkv"], p, want16=True)[1]
            return kvp16.hi, kvp16.lo, kvp16.ld, {}

        x32 = self._layers(ctx, p, x32, B=B, L=L, E=E, Lp=Lp, omask=omask, pmask=pmask, prompt_kv=prompt_kv, cache=cache)
        if cache is not None and not slots:
            cache.L += L
        out = x32.view(B, L, E)
        return out if batch_first else out.transpose(0, 1)

    def _layers(self, ctx, p, x32, *, B, L, E, Lp, omask, pmask, prompt_kv, cache=None, kv_scatter=None) -> torch.Tensor:
        """The decoder stack over the residual stream x32 [B*L, E] (tokens + position embeddings) -> the last block's output [B*L, E]:
        per layer cross-attention to the prompt keys/values prompt_kv(layer, packed weights) -> (hi, lo, ld, paged attention
        arguments) under the key mask pmask, then the causal block (run_block with `cache` / `kv_scatter`)."""
        M, H, Hx = B * L, self.n_head, self.xattn_n_head
        d_x = E // Hx
        dev = x32.device
        layers = self._packed(ctx, p)
        lnw = lambda ln: (ln.weight.detach(), ln.bias.detach())
        # first layer's query LayerNorm; later ones are chained onto the previous block's LN2
        w, b = lnw(self.xattns[0].layernorm)
        _, _, qin16 = eng.norm(ctx, x32, p, rows=M, cols=E, w=w, b=b, eps=self.xattns[0].layernorm.eps, want16=True, out_f8=True)
        for i, (blk, xa, W) in enumerate(zip(self.h, self.xattns, layers)):
            # ---------------- XAttention ----------------
            _, q16 = eng.gemm(ctx, qin16, W["wq"], p, want16=True)
            khi, klo, kld, paged = prompt_kv(i, W)
            c16 = eng.Opnd(M, E, dev, p.split, f8=p.f8)
            ctx.attention(q=(q16.hi, q16.lo, q16.ld, 0), k=(khi, klo, kld, 0), v=(khi, klo, kld, E), o=(c16.hi, c16.lo, c16.ld, 0), B=B,
                          H=Hx, Lq=L, Lk=Lp, D=d_x, scale=1.0 / math.sqrt(d_x), causal=False, key_mask=pmask, dtype=p.dtype,
                          o8=None if c16.lo8 is None else (c16.lo8, c16.hi8), **paged)
            part = eng.stats_buffer(ctx, M, W["wo"], dev)
            a32, a16 = eng.gemm(ctx, c16, W["wo"], p, residual=x32, want_f32=True, want16=True, out_f8=True, stats_out=part)
            st = eng.row_stats_of(ctx, part, M, E, xa.ln.eps)
            _, h16 = eng.gemm(ctx, a16, W["w1g"] if "w1g" in W else W["w1"], p, act=_C.ACT_GELU, want16=True, out_f8=True, row_stats=st)
            xb32, xb16 = eng.gemm(ctx, h16, W["w2"], p, residual=a32, want_f32=True, want16=True, out_f8=True)
            del h16, a32, a16
            # ---------------- causal Block ----------------
            nxt = self.xattns[i + 1].layernorm if i + 1 < self.n_layer else None
            x32, qin16 = run_block(ctx, p, W, blk, xb32, xb16, c16, B=B, L=L, E=E, H=H, omask=omask, chain_ln=nxt, out_f32=x32, cache=cache,
                                   layer=i, kv_scatter=kv_scatter)
        return x32


class _OpenAIGPTModel(nn.Module):
    """Parameter holder with the key layout of the reference's OpenAIGPTModel (gpt.py:83-101)."""

    def __init__(self, vocab_size, n_positions, n_embd, n_layer, n_head, geglu):
        super().__init__()
        self.tokens_embed = nn.Embedding(vocab_size, n_embd)
        self.positions_embed = nn.Embedding(n_positions, n_embd)
        self.h = nn.ModuleList([Block(n_embd, n_positions, n_head, geglu) for _ in range(n_layer)])
        for blk in self.h:  # HF >= 4.3x keeps the causal buffer out of the state dict (checked against the reference here)
            buf = blk.attn._buffers.pop("bias")
            blk.attn.register_buffer("bias", buf, persistent=False)
        self.register_buffer("position_ids", torch.arange(n_positions))


class HFGPT(nn.Module):
    """Decoder-only GPT-1 stack, GEGLU or plain gelu_new MLPs (reference: vima/nn/seq_modeling/gpt/gpt.py:15-301) -- the VIMA-Gato baseline's
    sequence model.  Same Block kernels as XAttnGPT (causal-only path, BASELINE.json configs[4])."""

    def __init__(self, *, vocab_size=40478, n_positions=512, n_embd=768, n_layer=12, n_head=12, dropout: float = 0.1, use_geglu: bool = False):
        super().__init__()
        self.n_embd, self.n_layer, self.n_head, self.n_positions = n_embd, n_layer, n_head, n_positions
        self.lm = _OpenAIGPTModel(vocab_size, n_positions, n_embd, n_layer, n_head, use_geglu)
        for m in self.modules():
            if isinstance(m, (nn.Linear, nn.Embedding)):
                nn.init.normal_(m.weight, std=0.02)
        self._wc = eng.WeightCache(self)
        # checkpoints written with transformers 4.x carry `lm.h.N.attn.bias`; accept and ignore it
        self._register_load_state_dict_pre_hook(self._drop_causal_buffers)

    @staticmethod
    def _drop_causal_buffers(state_dict, prefix, *args):
        for k in [k for k in state_dict if k.startswith(prefix + "lm.h.") and k.endswith(".attn.bias")]:
            del state_dict[k]

    def forward(self, x: torch.Tensor, *, custom_mask: Optional[torch.Tensor] = None, position_ids: Optional[torch.Tensor] = None,
                batch_first: bool = False, cache=None):
        """x: (L,B,E) if not batch_first else (B,L,E); custom_mask (B,L) or (B,1,L) combined with the causal mask (gpt.py:46-79).
        With `cache` (DecodeCache or SlotDecodeCache, opened by `prefill`) x, custom_mask and absolute position_ids describe only the
        tokens appended this step and only their rows are returned: a DecodeCache takes their mask columns and advances `L`; for a
        SlotDecodeCache x is one step block per slot as vima_slot_step_begin lays it out (it has written the mask columns)."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        ctx = eng.ctx_for(x)
        p = eng.prec()
        if batch_first:
            B, L, E = x.shape
        else:
            L, B, E = x.shape
        assert E == self.n_embd and L <= self.n_positions
        slots = isinstance(cache, SlotDecodeCache)
        if cache is not None:
            if position_ids is None or custom_mask is None:
                raise ValueError("cached decode needs absolute position ids and masks for the appended tokens")
            if slots:
                cache.check_step(B, L - 1, E, p)
            else:
                check_cache_append(cache, B, L, E, p)
        omask = None
        if custom_mask is not None:
            if custom_mask.dim() == 3:
                custom_mask = custom_mask.squeeze(dim=1)
            omask = eng.as_u8(custom_mask != 0)
        if cache is not None and not slots:
            cache.mask[:, cache.L:cache.L + L].copy_(omask)
        out = self._stack(ctx, p, x, omask, position_ids, batch_first, cache=cache)
        if cache is not None and not slots:
            cache.L += L
        return out

    @torch.no_grad()
    def prefill(self, cache, slots: list, x: torch.Tensor, custom_mask_u8: torch.Tensor, position_ids: torch.Tensor, history=None) -> None:
        """Decoder-only prompt prefill.  x (L,n,E) holds n new sequences [prompt | separator] (custom_mask_u8 / position_ids (n,L);
        the separator, last, is valid).  They run through every block with local causal attention -- the arithmetic of `forward` --
        and after each layer's c_attn GEMM their keys / values go to cache columns [0, L) of slots[j] (vima_slot_kv_scatter; into the
        pages the slots take first for a SlotDecodeCache, whose earlier pages go back to the pool).  Then the mask columns [0, L)
        and the state are set: a SlotDecodeCache's by vima_slot_admit_prefix (len = L, n_valid = valid tokens, no action, active), a
        DecodeCache's (slots = all its rows, in order) by copying the mask and setting L and n_valid.  The caller has validated
        shapes, slots, capacity (for a SlotDecodeCache also check_prefix) and the precision mode.

        With `history` = (steps int32 [n] on the device, actions (T,n,E), Q, P) the n sequences are [prompt | separator | recorded
        history] of slot episodes admitted mid-way, padded to the longest (vima_slot_assemble_history; P = Lp+1 prefix columns, padding
        columns masked): the caller has taken their pages (SlotDecodeCache.reserve_history; padding columns past a slot's pages land
        on the zero page and are skipped), and vima_slot_admit_history sets the mask rows, state and fed-back actions."""
        eng.uses(self)  # fp32 parameters read by the kernels directly
        ctx = eng.ctx_for(x)
        p = eng.prec()
        L, n, E = x.shape
        if isinstance(cache, SlotDecodeCache):
            if history is None:
                cache.free_slots(slots, L)
            sl = cache.device_ints(slots).to(torch.int32)
        else:
            sl = torch.tensor(slots, dtype=torch.int32, device=x.device)
        self._stack(ctx, p, x, custom_mask_u8, position_ids, False, kv_scatter=(sl, cache))
        if history is not None:
            steps, actions, Q, P = history
            ctx.slot_admit_history(sl, steps, Q, P, custom_mask_u8, actions, cache.Lmax, cache.mask, len_=cache.len, n_valid=cache.n_valid,
                                   has_action=cache.has_action, active=cache.active, action_token=cache.action_token)
        elif isinstance(cache, SlotDecodeCache):
            ctx.slot_admit_prefix(sl, custom_mask_u8[:, :L - 1].contiguous(), cache.Lmax, cache.mask, len_=cache.len, n_valid=cache.n_valid,
                                  has_action=cache.has_action, active=cache.active)
            for b in slots:
                cache.len_host[b], cache.has_action_host[b], cache.active_host[b] = L, False, True
        else:
            cache.mask[:, :L].copy_(custom_mask_u8)
            cache.n_valid.copy_(custom_mask_u8.sum(dim=1))
            cache.L = L

    def _stack(self, ctx, p, x, omask, position_ids, batch_first, *, cache=None, kv_scatter=None):
        if batch_first:
            B, L, E = x.shape
        else:
            L, B, E = x.shape
        dev = x.device
        xf = x.float()
        if xf.stride(-1) != 1:
            xf = xf.contiguous()
        sb, sl = (xf.stride(0), xf.stride(1)) if batch_first else (xf.stride(1), xf.stride(0))
        if position_ids is None:
            position_ids = self.lm.position_ids[None, :L].expand(B, L)
        ids = position_ids.to(torch.int64).contiguous()
        M, H = B * L, self.n_head
        x32 = torch.empty((M, E), dtype=torch.float32, device=dev)
        x16 = eng.Opnd(M, E, dev, p.split, f8=p.f8)
        ctx.add_pos_embed(xf, sb, sl, ids, self.lm.positions_embed.weight.detach(), B, L, E, out_f32=x32, hi=x16.hi, lo=x16.lo, dtype=p.dtype)
        if p.f8:
            ctx.split_f8(x32, x16.lo8, x16.hi8)
        layers = self._wc.get("blocks", tuple(self.lm.h.parameters()), lambda: [pack_block(ctx, blk, p) for blk in self.lm.h])
        c16 = eng.Opnd(M, E, dev, p.split, f8=p.f8)
        for i, (blk, W) in enumerate(zip(self.lm.h, layers)):
            x32, x16 = run_block(ctx, p, W, blk, x32, x16, c16, B=B, L=L, E=E, H=H, omask=omask, want16=i + 1 < self.n_layer, cache=cache,
                                 layer=i, kv_scatter=kv_scatter)
        out = x32.view(B, L, E)
        return out if batch_first else out.transpose(0, 1)
