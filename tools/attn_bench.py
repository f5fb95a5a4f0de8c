"""GPU microbenchmark of decoder attention at the cfg3 shapes (B=256, H=24, d=32, L=263, Lp=256).

Environment: AB_B episodes, AB_L history keys (causal self-attention, Lq = Lk = L), AB_LP cross-attention keys (prompt tokens, Lq = L),
AB_LQ > 0 adds a decode case (AB_LQ new query rows over AB_L cached keys, queries last), AB_SPLIT formats, AB_MASKED.
--paged: the decode case also runs as slot decode does (per-element q_pos), from contiguous K/V and from a pool of 64-row pages
through a shuffled page table (seed 0), both printed (e.g. AB_LQ=33 AB_L=1024 python tools/attn_bench.py --paged).  --paged also
adds the slot step's cross-attention (AB_XQ = 33 query rows per slot over AB_LP prompt keys), timed three ways: contiguous, paged through
a shuffled page table, and paged with ragged per-slot key counts (kv_len uniform in 1..AB_LP, seed 0) as prompts of different lengths.
"""
import sys, os, math
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vima_b200 import _C
ctx = _C.Context.get(torch.device("cuda", 0))
B, H, D, L, Lp = int(os.environ.get("AB_B", 256)), 24, 32, int(os.environ.get("AB_L", 263)), int(os.environ.get("AB_LP", 256))
Ld = int(os.environ.get("AB_LQ", 0))
E = H * D
cases = [("self causal", L, L, True), ("cross", L, Lp, False)] + ([(f"decode Lq={Ld}", Ld, L, True)] if Ld > 0 else [])
if "--paged" in sys.argv:
    cases.append(("slot cross", int(os.environ.get("AB_XQ", 33)), Lp, False))
for split in [int(x) for x in os.environ.get("AB_SPLIT", "0,1").split(",")]:
    for name, Lq, Lk, causal in cases:
        mk = lambda r, c: torch.randint(-3000, 3000, (r, c), dtype=torch.int16, device="cuda")
        if causal and Lq < Lk:  # decode: the new rows' queries over the cached keys
            qq = mk(B * Lq, E); ql = mk(B * Lq, E) if split else None
            kv = mk(B * Lk, 2 * E); kl = mk(B * Lk, 2 * E) if split else None
            q = (qq, ql, E, 0); k = (kv, kl, 2 * E, 0); v = (kv, kl, 2 * E, E)
        elif causal:
            qkv = mk(B * Lq, 3 * E); qkl = mk(B * Lq, 3 * E) if split else None
            q = (qkv, qkl, 3 * E, 0); k = (qkv, qkl, 3 * E, E); v = (qkv, qkl, 3 * E, 2 * E)
        else:
            qq = mk(B * Lq, E); ql = mk(B * Lq, E) if split else None
            kv = mk(B * Lk, 2 * E); kl = mk(B * Lk, 2 * E) if split else None
            q = (qq, ql, E, 0); k = (kv, kl, 2 * E, 0); v = (kv, kl, 2 * E, E)
        o_hi = torch.empty(B * Lq, E, dtype=torch.int16, device="cuda"); o_lo = torch.empty_like(o_hi) if split else None
        mask = torch.ones(B, Lk, dtype=torch.uint8, device="cuda")
        if causal and os.environ.get("AB_MASKED", "1") == "1":  # the bench workload pads ~10 % of the history's object slots
            mask = (torch.rand(B, Lk, device="cuda") > 0.1).to(torch.uint8)
            mask[:, 0] = 1
        kw = dict(q=q, k=k, v=v, o=(o_hi, o_lo, E, 0), B=B, H=H, Lq=Lq, Lk=Lk, D=D, scale=1 / math.sqrt(D), causal=causal, key_mask=mask, dtype=0,
                  q_pos0=Lk - Lq if causal else 0)
        ctx.attention(**kw); torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5): ctx.attention(**kw)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        timed = [("", ms)]
        if "--paged" in sys.argv and causal and Lq < Lk:
            pl = -(-Lk // 64)
            perm = torch.randperm(B * pl, generator=torch.Generator().manual_seed(0)).to(torch.int32) + 1
            table = perm.view(B, pl).cuda()
            rows = (table.long()[:, torch.arange(Lk) // 64] * 64 + torch.arange(Lk, device="cuda") % 64).view(-1)
            pool = torch.zeros((B * pl + 1) * 64, 2 * E, dtype=torch.int16, device="cuda")
            pool_lo = torch.zeros_like(pool) if split else None
            pool[rows] = kv
            if split:
                pool_lo[rows] = kl
            qp = torch.full((B,), Lk - Lq, dtype=torch.int32, device="cuda")
            base = dict(kw, q_pos0=0, q_pos=qp, mask_ld=Lk)
            for label, extra in (("q_pos contiguous", dict(kv_batch_rows=Lk)),
                                 ("q_pos paged", dict(k=(pool, pool_lo, 2 * E, 0), v=(pool, pool_lo, 2 * E, E), kv_pages=table,
                                                      kv_pool_pages=B * pl + 1))):
                ctx.attention(**{**base, **extra}); torch.cuda.synchronize()
                e0.record()
                for _ in range(20): ctx.attention(**{**base, **extra})
                e1.record(); torch.cuda.synchronize()
                timed.append((" " + label, e0.elapsed_time(e1) / 20))
        if name == "slot cross":  # the prompt K/V as the slot cache keeps it: 64-row pages of a pool, prompt_len keys per slot
            pl = -(-Lk // 64)
            perm = torch.randperm(B * pl, generator=torch.Generator().manual_seed(0)).to(torch.int32) + 1
            table = perm.view(B, pl).cuda()
            rows = (table.long()[:, torch.arange(Lk) // 64] * 64 + torch.arange(Lk, device="cuda") % 64).view(-1)
            pool = torch.zeros((B * pl + 1) * 64, 2 * E, dtype=torch.int16, device="cuda")
            pool_lo = torch.zeros_like(pool) if split else None
            pool[rows] = kv
            if split:
                pool_lo[rows] = kl
            full = torch.full((B,), Lk, dtype=torch.int32, device="cuda")
            ragged = torch.randint(1, Lk + 1, (B,), generator=torch.Generator().manual_seed(0), dtype=torch.int32).cuda()
            paged = dict(kw, k=(pool, pool_lo, 2 * E, 0), v=(pool, pool_lo, 2 * E, E), kv_pages=table, kv_pool_pages=B * pl + 1)
            timed = []
            for label, args in (("contiguous", kw), ("paged", dict(paged, kv_len=full)), ("paged ragged kv_len", dict(paged, kv_len=ragged))):
                ctx.attention(**args); torch.cuda.synchronize()
                e0.record()
                for _ in range(20): ctx.attention(**args)
                e1.record(); torch.cuda.synchronize()
                timed.append((" " + label, e0.elapsed_time(e1) / 20))
            print(f"split={split} slot cross: ragged kv_len mean {ragged.float().mean().item():.1f} of {Lk} keys (the FLOP/s below count all {Lk})",
                  flush=True)
        # causal: the cached keys in full plus half the square of the new rows (half of Lq * Lk for Lq = Lk)
        pairs = Lq * (Lk - Lq) + Lq * Lq / 2 if causal else Lq * Lk
        fl = 4.0 * B * H * pairs * D
        for label, ms in timed:
            print(f"split={split} {name + label:12s} Lq={Lq:5d} Lk={Lk:5d} {ms:8.3f} ms   {fl/ms/1e9:7.1f} TF/s algorithmic (causal: visible half of the new rows' square)",
                  flush=True)
