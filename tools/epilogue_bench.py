"""Epilogue time of the 128 x 256 f16f8 GEMM (gemm_wide_kernel) on the decoder's GEMM shapes, measured by varying K.

Each CTA of the persistent kernel runs its tiles back to back: per tile a main loop whose time grows with K, then an epilogue
whose time does not.  So a GEMM of T tiles on S SMs takes t(K) = ceil(T / S) * (ML * K / 768 + E).  The script times every
shape at K = 384, 768 and 1152 (M = 67328, the prompt K/V GEMM 65536; median of EB_ROUNDS rounds of EB_REPS calls), fits a line
to t(K) by least squares and reports, per tile, the main loop per K = 768 (ML) and the epilogue (E), E's share of the call at
K = 768 and of the decoder's own K, and the bytes the epilogue moves (residual / multiplier reads, output writes) with the rate
they reach while it runs.  The card's name, power limit and the median SM clock during the timed calls are printed with them.

    python tools/epilogue_bench.py            # EB_ROUNDS=5 EB_REPS=10 by default
"""
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from vima_b200 import _C

M = 67328  # cfg3: 256 episodes x 263 tokens
KS = (384, 768, 1152)  # at K = 3072 the GEGLU / QKV weights outgrow L2 and the main loop stops being linear in K
SHAPES = [  # (name, M, N (accumulator columns), the decoder's K, GLU, epilogue)
    ("GEGLU 6144, LN folded -> f16f8", M, 6144, 768, 1, "o16_lna"),
    ("down proj 768, +LN(res) -> f32", M, 768, 3072, 0, "res32_lnr"),
    ("QKV 2304 -> f16f8", M, 2304, 768, 0, "o16"),
    ("out proj 768, +res +stats -> f32, f16f8", M, 768, 768, 0, "res32_16_stats"),
    ("prompt K/V 1536 -> f16f8", 65536, 1536, 768, 0, "o16"),
]


def make_kwargs(ctx, m, n, k, glu, epi):
    """Arguments of one f16f8 ctx.gemm call: random operands, the epilogue's inputs and outputs."""
    dev = "cuda"
    i16 = lambda r: torch.randint(-2000, 2000, (r, k), dtype=torch.int16, device=dev)
    u8 = lambda r: torch.randint(0, 100, (r, k), dtype=torch.uint8, device=dev)
    n_out = n // 2 if glu else n
    kw = dict(M=m, N=n, K=k, a_hi=i16(m), a_lo=None, lda=k, b_hi=i16(n), b_lo=None, ldb=k, dtype=0, glu=glu, act=3 if glu else 0,
              a_lo8=u8(m), a_hi8=u8(m), b_hi8=u8(n), b_lo8=u8(n))
    if epi.startswith("res32"):
        kw["residual"] = torch.randn(m, n_out, device=dev)
        kw["out_f32"] = torch.empty(m, n_out, device=dev)
    if epi == "res32_lnr":
        kw["res_stats"] = torch.ones(m, 2, device=dev)
        kw["res_gamma"] = torch.ones(n_out, device=dev)
        kw["res_beta"] = torch.zeros(n_out, device=dev)
    if epi == "res32_16_stats":
        kw["stats_out"] = torch.empty(m, ctx.gemm_stats_parts(n, glu), 2, device=dev)
    if epi == "o16_lna":
        kw["row_stats"] = torch.ones(m, 2, device=dev)
        kw["ln_c1"] = torch.zeros(n, device=dev)
        kw["ln_cols"] = 2
    if epi in ("o16", "o16_lna", "res32_16_stats"):
        kw["out_hi"] = torch.empty(m, n_out, dtype=torch.int16, device=dev)
        kw["out_lo8"] = torch.empty(m, n_out, dtype=torch.uint8, device=dev)
        kw["out_hi8"] = torch.empty_like(kw["out_lo8"])
    if glu:
        kw["block_n"] = 128
    return kw


def epilogue_bytes(m, n, glu, epi):
    """Global bytes the epilogue of one call moves: residual reads and output writes (row statistics and column vectors are
    under 1 % and left out)."""
    n_out = n // 2 if glu else n
    per = 0
    if epi.startswith("res32"):
        per += 4 + 4                       # fp32 residual in, fp32 out
    if epi in ("o16", "o16_lna", "res32_16_stats"):
        per += 2 + 1 + 1                   # fp16 hi + two e4m3 views
    return m * n_out * per


def main():
    rounds, reps = int(os.environ.get("EB_ROUNDS", 5)), int(os.environ.get("EB_REPS", 10))
    assert torch.cuda.is_available(), "epilogue_bench needs a GPU"
    ctx = _C.Context.get(torch.device("cuda", 0))
    ctx.set_option("gemm_wide", "1")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    info = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {info}; {sms} SMs", flush=True)
    clk = subprocess.Popen(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-lms", "200"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    try:
        for name, m, n, k_dec, glu, epi in SHAPES:
            tiles = -(-m // 128) * (n // 256)
            per_sm = -(-tiles // sms)
            ts = []
            for k in KS:
                kw = make_kwargs(ctx, m, n, k, glu, epi)
                ctx.gemm(**kw)
                torch.cuda.synchronize()
                times = []
                for _ in range(rounds):
                    e0 = torch.cuda.Event(enable_timing=True)
                    e1 = torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps):
                        ctx.gemm(**kw)
                    e1.record()
                    torch.cuda.synchronize()
                    times.append(e0.elapsed_time(e1) / reps)
                ts.append(statistics.median(times))
                del kw
            slope, icpt = np.polyfit(np.array(KS, dtype=float), np.array(ts), 1)  # ms per unit K, ms at K = 0
            resid = max(abs(t - (slope * k + icpt)) for k, t in zip(KS, ts))
            ml = slope * 768 / per_sm * 1e3                                      # us per tile per K = 768
            e = icpt / per_sm * 1e3                                              # us per tile
            t_dec = per_sm * (ml * k_dec / 768 + e) * 1e-3
            eb = epilogue_bytes(m, n, glu, epi)
            rate = eb / (icpt * 1e-3) / 1e12 if icpt > 0 else float("nan")
            print(f"{name:40s} tiles/SM {per_sm:3d}  t(K=384/768/1152) {ts[0]:6.3f} {ts[1]:6.3f} {ts[2]:6.3f} ms (fit residual {resid:5.3f})  "
                  f"ML {ml:5.1f} us  E {e:5.1f} us/tile  E share {e / (ml + e):4.0%} at K=768, "
                  f"{per_sm * e * 1e-3 / t_dec:4.0%} at K={k_dec}  epilogue {eb / 1e6:6.1f} MB at {rate:4.2f} TB/s", flush=True)
    finally:
        clk.terminate()
        out = clk.communicate(timeout=10)[0]
    mhz = [int(x) for x in out.split() if x.isdigit()]
    print(f"median SM clock during the timed calls: {statistics.median(mhz) if mhz else 'n/a'} MHz ({len(mhz)} samples)", flush=True)


if __name__ == "__main__":
    main()
