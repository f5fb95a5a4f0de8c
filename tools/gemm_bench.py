"""GPU microbenchmark of the wgmma GEMM on the decoder's GEMM shapes (cfg3: M = 256*263).

GB_WIDE=1: the f16f8 decoder GEMMs with the context option gemm_wide = 0 and 1 alternated (GB_ROUNDS rounds of GB_REPS calls per
setting), with the card's name, power limit and the median SM clock sampled during the timed calls."""
import sys, os, math, json, statistics, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vima_b200 import _C
ctx = _C.Context.get(torch.device("cuda", 0))
M = int(os.environ.get("GB_M", 67328))


def wide_ab():
    """Median ms per call of each decoder GEMM on the 128-wide and the 128 x 256 kernel, and the operand bytes per call each
    kernel moves from L2 into shared memory (A once per n-tile, B once per m-tile; fp16 + 2 e4m3 bytes per element)."""
    rounds, reps = int(os.environ.get("GB_ROUNDS", 7)), int(os.environ.get("GB_REPS", 20))
    shapes = [  # (name, M, N, K, glu, epilogue kwargs)
        ("GEGLU LN-folded 6144x768", M, 6144, 768, 1, "o16_lna"),
        ("down proj 768x3072 +LN(res)", M, 768, 3072, 0, "res32_lnr"),
        ("QKV 2304x768", M, 2304, 768, 0, "o16"),
        ("out proj 768x768 +res +stats", M, 768, 768, 0, "res32_16_stats"),
        ("prompt K/V 1536x768", 65536, 1536, 768, 0, "o16"),
    ]
    info = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {info}", flush=True)
    clk = subprocess.Popen(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-lms", "200"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    try:
        for name, m, N, K, glu, epi in shapes:
            kw = make_kwargs(m, N, K, glu, epi, 2)
            times = {"0": [], "1": []}
            for w in ("0", "1"):  # warm both
                ctx.set_option("gemm_wide", w); ctx.gemm(**kw)
            torch.cuda.synchronize()
            for _ in range(rounds):
                for w in ("0", "1"):
                    ctx.set_option("gemm_wide", w)
                    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps): ctx.gemm(**kw)
                    e1.record(); torch.cuda.synchronize()
                    times[w].append(e0.elapsed_time(e1) / reps)
            t0, t1 = statistics.median(times["0"]), statistics.median(times["1"])
            tm = -(-m // 128)
            b128 = (tm * (N // 128) * 2 * 128 * K * 4)  # A and B tile bytes per tile: (128 + 128) rows x K x 4 B (fp16 + 2 x e4m3)
            b256 = (tm * (N // 256) * (128 + 256) * K * 4)
            fl = 2.0 * m * N * K
            print(f"{name:32s} M={m} 128-wide {t0:7.3f} ms ({b128 / t0 / 1e9:5.2f} TB/s L2->smem)  128x256 {t1:7.3f} ms "
                  f"({b256 / t1 / 1e9:5.2f} TB/s, {2 * fl / t1 / 1e9:6.1f} TF/s fp16-pass-equiv)  ratio {t1 / t0:.3f}  "
                  f"spread 128 {min(times['0']):.3f}-{max(times['0']):.3f} wide {min(times['1']):.3f}-{max(times['1']):.3f}", flush=True)
            del kw
    finally:
        ctx.set_option("gemm_wide", "1")
        clk.terminate(); out = clk.communicate(timeout=10)[0]
    mhz = [int(x) for x in out.split() if x.isdigit()]
    print(f"median SM clock during the timed calls: {statistics.median(mhz) if mhz else 'n/a'} MHz ({len(mhz)} samples)", flush=True)


def make_kwargs(M, N, K, glu, epi, split):
    a_hi = torch.randint(-2000, 2000, (M, K), dtype=torch.int16, device="cuda"); a_lo = torch.randint(-50, 50, (M, K), dtype=torch.int16, device="cuda") if split == 1 else None
    b_hi = torch.randint(-2000, 2000, (N, K), dtype=torch.int16, device="cuda"); b_lo = torch.randint(-50, 50, (N, K), dtype=torch.int16, device="cuda") if split == 1 else None
    f8 = {}
    if split == 2:
        mk8 = lambda r: torch.randint(0, 100, (r, K), dtype=torch.uint8, device="cuda")
        f8 = dict(a_lo8=mk8(M), a_hi8=mk8(M), b_hi8=mk8(N), b_lo8=mk8(N))
    n_out = N // 2 if glu else N
    kw = dict(M=M, N=N, K=K, a_hi=a_hi, a_lo=a_lo, lda=K, b_hi=b_hi, b_lo=b_lo, ldb=K, dtype=0, glu=glu, act=3 if (glu or epi == "mul16") else 0, **f8)
    if epi in ("res32_16", "res32", "res32_16_stats", "res32_lnr"): kw["residual"] = torch.zeros(M, n_out, device="cuda")
    if epi in ("res32_16", "res32", "o32", "res32_16_stats", "res32_lnr"): kw["out_f32"] = torch.empty(M, n_out, device="cuda")
    if epi == "mul16": kw["mul"] = torch.ones(M, n_out, device="cuda")
    if epi == "res32_16_stats": kw["stats_out"] = torch.empty(M, ctx.gemm_stats_parts(N, glu), 2, device="cuda")
    if epi == "o16_lna":
        kw["row_stats"] = torch.ones(M, 2, device="cuda"); kw["ln_c1"] = torch.zeros(N, device="cuda"); kw["ln_cols"] = 2
    if epi == "res32_lnr":
        kw["res_stats"] = torch.ones(M, 2, device="cuda"); kw["res_gamma"] = torch.ones(n_out, device="cuda"); kw["res_beta"] = torch.zeros(n_out, device="cuda")
    if epi in ("res32_16", "o16", "mul16", "res32_16_stats", "o16_lna"):
        kw["out_hi"] = torch.empty(M, n_out, dtype=torch.int16, device="cuda"); kw["out_lo"] = torch.empty_like(kw["out_hi"]) if split == 1 else None
        if split == 2:
            kw["out_lo8"] = torch.empty(M, n_out, dtype=torch.uint8, device="cuda"); kw["out_hi8"] = torch.empty_like(kw["out_lo8"])
    if glu: kw["block_n"] = 128
    return kw


if os.environ.get("GB_WIDE") == "1":
    wide_ab()
    sys.exit(0)
shapes = [  # (name, N_acc, K, glu, epilogue)
    ("q/out-proj N768 K768 +res f32+16", 768, 768, 0, "res32_16"),
    ("c_attn N2304 K768 ->16", 2304, 768, 0, "o16"),
    ("w1 N3072 K768 gelu*mul ->16", 3072, 768, 0, "mul16"),
    ("gate N3072 K768 ->f32", 3072, 768, 0, "o32"),
    ("fc_glu N6144 K768 ->16", 6144, 768, 1, "o16"),
    ("mlp_proj N768 K3072 +res f32", 768, 3072, 0, "res32"),
    # round 2: LayerNorm folded into the GEMMs
    ("wo/c_proj N768 K768 +res f32+16 +rowstats", 768, 768, 0, "res32_16_stats"),
    ("w1||gate N6144 K768 GEGLU, LN folded ->16", 6144, 768, 1, "o16_lna"),
    ("mlp_proj N768 K3072 +LN(res) f32", 768, 3072, 0, "res32_lnr"),
]
only = os.environ.get("GB_ONLY")
reps = int(os.environ.get("GB_REPS", 3))
splits = [int(x) for x in os.environ.get("GB_SPLIT", "0,1,2").split(",")]
for split in splits:
    for name, N, K, glu, epi in shapes:
        if only and only not in name: continue
        kw = make_kwargs(M, N, K, glu, epi, split)
        ctx.gemm(**kw); torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps): ctx.gemm(**kw)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        fl = 2.0 * M * N * K
        print(f"split={split} {name:40s} {ms:8.3f} ms  alg {fl/ms/1e9:8.1f} TF/s  tensor-work(fp16-pass-equiv) {fl*({0: 1, 1: 3, 2: 2}[split])/ms/1e9:8.1f} TF/s", flush=True)
        del kw
