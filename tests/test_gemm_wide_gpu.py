"""The 128 x 256 f16f8 GEMM (gemm_wide_kernel) against fp64, against the 128-wide kernel, and across operand magnitudes.

vima_gemm runs an f16f8 GEMM on the wide kernel when the context option gemm_wide is on (the default), its tiles are 128 wide and
N % 256 == 0.  The wide kernel carries the e4m3 cross terms in an fp16 accumulator (the hi*hi sum stays fp32), so its results
differ from the 128-wide kernel's by that sum's rounding only, and fp16's range is the one new risk.

  1. Every specialised epilogue against fp64 at the f16f8 bars, with sentinels past M and N, at K = 32, 64, 96, 392 (ragged), 768
     and 3072 (1 to 96 k blocks: tiles that end mid-ring and a producer a tile ahead), M not a multiple of 128, and grids where a
     CTA walks 1, 2 and many tiles.  Each GEMM also runs with gemm_wide = 0 on the same inputs: the fp32 outputs agree to rel-L2 2e-6
     (measured worst 5.9e-7), the fp16 + e4m3 views to 1e-5 (5.1e-6), and the row-statistics parts sit in the same places.
  2. The operand-magnitude rows of test_numeric_range_gpu.py (2^-16 .. 2^12, outlier channels, mean 1e3) through both kernels:
     the wide kernel stays finite and holds the f16f8 bar wherever the 128-wide kernel does.
  3. The kernel that runs: gemm_wide_kernel with the option on, gemm_tc_kernel with it off or for a shape it does not take.
"""
import math

import pytest
import torch

from tests.test_kernel_variants_gpu import GemmOperands, VARIANTS, _row_id, assert_canary, rel, run_gemm_variant, sentinel
from tests.test_numeric_range_gpu import F8_LIMIT, GEMM_BAR, decoded_a, magnitude_rows

OUTS = ("out_f32", "out_hi", "out_lo8", "out_hi8", "stats_out")
AB_BAR = 2e-6  # rel-L2 between the two kernels' fp32 outputs and row statistics: the fp16 carry of the cross terms (~2^-22)
# fp16 hi + e4m3 lo8 outputs are rounded twice: a last-bit change of the fp32 value can move hi by one fp16 ulp, and lo8 (3 mantissa
# bits) takes the new residual back only to ~2^-4 of it, so the two reconstructions differ by up to the format's own step
AB_BAR_F8_VIEWS = 1e-5


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    c = _C.Context.get(torch.device("cuda", 0))
    yield c
    c.set_option("gemm_wide", "1")


class BothKernels:
    """A Context whose gemm() runs every call twice on the same inputs: on the 128-wide kernel into copies of the output buffers
    (sentinels included), then on the wide kernel into the caller's buffers.  The pairs are kept for comparison."""

    def __init__(self, ctx):
        self.ctx, self.pairs = ctx, []

    def __getattr__(self, name):
        return getattr(self.ctx, name)

    def gemm(self, **kw):
        narrow = {k: kw[k].clone() for k in OUTS if kw.get(k) is not None}
        try:
            self.ctx.set_option("gemm_wide", "0")
            self.ctx.gemm(**{**kw, **narrow})
        finally:
            self.ctx.set_option("gemm_wide", "1")
        self.ctx.gemm(**kw)
        self.pairs.append((kw, narrow))


def compare_kernels(pairs, M, what):
    errs = {}
    for kw, narrow in pairs:
        n = kw["N"] // 2 if kw["glu"] else kw["N"]  # output columns; past them both buffers keep their sentinels (NaN in fp32)
        for k, t in narrow.items():
            wide = kw[k]
            if k == "stats_out":  # the same parts written, the same sentinels left
                assert torch.equal(wide.view(torch.int32) == 0x7FBADBAD, t.view(torch.int32) == 0x7FBADBAD), what
                errs[k] = max(errs.get(k, 0.0), rel(wide[:M], t[:M]))
            if k == "out_f32":
                errs[k] = max(errs.get(k, 0.0), rel(wide[:M, :n], t[:M, :n]))
        if kw.get("out_lo8") is not None:  # fp16 hi + lo8 / 2^10 as the next GEMM reads it
            rec = lambda h, l8: h[:M, :n].view(torch.float16).double() + l8[:M, :n].view(torch.float8_e4m3fn).double() / 1024.0
            errs["hi16+lo8"] = max(errs.get("hi16+lo8", 0.0), rel(rec(kw["out_hi"], kw["out_lo8"]), rec(narrow["out_hi"], narrow["out_lo8"])))
    for k, e in errs.items():
        assert e < (AB_BAR_F8_VIEWS if k == "hi16+lo8" else AB_BAR), (what, errs)  # also false for NaN
    return errs


# (M, n_out, K): num_kb = 1, 2, 3 (a tile ends mid-ring), 13 (ragged K), 24, 96; 1 to 114 tiles (one per CTA), 133 tiles (one CTA
# walks two) and 471 tiles (every CTA walks 3 or 4, the producer a tile ahead of the epilogue)
WIDE_SHAPES = [(1, 256, 768), (200, 512, 32), (300, 256, 64), (130, 768, 96), (515, 256, 392), (4741, 768, 768), (257, 512, 3072),
               (17000, 256, 96), (20000, 768, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("row", VARIANTS, ids=[f"v{i:02d}-{_row_id(r)}" for i, r in enumerate(VARIANTS)])
def test_wide_gemm_variant(ctx, row):
    glu = row[1]
    worst = {}
    for i, (M, n, K) in enumerate(WIDE_SHAPES):
        n_out = n // 2 if glu else n  # accumulator columns N = n either way: a multiple of 256
        both = BothKernels(ctx)
        errs = run_gemm_variant(both, row, "f16f8", M, n_out, K, 0, seed=500 + i)
        errs.update({"ab " + k: v for k, v in compare_kernels(both.pairs, M, f"{row} M={M} N={n} K={K}").items()})
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
    print(f"wide gemm {_row_id(row)}: " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))


@pytest.mark.gpu
def test_wide_gemm_operand_magnitudes(ctx):
    """The rows of test_gemm_operand_magnitudes through both kernels at K = 768, 392 and 3072: finite everywhere, and the f16f8 bar
    held by the wide kernel on every row group where the 128-wide kernel holds it (lo8-saturated rows, max|x| >= 1024, excepted)."""
    bar = GEMM_BAR["f16f8"]
    failures, lines = [], []
    for K, seed in ((768, 11), (392, 12), (3072, 13)):
        A, names = magnitude_rows(K, seed)
        M, N = A.shape[0], 256
        g = torch.Generator(device="cuda").manual_seed(seed + 100)
        W = torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
        ops = GemmOperands(ctx, A, W, "f16f8")
        out = {}
        for wide in ("0", "1"):
            ctx.set_option("gemm_wide", wide)
            out[wide] = sentinel((M + 3, N + 8), "f32")
            ctx.gemm(M=M, N=N, K=K, out_f32=out[wide], **ops.kwargs())
        ctx.set_option("gemm_wide", "1")
        torch.cuda.synchronize()
        ref = A.double() @ W.double().t()
        fmt = decoded_a(ops, "f16f8") @ W.double().t()
        for wide in out:
            assert_canary(out[wide], M, N, f"gemm_wide={wide} K={K}")
        for i, name in enumerate(names):
            r = slice(i * 8, (i + 1) * 8)
            amax = A[r].abs().max().item()
            gw, gn = out["1"][:M, :N][r], out["0"][:M, :N][r]
            ew, en, ef = rel(gw, ref[r]), rel(gn, ref[r]), rel(fmt[r], ref[r])
            lines.append(f"  {str(name):>18} {K:>5} {amax:>9.3g} {en:>9.2e} {ew:>9.2e} {rel(gw, gn):>9.2e} {ef:>9.2e}")
            if not torch.isfinite(gw).all():
                failures.append(f"K={K} rows {name}: non-finite output from the wide kernel")
            elif amax < F8_LIMIT and en < bar <= ew:
                failures.append(f"K={K} rows {name} (max|x| {amax:.3g}): wide {ew:.2e} over the bar, 128-wide {en:.2e}")
    print(f"\nf16f8 rel-L2 against fp64 by row scale, 128-wide and wide kernels:\n  {'rows':>18} {'K':>5} {'max|x|':>9} {'128':>9} "
          f"{'wide':>9} {'wide/128':>9} {'format':>9}\n" + "\n".join(lines))
    assert not failures, "\n".join(failures)


def _kernels(ctx, **kw):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.gemm(**kw)
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if "gemm" in e.name}


@pytest.mark.gpu
def test_wide_gemm_dispatch(ctx):
    M, K = 300, 256
    A = torch.randn(M, K, device="cuda")
    for N, bn, wide, want in ((768, 0, "1", "gemm_wide_kernel"), (768, 0, "0", "gemm_tc_kernel"), (640, 0, "1", "gemm_tc_kernel"),
                              (768, 64, "1", "gemm_tc_kernel")):
        ops = GemmOperands(ctx, A, torch.randn(N, K, device="cuda") / 16, "f16f8")
        ctx.set_option("gemm_wide", wide)
        try:
            names = _kernels(ctx, M=M, N=N, K=K, out_f32=torch.empty(M, N, device="cuda"), block_n=bn, **ops.kwargs())
        finally:
            ctx.set_option("gemm_wide", "1")
        assert len(names) == 1 and want in next(iter(names)), (N, bn, wide, names)
    with pytest.raises(RuntimeError):
        ctx.set_option("gemm_wide", "2")
