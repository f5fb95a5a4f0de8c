"""The GEMM epilogue's derived outputs, bit for bit, against the fp32 output of the same call.

Every value epilogue_tile (gemm_tc.cuh) derives from a row's fp32 result is a deterministic function of that result: the operand
views of the next GEMM ((hi, lo) 16-bit pairs, or fp16 hi + the two e4m3 cross-term views in f16f8) and the per-row partial
(sum, sum of squares) that folded LayerNorms finalize into (mean, rstd).  So each is checked exactly against out_f32 from the
same call, with no tolerance:

  1. stats_statement() writes out the summation tree documented above epilogue_tile: per 4-column group q1 = (o0 + o1) + (o2 + o3)
     and q2 = fma(o0, o0, o1*o1) + fma(o2, o2, o3*o3); per statistics half (the chunks of one parity of an n-tile) and per group
     index kc in 0..3, S_kc = (...((+0 + q(k0, kc)) + q(k0, kc + 4)) + q(k1, kc)) + q(k1, kc + 4) ... over the half's 32-column
     chunks in ascending order; then (S0 + S1) + (S2 + S3).
  2. A sweep over every operand mode, tile width (32, 64, 96, 128, GLU 64 and 128), both f16f8 kernels (gemm_tc_kernel with
     gemm_wide = 0, gemm_wide_kernel), the specialised and generic epilogues that emit statistics or (fp32, 16-bit) pairs, M at
     every row residue of the transposed layout (rows 4*it + rq) and tile boundary, last n-tiles that end at every 4-column
     residue that exercises partial and dead chunks of both parities, and epi_prefetch 0 / 1: stats_out, the views and every
     sentinel bit for bit.
  3. The O16-only specialised epilogues against the generic one: the same descriptor with out_f32 added runs the generic
     variant, and the specialised call's views must be the statement of that fp32 output.
  4. Rows with large means through vima_row_stats_finalize: the mean bit for bit against the finalize kernel's fp64 statement,
     rstd within 2 fp32 ulp of rsqrt of its variance, and both the variance and rstd within DESIGN.md §5's bound
     1e-6 * (1 + mean^2 / var) of the fp64 statistics of the fp32 rows.
"""
import math

import pytest
import torch

from tests.test_gemm_schedule_gpu import fma32
from tests.test_kernel_variants_gpu import (ACT, MODES, VARIANTS, GemmOperands, as_bits16, assert_canary, f8_statement, fold_ln,
                                            interleave, sentinel, split_statement)

F8_LO_SCALE, F8_HI_SCALE = 1024.0, 0.125  # F8_ACT_LO_SCALE / F8_ACT_HI_SCALE (common.cuh): the e4m3 views of an activation


# ------------------------------------------------------------------------------------------------------------------------------
# 1. the statement of the row-statistics partials
# ------------------------------------------------------------------------------------------------------------------------------
def stats_statement(o, M, n_out, bn_out, parts):
    """fp32 [M, parts, 2] partial (sum, sum of squares) of the fp32 output rows o[:M, :n_out], in epilogue_tile's summation tree.

    Column c lies in n-tile t = c // bn_out and 32-column chunk k = (c % bn_out) // 32 of it; its part is 2t + (k & 1).  (The
    wide kernel's 256-wide tiles are two 128-wide tiles here: pass its 128-wide bn_out.)  Columns at or past n_out add +0; a
    half without columns is (+0, +0).  fp32 rounding throughout, fma correctly rounded (fma32)."""
    tiles = parts // 2
    assert parts == 2 * tiles and tiles == -(-n_out // bn_out) and bn_out % 32 == 0, (n_out, bn_out, parts)
    nch = bn_out // 32
    x = torch.zeros(M, tiles * bn_out, dtype=torch.float32, device=o.device)
    x[:, :n_out] = o[:M, :n_out]
    o0, o1, o2, o3 = x.view(M, tiles, nch, 8, 4).unbind(-1)  # [row, tile, chunk, 4-column group of the chunk]
    q1 = (o0 + o1) + (o2 + o3)
    q2 = fma32(o0, o0, o1 * o1) + fma32(o2, o2, o3 * o3)
    out = torch.zeros(M, tiles, 2, 2, dtype=torch.float32, device=o.device)
    for half in (0, 1):
        s = [torch.zeros(M, tiles, 4, dtype=torch.float32, device=o.device) for _ in range(2)]
        for k in range(half, nch, 2):
            for j, q in enumerate((q1, q2)):
                s[j] = (s[j] + q[:, :, k, :4]) + q[:, :, k, 4:]  # groups kc and kc + 4: the chunk's two 16-column halves
        for j in range(2):
            out[:, :, half, j] = (s[j][..., 0] + s[j][..., 1]) + (s[j][..., 2] + s[j][..., 3])
    return out.view(M, parts, 2)


def stats_difference(got, want, bn_out):
    """None if the int32 bit patterns agree, else where they first differ in (row, part) terms."""
    bad = (got.view(torch.int32) != want.view(torch.int32)).any(-1)
    if not bad.any():
        return None
    r, p = bad.nonzero()[0].tolist()
    t, h = p // 2, p % 2
    return (f"stats_out: {int(bad.sum())} of {bad.numel()} (row, part) entries differ from the documented tree; first at row {r} "
            f"part {p} (n-tile {t}, {('even', 'odd')[h]} chunks from column {t * bn_out}): got (sum, sumsq) = "
            f"({got[r, p, 0].item()!r}, {got[r, p, 1].item()!r}), want ({want[r, p, 0].item()!r}, {want[r, p, 1].item()!r})")


def bits_difference(got, want, x, what):
    """None if the bit patterns agree, else the first differing (row, column) with its fp32 value."""
    bad = got != want
    if not bad.any():
        return None
    i = tuple(bad.nonzero()[0].tolist())
    return (f"{what}: {int(bad.sum())} elements differ; first at {i}: out_f32 = {x[i].item()!r}, got 0x{int(got[i]):x}, "
            f"want 0x{int(want[i]):x}")


# ------------------------------------------------------------------------------------------------------------------------------
# 2. the sweep
# ------------------------------------------------------------------------------------------------------------------------------
# (ACT, GLU, MUL, RES, O32, O16, LNA, LNR, STATS), in the order of test_kernel_variants_gpu.VARIANTS; "v.." names a row of
# VIMA_GEMM_VARIANTS by its index, everything else runs the generic runtime-flag epilogue (test_gemm_epilogue_bits_cpu.py checks both)
EPILOGUES = {
    "v02-res-o32-o16-stats": ("ACT_NONE", 0, 0, 1, 1, 1, 0, 0, 1),
    "generic-relu-mul-o32-stats": ("ACT_RELU", 0, 1, 0, 1, 0, 0, 0, 1),
    "generic-none-lna-o32-stats": ("ACT_NONE", 0, 0, 0, 1, 0, 1, 0, 1),
    "generic-quickgelu-res-o32-o16-stats": ("ACT_QUICKGELU", 0, 0, 1, 1, 1, 0, 0, 1),
    "v01-res-o32-o16": ("ACT_NONE", 0, 0, 1, 1, 1, 0, 0, 0),
    "generic-relu-mul-o32-o16": ("ACT_RELU", 0, 1, 0, 1, 1, 0, 0, 0),
    "generic-gelu-glu-o32-o16-stats": ("ACT_GELU", 1, 0, 0, 1, 1, 0, 0, 1),
}
FLAT_EPIS = [k for k, r in EPILOGUES.items() if not r[1]]
GLU_EPIS = [k for k, r in EPILOGUES.items() if r[1]]
WIDE_EPIS = ["v02-res-o32-o16-stats", "v01-res-o32-o16"]  # gemm_wide_kernel takes the specialised epilogues only
WIDTHS = ["32", "64", "96", "128", "glu64", "glu128"]
# rows 4*it + rq of a 16-row warp slice: every residue of M mod 4 and mod 16, the warp-row and 64-row warpgroup boundaries, the
# 128-row tile boundary, and 38 m-tiles (with several n-tiles, more tiles than SMs: CTAs walk several)
M_LIST = [1, 3, 4, 5, 15, 16, 17, 63, 64, 65, 127, 129, 4741]
# where the last n-tile ends: partial 16-column halves, partial 32-column chunks and whole dead chunks of either parity
RESIDUES = [4, 8, 12, 16, 20, 28, 32, 36, 60, 64, 68, 92, 96, 100, 124]
EXTRA_TILES = [0, 1, 2, 5]  # n-tiles before the last one
GLU_TILES = [1, 2, 7]
K_LIST = [64, 200]  # the epilogue does not see K; 200 ends in a partial k block
SWEEP_GROUPS = MODES + ["f16f8-wide"]


def width_of(key):
    glu = key.startswith("glu")
    return glu, int(key[3:] if glu else key)


def sweep_cases(group):
    """The cases of one mode (or of the wide f16f8 kernel): dicts of mode, wide, width, bn, glu, epi, M, n_out, K, prefetch,
    residue (None in GLU and wide cases).  Deterministic; every (mode, width) runs every residue below its tile width, and each
    width walks M_LIST, the epilogues and epi_prefetch across the modes."""
    out = []
    if group == "f16f8-wide":  # N % 256 == 0: whole 256-wide tiles
        for i, (M, tiles256) in enumerate(((1, 1), (5, 3), (17, 2), (64, 5), (129, 1), (4741, 3), (4741, 5), (63, 2))):
            out.append(dict(mode="f16f8", wide=True, width="128", bn=128, glu=False, epi=WIDE_EPIS[i % 2], M=M, n_out=256 * tiles256,
                            K=K_LIST[i % 2], prefetch=(i // 2) % 2, residue=None))
        return out
    mi = MODES.index(group)
    big = M_LIST[-1]  # with the most n-tiles: more tiles than SMs
    for wi, key in enumerate(WIDTHS):
        glu, bn = width_of(key)
        if glu:
            for j, tiles in enumerate(GLU_TILES):
                n = len(GLU_TILES) * mi + j
                M = M_LIST[(n * 5 + wi) % len(M_LIST)]
                out.append(dict(mode=group, wide=False, width=key, bn=bn, glu=True, epi=GLU_EPIS[0], M=M,
                                n_out=(GLU_TILES[-1] if M == big else tiles) * bn // 2, K=K_LIST[n % 2], prefetch=0, residue=None))
            continue
        rs = [r for r in RESIDUES if r <= bn]
        for j, r in enumerate(rs):
            n = len(rs) * mi + j  # this width's running case index across the modes
            M = M_LIST[n % len(M_LIST)]
            extra = EXTRA_TILES[-1] if M == big else EXTRA_TILES[(n + wi) % len(EXTRA_TILES)]
            out.append(dict(mode=group, wide=False, width=key, bn=bn, glu=False, epi=FLAT_EPIS[(j + mi) % len(FLAT_EPIS)], M=M,
                            n_out=extra * bn + r, K=K_LIST[n % 2], prefetch=(n // len(FLAT_EPIS)) % 2, residue=r))
    return out


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    return _C.Context.get(torch.device("cuda", 0))


@pytest.fixture
def options(ctx):
    """Sets gemm_wide / epi_prefetch per call; the finaliser puts back the defaults (1 and 0)."""
    yield lambda wide, prefetch: (ctx.set_option("gemm_wide", str(int(wide))), ctx.set_option("epi_prefetch", str(int(prefetch))))
    ctx.set_option("gemm_wide", "1")
    ctx.set_option("epi_prefetch", "0")


class Problem:
    """One GEMM's inputs for an epilogue row: operands in `mode`, bias, and the multiplier / residual / folded-LayerNorm vectors
    the row reads.  launch() runs it into fresh sentinel-filled outputs."""

    def __init__(self, ctx, row, mode, M, n_out, K, bn, seed, ln_cols=1):
        act_name, glu, mul, res, o32, o16, lna, lnr, stats = row
        assert not lnr
        g = torch.Generator(device="cuda").manual_seed(seed)
        rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
        A = rn(M, K) * 2.0 + 0.7 if lna else rn(M, K)
        Wv, bv = rn(n_out, K) / math.sqrt(K), 0.5 * rn(n_out)
        Wg, bg = rn(n_out, K) / math.sqrt(K), 0.5 * rn(n_out)
        self.kw = {}
        if lna:
            gam, bet = 1.0 + 0.1 * rn(K), 0.1 * rn(K)
            Wv, c1v, bv = fold_ln(Wv, bv, gam, bet)
            if ln_cols == 1:  # both halves of a GLU tile read the normalised rows
                Wg, c1g, bg = fold_ln(Wg, bg, gam, bet)
            else:
                c1g = torch.zeros_like(c1v)
            A64 = A.double()
            st = torch.stack([A64.mean(1), 1.0 / torch.sqrt(A64.var(1, unbiased=False) + 1e-5)], 1).float().contiguous()
            self.kw.update(row_stats=st, ln_c1=interleave(c1v, c1g, bn) if glu else c1v, ln_cols=ln_cols)
        W, bias = (interleave(Wv, Wg, bn), interleave(bv, bg, bn)) if glu else (Wv, bv)
        self.N = W.shape[0]
        assert self.N == (2 * n_out if glu else n_out), "GLU cases take whole tiles"
        self.ops = GemmOperands(ctx, A, W, mode)
        self.kw.update(bias=bias, mul=rn(M, n_out + 4)[:, :n_out] if mul else None,
                       residual=(rn(M, n_out + 4) * 2.0 + 0.7)[:, :n_out] if res else None)
        self.ctx, self.row, self.M, self.n_out, self.K, self.bn, self.glu = ctx, row, M, n_out, K, bn, glu
        self.parts = ctx.gemm_stats_parts(self.N, glu, bn)

    def launch(self, o32, o16, stats):
        M, n = self.M, self.n_out
        out = {}
        if o32:
            out["out_f32"] = sentinel((M + 3, n + 8), "f32")
        if o16:
            out["out_hi"] = sentinel((M + 3, n + 8), "i16")
            if self.ops.f8:
                out["out_lo8"], out["out_hi8"] = sentinel((M + 3, n + 16), "u8"), sentinel((M + 3, n + 16), "u8")
            else:
                out["out_lo"] = sentinel((M + 3, n + 8), "i16")
        if stats:
            out["stats_out"] = sentinel((M + 3, self.parts, 2), "f32")
        self.ctx.gemm(M=M, N=self.N, K=self.K, glu=self.glu, act=ACT[self.row[0]], block_n=self.bn, **out, **self.ops.kwargs(), **self.kw)
        return out

    def check_outputs(self, out, x):
        """Sentinels past row M and column n_out (past parts in stats_out), then the views of out against their statements of the
        fp32 rows x.  -> list of failure strings."""
        M, n = self.M, self.n_out
        fails = []
        for name, t in out.items():
            try:
                if name == "stats_out":
                    assert_canary(t.view(M + 3, self.parts * 2), M, self.parts * 2, name)
                else:
                    assert_canary(t, M, n, name)
            except AssertionError as e:
                fails.append(str(e))
        if "out_hi" in out:
            if self.ops.f8:
                wl, wh = f8_statement(x, F8_LO_SCALE, F8_HI_SCALE)
                views = (("out_hi", as_bits16(out["out_hi"][:M, :n]), split_statement(x, 0)[0]),
                         ("out_lo8", out["out_lo8"][:M, :n].to(torch.int32), wl), ("out_hi8", out["out_hi8"][:M, :n].to(torch.int32), wh))
            else:
                hb, lb = split_statement(x, self.ops.dt)
                views = (("out_hi", as_bits16(out["out_hi"][:M, :n]), hb), ("out_lo", as_bits16(out["out_lo"][:M, :n]), lb))
            for name, got, want in views:
                msg = bits_difference(got, want, x, name)
                if msg:
                    fails.append(msg)
        return fails


def describe(c):
    return (f"{c['mode']}{' wide' if c['wide'] else ''} bn={c['width']} {c['epi']} M={c['M']} n_out={c['n_out']} K={c['K']} "
            f"epi_prefetch={c['prefetch']}")


def run_sweep_case(ctx, set_options, case, seed):
    """One call writing out_f32 and the row's other outputs -> list of failure strings."""
    row = EPILOGUES[case["epi"]]
    pb = Problem(ctx, row, case["mode"], case["M"], case["n_out"], case["K"], case["bn"], seed)
    set_options(case["wide"], case["prefetch"])
    out = pb.launch(o32=True, o16=row[5], stats=row[8])
    torch.cuda.synchronize()
    x = out["out_f32"][: case["M"], : case["n_out"]]
    fails = [] if torch.isfinite(x).all() else ["out_f32 is not finite"]
    fails += pb.check_outputs(out, x)
    if row[8]:
        bn_out = case["bn"] // 2 if case["glu"] else case["bn"]  # the wide kernel's halves are these 128-wide tiles
        want = stats_statement(x, case["M"], case["n_out"], bn_out, pb.parts)
        msg = stats_difference(out["stats_out"][: case["M"]], want, bn_out)
        if msg:
            fails.append(msg)
    return fails


@pytest.mark.gpu
@pytest.mark.parametrize("group", SWEEP_GROUPS)
def test_epilogue_outputs_are_statements_of_out_f32(ctx, options, group):
    cases = sweep_cases(group)
    failures = []
    for i, case in enumerate(cases):
        fails = run_sweep_case(ctx, options, case, seed=1000 * SWEEP_GROUPS.index(group) + i)
        failures += [f"{describe(case)}: {f}" for f in fails]
    print(f"\nepilogue bits {group}: {len(cases)} cases, {len(failures)} failures")
    assert not failures, f"{len(failures)} failures:\n" + "\n".join(failures[:40])


# ------------------------------------------------------------------------------------------------------------------------------
# 3. the O16-only specialised epilogues against the generic one
# ------------------------------------------------------------------------------------------------------------------------------
SPECIALISED_O16 = [0, 4, 7, 8, 9, 10, 11]  # the VARIANTS rows with a 16-bit output and no fp32 one


def specialised_cases(idx):
    """(M, n_out, bn, ln_cols) per specialised row: a few M and last-tile residues on every tile width the row takes."""
    glu = VARIANTS[idx][1]
    if glu:
        return [(5, 32, 64, 1), (129, 192, 128, 2), (4741, 128, 64, 2), (17, 448, 128, 1)]
    return [(1, 32 + 4, 32, 1), (17, 64 + 36, 64, 1), (65, 2 * 96 + 68, 96, 1), (4741, 5 * 128 + 124, 128, 1), (127, 128, 128, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("idx", SPECIALISED_O16, ids=[f"v{i:02d}" for i in SPECIALISED_O16])
def test_specialised_views_equal_the_generic_formula(ctx, options, idx):
    """The specialised call's views are the statement of the fp32 output of the same descriptor with out_f32 added (which runs
    the generic epilogue), in every mode; gemm_tc_kernel only (gemm_wide = 0: the wide kernel has no generic epilogue)."""
    row = VARIANTS[idx]
    failures, n = [], 0
    for mode in MODES:
        for j, (M, n_out, bn, ln_cols) in enumerate(specialised_cases(idx)):
            pb = Problem(ctx, row, mode, M, n_out, 64, bn, seed=100 * idx + 10 * MODES.index(mode) + j, ln_cols=ln_cols)
            options(False, j % 2)
            spec = pb.launch(o32=False, o16=True, stats=False)
            gen = pb.launch(o32=True, o16=True, stats=False)
            torch.cuda.synchronize()
            x = gen["out_f32"][:M, :n_out]
            fails = pb.check_outputs(spec, x) + [f"generic call: {f}" for f in pb.check_outputs(gen, x)]
            failures += [f"v{idx:02d} {mode} bn={bn} M={M} n_out={n_out} ln_cols={ln_cols}: {f}" for f in fails]
            n += 1
    print(f"\nv{idx:02d} specialised vs generic: {n} pairs, {len(failures)} failures")
    assert not failures, "\n".join(failures[:40])


# ------------------------------------------------------------------------------------------------------------------------------
# 4. rows with large means through vima_row_stats_finalize
# ------------------------------------------------------------------------------------------------------------------------------
LARGE_MEANS = (0.0, 1.0, 10.0, 100.0, 300.0)
VAR_COEF = 1e-6  # DESIGN.md §5: the variance's relative error is about VAR_COEF * (1 + mean^2 / var)


def finalize_statement(partial, cols, eps):
    """The finalize kernel in fp64: sums over the parts in order, mean = s1 * (1 / cols), var = max(s2 * (1 / cols) - mean^2, 0);
    -> (mean rounded to fp32, var fp64, the fp32 rstd argument (float)var + eps)."""
    p = partial.double()
    s1 = torch.zeros(p.shape[0], dtype=torch.float64, device=p.device)
    s2 = torch.zeros_like(s1)
    for i in range(p.shape[1]):
        s1 = s1 + p[:, i, 0]
        s2 = s2 + p[:, i, 1]
    inv_n = 1.0 / cols
    mean = s1 * inv_n
    var = (s2 * inv_n - mean * mean).clamp_min(0.0)
    return mean.float(), var, var.float() + torch.tensor(eps, dtype=torch.float32)


@pytest.mark.gpu
def test_large_mean_rows_through_finalize(ctx):
    """The out-projection shape (M = 263 * 9, E = 768, v02) with residual rows of mean mu in LARGE_MEANS and sigma 1."""
    M, E, eps = 263 * 9, 768, 1e-5
    lines, failures = [], []
    for mode in ("f16x3", "bf16x3", "f16f8"):  # f16f8 at N = 768 runs on gemm_wide_kernel
        g = torch.Generator(device="cuda").manual_seed(77)
        rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
        mu = torch.tensor(LARGE_MEANS, device="cuda")[torch.arange(M, device="cuda") % len(LARGE_MEANS)]
        res = (mu[:, None] + rn(M, E + 4))[:, :E]
        ops = GemmOperands(ctx, rn(M, E), rn(E, E) / math.sqrt(E), mode)
        parts = ctx.gemm_stats_parts(E, 0, 0)
        out32, hi = sentinel((M + 3, E + 8), "f32"), sentinel((M + 3, E + 8), "i16")
        views = dict(out_lo8=sentinel((M + 3, E + 16), "u8"), out_hi8=sentinel((M + 3, E + 16), "u8")) if ops.f8 else \
            dict(out_lo=sentinel((M + 3, E + 8), "i16"))
        part = sentinel((M + 3, parts, 2), "f32")
        ctx.gemm(M=M, N=E, K=E, bias=0.1 * rn(E), residual=res, out_f32=out32, out_hi=hi, stats_out=part, **views, **ops.kwargs())
        stats = sentinel((M + 3, 2), "f32")
        ctx.row_stats_finalize(part[:M], E, eps, stats)
        torch.cuda.synchronize()
        assert_canary(stats, M, 2, f"{mode} row_stats_finalize")
        x = out32[:M, :E]
        msg = stats_difference(part[:M], stats_statement(x, M, E, 128, parts), 128)
        if msg:
            failures.append(f"{mode}: {msg}")
        mean_f, var, arg = finalize_statement(part[:M], E, eps)
        got = stats[:M]
        if not torch.equal(got[:, 0].contiguous().view(torch.int32), mean_f.view(torch.int32)):
            r = int((got[:, 0].contiguous().view(torch.int32) != mean_f.view(torch.int32)).nonzero()[0])
            failures.append(f"{mode}: mean differs from the finalize statement at row {r}: {got[r, 0].item()!r} vs {mean_f[r].item()!r}")
        # rsqrtf is within 2 ulp of the exact 1 / sqrt of its fp32 argument
        want = torch.rsqrt(arg.double())
        ulp = torch.pow(2.0, torch.floor(torch.log2(want)) - 23)
        off = ((got[:, 1].double() - want).abs() / ulp).max().item()
        if off > 2:
            failures.append(f"{mode}: rstd {off:.2f} ulp from rsqrt((float)var + eps)")
        # against the fp64 statistics of the fp32 rows
        y = x.double()
        m64, v64 = y.mean(1), y.var(1, unbiased=False)
        r64 = 1.0 / torch.sqrt(v64 + eps)
        scale = 1.0 + m64 * m64 / v64
        e_var = (var - v64).abs() / v64
        e_rstd = (got[:, 1].double() - r64).abs() / r64
        for i, m in enumerate(LARGE_MEANS):
            sel = torch.arange(M, device="cuda") % len(LARGE_MEANS) == i
            ratio = (m64[sel].abs() / v64[sel].sqrt()).max().item()
            cv, cr = (e_var[sel] / scale[sel]).max().item(), (e_rstd[sel] / scale[sel]).max().item()
            lines.append(f"  {mode:>7} {m:>6g} {ratio:>8.1f} {e_var[sel].max().item():>10.2e} {cv:>10.2e} {e_rstd[sel].max().item():>10.2e} "
                         f"{cr:>10.2e}")
            assert ratio <= 300, "rows past the stated contract (|mean| / sigma <= ~300)"
            if cv > VAR_COEF or cr > VAR_COEF:
                failures.append(f"{mode} mu={m}: error / (1 + mean^2/var) = {cv:.2e} (variance), {cr:.2e} (rstd) > {VAR_COEF:g}")
    print(f"\nrow statistics through finalize, M = {M}, E = {E} (max over rows of each group):\n  {'mode':>7} {'mu':>6} "
          f"{'|mean|/sd':>8} {'var err':>10} {'var coef':>10} {'rstd err':>10} {'rstd coef':>10}\n" + "\n".join(lines))
    assert not failures, "\n".join(failures)
