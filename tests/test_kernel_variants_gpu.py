"""Kernel variants, output formats and operand producers against fp64 (or bit-exact) torch statements of the same operation.

The policy-level suites hold whole policies to rel-L2 bars of 1e-3 .. 5e-5; a localised error in one compiled epilogue, one output
format or one operand producer disappears in those.  Here every such path is called through the C ABI with explicit descriptor
fields, so each case runs the kernel variant it names:

  1. every row of VIMA_GEMM_VARIANTS (gemm_tc_variants.cuh) plus combinations that fall to the generic epilogue, in every operand
     mode, at decode-sized, ragged and multi-tile shapes, with sentinels around every output and NaN in every operand column past K;
  2. the activations elementwise (A = 0, so the epilogue evaluates act(bias)) over a dense grid and the fp32 extremes;
  3. every 16-bit and e4m3 operand producer bit for bit against one statement of the saturating split;
  4. attention in every kernel (wgmma, mma.sync, SIMT tail), format and output layout at the tail-split and capacity boundaries;
  5. the norm kernel's formats and strides;
  6. the entry points no other test calls (latent / small attention sizes, vit_tokens, gato_positions, row_stats_finalize rms).

Bars that rest on a measurement say so where they are defined; the measurements were taken on an H100 80GB HBM3 (700 W power
limit).
"""
import math
import os
import re

import pytest
import torch

F = torch.nn.functional
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = {"f16": (0, torch.float16), "bf16": (1, torch.bfloat16)}
NAN16 = {0: 0x7E00, 1: 0x7FC0}  # a quiet NaN of each 16-bit format
NAN8 = 0x7F                      # e4m3fn NaN
S16, S32, S8 = 0x7BAD, 0x7FBADBAD, 0xA5  # output sentinels (int16, fp32 bit pattern, byte)
ACT = {"ACT_NONE": 0, "ACT_RELU": 1, "ACT_QUICKGELU": 2, "ACT_GELU": 3, "ACT_GELU_TANH": 4}

# (ACT, GLU, MUL, RES, O32, O16, LNA, LNR, STATS): the rows of VIMA_GEMM_VARIANTS, in order
VARIANTS = [
    ("ACT_NONE", 0, 0, 0, 0, 1, 0, 0, 0),
    ("ACT_NONE", 0, 0, 1, 1, 1, 0, 0, 0),
    ("ACT_NONE", 0, 0, 1, 1, 1, 0, 0, 1),
    ("ACT_NONE", 0, 0, 0, 1, 0, 0, 0, 0),
    ("ACT_GELU", 0, 1, 0, 0, 1, 0, 0, 0),
    ("ACT_NONE", 0, 0, 1, 1, 0, 0, 0, 0),
    ("ACT_NONE", 0, 0, 1, 1, 0, 0, 1, 0),
    ("ACT_GELU", 1, 0, 0, 0, 1, 0, 0, 0),
    ("ACT_GELU", 1, 0, 0, 0, 1, 1, 0, 0),
    ("ACT_RELU", 0, 0, 0, 0, 1, 0, 0, 0),
    ("ACT_QUICKGELU", 0, 0, 0, 0, 1, 0, 0, 0),
    ("ACT_QUICKGELU", 0, 0, 0, 0, 1, 1, 0, 0),
    ("ACT_NONE", 0, 0, 0, 1, 0, 1, 0, 0),
]
# combinations that must run the generic runtime-flag epilogue
GENERIC = [
    ("ACT_RELU", 0, 1, 0, 1, 1, 0, 0, 0),
    ("ACT_GELU_TANH", 0, 0, 0, 0, 1, 1, 0, 0),  # the GPT-baseline MLP: gelu_tanh(LN folded) -> fp16 + e4m3 views
    ("ACT_QUICKGELU", 0, 0, 1, 1, 0, 0, 0, 0),
]
MODES = ["f16", "f16x3", "f16f8", "bf16", "bf16x3"]


def test_variant_table_matches_the_compiled_list():
    """A specialisation added to (or removed from) VIMA_GEMM_VARIANTS without a matching row here fails the CPU suite."""
    lines = open(os.path.join(ROOT, "vima_b200", "csrc", "gemm_tc_variants.cuh")).read().splitlines()
    start = next(i for i, ln in enumerate(lines) if ln.startswith("#define VIMA_GEMM_VARIANTS("))
    body = []
    for ln in lines[start + 1:]:
        body.append(ln)
        if not ln.rstrip().endswith("\\"):
            break
    rows = []
    for args in re.findall(r"X\(([^)]*)\)", "\n".join(body)):
        f = [a.strip() for a in args.split(",")]
        assert len(f) == 10 and f[6] == "DT", f
        rows.append((f[0],) + tuple({"true": 1, "false": 0}[v] for v in f[1:6] + f[7:]))
    assert rows == VARIANTS
    assert not set(GENERIC) & set(rows)


# ------------------------------------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    return _C.Context.get(torch.device("cuda", 0))


def rup(x, m):
    return (x + m - 1) // m * m


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def f16view(t, dt):
    return t.view(torch.float16 if dt == 0 else torch.bfloat16)


def sentinel(shape, kind):
    """An output buffer pre-filled with a bit pattern no kernel writes: kind 'f32' | 'i16' | 'u8'."""
    if kind == "f32":
        return torch.full(shape, S32, dtype=torch.int32, device="cuda").view(torch.float32)
    if kind == "i16":
        return torch.full(shape, S16, dtype=torch.int16, device="cuda")
    return torch.full(shape, S8, dtype=torch.uint8, device="cuda")


def assert_canary(buf, rows, cols, what):
    """Rows >= rows and columns >= cols of buf still hold the sentinel."""
    raw = {4: lambda t: t.view(torch.int32), 2: lambda t: t, 1: lambda t: t}[buf.element_size()](buf)
    want = {4: S32, 2: S16, 1: S8}[buf.element_size()]
    assert (raw[rows:] == want).all(), f"{what}: written past the last row"
    assert (raw[:, cols:] == want).all(), f"{what}: written past the last column"


def as_bits16(t):
    return t.view(torch.int16).to(torch.int32) & 0xFFFF


def assert_bits(got, want, x, what):
    bad = got != want
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ; first at {i}: x = {x[i].item()!r}, "
                             f"got 0x{int(got[i]) & 0xFFFF:04x}, want 0x{int(want[i]) & 0xFFFF:04x}")


def assert_hi8(hi8, x, what):
    """hi8 = e4m3(x / 8) elementwise, x the value the kernel split (fp64): within e4m3 round-to-nearest, i.e. 2^-4 relative and, in
    e4m3's subnormal range, 2^-10 absolute of x / 8 (a little slack for x itself).  A swapped byte or column fails it."""
    got = hi8.view(torch.float8_e4m3fn).double() * 8.0
    err = (got - x).abs() - (0.0625 * 1.01 * x.abs() + 8 * 2.0 ** -10 * 1.01)
    if (err > 0).any():
        raise AssertionError(f"{what}: hi8 off e4m3(x/8) at {int((err > 0).sum())} elements; worst x = "
                             f"{x.flatten()[err.argmax()].item()!r}, got {got.flatten()[err.argmax()].item()!r}")


def act_ref(act, x):
    return {0: lambda t: t, 1: torch.relu, 2: lambda t: t * torch.sigmoid(1.702 * t), 3: lambda t: F.gelu(t),
            4: lambda t: F.gelu(t, approximate="tanh")}[act](x)


def block_n_for(N, glu):
    """The block_n vima_gemm picks when the descriptor leaves it 0 (api.cu choose_block_n)."""
    step = 64 if glu else 32
    best, best_pad = step, 1 << 30
    for bn in range(step, 129, step):
        padded = -(-N // bn) * bn
        if padded < best_pad or (padded == best_pad and bn > best):
            best, best_pad = bn, padded
    return best


def interleave(val, gate, bn):
    """Value / gate rows (or vector entries) -> the accumulator-column order of a GLU GEMM: per tile of bn, value half | gate half."""
    half = bn // 2
    n = val.shape[0]
    tiles = -(-n // half)
    pad = (0, 0) * (val.dim() - 1) + (0, tiles * half - n)
    v = F.pad(val, pad).reshape(tiles, half, *val.shape[1:])
    g = F.pad(gate, pad).reshape(tiles, half, *val.shape[1:])
    return torch.stack([v, g], 1).reshape(tiles * bn, *val.shape[1:]).contiguous()


def deinterleave(acc, bn, n_out):
    """[M, tiles*bn] accumulator columns -> (value [M, n_out], gate [M, n_out])."""
    M = acc.shape[0]
    t = acc.reshape(M, -1, 2, bn // 2)
    return t[:, :, 0].reshape(M, -1)[:, :n_out], t[:, :, 1].reshape(M, -1)[:, :n_out]


def fold_ln(w, b, gamma, beta):
    """LayerNorm folded into the Linear after it (fp64, rounded to fp32): W*gamma, rowsum(W*gamma), b + W beta."""
    w64 = w.double()
    wp = w64 * gamma.double()[None, :]
    return wp.float(), wp.sum(1).float(), (b.double() + w64 @ beta.double()).float()


def ln64(x, w, b, eps=1e-5):
    return F.layer_norm(x.double(), (x.shape[-1],), w.double(), b.double(), eps)


# ------------------------------------------------------------------------------------------------------------------------------
# 1. GEMM epilogue variants
# ------------------------------------------------------------------------------------------------------------------------------
# rel-L2 of the fp32 output against fp64: the split modes against the exact product, the single-pass modes against the product of
# the rounded operands (the accumulation and the epilogue are what is checked there).  Twice the bar for a folded LayerNorm.
# Measured worst over every row and shape: f16 9.0e-7, f16x3 2.7e-6, f16f8 1.05e-5, bf16 7.1e-7, bf16x3 4.9e-6 (fp32 output);
# (hi, lo) against fp64 up to 8.8e-6 in bf16x3 (GEGLU with the LayerNorm folded in), fp16 hi + lo8 / 1024 up to 1.55e-5 in f16f8.
GEMM_TOL = {"f16": 3e-6, "f16x3": 6e-6, "f16f8": 2.5e-5, "bf16": 3e-6, "bf16x3": 1.5e-5}
REP = {0: 3e-7, 1: 6e-6}  # rel-L2 of a (hi, lo) pair against the fp32 value it stands for (22 / 16 bits; measured 4.8e-8 / 2.6e-6)
HI_ONLY = {0: 1e-3, 1: 8e-3}
GEMM_SHAPES = [(1, 256, 768, 0), (33, 256, 768, 0), (515, 288, 392, 96), (4741, 768, 768, 0)]  # (M, N or n_out, K, block_n)


class GemmOperands:
    """A [M, K] and W [N, K] as the kernel's operands in `mode`, with NaN in every column in [K, ld) (and in A's rows past M):
    a finite result proves the kernel never reads them."""

    def __init__(self, ctx, A, W, mode):
        M, K = A.shape
        N = W.shape[0]
        self.dt = 1 if mode.startswith("bf16") else 0
        self.split = mode.endswith("x3")
        self.f8 = mode == "f16f8"
        self.ws = 1.0 if self.dt == 1 else 2.0 ** math.floor(math.log2(1024.0 / W.abs().max().item()))  # engine._pow2_scale
        ld = rup(K, 8) + 8
        self.ld = ld
        self.a_hi = torch.empty(M + 3, ld, dtype=torch.int16, device="cuda")
        self.a_lo = torch.empty_like(self.a_hi) if self.split else None
        ctx.split(A, self.a_hi, self.a_lo, cols=K, pad_cols=ld, dtype=self.dt)
        self.b_hi = torch.empty(N, ld, dtype=torch.int16, device="cuda")
        self.b_lo = torch.empty_like(self.b_hi) if self.split else None
        ctx.pack_weight(W, self.b_hi, self.b_lo, transposed=False, scale=self.ws, dtype=self.dt)
        for t in (self.a_hi, self.a_lo, self.b_hi, self.b_lo):
            if t is not None:
                t[:, K:] = NAN16[self.dt]
        for t in (self.a_hi, self.a_lo):
            if t is not None:
                t[M:] = NAN16[self.dt]
        self.a8 = self.b8 = (None, None)
        if self.f8:
            ld8 = rup(K, 16) + 16
            a_lo8 = torch.zeros(M + 3, ld8, dtype=torch.uint8, device="cuda"); a_hi8 = torch.zeros_like(a_lo8)
            ctx.split_f8(A, a_lo8, a_hi8)
            b_hi8 = torch.zeros(N, ld8, dtype=torch.uint8, device="cuda"); b_lo8 = torch.zeros_like(b_hi8)
            ctx.pack_weight_f8(W, b_hi8, b_lo8, transposed=False, scale=self.ws)
            for t in (a_lo8, a_hi8, b_hi8, b_lo8):
                t[:, K:] = NAN8
            a_lo8[M:] = NAN8; a_hi8[M:] = NAN8
            self.a8, self.b8 = (a_lo8, a_hi8), (b_hi8, b_lo8)
        self.K, self.M = K, M

    def kwargs(self):
        return dict(a_hi=self.a_hi, a_lo=self.a_lo, lda=self.ld, b_hi=self.b_hi, b_lo=self.b_lo, ldb=self.ld, dtype=self.dt,
                    acc_scale=1.0 / self.ws, a_lo8=self.a8[0], a_hi8=self.a8[1], b_hi8=self.b8[0], b_lo8=self.b8[1])

    def rounded_product(self):
        """fp64 product of the operands a single-pass kernel multiplies: [M, N]."""
        a = f16view(self.a_hi[: self.M, : self.K], self.dt).double()
        b = f16view(self.b_hi[:, : self.K], self.dt).double() / self.ws
        return a @ b.t()


def run_gemm_variant(ctx, row, mode, M, n_out, K, bn, seed):
    act_name, glu, mul, res, o32, o16, lna, lnr, stats = row
    act = ACT[act_name]
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    A = rn(M, K) * 2.0 + 0.7 if lna else rn(M, K)
    Wv, bv = rn(n_out, K) / math.sqrt(K), 0.5 * rn(n_out)
    Wg, bg = rn(n_out, K) / math.sqrt(K), 0.5 * rn(n_out)
    gam, bet = 1.0 + 0.1 * rn(K), 0.1 * rn(K)
    if glu:
        bn = ctx.glu_block_n(n_out)
        W_acc, b_acc = interleave(Wv, Wg, bn), interleave(bv, bg, bn)
    else:
        bn = bn or block_n_for(n_out, False)
        W_acc, b_acc = Wv, bv
    N = W_acc.shape[0]
    kw = {}
    W_pack = W_acc
    if lna:  # the GEMM takes the un-normalised rows, W*gamma, their row sums, and (mean, rstd) of each row
        fv, c1v, fbv = fold_ln(Wv, bv, gam, bet)
        fg, c1g, fbg = fold_ln(Wg, bg, gam, bet)
        W_pack = interleave(fv, fg, bn) if glu else fv
        b_fold = interleave(fbv, fbg, bn) if glu else fbv
        c1 = interleave(c1v, c1g, bn) if glu else c1v
        A64 = A.double()
        st = torch.stack([A64.mean(1), 1.0 / torch.sqrt(A64.var(1, unbiased=False) + 1e-5)], 1).float().contiguous()
        kw.update(row_stats=st, ln_c1=c1, ln_cols=1)
    ops = GemmOperands(ctx, A, W_pack, mode)
    mul_t = rn(M, n_out + 4)[:, :n_out] if mul else None
    res_t = (rn(M, n_out + 4) * 2.0 + 0.7)[:, :n_out] if res else None
    if lnr:
        r64 = res_t.double()
        rst = torch.stack([r64.mean(1), 1.0 / torch.sqrt(r64.var(1, unbiased=False) + 1e-5)], 1).float().contiguous()
        rg, rb = 1.0 + 0.1 * rn(n_out), 0.1 * rn(n_out)
        kw.update(res_stats=rst, res_gamma=rg, res_beta=rb)
    out32 = sentinel((M + 3, n_out + 8), "f32") if o32 else None
    hi = lo = lo8 = hi8 = None
    f8_out = o16 and ops.f8
    if o16:
        hi = sentinel((M + 3, n_out + 8), "i16")
        if f8_out:
            lo8, hi8 = sentinel((M + 3, n_out + 16), "u8"), sentinel((M + 3, n_out + 16), "u8")
        else:
            lo = sentinel((M + 3, n_out + 8), "i16")
    parts = ctx.gemm_stats_parts(N, glu, bn)
    st_out = sentinel((M + 3, parts, 2), "f32") if stats else None
    ctx.gemm(M=M, N=N, K=K, glu=glu, act=act, bias=(b_fold if lna else b_acc), mul=mul_t, residual=res_t, out_f32=out32, out_hi=hi,
             out_lo=lo, block_n=bn, out_lo8=lo8, out_hi8=hi8, stats_out=st_out, **ops.kwargs(), **kw)
    torch.cuda.synchronize()

    # ---- fp64 statement of the epilogue ----
    if ops.split or ops.f8:  # against the exact operation
        x = ln64(A, gam, bet) if lna else A.double()
        pre = x @ W_acc.double().t() + b_acc.double()
    else:  # against the rounded operands, with the epilogue's own fp32 vectors
        acc = ops.rounded_product()
        if lna:
            pre = kw["row_stats"][:, 1:2].double() * (acc - kw["row_stats"][:, 0:1].double() * c1.double()[None]) + b_fold.double()
        else:
            pre = acc + b_acc.double()
    if glu:
        val, gate = deinterleave(pre, bn, n_out)
        ref = act_ref(act, val) * gate
    else:
        ref = act_ref(act, pre)
    if mul:
        ref = ref * mul_t.double()
    if res:
        r = res_t.double()
        if lnr:
            r = (r - kw["res_stats"][:, 0:1].double()) * kw["res_stats"][:, 1:2].double() * kw["res_gamma"].double() + kw["res_beta"].double()
        ref = ref + r
    tol = GEMM_TOL[mode] * (2 if lna else 1)
    what = f"{row} {mode} M={M} N={n_out} K={K}"
    errs = {}
    got = None
    if o32:
        assert_canary(out32, M, n_out, what + " out_f32")
        got = out32[:M, :n_out]
        assert torch.isfinite(got).all(), what
        errs["f32"] = rel(got, ref)
        assert errs["f32"] < tol, (what, errs)
    if o16:
        assert_canary(hi, M, n_out, what + " out_hi")
        h = f16view(hi[:M, :n_out], ops.dt).double()
        if f8_out:
            assert_canary(lo8, M, n_out, what + " out_lo8"); assert_canary(hi8, M, n_out, what + " out_hi8")
            rec = h + lo8[:M, :n_out].view(torch.float8_e4m3fn).double() / 1024.0
            errs["hi16+lo8"] = rel(rec, ref)
            assert errs["hi16+lo8"] < tol + 2e-5, (what, errs)
            assert_hi8(hi8[:M, :n_out], rec, what)
        else:
            assert_canary(lo, M, n_out, what + " out_lo")
            rec = h + f16view(lo[:M, :n_out], ops.dt).double()
            if got is not None:
                errs["hi+lo vs f32"] = rel(rec, got)
                assert errs["hi+lo vs f32"] < REP[ops.dt], (what, errs)
            errs["hi+lo"] = rel(rec, ref)
            assert errs["hi+lo"] < tol + REP[ops.dt], (what, errs)
        assert torch.isfinite(h).all(), what
        errs["hi"] = rel(h, ref)
        assert errs["hi"] < HI_ONLY[ops.dt] + tol, (what, errs)
    if stats:
        assert_canary(st_out.view(M + 3, parts * 2), M, parts * 2, what + " stats_out")
        # partial (sum, sum of squares) per (n-tile, 32-column half of the tile)
        bn_out = bn // 2 if glu else bn
        c = torch.arange(n_out, device="cuda")
        part = 2 * (c // bn_out) + ((c % bn_out) // 32) % 2
        s_ref = torch.zeros(M, parts, 2, dtype=torch.float64, device="cuda")
        s_ref[:, :, 0].index_add_(1, part, ref)
        s_ref[:, :, 1].index_add_(1, part, ref * ref)
        s_abs = torch.zeros(M, parts, dtype=torch.float64, device="cuda").index_add_(1, part, ref.abs())
        s = st_out[:M].double()
        errs["sum"] = ((s[:, :, 0] - s_ref[:, :, 0]).norm() / s_abs.norm()).item()
        errs["sumsq"] = rel(s[:, :, 1], s_ref[:, :, 1])
        assert errs["sum"] < 4 * tol and errs["sumsq"] < 4 * tol, (what, errs)
    return errs


def _row_id(row):
    act, glu, mul, res, o32, o16, lna, lnr, stats = row
    parts = [act[4:]] + [n for n, f in zip(("GLU", "MUL", "RES", "O32", "O16", "LNA", "LNR", "STATS"), row[1:]) if f]
    return "-".join(parts)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("row", VARIANTS + GENERIC, ids=[f"v{i:02d}-{_row_id(r)}" for i, r in enumerate(VARIANTS)] +
                         [f"generic-{_row_id(r)}" for r in GENERIC])
def test_gemm_variant(ctx, row, mode):
    worst = {}
    for i, (M, n, K, bn) in enumerate(GEMM_SHAPES):
        for k, v in run_gemm_variant(ctx, row, mode, M, n, K, bn, seed=1000 * i + 7).items():
            worst[k] = max(worst.get(k, 0.0), v)
    print(f"gemm {_row_id(row)} {mode}: " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))


# ------------------------------------------------------------------------------------------------------------------------------
# 2. activations, elementwise
# ------------------------------------------------------------------------------------------------------------------------------
# |got - ref| <= ACT_BAR * max(1, |x|).  Measured worst: 1.4e-7 (erf GELU), 9.9e-8 (quick GELU), 9.1e-8 (tanh GELU), 0 (ReLU); the
# specialised epilogues gave the same bits as the generic one for every activation and format.
ACT_BAR = 3e-7


def act_grid():
    special = [1e4, -1e4, 3e38, -3e38, 3.4028235e38, -3.4028235e38, 0.0, -0.0, 1e-40, -1e-40, 1.4e-45, -1.4e-45, 1.1754942e-38,
               -100.0, -1000.0, 100.0, 1000.0, 30.0, 6e4, -6e4, 9.0, -9.0, 5.5, -5.5, 1e-3, -1e-3]
    dense = torch.linspace(-40.0, 40.0, 4096 - len(special), dtype=torch.float64).float()
    return torch.cat([torch.tensor(special, dtype=torch.float32), dense]).cuda()


def act_launch(ctx, dt, x, row):
    """One GEMM with A = 0 and bias = x: the epilogue evaluates act(x) per column.  GLU: gate bias 1.  -> (fp32 | None, hi+lo fp64)."""
    act_name, glu, mul, res, o32, o16, lna, lnr, stats = row
    n = x.numel()
    M, K = 2, 64
    a_hi = torch.zeros(M, K, dtype=torch.int16, device="cuda")
    if glu:
        bn = ctx.glu_block_n(n)
        bias = interleave(x, torch.ones_like(x), bn)
    else:
        bn, bias = 0, x
    N = bias.numel()
    b_hi = torch.zeros(N, K, dtype=torch.int16, device="cuda")
    kw = {}
    if lna:
        kw = dict(row_stats=torch.tensor([[0.0, 1.0]] * M, device="cuda"), ln_c1=torch.zeros(N, device="cuda"), ln_cols=1)
    mul_t = torch.ones(M, n, device="cuda") if mul else None
    out32 = torch.empty(M, n, device="cuda") if o32 else None
    hi = torch.empty(M, n, dtype=torch.int16, device="cuda"); lo = torch.empty_like(hi)
    ctx.gemm(M=M, N=N, K=K, a_hi=a_hi, a_lo=None, lda=K, b_hi=b_hi, b_lo=None, ldb=K, dtype=dt, glu=glu, act=ACT[act_name], bias=bias,
             mul=mul_t, out_f32=out32, out_hi=hi, out_lo=lo, block_n=bn, **kw)
    torch.cuda.synchronize()
    rec = f16view(hi[0], dt).double() + f16view(lo[0], dt).double()
    assert torch.equal(hi[0], hi[1]) and torch.equal(lo[0], lo[1])
    return (None if out32 is None else out32[0]), rec


@pytest.mark.gpu
@pytest.mark.parametrize("dtname", ["f16", "bf16"])
@pytest.mark.parametrize("act", [1, 2, 3, 4])
def test_activation_elementwise(ctx, dtname, act):
    dt, _ = DT[dtname]
    x = act_grid()
    x64 = x.double()
    ref = act_ref(act, x64)
    scale = x64.abs().clamp_min(1.0)
    rep = (2.0 ** -22 if dt == 0 else 2.0 ** -16) * ref.abs() + 2.0 ** -24  # (hi, lo) representation error
    small = x64.abs() <= 6e4  # beyond that the 16-bit operands saturate by design
    name = [k for k, v in ACT.items() if v == act][0]
    report = {}
    generic = {}
    for glu in (0, 1):
        row = (name, glu, 0, 0, 1, 1, 0, 0, 0)  # fp32 + (hi, lo): never a specialisation
        got, rec = act_launch(ctx, dt, x, row)
        g64 = got.double()
        err = (g64 - ref).abs() / scale
        report[f"generic glu={glu}"] = err.max().item()
        assert err.max().item() <= ACT_BAR, (row, x[err.argmax()].item(), err.max().item())
        assert not torch.isnan(got).any()
        big, neg = x >= 30, x <= -100
        assert torch.equal(got[big], x[big]), (row, x[big][got[big] != x[big]])
        assert (got[neg] == 0).all(), (row, x[neg][got[neg] != 0])
        assert ((rec - ref).abs() <= ACT_BAR * scale + rep)[small].all(), row
        generic[glu] = rec
    for row in VARIANTS:
        if ACT[row[0]] != act:
            continue
        _, rec = act_launch(ctx, dt, x, row)
        e = ((rec - ref).abs() - rep) / scale
        report[_row_id(row)] = e[small].max().item()
        assert e[small].max().item() <= ACT_BAR, (row, x[small][e[small].argmax()].item())
        other = generic[row[1]]
        report[_row_id(row) + " bit-identical to generic"] = bool(torch.equal(rec[small], other[small]))
        assert (((rec - other).abs() - 2 * rep) <= 2 * ACT_BAR * scale)[small].all(), row
    print(f"act {name} {dtname}: {report}")


# ------------------------------------------------------------------------------------------------------------------------------
# 3. operand producers, bit for bit
# ------------------------------------------------------------------------------------------------------------------------------
def split_statement(v, dt):
    """The operand pair of an fp32 value: hi = rn(clamp(v, +-MAX)), lo = rn(clamp(v - hi, +-MAX)) in the 16-bit format (MAX its
    largest finite value, so +-inf saturates); a NaN gives the canonical NaN 0x7FFF in both.  -> (hi bits, lo bits) as int32."""
    tdt = torch.float16 if dt == 0 else torch.bfloat16
    mx = torch.finfo(tdt).max
    hi = v.clamp(-mx, mx).to(tdt)
    lo = (v - hi.float()).clamp(-mx, mx).to(tdt)
    hb, lb = as_bits16(hi), as_bits16(lo)
    nan = torch.isnan(v)
    hb[nan] = 0x7FFF
    lb[nan] = 0x7FFF
    return hb, lb


def e4m3_statement(v):
    """e4m3fn(clamp(v, +-448)); NaN -> 0x7F.  -> bits as int32."""
    b = v.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8).to(torch.int32)
    b[torch.isnan(v)] = NAN8
    return b


def f8_statement(v, lo_scale, hi_scale):
    """The e4m3 cross-term views: lo8 = e4m3((v - hi16) * lo_scale), hi8 = e4m3(v * hi_scale), hi16 the fp16 operand of v."""
    h16 = v.clamp(-65504.0, 65504.0).to(torch.float16).float()
    return e4m3_statement((v - h16) * lo_scale), e4m3_statement(v * hi_scale)


def edge_matrix(rows, cols, seed):
    """fp32 [rows, cols]: every edge value with both signs, then random normal values over a wide exponent range."""
    e = [0.0, 2.0 ** -24, 3 * 2.0 ** -24, 2.0 ** -20, 1023 * 2.0 ** -24, 2.0 ** -14, 2.0 ** -15 + 2.0 ** -24, 65504.0, 65519.0, 65520.0,
         65536.0, 1e5, 131023.0, 131024.0, 131040.0, 1e6, 3e38, 3.3895314e38, 3.39e38, 3.4028235e38, float("inf"), float("nan"),
         1e-40, 1.4e-45, 1.1754942e-38, 448.0, 464.0, 480.0, 3584.0, 2.0 ** -9, 2.0 ** -10, 0.1, 1.0 / 3.0, 1.0, 7.5e-5]
    vals = torch.tensor(e + [-v for v in e], dtype=torch.float32)
    g = torch.Generator().manual_seed(seed)
    n = rows * cols - vals.numel()
    rnd = torch.randn(n, generator=g) * torch.pow(2.0, torch.randint(-20, 21, (n,), generator=g).float())
    return torch.cat([vals, rnd]).reshape(rows, cols).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("dtname", ["f16", "bf16"])
def test_split_producers_bit_exact(ctx, dtname):
    """split (scale, pad_cols > cols), pack_weight (both orientations, scale), fill_ee, the norm in pure-convert mode and the GEMM
    epilogue (A = 0, residual = X) all emit split_statement() bit for bit."""
    dt, _ = DT[dtname]
    R, C = 8, 64
    X = edge_matrix(R, C, 1)
    # split, with padding columns [C, pad) zero and [pad, ld) untouched
    for scale in (1.0, 0.25):
        hi, lo = sentinel((R + 2, C + 16), "i16"), sentinel((R + 2, C + 16), "i16")
        ctx.split(X, hi, lo, cols=C, pad_cols=C + 8, scale=scale, dtype=dt)
        want = split_statement(X * scale, dt)
        for got, w, nm in ((hi, want[0], "hi"), (lo, want[1], "lo")):
            assert_bits(as_bits16(got[:R, :C]), w, X, f"split scale={scale} {nm}")
            assert (got[:R, C:C + 8] == 0).all()
            assert_canary(got, R, C + 8, f"split {nm}")
    # pack_weight: [n, k] or, transposed, [k, n] -> K-major [n, ld16] zero padded
    for transposed in (False, True):
        for scale in (1.0, 8.0):
            W = X.t().contiguous() if transposed else X
            hi, lo = sentinel((R + 2, C + 8), "i16"), sentinel((R + 2, C + 8), "i16")
            ctx.pack_weight(W, hi, lo, transposed=transposed, scale=scale, dtype=dt)
            want = split_statement(X * scale, dt)
            for got, w, nm in ((hi, want[0], "hi"), (lo, want[1], "lo")):
                assert_bits(as_bits16(got[:R, :C]), w, X, f"pack_weight transposed={transposed} scale={scale} {nm}")
                assert (got[:R, C:] == 0).all()
                assert_canary(got, R, C + 8, "pack_weight")
    # fill_ee: rows te*Q + q, columns [col0, col0 + 2) = table[ee[te]], then n_pad zero columns
    table = X.reshape(-1, 2).contiguous()
    ee = torch.arange(table.shape[0], device="cuda", dtype=torch.int64).flip(0).contiguous()
    Q, col0, n_pad = 3, 4, 2
    rows = ee.numel() * Q
    hi, lo = sentinel((rows + 2, 16), "i16"), sentinel((rows + 2, 16), "i16")
    ctx.fill_ee(ee, table, ee.numel(), Q, hi, lo, col0, n_pad, dtype=dt)
    tv = table[ee].repeat_interleave(Q, 0)
    want = split_statement(tv, dt)
    for got, w, nm in ((hi, want[0], "hi"), (lo, want[1], "lo")):
        assert_bits(as_bits16(got[:rows, col0:col0 + 2]), w, tv, f"fill_ee {nm}")
        assert (got[:rows, col0 + 2:col0 + 2 + n_pad] == 0).all()
        assert (got[:rows, :col0] == S16).all()
        assert_canary(got, rows, col0 + 2 + n_pad, "fill_ee")
    # norm, pure convert (no weights)
    hi, lo = sentinel((R + 2, C + 8), "i16"), sentinel((R + 2, C + 8), "i16")
    ctx.norm(X, rows=R, cols=C, ldx=C, out_hi=hi, out_lo=lo, dtype=dt)
    want = split_statement(X, dt)
    for got, w, nm in ((hi, want[0], "hi"), (lo, want[1], "lo")):
        assert_bits(as_bits16(got[:R, :C]), w, X, f"norm {nm}")
        assert_canary(got, R, C, "norm")
    # GEMM epilogue: 0 * W + X (row 2 of the variant table, and the generic epilogue without the fp32 output)
    K = 64
    a0 = torch.zeros(R, K, dtype=torch.int16, device="cuda")
    b = torch.randn(C, K, device="cuda").to(torch.float16 if dt == 0 else torch.bfloat16).view(torch.int16).contiguous()
    v = X + 0.0  # the epilogue adds the residual to a zero accumulator: -0 becomes +0
    want = split_statement(v, dt)
    for o32 in (True, False):
        hi, lo = sentinel((R + 2, C + 8), "i16"), sentinel((R + 2, C + 8), "i16")
        out = torch.empty(R, C, device="cuda") if o32 else None
        ctx.gemm(M=R, N=C, K=K, a_hi=a0, a_lo=None, lda=K, b_hi=b, b_lo=None, ldb=K, dtype=dt, residual=X, out_f32=out, out_hi=hi, out_lo=lo)
        for got, w, nm in ((hi, want[0], "hi"), (lo, want[1], "lo")):
            assert_bits(as_bits16(got[:R, :C]), w, X, f"gemm o32={o32} {nm}")
            assert_canary(got, R, C, "gemm")


@pytest.mark.gpu
def test_e4m3_producers_bit_exact(ctx):
    """split_f8, pack_weight_f8 (weight scales, both orientations), the norm and the GEMM epilogue emit e4m3(clamp(v, +-448)) views."""
    R, C = 8, 64
    X = edge_matrix(R, C, 2)
    lo8, hi8 = sentinel((R + 2, C + 16), "u8"), sentinel((R + 2, C + 16), "u8")
    ctx.split_f8(X, lo8, hi8)
    wl, wh = f8_statement(X, 1024.0, 0.125)
    assert_bits(lo8[:R, :C].to(torch.int32), wl, X, "split_f8 lo8")
    assert_bits(hi8[:R, :C].to(torch.int32), wh, X, "split_f8 hi8")
    assert_canary(lo8, R, C, "split_f8"); assert_canary(hi8, R, C, "split_f8")
    for transposed in (False, True):
        for scale in (1.0, 512.0):
            W = X.t().contiguous() if transposed else X
            h8, l8 = sentinel((R + 2, C + 16), "u8"), sentinel((R + 2, C + 16), "u8")
            ctx.pack_weight_f8(W, h8, l8, transposed=transposed, scale=scale)
            wl, wh = f8_statement(X * scale, 8.0, 1.0 / 1024.0)
            assert_bits(l8[:R, :C].to(torch.int32), wl, X, f"pack_weight_f8 lo8 transposed={transposed} scale={scale}")
            assert_bits(h8[:R, :C].to(torch.int32), wh, X, f"pack_weight_f8 hi8 transposed={transposed} scale={scale}")
            assert (l8[:R, C:] == 0).all() and (h8[:R, C:] == 0).all()
            assert_canary(l8, R, C + 16, "pack_weight_f8")
    # norm (pure convert) and GEMM epilogue: fp16 hi + the two views
    K = 64
    a0 = torch.zeros(R, K, dtype=torch.int16, device="cuda")
    b = torch.randn(C, K, device="cuda").half().view(torch.int16).contiguous()
    for who in ("norm", "gemm"):
        hi = sentinel((R + 2, C + 8), "i16")
        lo8, hi8 = sentinel((R + 2, C + 16), "u8"), sentinel((R + 2, C + 16), "u8")
        if who == "norm":
            v = X
            ctx.norm(X, rows=R, cols=C, ldx=C, out_hi=hi, out_lo8=lo8, out_hi8=hi8, dtype=0)
        else:
            v = X + 0.0
            ctx.gemm(M=R, N=C, K=K, a_hi=a0, a_lo=None, lda=K, b_hi=b, b_lo=None, ldb=K, dtype=0, residual=X, out_hi=hi, out_lo8=lo8, out_hi8=hi8)
        wl, wh = f8_statement(v, 1024.0, 0.125)
        assert_bits(as_bits16(hi[:R, :C]), split_statement(v, 0)[0], X, f"{who} hi16")
        assert_bits(lo8[:R, :C].to(torch.int32), wl, X, f"{who} lo8")
        assert_bits(hi8[:R, :C].to(torch.int32), wh, X, f"{who} hi8")
        for t in (hi, lo8, hi8):
            assert_canary(t, R, C, who)


# ------------------------------------------------------------------------------------------------------------------------------
# 4. attention formats and boundaries
# ------------------------------------------------------------------------------------------------------------------------------
def ref_attention(q, k, v, scale, causal, key_mask, q_pos0=0):
    """q (B,H,Lq,D) etc. in float64; reference mask semantics (soft causal -1e4, finfo(fp32).min for padded keys); query row i sits
    at key position q_pos0 + i."""
    s = torch.matmul(q, k.transpose(-1, -2)) * scale
    Lq, Lk = s.shape[-2:]
    if causal:
        tril = torch.tril(torch.ones(Lq, Lk, dtype=s.dtype, device=s.device), diagonal=q_pos0)
        s = s * tril + -1e4 * (1 - tril)
    if key_mask is not None:
        s = s + (1.0 - key_mask[:, None, None, :].to(s.dtype)) * torch.finfo(torch.float32).min
    return torch.matmul(torch.softmax(s, -1), v)


def attn_shapes(f8):
    """(Lq, Lk, D, causal): the wgmma tail split (Lq % 128 of 1, 8, 9 -> tail kernel, tail kernel, full tile), one key, a partial key
    chunk, the wgmma kernel's key limit (512) and one past it (mma.sync).  Causal cases with Lq < Lk put the queries last."""
    out = []
    for D in ((32,) if f8 else (32, 64)):
        for Lq in (1, 129, 136, 137, 263):
            for Lk in ((65, 513) if f8 else (1, 64, 65, 512, 513)):
                out.append((Lq, Lk, D, False))
                if Lk >= Lq:
                    out.append((Lq, Lk, D, True))
            if (Lq, Lq, D, True) not in out:
                out.append((Lq, Lq, D, True))
    return out


# rel-L2 against fp64 (fp16: the bars of test_kernels_gpu.py).  Measured worst over every kernel and shape: f16x3 2.0e-6 ((hi, lo)),
# 9.5e-6 (hi + lo8 / 1024), bf16x3 8.3e-6, single-pass f16 2.0e-4, single-pass bf16 1.3e-3.
ATTN_TOL = {(0, True): 1e-5, (1, True): 2e-5, (0, False): 2e-3, (1, False): 4e-3}


@pytest.fixture(params=["mma", "tc", "tc+tail_off"])
def attn_impl(request, ctx):
    impl, _, tail = request.param.partition("+tail_")
    ctx.set_option("attn", impl)
    ctx.set_option("attn_tail", tail or "kernel")
    yield request.param
    ctx.set_option("attn", "tc")
    ctx.set_option("attn_tail", "kernel")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f16-x3-hilo", "f16-x3-hi8", "f16-x3-hilo8", "f16-single-hilo", "f16-single-hi8", "f16-single-hilo8",
                                 "bf16-x3-hilo", "bf16-single-hilo"])
def test_attention_formats(ctx, attn_impl, fmt):
    """Batch element 0 has random padded keys (key 0 valid), batch element 1 has every key padded (uniform weights over all keys).
    Outputs: (hi, lo); fp16 hi + e4m3 views; (hi, lo) + e4m3 views.  Shapes past the mma.sync kernel's shared memory are refused
    with the capacity message and nothing is written."""
    dtname, mode, out = fmt.split("-")
    dt, tdt = DT[dtname]
    split = mode == "x3"
    want_lo, want8 = out in ("hilo", "hilo8"), out in ("hi8", "hilo8")
    tol = ATTN_TOL[(dt, split)]
    B, H = 2, 2
    worst = 0.0
    for Lq, Lk, D, causal in attn_shapes(want8):
        E = H * D
        q_pos0 = Lk - Lq if causal else 0
        g = torch.Generator(device="cuda").manual_seed(Lq * 1000 + Lk + D + causal)
        Qm = torch.randn(B * Lq, E, device="cuda", generator=g)
        KV = torch.randn(B * Lk, 2 * E, device="cuda", generator=g)

        def ops(x):  # 16-bit operands, ld padded with NaN columns the kernels must not read
            rows, cols = x.shape
            hi = torch.empty(rows, cols + 8, dtype=torch.int16, device="cuda")
            lo = torch.empty_like(hi) if split else None
            ctx.split(x, hi, lo, cols=cols, pad_cols=cols + 8, dtype=dt)
            for t in (hi, lo):
                if t is not None:
                    t[:, cols:] = NAN16[dt]
            return hi, lo

        qh, ql = ops(Qm)
        kh, kl = ops(KV)
        key_mask = torch.rand(B, Lk, device="cuda", generator=g) > 0.2
        key_mask[0, 0] = True
        key_mask[1] = False
        o_hi = sentinel((B * Lq + 3, E + 8), "i16")
        o_lo = sentinel((B * Lq + 3, E + 8), "i16") if want_lo else None
        o8 = (sentinel((B * Lq + 3, E + 16), "u8"), sentinel((B * Lq + 3, E + 16), "u8")) if want8 else None
        args = dict(q=(qh, ql, E + 8, 0), k=(kh, kl, 2 * E + 8, 0), v=(kh, kl, 2 * E + 8, E), o=(o_hi, o_lo, E + 8, 0), B=B, H=H, Lq=Lq,
                    Lk=Lk, D=D, scale=1 / math.sqrt(D), causal=causal, key_mask=key_mask.to(torch.uint8), dtype=dt, o8=o8, q_pos0=q_pos0)
        what = f"{attn_impl} {fmt} Lq={Lq} Lk={Lk} D={D} causal={causal}"
        if D == 64 and split and Lk > 384:
            with pytest.raises(RuntimeError, match=r"resident-K/V kernel takes Lk <= 384"):
                ctx.attention(**args)
            torch.cuda.synchronize()
            assert (o_hi == S16).all(), what
            continue
        ctx.attention(**args)
        torch.cuda.synchronize()

        def heads(x, L):
            return x.reshape(B, L, H, D).permute(0, 2, 1, 3).double()

        Q, K, V = Qm, KV[:, :E], KV[:, E:]
        if not split:
            Q, K, V = (t.to(tdt).float() for t in (Q, K, V))
        ref = ref_attention(heads(Q, Lq), heads(K, Lk), heads(V, Lk), 1 / math.sqrt(D), causal, key_mask, q_pos0)
        ref = ref.permute(0, 2, 1, 3).reshape(B * Lq, E)
        h = f16view(o_hi[: B * Lq, :E], dt).double()
        assert_canary(o_hi, B * Lq, E, what)
        if want_lo:
            assert_canary(o_lo, B * Lq, E, what)
            got = h + f16view(o_lo[: B * Lq, :E], dt).double()
            e = rel(got, ref)
            worst = max(worst, e)
            assert torch.isfinite(got).all() and e < tol, (what, e)
        if want8:
            lo8, hi8 = o8
            assert_canary(lo8, B * Lq, E, what); assert_canary(hi8, B * Lq, E, what)
            rec = h + lo8[: B * Lq, :E].view(torch.float8_e4m3fn).double() / 1024.0
            e = rel(rec, ref)
            worst = max(worst, e)
            assert torch.isfinite(rec).all() and e < tol + 2e-5, (what, e)
            assert_hi8(hi8[: B * Lq, :E], rec, what)
    print(f"attention {attn_impl} {fmt}: worst rel-L2 {worst:.2e}")


# ------------------------------------------------------------------------------------------------------------------------------
# 5. norm formats
# ------------------------------------------------------------------------------------------------------------------------------
NORM_HILO = {0: 3e-7, 1: 6e-6}  # rel-L2 of (hi, lo) against the fp32 row it stands for (measured 6.2e-8 / 3.1e-6)
# LayerNorm of rows with mean 1e3, sigma 1: the fp32 row mean carries the 1e3 magnitude (measured 6.1e-5; 1.2e-5 after the chained
# second LayerNorm).  A one-pass variance, E[x^2] - mean^2 in fp32, is off by whole percent there.
NORM_OFFSET_TOL = 1.5e-4


@pytest.mark.gpu
@pytest.mark.parametrize("dtname", ["f16", "bf16"])
@pytest.mark.parametrize("kind", ["ln", "rms", "none", "chain"])
def test_norm_formats(ctx, dtname, kind):
    """LayerNorm / RMSNorm / pure convert / LayerNorm chained into a second LayerNorm (eps2 != eps), of x + add, with strided
    inputs (NaN in the padding) and outputs (sentinels in the padding), (hi, lo) [+ e4m3 views in fp16] and the row statistics."""
    dt, _ = DT[dtname]
    eps, eps2 = (1e-6 if kind == "rms" else 1e-5), 1e-3
    worst = {}
    for cols in (4, 36, 1020, 1024):
        for rows in (1, 7, 1037):
            g = torch.Generator(device="cuda").manual_seed(cols * 10 + rows)
            rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
            xb = rn(rows, cols + 4) * 3 + 0.5
            offset = torch.arange(rows, device="cuda") % 3 == 1  # rows with mean 1e3 and sigma 1
            xb[offset] = 1e3 + rn(int(offset.sum()), cols + 4) * 0.7
            ab = rn(rows, cols + 8)
            xb[:, cols:] = float("nan"); ab[:, cols:] = float("nan")
            w, b, w2, b2 = 1.0 + 0.2 * rn(cols), 0.2 * rn(cols), 1.0 + 0.2 * rn(cols), 0.2 * rn(cols)
            o32 = sentinel((rows + 3, cols + 12), "f32")
            o2 = sentinel((rows + 3, cols + 4), "f32") if kind == "chain" else None
            hi, lo = sentinel((rows + 3, cols + 4), "i16"), sentinel((rows + 3, cols + 4), "i16")
            lo8 = hi8 = None
            if dt == 0:
                lo8, hi8 = sentinel((rows + 3, cols + 8), "u8"), sentinel((rows + 3, cols + 8), "u8")
            st = sentinel((rows + 3, 2), "f32")
            ctx.norm(xb, rows=rows, cols=cols, ldx=cols + 4, add=ab, w=None if kind == "none" else w, b=b if kind in ("ln", "chain") else None,
                     eps=eps, rms=int(kind == "rms"), w2=w2 if kind == "chain" else None, b2=b2 if kind == "chain" else None, eps2=eps2,
                     out_f32=o32, out2_f32=o2, out_hi=hi, out_lo=lo, dtype=dt, out_lo8=lo8, out_hi8=hi8, stats_out=st, stats_eps=1e-5)
            torch.cuda.synchronize()
            what = f"{kind} {dtname} rows={rows} cols={cols}"
            s = xb[:, :cols] + ab[:, :cols]  # fp32, as the kernel adds
            s64 = s.double()
            if kind == "none":
                y1 = s64
            elif kind == "rms":
                y1 = w.double() * s64 * torch.rsqrt(s64.pow(2).mean(-1, keepdim=True) + eps)
            else:
                y1 = ln64(s, w, b, eps)
            got1 = o32[:rows, :cols]
            for t, c in ((o32, cols), (hi, cols), (lo, cols), (st, 2)):
                assert_canary(t, rows, c, what)

            def check_rows(got, ref, tol, name):
                for sel, bar, key in ((~offset, tol, name), (offset, NORM_OFFSET_TOL, name + " mean-1e3 rows")):
                    if sel.any():
                        e = rel(got[sel], ref[sel])
                        worst[key] = max(worst.get(key, 0.0), e)
                        assert e < bar, (what, name, e)

            if kind == "none":
                assert torch.equal(got1, s), what
            else:
                check_rows(got1, y1, 2e-6, "out_f32")
            last = got1
            if kind == "chain":
                assert_canary(o2, rows, cols, what)
                last = o2[:rows, :cols]
                check_rows(last, ln64(y1, w2, b2, eps2), 5e-6, "out2_f32")
            rec = f16view(hi[:rows, :cols], dt).double() + f16view(lo[:rows, :cols], dt).double()
            worst["hi+lo"] = max(worst.get("hi+lo", 0.0), rel(rec, last))
            assert rel(rec, last) < NORM_HILO[dt], (what, rel(rec, last))
            if dt == 0:
                assert_canary(lo8, rows, cols, what); assert_canary(hi8, rows, cols, what)
                rec8 = f16view(hi[:rows, :cols], 0).double() + lo8[:rows, :cols].view(torch.float8_e4m3fn).double() / 1024.0
                assert rel(rec8, last) < 2e-5, what
                assert_hi8(hi8[:rows, :cols], last.double(), what)
            # (mean, rstd) of the first norm's output rows (rms: (0, 1 / rms))
            y = got1.double()
            if kind == "rms":
                mean_ref = torch.zeros(rows, dtype=torch.float64, device="cuda")
                rstd_ref = torch.rsqrt(y.pow(2).mean(1) + 1e-5)
            else:
                mean_ref = y.mean(1)
                rstd_ref = torch.rsqrt(y.var(1, unbiased=False) + 1e-5)
            sd = st[:rows].double()
            assert ((sd[:, 0] - mean_ref).abs() <= 2e-5 * (1 + mean_ref.abs())).all(), what
            assert ((sd[:, 1] - rstd_ref).abs() <= 2e-5 * rstd_ref).all(), what
    print(f"norm {kind} {dtname}: " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))


# ------------------------------------------------------------------------------------------------------------------------------
# 6. entry points without another test
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["shared_q", "batched_q", "perceiver_self"])
def test_latent_attention(ctx, layout):
    """Perceiver attention in fp32: latent queries shared by every image (q_batch_stride 0), per-image queries, and the self-attention
    layout of nn/perceiver.py (q | k | v column blocks of one [N*nl, 3E] buffer)."""
    N, H = 7, 3
    for Lk in (1, 5, 16):
        for d in (16, 48, 64, 128):
            E = H * d
            Lq = Lk if layout == "perceiver_self" else 4
            g = torch.Generator(device="cuda").manual_seed(Lk * 1000 + d)
            if layout == "perceiver_self":
                qkv = torch.randn(N * Lq, 3 * E, device="cuda", generator=g)
                q, ldq, qbs = qkv, 3 * E, Lq * 3 * E
                k, v, ldk = qkv[:, E:], qkv[:, 2 * E:], 3 * E
                Qr = qkv[:, :E].reshape(N, Lq, H, d)
                Kr, Vr = qkv[:, E:2 * E].reshape(N, Lk, H, d), qkv[:, 2 * E:].reshape(N, Lk, H, d)
            else:
                kv = torch.randn(N * Lk, 2 * E + 4, device="cuda", generator=g)
                k, v, ldk = kv, kv[:, E:], 2 * E + 4
                Kr, Vr = kv[:, :E].reshape(N, Lk, H, d), kv[:, E:2 * E].reshape(N, Lk, H, d)
                if layout == "shared_q":
                    q = torch.randn(Lq, E + 4, device="cuda", generator=g)
                    ldq, qbs = E + 4, 0
                    Qr = q[:, :E].reshape(1, Lq, H, d).expand(N, Lq, H, d)
                else:
                    q = torch.randn(N * Lq, E + 4, device="cuda", generator=g)
                    ldq, qbs = E + 4, Lq * (E + 4)
                    Qr = q[:, :E].reshape(N, Lq, H, d)
            o = sentinel((N * Lq + 3, E + 4), "f32")
            scale = 1.0 / math.sqrt(d)
            ctx.latent_attention(q=q, ldq=ldq, q_batch_stride=qbs, k=k, ldk=ldk, v=v, ldv=ldk, o=o, ldo=E + 4, N=N, Lq=Lq, Lk=Lk, H=H, d=d,
                                 scale=scale)
            torch.cuda.synchronize()
            qh, kh, vh = (t.permute(0, 2, 1, 3).double() for t in (Qr, Kr, Vr))
            ref = (torch.softmax(qh @ kh.transpose(-1, -2) * scale, -1) @ vh).permute(0, 2, 1, 3).reshape(N * Lq, E)
            what = f"{layout} Lk={Lk} d={d}"
            assert_canary(o, N * Lq, E, what)
            assert rel(o[: N * Lq, :E], ref) < 2e-6, (what, rel(o[: N * Lq, :E], ref))


@pytest.mark.gpu
@pytest.mark.parametrize("dtname", ["f16", "bf16"])
def test_small_attention_sizes(ctx, dtname):
    """ViT crops of 1 .. 16 tokens (the kernel's range; the encoders use 5, 8 and 9)."""
    dt, _ = DT[dtname]
    N, H = 13, 4
    W = 32 * H
    for S in (1, 5, 8, 9, 16):
        g = torch.Generator(device="cuda").manual_seed(S)
        qkv = torch.randn(N * S, 3 * W + 4, device="cuda", generator=g)
        o32 = sentinel((N * S + 3, W + 8), "f32")
        hi, lo = sentinel((N * S + 3, W + 8), "i16"), sentinel((N * S + 3, W + 8), "i16")
        ctx.small_attention(qkv, N=N, S=S, H=H, W=W, scale=1 / math.sqrt(32), o_hi=hi, o_lo=lo, o_f32=o32, dtype=dt)
        torch.cuda.synchronize()
        q, k, v = [qkv[:, i * W:(i + 1) * W].reshape(N, S, H, 32).transpose(1, 2).double() for i in range(3)]
        ref = (torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(32), -1) @ v).transpose(1, 2).reshape(N * S, W)
        got = o32[: N * S, :W]
        for t in (o32, hi, lo):
            assert_canary(t, N * S, W, f"S={S}")
        assert rel(got, ref) < 2e-6, (S, rel(got, ref))
        rec = f16view(hi[: N * S, :W], dt).double() + f16view(lo[: N * S, :W], dt).double()
        assert rel(rec, got) < NORM_HILO[dt], (S, rel(rec, got))


@pytest.mark.gpu
def test_vit_tokens(ctx):
    """x[n, 0] = cls + pos[0], x[n, 1 + p] = patch[n, p] + pos[1 + p]; without cls x[n, s] = patch[n, s] + pos[s]: bit for bit."""
    N, S, W = 6, 9, 64
    g = torch.Generator(device="cuda").manual_seed(3)
    pos = torch.randn(S, W, device="cuda", generator=g)
    cls = torch.randn(W, device="cuda", generator=g)
    for with_cls in (True, False):
        patch = torch.randn(N * (S - 1 if with_cls else S), W, device="cuda", generator=g)
        flat = sentinel((N * S * W + 64,), "f32")
        ctx.vit_tokens(patch, cls if with_cls else None, pos, N, S, W, flat)
        torch.cuda.synchronize()
        if with_cls:
            tok = torch.cat([cls.expand(N, 1, W), patch.view(N, S - 1, W)], 1)
        else:
            tok = patch.view(N, S, W)
        assert torch.equal(flat[: N * S * W].view(N, S, W), tok + pos[None]), with_cls
        assert (flat[N * S * W:].view(torch.int32) == S32).all()


@pytest.mark.gpu
def test_gato_positions(ctx):
    """Mask [prompt_mask | ones] and position ids [arange(n), (n - 1) on the rest of the prompt, n, n + 1, ...] of the Gato sequence,
    n = valid prompt tokens: bit for bit, including an all-padded prompt (ids -1), Lp > 256 (several columns per thread) and L == Lp."""
    B = 5
    g = torch.Generator().manual_seed(4)
    for Lp in (1, 7, 300):
        for L in (Lp, Lp + 1, Lp + 40):
            pm = torch.rand(B, Lp, generator=g) > 0.4
            pm[0] = True
            pm[1] = False
            mask = torch.full((B, L), 0xA5, dtype=torch.uint8, device="cuda")
            pos = torch.full((B, L), -7, dtype=torch.int64, device="cuda")
            ctx.gato_positions(pm.to(torch.uint8).cuda(), L, mask, pos)
            torch.cuda.synchronize()
            m_ref = torch.cat([pm, torch.ones(B, L - Lp, dtype=torch.bool)], 1)
            ids = []
            for n in pm.sum(1).tolist():
                ids.append(torch.cat([torch.arange(n), torch.full((Lp - n,), n - 1), torch.arange(n, n + L - Lp)]))
            assert torch.equal(mask.cpu(), m_ref.to(torch.uint8)), (Lp, L)
            assert torch.equal(pos.cpu(), torch.stack(ids)), (Lp, L)


@pytest.mark.gpu
@pytest.mark.parametrize("rms", [False, True])
def test_row_stats_finalize(ctx, rms):
    """(sum, sum of squares) partials -> (mean, rstd), LayerNorm form or T5 RMSNorm form (0, 1/sqrt(mean(x^2) + eps))."""
    rows, parts, cols = 1037, 12, 768
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(rows, cols, device="cuda", generator=g) * 2 + 0.3
    xp = x.view(rows, parts, cols // parts)
    partial = torch.stack([xp.sum(2), (xp * xp).sum(2)], 2).contiguous()
    st = sentinel((rows + 3, 2), "f32")
    ctx.row_stats_finalize(partial, cols, 1e-5, st, rms=rms)
    torch.cuda.synchronize()
    assert_canary(st, rows, 2, "row_stats_finalize")
    p64 = partial.double()
    s1, s2 = p64[:, :, 0].sum(1) / cols, p64[:, :, 1].sum(1) / cols
    mean = torch.zeros_like(s1) if rms else s1
    rstd = torch.rsqrt(s2 - mean * mean + 1e-5)
    got = st[:rows].double()
    assert ((got[:, 0] - mean).abs() <= 1e-6 * (1 + mean.abs())).all()
    assert ((got[:, 1] - rstd).abs() <= 1e-6 * rstd).all()
