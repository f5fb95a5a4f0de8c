"""Kernels against fp64 across operand magnitudes and score distributions, not only unit-variance noise.

The other kernel suites feed torch.randn operands: O(1) values, attention scores with a spread of about one nat, no dominant key,
a softmax maximum that hardly moves from one key chunk to the next.  The numerics here depend on magnitude:

  1. the split operand formats across row scales 2^-16 .. 2^12, an outlier channel, a large row offset, and the LayerNorm fold
     on rows with large means (the (1 + mean^2/var)^1/2 cancellation bound of DESIGN.md section 5);
  2. every attention kernel on constructed score distributions: a maximum that rises (or falls) by 3 nats per 64-key chunk, one
     key 10 / 30 / 80 nats above the rest in the first or last chunk or past the causal diagonal, a common offset of 1e3, T5's
     unscaled scores with relative bias, and Q/K/V scaled by 2^-10 .. 2^8;
  3. head_select on ties, one-wide heads, equal and -inf logits and logits around +-1e4;
  4. the largest |x| of every operand that reaches an e4m3 view while the 200M policy runs in f16f8.

Every bar that rests on a measurement says so where it is defined; the measurements were taken on an H100 80GB HBM3 (700 W power
limit).  Each test prints its table of worst errors.
"""
import math
import os
import sys

import pytest
import torch

from tests.test_kernel_variants_gpu import (ATTN_TOL, DT, NAN16, GemmOperands, as_bits16, assert_canary, f16view, fold_ln, ln64, rel,
                                            sentinel, split_statement)

F = torch.nn.functional


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    return _C.Context.get(torch.device("cuda", 0))


# ------------------------------------------------------------------------------------------------------------------------------
# 1. split operand formats and the GEMM across magnitudes
# ------------------------------------------------------------------------------------------------------------------------------
GEMM_BAR = {"f16x3": 2e-5, "bf16x3": 1e-4, "f16f8": 4e-5}  # test_kernels_gpu.py: test_gemm_plain (split), test_gemm_f16f8
EXPS = list(range(-16, 13, 2))  # rows ~ 2^e N(0, 1)
# Row scales 2^e at which each format holds its bar (the table in DESIGN.md section 3).  fp16 (hi, lo): lo turns subnormal below
# |x| ~ 2^-3 and the pair's absolute error floors at 2^-25; e4m3 lo8 = e4m3((x - hi) 2^10) floors at 2^-20 absolute and saturates
# once |x| >= 1024.  bf16 has fp32's exponent range.  Measured worst rel-L2 inside the range: f16x3 1.72e-5 (at 2^-10; 2.9e-6 from
# 2^-6 up), bf16x3 5.4e-6, f16f8 1.96e-5 (at 2^-4; 1.1e-5 from 2^-2 up).  Just outside: f16x3 6.7e-5 at 2^-12, f16f8 7.0e-5 at 2^-6.
IN_RANGE = {"f16x3": (-10, 12), "bf16x3": (-16, 12), "f16f8": (-4, 6)}
# Outside the range the kernel's error stays within FMT_FACTOR x the operand format's own error plus the bar.  The weight side of
# f16f8 carries e4m3 views of the same precision as the activation's, so the kernel's error there is twice the activation format's
# alone (measured 2.0x at 2^-8); the 16-bit pairs measure 1.0x.
FMT_FACTOR = 3.0
F8_LIMIT = 1024.0  # |x| at which lo8 saturates (e4m3 max 448 = (x - hi16) * 2^10 with fp16 ulp 1)
ROWS = 8


def magnitude_rows(K, seed):
    """[groups * ROWS, K] fp32 and the group labels: one group per 2^e, an outlier channel 2^10 above rows at 2^-4 and at 2^0, and
    rows with mean 1e3, sigma 1."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    blocks, names = [], []
    for e in EXPS:
        blocks.append(rn(ROWS, K) * 2.0 ** e)
        names.append(e)
    for base in (-4, 0):
        x = rn(ROWS, K) * 2.0 ** base
        x[:, K // 3] *= 1024.0
        blocks.append(x)
        names.append(f"outlier 2^{base}+10")
    blocks.append(1e3 + rn(ROWS, K))
    names.append("mean 1e3")
    return torch.cat(blocks), names


def decoded_a(ops, mode):
    """The A operand as the kernel's format carries it, fp64 [M, K] (hi + lo, or hi16 + lo8 / 2^10)."""
    h = f16view(ops.a_hi[: ops.M, : ops.K], ops.dt).double()
    if mode == "f16f8":
        return h + ops.a8[0][: ops.M, : ops.K].view(torch.float8_e4m3fn).double() / 1024.0
    return h + f16view(ops.a_lo[: ops.M, : ops.K], ops.dt).double()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["f16x3", "bf16x3", "f16f8"])
def test_gemm_operand_magnitudes(ctx, mode):
    """Plain GEMM (K = 768 and a ragged 392) on rows scaled by 2^e, against fp64 A @ W^T.  Inside IN_RANGE the bar holds; outside
    it the error stays within what the operand format itself carries (the exact product of the decoded operand, 'fmt') plus the bar,
    grows monotonically as the rows shrink, and the output stays finite wherever hi does not saturate.  f16f8 past |x| = 1024
    (lo8 saturated) must stay finite only."""
    lo_e, hi_e = IN_RANGE[mode]
    bar = GEMM_BAR[mode]
    table = {}
    failures = []
    for K, seed in ((768, 11), (392, 12)):
        A, names = magnitude_rows(K, seed)
        M, N = A.shape[0], 256
        g = torch.Generator(device="cuda").manual_seed(seed + 100)
        W = torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
        ops = GemmOperands(ctx, A, W, mode)
        out = sentinel((M + 3, N + 8), "f32")
        ctx.gemm(M=M, N=N, K=K, out_f32=out, **ops.kwargs())
        torch.cuda.synchronize()
        assert_canary(out, M, N, f"{mode} K={K}")
        got = out[:M, :N]
        ref = A.double() @ W.double().t()
        fmt = decoded_a(ops, mode) @ W.double().t()
        for i, name in enumerate(names):
            r = slice(i * ROWS, (i + 1) * ROWS)
            amax = A[r].abs().max().item()
            e, ef = rel(got[r], ref[r]), rel(fmt[r], ref[r])
            key = (name, K)
            table[key] = (e, ef, amax)
            what = f"{mode} K={K} rows {name} (max|x| {amax:.3g}): err {e:.2e}, format alone {ef:.2e}"
            if not torch.isfinite(got[r]).all():
                failures.append(what + ": non-finite output")
                continue
            if mode == "f16f8" and amax >= F8_LIMIT:  # lo8 saturated: the documented end of the format's range
                continue
            if isinstance(name, int) and lo_e <= name <= hi_e and e >= bar:
                failures.append(what + f": over the bar {bar:.0e} inside the documented range")
            if e > bar + FMT_FACTOR * ef:
                failures.append(what + ": more than the format's own error plus the bar")
        # below the range the error only grows as the rows shrink (monotone within 20 %)
        below = [e for e in EXPS if e < lo_e]
        for e_small, e_big in zip(below, below[1:] + [lo_e]):
            if table[(e_small, K)][0] < 0.8 * table[(e_big, K)][0]:
                failures.append(f"{mode} K={K}: error at 2^{e_small} ({table[(e_small, K)][0]:.2e}) below the one at 2^{e_big} "
                                f"({table[(e_big, K)][0]:.2e})")
    print(f"\n{mode} GEMM rel-L2 against fp64 by row scale (bar {bar:.0e} on 2^{lo_e} .. 2^{hi_e}):")
    print(f"  {'rows':>18} {'K':>4} {'max|x|':>9} {'kernel':>9} {'format':>9}")
    for (name, K), (e, ef, amax) in table.items():
        label = f"2^{name}" if isinstance(name, int) else name
        print(f"  {label:>18} {K:>4} {amax:>9.3g} {e:>9.2e} {ef:>9.2e}")
    assert not failures, "\n".join(failures)


MEANS = [0.0, 10.0, 1e2, 1e3, 1e4]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["f16x3", "bf16x3", "f16f8"])
def test_folded_layernorm_on_large_means(ctx, mode):
    """W LN(x) + b with the LayerNorm folded into the GEMM (row_stats / ln_c1) on rows of mean mu and sigma 1.  The epilogue's
    rstd (W*gamma x - mean c1) cancels mean c1, so the product error grows by (1 + mu^2 / var)^1/2 (DESIGN.md section 5): the bar is
    2 x GEMM_BAR times that factor.  f16f8 rows past |x| = 1024 saturate lo8 and are held to finiteness only."""
    bar = GEMM_BAR[mode]
    K, N = 768, 256
    g = torch.Generator(device="cuda").manual_seed(21)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    A = torch.cat([mu + rn(ROWS, K) for mu in MEANS])
    W, b = rn(N, K) / math.sqrt(K), 0.5 * rn(N)
    gam, bet = 1.0 + 0.1 * rn(K), 0.1 * rn(K)
    wf, c1, bf = fold_ln(W, b, gam, bet)
    A64 = A.double()
    st = torch.stack([A64.mean(1), 1.0 / torch.sqrt(A64.var(1, unbiased=False) + 1e-5)], 1).float().contiguous()
    ops = GemmOperands(ctx, A, wf, mode)
    M = A.shape[0]
    out = sentinel((M + 3, N + 8), "f32")
    ctx.gemm(M=M, N=N, K=K, bias=bf, out_f32=out, row_stats=st, ln_c1=c1, ln_cols=1, **ops.kwargs())
    torch.cuda.synchronize()
    assert_canary(out, M, N, mode)
    got = out[:M, :N]
    ref = ln64(A, gam, bet) @ W.double().t() + b.double()
    rows = []
    for i, mu in enumerate(MEANS):
        r = slice(i * ROWS, (i + 1) * ROWS)
        var = A64[r].var(1, unbiased=False).mean().item()
        allowed = 2 * bar * math.sqrt(1.0 + mu * mu / var)
        e = rel(got[r], ref[r])
        rows.append((mu, e, allowed))
        assert torch.isfinite(got[r]).all(), (mode, mu)
        if mode == "f16f8" and A[r].abs().max().item() >= F8_LIMIT:
            continue
        assert e < allowed, (mode, mu, e, allowed)
    print(f"\n{mode} folded LayerNorm: " + "  ".join(f"mean {mu:g}: {e:.2e} (bound {a:.1e})" for mu, e, a in rows))


# ------------------------------------------------------------------------------------------------------------------------------
# 2. attention on constructed score distributions
# ------------------------------------------------------------------------------------------------------------------------------
# A case passes when its rel-L2 against fp64 is at most max(ATTN_TOL, C32 * e32), and for bf16 pairs max(.., CFMT * efmt):
#   e32  = rel-L2 of the same formula evaluated by torch in fp32 on the same operands (fp32 itself loses bits at a score offset of 1e3);
#   efmt = rel-L2 of exact attention on the operands as the (hi, lo) format carries them, with the output rounded to that format.
# A bf16 pair carries 16 significand bits and the kernels drop its lo*lo product (2^-16 of each score): with scores of ~1e3 nats
# (offset 1e3, Q/K at 2^5) that alone exceeds ATTN_TOL, and efmt measures it.  fp16 pairs get no such term: they carry 22 bits
# wherever |x| >= 2^-3, and operands below that are split with a power-of-two scale (run_attention's pow2), as weights are.
# Measured: err / e32 reaches 1.2 at the 1e3 offset in f16x3 (err 1.1e-4, fp32 8.9e-5) and 3 in single-pass f16; err / efmt
# reaches 3.7 in bf16x3 with Q/K/V at 2^5 (mma.sync, D = 64).  fp16 pairs split with the power-of-two scale: at most 2.0e-6 from
# 2^-10 to 2^-2, 5.7e-6 at 2^2.  Unscaled they would give 2.2e-5 at 2^-6 and 1.0e-4 at 2^-10, exactly efmt: the loss is the
# split's, before any kernel runs.  Worst err / allowed over every kernel: 0.86 (bf16x3 at 2^5, mma.sync with bias).
C32, CFMT = 4.0, 5.0
B_ATT, H_ATT = 2, 2


def attn_reference(Q, K, V, *, B, H, Lq, Lk, D, scale, causal, q_pos, key_mask, rel_bias, dtype):
    """The kernels' formula in `dtype`: s = q k^T scale (+ bias[h][j - i + Lk - 1]); causal: key j > q_pos[b] + i gets -1e4 (the
    reference's soft mask); padded key: + finfo(fp32).min; softmax; @ v.  Q [B*Lq, H*D], K / V [B*Lk, H*D] -> [B*Lq, H*D]."""
    heads = lambda x, L: x.to(dtype).reshape(B, L, H, D).permute(0, 2, 1, 3)
    s = heads(Q, Lq) @ heads(K, Lk).transpose(-1, -2) * scale
    ii = torch.arange(Lq, device=Q.device)[:, None]
    jj = torch.arange(Lk, device=Q.device)[None, :]
    if rel_bias is not None:
        s = s + rel_bias.to(dtype)[:, jj - ii + Lk - 1][None]
    if causal:
        allowed = jj[None] <= ii[None] + q_pos.to(Q.device).long()[:, None, None]  # [B, Lq, Lk]
        s = torch.where(allowed[:, None], s, torch.tensor(-1e4, dtype=dtype, device=Q.device))
    if key_mask is not None:
        s = s + (1.0 - key_mask[:, None, None, :].to(dtype)) * torch.finfo(torch.float32).min
    o = torch.softmax(s, -1) @ heads(V, Lk)
    return o.permute(0, 2, 1, 3).reshape(B * Lq, H * D)


def pow2_scale(x):
    """The power of two that puts max|x| in [512, 1024), as weights are packed (engine._pow2_scale)."""
    return 2.0 ** math.floor(math.log2(1024.0 / x.abs().max().item()))


def run_attention(ctx, dtname, split, Q, K, V, *, Lq, Lk, D, scale, causal=False, q_pos0=0, q_pos=None, rel_bias=None, key_mask=None,
                  pow2=False):
    """One call through the C ABI with NaN in every operand column past the head block and sentinels around the output.
    pow2: Q, K and V are split with power-of-two scales sq, sk, sv that put each one's max|x| in [512, 1024); the kernel gets
    scale / (sq sk), and its output, a convex combination of V's rows, comes back scaled by sv (a consumer GEMM folds 1 / sv into
    acc_scale).  Nothing in the kernel changes: the scales fold into its score scale and pass through its normaliser exactly.
    -> (kernel error, fp32 formula error, format error) against fp64."""
    dt, tdt = DT[dtname]
    B, H = B_ATT, H_ATT
    E = H * D
    sq, sk, sv = (pow2_scale(Q), pow2_scale(K), pow2_scale(V)) if pow2 else (1.0, 1.0, 1.0)

    def ops(x, ld, parts):
        """parts: [(tensor, power-of-two scale)] side by side in one [rows, ld] operand; NaN in the columns past them."""
        rows = x.shape[0]
        hi = torch.empty(rows, ld, dtype=torch.int16, device="cuda")
        lo = torch.empty_like(hi) if split else None
        c0 = 0
        for t, s in parts:
            ctx.split(t.contiguous(), hi[:, c0:], None if lo is None else lo[:, c0:], cols=E, pad_cols=E, scale=s, dtype=dt)
            c0 += E
        for t in (hi, lo):
            if t is not None:
                t[:, c0:] = NAN16[dt]
        return hi, lo

    def decode(hi, lo, c0, s):
        x = f16view(hi[:, c0:c0 + E], dt).double()
        return (x if lo is None else x + f16view(lo[:, c0:c0 + E], dt).double()) / s

    qh, ql = ops(Q, E + 8, [(Q, sq)])
    kvh, kvl = ops(K, 2 * E + 8, [(K, sk), (V, sv)])
    o_hi, o_lo = sentinel((B * Lq + 3, E + 8), "i16"), sentinel((B * Lq + 3, E + 8), "i16")
    qp = None if q_pos is None else torch.tensor(q_pos, dtype=torch.int32, device="cuda")
    ctx.attention(q=(qh, ql, E + 8, 0), k=(kvh, kvl, 2 * E + 8, 0), v=(kvh, kvl, 2 * E + 8, E), o=(o_hi, o_lo, E + 8, 0), B=B, H=H,
                  Lq=Lq, Lk=Lk, D=D, scale=scale / (sq * sk), causal=causal,
                  key_mask=None if key_mask is None else key_mask.to(torch.uint8), rel_bias=rel_bias, dtype=dt, q_pos0=q_pos0, q_pos=qp)
    torch.cuda.synchronize()
    assert_canary(o_hi, B * Lq, E, "o_hi"); assert_canary(o_lo, B * Lq, E, "o_lo")
    got = decode(o_hi[: B * Lq], o_lo[: B * Lq], 0, sv)
    assert torch.isfinite(got).all()
    dec = (decode(qh, ql, 0, sq), decode(kvh, kvl, 0, sk), decode(kvh, kvl, E, sv))
    # the single-pass kernels multiply the rounded operands: that is their exact operation
    exact = (Q, K, V) if split else tuple(t.to(tdt).float() for t in (Q, K, V))
    qpos_t = torch.tensor(q_pos if q_pos is not None else [q_pos0] * B)
    kw = dict(B=B, H=H, Lq=Lq, Lk=Lk, D=D, scale=scale, causal=causal, q_pos=qpos_t, key_mask=key_mask, rel_bias=rel_bias)
    ref = attn_reference(*exact, dtype=torch.float64, **kw)
    e32 = rel(attn_reference(*exact, dtype=torch.float32, **kw), ref)
    efmt = 0.0
    if split:
        r = (attn_reference(*dec, dtype=torch.float64, **kw) * sv).float()
        hb, lb = split_statement(r, dt)
        pair = (hb.to(torch.int16).view(tdt).double() + lb.to(torch.int16).view(tdt).double()) / sv
        efmt = rel(pair, ref)
    return rel(got, ref), e32, efmt


def logits_qk(g, L_q, Lk, D, scale, target, a=4.0, noise=0.5):
    """Q [B*Lq, H*D], K [B*Lk, H*D] whose scores s_ij = scale q_i . k_j are target[j] + O(noise^2): per head a unit direction u, q_i =
    a u + eps_i and k_j = target[j] / (scale a) u + eta_j with eps, eta orthogonal to u."""
    B, H = B_ATT, H_ATT
    Q = torch.empty(B, L_q, H, D, device="cuda")
    K = torch.empty(B, Lk, H, D, device="cuda")
    for h in range(H):
        u = torch.randn(D, device="cuda", generator=g, dtype=torch.float64)
        u = u / u.norm()
        eps = torch.randn(B, L_q, D, device="cuda", generator=g, dtype=torch.float64) * noise
        eta = torch.randn(B, Lk, D, device="cuda", generator=g, dtype=torch.float64) * noise
        eps = eps - (eps @ u)[..., None] * u
        eta = eta - (eta @ u)[..., None] * u
        Q[:, :, h] = (a * u + eps).float()
        K[:, :, h] = (target.double()[None, :, None] / (scale * a) * u + eta).float()
    return Q.reshape(B * L_q, H * D), K.reshape(B * Lk, H * D)


def distributions(Lk, t5=False):
    """name -> per-key target logits (or ('mag', e) for plain noise at 2^e)."""
    j = torch.arange(Lk, device="cuda", dtype=torch.float64)
    chunk = torch.div(j, 64, rounding_mode="floor")
    d = {"rise 3/chunk": 3.0 * chunk, "fall 3/chunk": 3.0 * (chunk.max() - chunk)}
    for p in (10, 30, 80):
        for where, k in (("first", 3), ("last", Lk - 2)):
            t = torch.zeros(Lk, device="cuda", dtype=torch.float64)
            t[k] = p
            d[f"peak {p} {where}"] = t
    g = torch.Generator(device="cuda").manual_seed(Lk)
    d["offset 1e3"] = 1e3 + torch.randn(Lk, device="cuda", generator=g, dtype=torch.float64)
    if t5:
        d["t5 20..50"] = 20.0 + 30.0 * torch.rand(Lk, device="cuda", generator=g, dtype=torch.float64)
    for e in (-10, -6, -2, 2, 5, 8):
        d[f"mag 2^{e}"] = ("mag", e)
    return d


def make_case(seed, Lq, Lk, D, scale, target):
    g = torch.Generator(device="cuda").manual_seed(seed)
    E = H_ATT * D
    if isinstance(target, tuple):
        s = 2.0 ** target[1]
        Q = torch.randn(B_ATT * Lq, E, device="cuda", generator=g) * s
        K = torch.randn(B_ATT * Lk, E, device="cuda", generator=g) * s
        V = torch.randn(B_ATT * Lk, E, device="cuda", generator=g) * s
    else:
        Q, K = logits_qk(g, Lq, Lk, D, scale, target)
        V = torch.randn(B_ATT * Lk, E, device="cuda", generator=g)
    return Q, K, V


# (name, options, D, Lq, Lk, relative bias, formats): every kernel vima_attention dispatches to
ATTN_KERNELS = {
    "tc": (dict(attn="tc"), 32, 256, 512, False, ("f16-x3", "bf16-x3")),
    "tc_tail": (dict(attn="tc"), 32, 136, 512, False, ("f16-x3", "bf16-x3")),  # 128 rows on wgmma, 8 on the SIMT tail kernel
    "tc_tail129": (dict(attn="tc"), 32, 129, 512, False, ("f16-x3",)),
    "tc_tail_off": (dict(attn="tc", attn_tail="off"), 32, 136, 512, False, ("f16-x3", "bf16-x3")),
    "mma_d32": (dict(attn="mma"), 32, 256, 512, False, ("f16-x3", "bf16-x3", "f16-single", "bf16-single")),
    "mma_d64": (dict(attn="mma"), 64, 200, 384, False, ("f16-x3", "bf16-x3", "f16-single", "bf16-single")),
    "mma_bias": (dict(attn="mma"), 64, 384, 384, True, ("f16-x3", "bf16-x3", "f16-single", "bf16-single")),
    "bias_tc": (dict(attn="tc", attn_bias="tc"), 64, 512, 512, True, ("f16-x3", "bf16-x3", "f16-single", "bf16-single")),
}


@pytest.fixture
def attn_options(ctx):
    def set_(**kw):
        for k, v in kw.items():
            ctx.set_option(k, v)

    yield set_
    set_(attn="tc", attn_tail="kernel", attn_bias="auto")


def check_attention_cases(cases, label):
    """cases: list of (what, err, e32, efmt, tol, cfmt).  Prints the table and the worst ratio err / allowed; asserts every case."""
    failures, worst = [], (0.0, "")
    for what, e, e32, efmt, tol, cfmt in cases:
        allowed = max(tol, C32 * e32, cfmt * efmt)
        if e / allowed > worst[0]:
            worst = (e / allowed, what)
        if not e <= allowed:
            failures.append(f"{what}: err {e:.2e} > allowed {allowed:.2e} (bar {tol:.0e}, fp32 {e32:.2e}, format {efmt:.2e})")
    print(f"\n{label}: {len(cases)} cases, worst err / allowed {worst[0]:.2f} at {worst[1]}")
    for what, e, e32, efmt, tol, cfmt in cases:
        print(f"  {what:<48} err {e:.2e}  fp32 {e32:.2e}  format {efmt:.2e}")
    assert not failures, "\n".join(failures)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", list(ATTN_KERNELS))
def test_attention_score_distributions(ctx, attn_options, kernel):
    """Every kernel and format it supports on every constructed distribution; the non-bias kernels also causally with the queries
    last (q_pos0 = Lk - Lq), so a peak in the last chunk sits past the diagonal of most rows, and with per-batch q_pos (tc, mma)."""
    opts, D, Lq, Lk, bias, formats = ATTN_KERNELS[kernel]
    attn_options(**opts)
    t5 = bias
    scale = 1.0 if t5 else 1.0 / math.sqrt(D)
    cases = []
    for fmt in formats:
        dtname, mode = fmt.split("-")
        split = mode == "x3"
        tol = ATTN_TOL[(DT[dtname][0], split)]
        for n, (name, target) in enumerate(distributions(Lk, t5).items()):
            Q, K, V = make_case(1000 * n + Lq, Lq, Lk, D, scale, target)
            kw = {}
            if bias:
                g = torch.Generator(device="cuda").manual_seed(n)
                kw["rel_bias"] = (torch.rand(H_ATT, 2 * Lk - 1, device="cuda", generator=g) * 20.0 - 10.0)
            runs = [("", kw)]
            if not bias and not name.startswith("mag"):
                runs.append((" causal q_pos0", dict(causal=True, q_pos0=Lk - Lq)))
                if kernel in ("tc", "mma_d32"):
                    runs.append((" causal q_pos", dict(causal=True, q_pos=[Lk - Lq - 100, Lk - Lq])))
            if fmt == "f16-x3" and name.startswith("mag"):
                # fp16 pairs hold 22 bits only above |x| ~ 2^-3: operands below that are split with a power-of-two scale, as weights are
                runs = [(" pow2", dict(kw, pow2=True))] + (runs if target[1] >= -2 else [])
            for suffix, extra in runs:
                e, e32, efmt = run_attention(ctx, dtname, split, Q, K, V, Lq=Lq, Lk=Lk, D=D, scale=scale, **extra)
                cases.append((f"{fmt} {name}{suffix}", e, e32, efmt, tol, CFMT if fmt == "bf16-x3" else 0.0))
    check_attention_cases(cases, f"attention {kernel} (D={D}, Lq={Lq}, Lk={Lk})")


@pytest.mark.gpu
def test_small_and_latent_attention_score_distributions(ctx):
    """The fp32 full-width softmax kernels (ViT crops: small_attention, 16 tokens; Perceiver: latent_attention, 16 keys, d = 64) on
    the same distributions, against max(2e-6, C32 x the fp32 formula's own error)."""
    S, D = 16, 32
    cases = []
    for n, (name, target) in enumerate(distributions(S).items()):
        if not isinstance(target, tuple):  # 'last' is key 14 of 16; 'rise' is flat over one chunk: spread it over the 16 keys
            target = target if not name.startswith(("rise", "fall")) else 3.0 * torch.arange(S, device="cuda", dtype=torch.float64) * (
                1 if name.startswith("rise") else -1)
        # small_attention: qkv [N*S, 3W] with W = H*32, scale 1/sqrt(32); here N = B_ATT, H = H_ATT
        Q, K, V = make_case(7 + n, S, S, D, 1 / math.sqrt(D), target)
        W = H_ATT * D
        qkv = torch.cat([Q, K, V, torch.zeros(B_ATT * S, 4, device="cuda")], 1).contiguous()
        o32 = sentinel((B_ATT * S + 3, W + 8), "f32")
        hi, lo = sentinel((B_ATT * S + 3, W + 8), "i16"), sentinel((B_ATT * S + 3, W + 8), "i16")
        ctx.small_attention(qkv, N=B_ATT, S=S, H=H_ATT, W=W, scale=1 / math.sqrt(D), o_hi=hi, o_lo=lo, o_f32=o32, dtype=0)
        torch.cuda.synchronize()
        assert_canary(o32, B_ATT * S, W, "small_attention")
        assert_canary(hi, B_ATT * S, W, "small_attention o_hi"); assert_canary(lo, B_ATT * S, W, "small_attention o_lo")
        # the (hi, lo) pair is the saturating split of the fp32 output, bit for bit
        want_hi, want_lo = split_statement(o32[: B_ATT * S, :W], 0)
        assert torch.equal(as_bits16(hi[: B_ATT * S, :W]), want_hi) and torch.equal(as_bits16(lo[: B_ATT * S, :W]), want_lo), name
        kw = dict(B=B_ATT, H=H_ATT, Lq=S, Lk=S, D=D, scale=1 / math.sqrt(D), causal=False, q_pos=None, key_mask=None, rel_bias=None)
        ref = attn_reference(Q, K, V, dtype=torch.float64, **kw)
        got = o32[: B_ATT * S, :W]
        assert torch.isfinite(got).all(), name
        cases.append((f"small S=16 {name}", rel(got, ref), rel(attn_reference(Q, K, V, dtype=torch.float32, **kw), ref), 0.0, 2e-6, 0.0))
        # latent_attention, d = 64: 4 latent queries against 16 keys
        d, Lq = 64, 4
        Q, K, V = make_case(77 + n, Lq, S, d, 1 / math.sqrt(d), target)
        E = H_ATT * d
        o = sentinel((B_ATT * Lq + 3, E + 4), "f32")
        ctx.latent_attention(q=Q, ldq=E, q_batch_stride=Lq * E, k=K, ldk=E, v=V, ldv=E, o=o, ldo=E + 4, N=B_ATT, Lq=Lq, Lk=S, H=H_ATT, d=d,
                             scale=1 / math.sqrt(d))
        torch.cuda.synchronize()
        assert_canary(o, B_ATT * Lq, E, "latent_attention")
        kw.update(Lq=Lq, D=d, scale=1 / math.sqrt(d))
        ref = attn_reference(Q, K, V, dtype=torch.float64, **kw)
        got = o[: B_ATT * Lq, :E]
        assert torch.isfinite(got).all(), name
        cases.append((f"latent d=64 {name}", rel(got, ref), rel(attn_reference(Q, K, V, dtype=torch.float32, **kw), ref), 0.0, 2e-6, 0.0))
    check_attention_cases(cases, "small / latent attention")


# ------------------------------------------------------------------------------------------------------------------------------
# 3. head_select: ties and extremes
# ------------------------------------------------------------------------------------------------------------------------------
HEAD_WIDTHS = [1, 33, 64, 100, 7, 50, 130]


def head_select_rows():
    """[rows, sum(HEAD_WIDTHS)] fp32, each row one kind of logits in every head, and the row names."""
    g = torch.Generator().manual_seed(31)
    total = sum(HEAD_WIDTHS)
    rows, names = [], []

    def per_head(fn):
        parts = [fn(w) for w in HEAD_WIDTHS]
        return torch.cat(parts).float()

    def ties(w, gap):  # the maximum at index 1 and again 'gap' (and 2 gap) further on
        x = torch.randn(w, generator=g)
        for k in range(1, w, gap):
            x[k] = 5.0
        return x

    def last(w):
        x = torch.randn(w, generator=g)
        x[-1] = 6.0
        return x

    def some_neg_inf(w):
        x = torch.randn(w, generator=g)
        x[torch.arange(w) % 3 == 0] = -math.inf
        if w == 1:
            x[0] = 0.5
        return x

    def first_last_tie(w):
        x = torch.randn(w, generator=g)
        x[0] = x[-1] = 7.0
        return x

    kinds = {
        "randn": lambda w: torch.randn(w, generator=g),
        "tie 32 apart (same lane)": lambda w: ties(w, 32),
        "tie 64 apart": lambda w: ties(w, 64),
        "tie 5 apart (other lanes)": lambda w: ties(w, 5),
        "max at last index": last,
        "tie first and last": first_last_tie,
        "all equal": lambda w: torch.full((w,), 0.25),
        "all equal 1e4": lambda w: torch.full((w,), 1e4),
        "some -inf": some_neg_inf,
        "all -inf": lambda w: torch.full((w,), -math.inf),
        "1e4 + randn": lambda w: 1e4 + torch.randn(w, generator=g),
        "-1e4 + randn": lambda w: -1e4 + torch.randn(w, generator=g),
        "+-1e4 + randn": lambda w: torch.sign(torch.randn(w, generator=g)) * 1e4 + torch.randn(w, generator=g),
        "1e4 + ties": lambda w: 1e4 + ties(w, 7),
    }
    for name, fn in kinds.items():
        rows.append(per_head(fn))
        names.append(name)
    x = torch.stack(rows)
    assert x.shape[1] == total
    return x, names


@pytest.mark.gpu
def test_head_select_ties_and_extremes(ctx):
    """Modes equal torch.distributions.Categorical(logits=...).probs.argmax(-1) (the reference's mode, dists.py) bit for bit, exact
    ties included (first index wins, across lanes and within one lane); normalised logits equal fp64 log_softmax within a few fp32
    ulps of the head's largest |logit|.  A head of all -inf logits has NaN probabilities: mode 0 (torch's argmax of them) and NaN
    normalised logits (log_softmax's value)."""
    x, names = head_select_rows()
    B, total, n_heads = x.shape[0], x.shape[1], len(HEAD_WIDTHS)
    off = torch.tensor([0] + list(torch.cumsum(torch.tensor(HEAD_WIDTHS), 0)), dtype=torch.int32)
    norm = torch.full((B, total), 123.0, device="cuda")
    modes = torch.full((B, n_heads), -5, dtype=torch.int64, device="cuda")
    ctx.head_select(x.cuda(), B, n_heads, off.cuda(), norm, modes)
    torch.cuda.synchronize()
    norm, modes = norm.cpu(), modes.cpu()
    failures = []
    worst = 0.0
    for h, (o0, o1) in enumerate(zip(off[:-1].tolist(), off[1:].tolist())):
        xs = x[:, o0:o1]
        want = torch.distributions.Categorical(logits=xs, validate_args=False).probs.argmax(-1)
        ref = torch.log_softmax(xs.double(), -1)
        for r in range(B):
            what = f"row '{names[r]}' head {h} (width {o1 - o0})"
            if modes[r, h].item() != want[r].item():
                failures.append(f"{what}: mode {modes[r, h].item()}, torch {want[r].item()}")
            got, rr = norm[r, o0:o1].double(), ref[r]
            if torch.isnan(rr).all():
                if not torch.isnan(got).all():
                    failures.append(f"{what}: normalised logits {got[:4].tolist()}, want NaN")
                continue
            ninf = torch.isinf(rr)
            if not torch.equal(got[ninf], rr[ninf]):
                failures.append(f"{what}: -inf logits not normalised to -inf")
            big = xs[r][~ninf].abs().max().item() if (~ninf).any() else 0.0
            err = (got[~ninf] - rr[~ninf]).abs()
            allowed = 8 * 2.0 ** -24 * (big + rr[~ninf].abs() + 8.0)
            worst = max(worst, (err / allowed).max().item() if err.numel() else 0.0)
            if (err > allowed).any():
                failures.append(f"{what}: normalised logits off by {err.max().item():.3g}")
    print(f"\nhead_select: {B} rows x {n_heads} heads, modes exact, worst normalised-logit error {worst:.2f} of its bound")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------------------------------------
# 4. the operand range the f16f8 format assumes, measured on the 200M policy
# ------------------------------------------------------------------------------------------------------------------------------
# DESIGN.md section 3: lo8 saturates once |x| >= 1024; the decoder's and the ViT's un-normalised streams are said to stay O(10).  The
# largest |x| at any e4m3 site of cfg3_small on the deterministic detgen weights must stay below 1024 / F8_MARGIN.  Measured: 13.8
# (the decoder's c_proj input after the GEGLU, xattn_gpt.py forward), 10.3 (the ViT's folded-LN c_fc input), 74x below saturation.
F8_MARGIN = 8.0


SITE_CLASSES = ("folded-LN input", "attention output", "GEGLU output")


@pytest.fixture
def e4m3_site_maxima(monkeypatch):
    """Wraps _C.Context.gemm / attention / norm: for every GEMM whose A operand carries e4m3 views, the largest |hi16| of A, by
    calling site, with the site's class: a folded-LN input (the GEMM applies row statistics), an attention output or a GEGLU output
    (the last kernel that wrote A's storage was an attention call with e4m3 views or a GLU GEMM), or 'other'."""
    from vima_b200 import _C

    sites = {}
    producer = {}  # storage pointer -> class of the last kernel that wrote it
    orig = {n: getattr(_C.Context, n) for n in ("gemm", "attention", "norm")}
    pkg = os.path.dirname(os.path.abspath(_C.__file__))
    root = os.path.dirname(pkg)
    here = {os.path.join(pkg, "_C.py"), os.path.join(pkg, "engine.py"), os.path.abspath(__file__)}
    store = lambda t: t.untyped_storage().data_ptr()

    def gemm(self, **kw):
        if kw.get("a_lo8") is not None:
            f = sys._getframe(1)
            while os.path.abspath(f.f_code.co_filename) in here:
                f = f.f_back
            cls = "folded-LN input" if kw.get("row_stats") is not None else producer.get(store(kw["a_hi"]), "other")
            key = (f"{os.path.relpath(f.f_code.co_filename, root)}:{f.f_lineno} ({f.f_code.co_name})", cls)
            a = kw["a_hi"][: kw["M"], : kw["K"]].view(torch.float16)
            m = a.float().abs().max()
            sites[key] = torch.maximum(sites[key], m) if key in sites else m
        out = orig["gemm"](self, **kw)
        if kw.get("out_hi") is not None:
            producer[store(kw["out_hi"])] = "GEGLU output" if kw.get("glu") and kw.get("out_lo8") is not None else "other"
        return out

    def attention(self, **kw):
        out = orig["attention"](self, **kw)
        producer[store(kw["o"][0])] = "attention output" if kw.get("o8") is not None else "other"
        return out

    def norm(self, x, **kw):
        out = orig["norm"](self, x, **kw)
        if kw.get("out_hi") is not None:
            producer[store(kw["out_hi"])] = "other"
        return out

    for n, fn in (("gemm", gemm), ("attention", attention), ("norm", norm)):
        monkeypatch.setattr(_C.Context, n, fn)
    return sites


@pytest.mark.gpu
def test_f16f8_operand_range_on_the_200m_policy(e4m3_site_maxima):
    """cfg3_small (200M shapes) through the policy in f16f8: the folded-LayerNorm GEMM inputs, the attention outputs and the GEGLU
    outputs that reach an e4m3 view all stay below 1024 / F8_MARGIN.  Prints the maximum per site."""
    import vima_b200
    from oracle import synth
    from tests.policy_runner import build_policy, run_policy_case

    case = synth.CASES["cfg3_small"]
    pol = build_policy(case.model)
    vima_b200.set_precision("f16f8")
    try:
        run_policy_case(pol, case)
    finally:
        vima_b200.set_precision("f16x3")
    torch.cuda.synchronize()
    maxima = {k: v.item() for k, v in e4m3_site_maxima.items()}
    print(f"\nf16f8 operand maxima on cfg3_small (saturation at {F8_LIMIT:g}, bar {F8_LIMIT / F8_MARGIN:g}):")
    for (site, cls), v in sorted(maxima.items(), key=lambda kv: -kv[1]):
        print(f"  {v:>9.3f}  {cls:<17} {site}")
    seen = {cls for _, cls in maxima}
    assert set(SITE_CLASSES) <= seen, f"no e4m3 operand of class {sorted(set(SITE_CLASSES) - seen)} was measured"
    assert all(math.isfinite(v) for v in maxima.values())
    worst = max(maxima.values())
    assert worst < F8_LIMIT / F8_MARGIN, (worst, maxima)
