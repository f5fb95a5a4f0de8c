"""How the GEMMs walk their work: the persistent wgmma GEMM across tile schedules and ring phases, and the exact-fp32 grouped GEMM
held to its fmaf order.

gemm_tc_kernel is persistent and warp-specialised: grid = min(tiles, SMs), each CTA walks tiles blockIdx.x, +gridDim.x, ...; the
producer and the consumers each keep one (stage, phase) counter across all of a CTA's tiles, so a CTA's second tile starts in ring
slot (num_kb mod n_stages), and with num_kb < n_stages the producer fills the next tile's stages during the epilogue.  The per-tile
column vectors (bias, ln_c1, res_gamma, res_beta) sit in a two-buffer ring that warpgroup 0 fills and both warpgroups read.

  1. Every operand mode and tile width, at K = 64 kb - 24 | 64 kb (kb = 1 .. 9: every residue of num_kb mod n_stages) and at
     every K the policy runs, with fewer tiles than SMs, SMs + 1 tiles, ~2.5 tiles per SM (uneven per CTA) and > 4 tiles per CTA,
     through the epilogues that read the column-vector ring, with vectors that differ from one n-tile to the next.  The primary
     assertion: the same rows computed again in row blocks that give every CTA at most one tile (every tile starts at ring slot 0)
     are bit-identical, in every output.  Each output element depends only on its own A row and B row, so the schedule must not
     change a bit.  Then fp64 with the bars of test_kernel_variants_gpu.py, and epi_prefetch = 1 bit-identical to 0.
  2. simt_gemm against a CPU-exact statement of its contract: acc = fma(x_k, w_k, acc) in ascending k from 0, then + b in fp32,
     then the activation.  Bit for bit at k across the 32-wide k step, M and n across the 64-wide tiles, 1 .. 33 groups (the host
     entry point launches 16 per call), and descriptors that share one x through column windows, as nn/action.py's grouped MLPs do.
  3. The sweep's K list and (mode, tile width) pairs against the GEMMs cfg1 and cfg3_small actually run.

Bars that rest on a measurement were measured on an H100 80GB HBM3 (700 W power limit).
"""
import math
import os
import random
import re
from fractions import Fraction

import pytest
import torch

F = torch.nn.functional
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN16 = {0: 0x7E00, 1: 0x7FC0}  # a quiet NaN of each 16-bit format
NAN8 = 0x7F                      # e4m3fn NaN
S16, S32, S8 = 0x7BAD, 0x7FBADBAD, 0xA5  # output sentinels (int16, fp32 bit pattern, byte)
ACT = {"ACT_NONE": 0, "ACT_RELU": 1, "ACT_QUICKGELU": 2, "ACT_GELU": 3, "ACT_GELU_TANH": 4}
MODES = ["f16", "f16x3", "f16f8", "bf16", "bf16x3"]

# (ACT, GLU, MUL, RES, O32, O16, LNA, LNR, STATS): rows of VIMA_GEMM_VARIANTS (index in the compiled list) and one generic combination
EPILOGUES = {
    "v00-plain": (0, ("ACT_NONE", 0, 0, 0, 0, 1, 0, 0, 0)),
    "v02-res-stats": (2, ("ACT_NONE", 0, 0, 1, 1, 1, 0, 0, 1)),
    "v06-ln-res": (6, ("ACT_NONE", 0, 0, 1, 1, 0, 0, 1, 0)),
    "v07-geglu": (7, ("ACT_GELU", 1, 0, 0, 0, 1, 0, 0, 0)),
    "v08-geglu-ln": (8, ("ACT_GELU", 1, 0, 0, 0, 1, 1, 0, 0)),
    "generic-relu-mul": (None, ("ACT_RELU", 0, 1, 0, 1, 1, 0, 0, 0)),
}
EPIS = ["v02-res-stats", "v06-ln-res", "v00-plain", "generic-relu-mul"]
GLU_EPIS = ["v08-geglu-ln", "v07-geglu"]

# rel-L2 against fp64: test_kernel_variants_gpu.py's GEMM_TOL, set at K <= 768, twice the bar with a folded LayerNorm.  Past K = 768
# the bar grows in proportion to K, as the fp32 accumulation's error does.  Measured worst: f16x3 1.1e-6 at K = 768, 6.2e-6 at
# 2560; f16x3 GEGLU (hi, lo) 4.1e-6 at 768, 1.6e-5 at 3072; f16 GEGLU 1.3e-6 at 768, 5.2e-6 at 3072; f16f8 and bf16 flat in K.
GEMM_TOL = {"f16": 3e-6, "f16x3": 6e-6, "f16f8": 2.5e-5, "bf16": 3e-6, "bf16x3": 1.5e-5}
TOL_K = 768
REP = {0: 3e-7, 1: 6e-6}  # rel-L2 of a (hi, lo) pair against the fp32 value it stands for

# ------------------------------------------------------------------------------------------------------------------------------
# the sweep
# ------------------------------------------------------------------------------------------------------------------------------
BN_KEYS = ["32", "64", "96", "128", "glu64", "glu128"]
KB_KS = [64 * kb - (24 if kb % 2 else 0) for kb in range(1, 10)]  # num_kb = 1 .. 9; odd kb end in a partial k-block
# the policy's GEMM widths at every MODEL_CFGS embed_dim E = 256 .. 768 (E, the observation fusion's E + 2, the MLPs' 4E) and the
# ViT / T5 widths 768, 1536, 3072; test_sweep_covers_the_policy_gemms checks them against the GEMMs cfg1 and cfg3_small run
POLICY_KS = [256, 258, 320, 322, 384, 386, 512, 514, 640, 642, 768, 770, 1024, 1280, 1536, 2048, 2560, 3072]
SWEEP_KS = KB_KS + [k for k in POLICY_KS if k not in KB_KS]
CLASSES = ("lt", "sm+1", "2.5x", "many")  # fewer tiles than SMs, SMs + 1, ~2.5 per SM, > 4 per CTA

# shared-memory carve of gemm_smem_bytes (gemm_tc.cuh): align slack, transpose staging, column-vector ring, barriers
GEMM_FIXED_SMEM = 1024 + 8 * 16 * 16 * 4 + 2 * 4 * 256 * 4 + 2 * 8 * 8 + 16


def rup(x, m):
    return (x + m - 1) // m * m


def n_stages(mode, bn, smem_optin):
    """The ring depth vima_gemm picks (api.cu): as many stages as the opt-in shared memory holds, at most 8.  Used to classify and
    report the cases; the K list does not depend on it."""
    stage = (128 * 128 + bn * 128) * (1 if mode in ("f16", "bf16") else 2)
    return min(8, (smem_optin - GEMM_FIXED_SMEM) // stage)


def tile_offset(t):
    """A per-n-tile offset in [-2, 2), distinct for every tile index (golden-ratio sequence): a tile that reads a neighbour's
    column vectors is off by O(1) of the output's own spread."""
    return 4.0 * torch.frac(t.double() * 0.6180339887498949).float() - 2.0


def pick_tiles_n(T, total=None):
    """A few n-tiles, coprime to the SM count so that consecutive tiles of one CTA (tile, tile + grid) sit in different n-tiles and
    read different column vectors; with `total`, a count that divides it if there is one."""
    cands = [n for n in range(3, 12) if math.gcd(n, T) == 1]
    if total is not None:
        exact = [n for n in cands if total % n == 0]
        if exact:
            return exact[0]
    return cands[0]


def sweep_cases(mode, bnkey, T):
    """The cases of one (mode, tile width) for a device with T SMs: dicts of K, class, epilogue, M, N, tiles."""
    glu = bnkey.startswith("glu")
    bn = int(bnkey[3:] if glu else bnkey)
    epis = GLU_EPIS if glu else EPIS
    out = []
    for i, K in enumerate(SWEEP_KS):
        num_kb = -(-K // 64)
        if i < len(KB_KS):
            cls = "many" if num_kb <= 2 else ("2.5x", "sm+1", "many")[i % 3]
        else:
            cls = CLASSES[i % 4]
            if cls == "many" and K > 1024:
                cls = "2.5x"
        target = {"lt": T // 2, "sm+1": T + 1, "2.5x": (5 * T) // 2, "many": (11 * T) // 2}[cls]
        tiles_n = pick_tiles_n(T, target if cls == "sm+1" else None)
        tiles_m = max(1, -(-target // tiles_n)) if cls != "lt" else max(1, target // tiles_n)
        ragged = i % 2 == 1
        M = tiles_m * 128 - ((1 + 37 * i) % 127 if ragged else 0)
        N = tiles_n * bn - (8 if (not glu and i % 3 == 1) else 0)  # a ragged last n-tile in every third non-GLU case
        out.append(dict(i=i, K=K, num_kb=num_kb, cls=cls, epi=epis[(i + i // len(epis)) % len(epis)], glu=glu, bn=bn, M=M, N=N,
                        n_out=N // 2 if glu else N, tiles_n=tiles_n, tiles=tiles_m * tiles_n, ragged=ragged))
    return out


def schedule(case, mode, T, smem_optin):
    """(n_stages, grid, fewest and most tiles per CTA, a tile starts mid-ring, the producer runs a whole tile ahead)."""
    ns = n_stages(mode, case["bn"], smem_optin)
    grid = min(case["tiles"], T)
    lo, hi = case["tiles"] // grid, -(-case["tiles"] // grid)
    return dict(ns=ns, grid=grid, lo=lo, hi=hi, mid_ring=hi > 1 and case["num_kb"] % ns != 0, ahead=hi > 1 and case["num_kb"] < ns)


def coverage_problems(mode, bnkey, T, smem_optin):
    """What the cases of one (mode, tile width) fail to cover; empty when the sweep does its job on this device."""
    cases = sweep_cases(mode, bnkey, T)
    sch = [schedule(c, mode, T, smem_optin) for c in cases]
    ns = sch[0]["ns"]
    bad = []
    if not any(s["mid_ring"] for s in sch):
        bad.append("no tile starts mid-ring")
    if not any(s["ahead"] and s["lo"] > 4 for s in sch):
        bad.append("no case with > 4 tiles per CTA and num_kb < n_stages")
    if {c["num_kb"] % ns for c, s in zip(cases, sch) if s["hi"] > 1} != set(range(ns)):
        bad.append("not every residue of num_kb mod n_stages runs with several tiles per CTA")
    for cls in CLASSES:
        if not any(c["cls"] == cls for c in cases):
            bad.append(f"no case of class {cls}")
    if not any(c["tiles"] < T for c in cases) or not any(T < c["tiles"] < 2 * T for c in cases):
        bad.append("no case with fewer tiles than SMs or with just over one tile per SM")
    for epi in (GLU_EPIS if bnkey.startswith("glu") else EPIS):
        if not any(c["epi"] == epi and s["lo"] != s["hi"] for c, s in zip(cases, sch)):
            bad.append(f"{epi} never runs with uneven tile counts per CTA")
        if not any(c["epi"] == epi and s["mid_ring"] for c, s in zip(cases, sch)):
            bad.append(f"{epi} never runs a tile that starts mid-ring")
    if not 0.3 <= sum(c["ragged"] for c in cases) / len(cases) <= 0.7:
        bad.append("ragged M in too few or too many cases")
    return bad


def test_sweep_covers_every_schedule_class():
    """On an H100 (132 SMs, 232448 bytes of opt-in shared memory) every (mode, tile width) of the sweep runs a tile that starts
    mid-ring, > 4 tiles per CTA with num_kb < n_stages, every residue of num_kb mod n_stages, every tile-count class, and every
    epilogue with uneven tile counts per CTA.  The GPU test repeats the check with the device's own numbers."""
    for mode in MODES:
        for bnkey in BN_KEYS:
            assert not coverage_problems(mode, bnkey, 132, 232448), (mode, bnkey, coverage_problems(mode, bnkey, 132, 232448))
            assert any(c["tiles"] == 133 for c in sweep_cases(mode, bnkey, 132)), (mode, bnkey)
    # the ring depths the kernel's shared-memory formula gives on that card (split / f16f8 modes, then single-pass)
    assert [n_stages("f16x3", bn, 232448) for bn in (128, 96, 64, 32)] == [3, 3, 4, 5]
    assert [n_stages("f16", bn, 232448) for bn in (128, 96, 64, 32)] == [6, 7, 8, 8]


def test_sweep_epilogues_are_the_compiled_rows():
    """The v.. epilogues are the VIMA_GEMM_VARIANTS rows of that index (so they run the specialised epilogue they name), and the
    generic one is none of them."""
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
        rows.append((f[0],) + tuple({"true": 1, "false": 0}[v] for v in f[1:6] + f[7:]))
    for name, (idx, row) in EPILOGUES.items():
        if idx is None:
            assert row not in rows, name
        else:
            assert rows[idx] == row, (name, rows[idx], row)


# ------------------------------------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    return _C.Context.get(torch.device("cuda", 0))


@pytest.fixture
def epi_prefetch(ctx):
    """Sets the context's epi_prefetch option; the finaliser puts it back to the default, 0."""
    ctx.set_option("epi_prefetch", "0")
    yield lambda v: ctx.set_option("epi_prefetch", v)
    ctx.set_option("epi_prefetch", "0")


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


def raw(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def assert_canary(buf, rows, cols, what):
    """Rows >= rows and columns >= cols of buf still hold the sentinel."""
    r = raw(buf)
    want = {4: S32, 2: S16, 1: S8}[buf.element_size()]
    assert (r[rows:] == want).all(), f"{what}: written past the last row"
    assert (r[:, cols:] == want).all(), f"{what}: written past the last column"


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


def deinterleave(acc, bn, n_out):
    """[M, tiles*bn] accumulator columns -> (value [M, n_out], gate [M, n_out])."""
    M = acc.shape[0]
    t = acc.reshape(M, -1, 2, bn // 2)
    return t[:, :, 0].reshape(M, -1)[:, :n_out], t[:, :, 1].reshape(M, -1)[:, :n_out]


class Operands:
    """A [M, K] and W [N, K] as the kernel's operands in `mode`, with NaN in every column in [K, ld) and in A's rows past M."""

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
            ctx.split_f8(F.pad(A, (0, rup(K, 4) - K)), a_lo8, a_hi8)  # split_f8 takes whole 4-column groups (K = E + 2)
            b_hi8 = torch.zeros(N, ld8, dtype=torch.uint8, device="cuda"); b_lo8 = torch.zeros_like(b_hi8)
            ctx.pack_weight_f8(W, b_hi8, b_lo8, transposed=False, scale=self.ws)
            for t in (a_lo8, a_hi8, b_hi8, b_lo8):
                t[:, K:] = NAN8
            a_lo8[M:] = NAN8; a_hi8[M:] = NAN8
            self.a8, self.b8 = (a_lo8, a_hi8), (b_hi8, b_lo8)
        self.K, self.M = K, M

    def kwargs(self, r0=0):
        """Operands of rows [r0, ...): views into the same buffers (every row pitch keeps 16-byte alignment)."""
        a = lambda t: None if t is None else t[r0:]
        return dict(a_hi=a(self.a_hi), a_lo=a(self.a_lo), lda=self.ld, b_hi=self.b_hi, b_lo=self.b_lo, ldb=self.ld, dtype=self.dt,
                    acc_scale=1.0 / self.ws, a_lo8=a(self.a8[0]), a_hi8=a(self.a8[1]), b_hi8=self.b8[0], b_lo8=self.b8[1])

    def product(self, A, W):
        """fp64 [M, N]: the exact product for the split modes, the product of the rounded operands for the single-pass ones."""
        if self.split or self.f8:
            return A.double() @ W.double().t()
        a = f16view(self.a_hi[: self.M, : self.K], self.dt).double()
        b = f16view(self.b_hi[:, : self.K], self.dt).double() / self.ws
        return a @ b.t()


def first_difference(got, want, case, T, what):
    """Where the bits first differ, in schedule terms: the tile, the CTA that ran it, its place in the CTA's walk."""
    bad = raw(got) != raw(want)
    if bad.dim() == 3:
        bad = bad.flatten(1)
    n = int(bad.sum())
    r, c = bad.nonzero()[0].tolist()
    bn_out = case["bn"] // 2 if case["glu"] else case["bn"]
    if what == "stats_out":  # [parts, 2] -> the first column of that (n-tile, 32-column half)
        part = c // 2
        c = (part // 2) * bn_out + (part % 2) * 32
    tile = (r // 128) * case["tiles_n"] + c // bn_out
    grid = min(case["tiles"], T)
    return (f"{what}: {n} elements differ from the one-tile-per-CTA schedule; first at row {r} column {c}: tile {tile} (m-tile {r // 128}, "
            f"n-tile {c // bn_out}), run by CTA {tile % grid} as its tile {tile // grid} of {-(-case['tiles'] // grid)}")


def run_case(ctx, set_prefetch, mode, case, seed):
    """One case: the GEMM at full size (several tiles per CTA), again in row blocks with at most one tile per CTA, and with
    epi_prefetch = 1 when the epilogue reads rows; bit-identity between them, then fp64.  Returns the fp64 errors."""
    T = ctx.sm_count
    idx, row = EPILOGUES[case["epi"]]
    act_name, glu, mul, res, o32, o16, lna, lnr, stats = row
    act = ACT[act_name]
    M, N, K, bn, n_out = case["M"], case["N"], case["K"], case["bn"], case["n_out"]
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    A = rn(M, K) * 2.0 + 0.7 if lna else rn(M, K)
    W = rn(N, K) / math.sqrt(K)  # accumulator-column order (value | gate halves per tile with GLU)
    acc_off = tile_offset(torch.arange(N, device="cuda") // bn)
    bias = 0.5 * rn(N) + acc_off
    kw = {}
    if lna:  # LayerNorm folded in (gamma = 1, beta = 0): the kernel takes the raw rows, their (mean, rstd) and the weight row sums
        A64 = A.double()
        st = torch.stack([A64.mean(1), 1.0 / torch.sqrt(A64.var(1, unbiased=False) + 1e-5)], 1).float().contiguous()
        c1 = (W.double().sum(1) + acc_off.double()).float()  # a per-tile offset on top, so a stale ln_c1 tile shows
        kw.update(row_stats=st, ln_c1=c1, ln_cols=1)
    ops = Operands(ctx, A, W, mode)
    mul_t = rn(M, n_out + 4)[:, :n_out] if mul else None
    res_t = (rn(M, n_out + 4) * 2.0 + 0.7)[:, :n_out] if res else None
    if lnr:
        out_off = tile_offset(torch.arange(n_out, device="cuda") // bn)
        r64 = res_t.double()
        rst = torch.stack([r64.mean(1), 1.0 / torch.sqrt(r64.var(1, unbiased=False) + 1e-5)], 1).float().contiguous()
        kw.update(res_stats=rst, res_gamma=1.0 + 0.1 * rn(n_out) + 0.25 * out_off, res_beta=0.1 * rn(n_out) + out_off)
    parts = ctx.gemm_stats_parts(N, glu, bn)
    f8_out = o16 and ops.f8

    def outputs():
        o = {}
        if o32:
            o["out_f32"] = sentinel((M + 3, n_out + 8), "f32")
        if o16:
            o["out_hi"] = sentinel((M + 3, n_out + 8), "i16")
            if f8_out:
                o["out_lo8"], o["out_hi8"] = sentinel((M + 3, n_out + 16), "u8"), sentinel((M + 3, n_out + 16), "u8")
            else:
                o["out_lo"] = sentinel((M + 3, n_out + 8), "i16")
        if stats:
            o["stats_out"] = sentinel((M + 3, parts, 2), "f32")
        return o

    def launch(o, r0=0, rows=M):
        sl = lambda t: None if t is None else t[r0:r0 + rows]
        rows_kw = {k: (sl(v) if k in ("row_stats", "res_stats") else v) for k, v in kw.items()}
        ctx.gemm(M=rows, N=N, K=K, glu=glu, act=act, bias=bias, mul=sl(mul_t), residual=sl(res_t), block_n=bn,
                 **{k: v[r0:] for k, v in o.items()}, **ops.kwargs(r0), **rows_kw)

    what = f"{mode} bn={bn}{' GLU' if glu else ''} {case['epi']} M={M} N={N} K={K} tiles={case['tiles']} ({case['cls']})"
    big = outputs()
    launch(big)
    chunked = outputs()
    step = 128 * (T // case["tiles_n"])  # at most T tiles per call: one tile per CTA, every tile starts at ring slot 0
    for r0 in range(0, M, step):
        launch(chunked, r0, min(step, M - r0))
    torch.cuda.synchronize()
    for name in big:
        if not torch.equal(raw(big[name]), raw(chunked[name])):
            raise AssertionError(what + ": " + first_difference(big[name], chunked[name], case, T, name))
    if mul or res:
        set_prefetch("1")
        pre = outputs()
        launch(pre)
        set_prefetch("0")
        torch.cuda.synchronize()
        for name in big:
            if not torch.equal(raw(big[name]), raw(pre[name])):
                raise AssertionError(what + ": epi_prefetch=1: " + first_difference(pre[name], big[name], case, T, name))

    # ---- fp64 statement of the epilogue, with the vectors as given ----
    P = ops.product(A, W)
    if lna:
        pre_act = st[:, 1:2].double() * (P - st[:, 0:1].double() * c1.double()[None]) + bias.double()
    else:
        pre_act = P + bias.double()
    if glu:
        val, gate = deinterleave(pre_act, bn, n_out)
        ref = act_ref(act, val) * gate
    else:
        ref = act_ref(act, pre_act[:, :n_out])
    if mul:
        ref = ref * mul_t.double()
    if res:
        r = res_t.double()
        if lnr:
            r = (r - rst[:, 0:1].double()) * rst[:, 1:2].double() * kw["res_gamma"].double() + kw["res_beta"].double()
        ref = ref + r
    tol = GEMM_TOL[mode] * (2 if lna else 1) * max(1.0, K / TOL_K)
    errs = {}
    if o32:
        got = big["out_f32"]
        assert_canary(got, M, n_out, what + " out_f32")
        assert torch.isfinite(got[:M, :n_out]).all(), what
        errs["f32"] = rel(got[:M, :n_out], ref)
        assert errs["f32"] < tol, (what, errs)
    if o16:
        hi = big["out_hi"]
        assert_canary(hi, M, n_out, what + " out_hi")
        h = f16view(hi[:M, :n_out], ops.dt).double()
        if f8_out:
            for nm in ("out_lo8", "out_hi8"):
                assert_canary(big[nm], M, n_out, what + " " + nm)
            rec = h + big["out_lo8"][:M, :n_out].view(torch.float8_e4m3fn).double() / 1024.0
            errs["hi16+lo8"] = rel(rec, ref)
            assert errs["hi16+lo8"] < tol + 2e-5, (what, errs)
        else:
            assert_canary(big["out_lo"], M, n_out, what + " out_lo")
            rec = h + f16view(big["out_lo"][:M, :n_out], ops.dt).double()
            errs["hi+lo"] = rel(rec, ref)
            assert errs["hi+lo"] < tol + REP[ops.dt], (what, errs)
        assert torch.isfinite(rec).all(), what
    if stats:
        so = big["stats_out"]
        assert_canary(so.view(M + 3, parts * 2), M, parts * 2, what + " stats_out")
        c = torch.arange(n_out, device="cuda")
        part = 2 * (c // bn) + ((c % bn) // 32) % 2  # (n-tile, 32-column half of the tile)
        s_ref = torch.zeros(M, parts, 2, dtype=torch.float64, device="cuda")
        s_ref[:, :, 0].index_add_(1, part, ref)
        s_ref[:, :, 1].index_add_(1, part, ref * ref)
        s_abs = torch.zeros(M, parts, dtype=torch.float64, device="cuda").index_add_(1, part, ref.abs())
        s = so[:M].double()
        errs["sum"] = ((s[:, :, 0] - s_ref[:, :, 0]).norm() / s_abs.norm()).item()
        errs["sumsq"] = rel(s[:, :, 1], s_ref[:, :, 1])
        assert errs["sum"] < 4 * tol and errs["sumsq"] < 4 * tol, (what, errs)
    return errs


@pytest.mark.gpu
@pytest.mark.parametrize("bnkey", BN_KEYS)
@pytest.mark.parametrize("mode", MODES)
def test_gemm_schedule_sweep(ctx, epi_prefetch, mode, bnkey):
    T = ctx.sm_count
    optin = torch.cuda.get_device_properties(ctx.device).shared_memory_per_block_optin
    problems = coverage_problems(mode, bnkey, T, optin)
    assert not problems, (T, optin, problems)
    worst = {}
    cases = sweep_cases(mode, bnkey, T)
    sch = [schedule(c, mode, T, optin) for c in cases]
    for case in cases:
        seed = 100000 * MODES.index(mode) + 1000 * BN_KEYS.index(bnkey) + case["i"]
        for k, v in run_case(ctx, epi_prefetch, mode, case, seed).items():
            worst[k] = max(worst.get(k, 0.0), v)
    mid = sorted({c["num_kb"] for c, s in zip(cases, sch) if s["mid_ring"]})
    ahead = sorted({c["num_kb"] for c, s in zip(cases, sch) if s["ahead"]})
    print(f"\nschedule {mode} bn={bnkey} n_stages={sch[0]['ns']}: {len(cases)} cases; num_kb with tiles starting mid-ring {mid}, with the "
          f"producer a tile ahead {ahead}; fp64 " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))


# ------------------------------------------------------------------------------------------------------------------------------
# 2. simt_gemm: ascending-k fmaf chains, bit for bit
# ------------------------------------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fp32 fma(a, b, c), correctly rounded, from float32 tensors (CPU or CUDA; numpy and Python 3.12 have no fma).  The product is
    exact in fp64 (24 + 24 bits); s = p + c is rounded to fp64 and TwoSum gives its exact error; rounding s to odd (one ulp toward
    the error when the error is non-zero and s is even) keeps the sticky information, so the final cast to fp32 rounds the exact
    a * b + c once."""
    p = a.double() * b.double()
    c = c.double()
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    fix = (err != 0) & ((s.view(torch.int64) & 1) == 0)
    toward = torch.where(err > 0, torch.full_like(s, math.inf), torch.full_like(s, -math.inf))
    return torch.where(fix, torch.nextafter(s, toward), s).float()


def round_f32(x: Fraction) -> float:
    """The rational x rounded to the nearest fp32 value, ties to even (normal and subnormal range)."""
    if x == 0:
        return 0.0
    sign = -1 if x < 0 else 1
    x = abs(x)
    e = x.numerator.bit_length() - x.denominator.bit_length()
    if Fraction(2) ** e > x:
        e -= 1
    ulp = Fraction(2) ** max(e - 23, -149)
    q = x / ulp
    n = q.numerator // q.denominator
    rem = q - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return sign * float(n * ulp)


def f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def test_fma_emulation_matches_exact_rounding():
    """fma32 equals the exactly rounded a * b + c on random triples (wide exponents, cancellation) and on constructed cases where
    a * b + c lies a hair off a halfway point between two fp32 values, where rounding the fp64 sum to fp32 rounds twice and
    goes the wrong way."""
    rng = random.Random(5)
    trip = []
    for _ in range(4000):
        a = f32(rng.gauss(0, 1) * 2.0 ** rng.randint(-30, 30))
        b = f32(rng.gauss(0, 1) * 2.0 ** rng.randint(-30, 30))
        kind = rng.randint(0, 2)
        if kind == 0:
            c = f32(rng.gauss(0, 1) * 2.0 ** rng.randint(-60, 60))
        elif kind == 1:  # near-total cancellation: c = -rn(a * b) (+ a few ulps)
            c = f32(-f32(a * b) * (1 + rng.randint(-3, 3) * 2.0 ** -23))
        else:  # c dominates by 2^20 .. 2^30: a * b lands among c's last bits
            c = f32(a * b * 2.0 ** rng.randint(20, 30) * rng.choice((1, -1)))
        trip.append((a, b, c))
    u = 2.0 ** -23
    halfway = []
    for s in (-40, 0, 17):
        for sa in (1, -1):
            for sc in (1, -1):
                for j in range(4):  # c = 1 + j ulp: both parities of c's last bit
                    for a0, b0 in ((1 + u, 1 - u), (1 + u, 1 + u), (1 - u, 1 - u), (1 + 3 * u, 1 - 5 * u)):
                        # a * b = 2^-24 (1 + O(2^-22)): the sum sits within 2^-45 ulp of the midpoint between c and c + 1 ulp
                        halfway.append((sa * a0 * 2.0 ** (s - 24), b0, sc * sa * (1 + j * u) * 2.0 ** s))
    trip += [(f32(a), f32(b), f32(c)) for a, b, c in halfway]
    a, b, c = (torch.tensor(v, dtype=torch.float32) for v in zip(*trip))
    got = fma32(a, b, c)
    naive = (a.double() * b.double() + c.double()).float()
    bad = []
    for i, (x, y, z) in enumerate(trip):
        want = round_f32(Fraction(x) * Fraction(y) + Fraction(z))
        if got[i].item() != want:
            bad.append((x, y, z, got[i].item(), want))
    assert not bad, bad[:5]
    n_double_rounding = int((naive[-len(halfway):] != got[-len(halfway):]).sum())
    assert n_double_rounding > 0, "no constructed case separates fma from the double-rounded fp64 sum"


SIMT_KS = (1, 2, 4, 31, 32, 33, 260, 768)  # across the 32-wide k step and its register prefetch
SIMT_NS = (50, 64, 100, 512)               # across the 64-wide column tiles
SIMT_GROUPS = (1, 12, 16, 17, 33)          # the host entry point launches 16 descriptors per call
ACT_BAR = 3e-7  # |got - act(v)| <= ACT_BAR * max(1, |v|): test_kernel_variants_gpu.py's bar for the same device activations


def simt_groups(M, G, seed):
    """G descriptors in the layout of nn/action.py's grouped MLPs: x is one [M, 811] buffer read through column windows (several
    groups at the same window, as every head reads the same input), or a tensor of the group's own; each group has its own
    weight with a padded row pitch; the outputs are column windows of one [M + 2, total] buffer with 3 unwritten columns between
    them; every third group has no bias."""
    from vima_b200 import _C

    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    x_shared = rn(M, 811)
    specs, keep = [], [x_shared]
    col = 0
    for i in range(G):
        k, n = SIMT_KS[(i + G) % len(SIMT_KS)], SIMT_NS[(i + G // 3) % len(SIMT_NS)]
        off = (0, 0, 3, 17, None)[i % 5]
        if off is None:
            x = rn(M, k)
            keep.append(x)
        else:
            x = x_shared[:, off:]
        w = rn(n, k + 3)[:, :k]
        b = None if i % 3 == 2 else rn(n)
        keep += [w] + ([] if b is None else [b])
        specs.append(dict(x=x, w=w, b=b, n=n, k=k, col=col))
        col += n + 3
    y = sentinel((M + 2, col), "f32")
    arr = (_C.F32GemmGroup * G)()
    for i, s in enumerate(specs):
        arr[i] = _C.F32GemmGroup(s["x"].data_ptr(), s["x"].stride(0), s["w"].data_ptr(), s["w"].stride(0),
                                 None if s["b"] is None else s["b"].data_ptr(), y.data_ptr() + 4 * s["col"], y.stride(0), s["n"], s["k"])
    return specs, y, arr, keep


def simt_reference(specs, M):
    """v = fl32(fma chain over ascending k from 0) + b (one fp32 add), per group: [M, n] fp32.  All groups in one chain over the
    longest k, zero-padded (fma(0, 0, acc) = acc exactly: the chain never holds -0)."""
    G = len(specs)
    kmax, nmax = max(s["k"] for s in specs), max(s["n"] for s in specs)
    X = torch.zeros(G, M, kmax, device="cuda")
    Wt = torch.zeros(G, nmax, kmax, device="cuda")
    B = torch.zeros(G, nmax, device="cuda")
    for i, s in enumerate(specs):
        X[i, :, : s["k"]] = s["x"][:, : s["k"]]
        Wt[i, : s["n"], : s["k"]] = s["w"]
        if s["b"] is not None:
            B[i, : s["n"]] = s["b"]
    acc = torch.zeros(G, M, nmax, device="cuda")
    for k in range(kmax):
        acc = fma32(X[:, :, k, None], Wt[:, None, :, k], acc)
    v = acc + B[:, None, :]  # a separate fp32 add, correctly rounded
    return [v[i, :, : s["n"]] for i, s in enumerate(specs)]


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 63, 64, 65, 200])
def test_simt_gemm_bit_exact(ctx, M):
    """Both entry points give the fmaf chain's bits for ACT_NONE and ACT_RELU and act(v) within the activation bar for the other
    codes; nothing outside the output windows changes."""
    worst = 0.0
    for G in SIMT_GROUPS:
        specs, y, arr, keep = simt_groups(M, G, seed=1000 * M + G)
        ref = simt_reference(specs, M)
        max_n = max(s["n"] for s in specs) + (100 if G % 2 else 0)  # a wider launch than needed: its extra column tiles do nothing
        gd = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).cuda()
        for act in ACT.values():
            for entry in ("device", "host"):
                y.view(torch.int32).fill_(S32)
                if entry == "device":
                    ctx.gemm_f32_grouped(gd, G, M, max_n, act)
                else:
                    ctx.gemm_f32_grouped_host(arr, G, M, max_n, act)
                torch.cuda.synchronize()
                what = f"{entry} M={M} groups={G} act={act}"
                written = torch.zeros(y.shape[1], dtype=torch.bool, device="cuda")
                for i, (s, v) in enumerate(zip(specs, ref)):
                    got = y[:M, s["col"]: s["col"] + s["n"]]
                    written[s["col"]: s["col"] + s["n"]] = True
                    gw = f"{what} group {i} (n={s['n']} k={s['k']})"
                    if act in (0, 1):
                        want = v if act == 0 else torch.relu(v)
                        if not torch.equal(got, want):
                            bad = (got != want).nonzero()[0].tolist()
                            raise AssertionError(f"{gw}: {int((got != want).sum())} outputs differ from the fmaf chain; first at "
                                                 f"{bad}: got {got[tuple(bad)].item()!r}, want {want[tuple(bad)].item()!r}")
                    else:
                        v64 = v.double()
                        e = ((got.double() - act_ref(act, v64)).abs() / v64.abs().clamp_min(1.0)).max().item()
                        worst = max(worst, e)
                        assert e <= ACT_BAR, (gw, e)
                assert (y.view(torch.int32)[M:] == S32).all(), what + ": written past row M"
                assert (y.view(torch.int32)[:, ~written] == S32).all(), what + ": written outside the output windows"
    print(f"\nsimt_gemm M={M}: bit-exact for ACT_NONE / ACT_RELU; worst activation error {worst:.2e} (bar {ACT_BAR:g})")


@pytest.mark.gpu
def test_simt_gemm_host_refuses_max_n_below_a_group(ctx):
    """max_n sets the launch's column tiles: a group wider than it would lose its last columns silently, so the host entry point
    refuses the call (and M < 0) before launching anything."""
    specs, y, arr, keep = simt_groups(65, 17, seed=7)
    widest = max(s["n"] for s in specs)
    before = ctx.launches
    with pytest.raises(RuntimeError, match=r"more than max_n"):
        ctx.gemm_f32_grouped_host(arr, 17, 65, widest - 1, 0)
    with pytest.raises(RuntimeError, match=r"M = -1"):
        ctx.gemm_f32_grouped_host(arr, 17, -1, widest, 0)
    torch.cuda.synchronize()
    assert ctx.launches == before
    assert (y.view(torch.int32) == S32).all(), "a refused call wrote its output"
    ctx.gemm_f32_grouped_host(arr, 17, 65, widest, 0)  # the same descriptors at max_n = the widest group run
    torch.cuda.synchronize()
    for s, v in zip(specs, simt_reference(specs, 65)):
        assert torch.equal(y[:65, s["col"]: s["col"] + s["n"]], v)


# ------------------------------------------------------------------------------------------------------------------------------
# 3. the sweep against the policy's own GEMMs
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def policy_gemm_shapes():
    """(mode, block_n key, K) of every wgmma GEMM one forward of cfg1 (2M) and of cfg3_small (200M shapes) issues, in f16x3 and in
    f16f8, recorded by wrapping Context.gemm."""
    import vima_b200
    from oracle import synth
    from vima_b200 import _C, engine
    from tests.policy_runner import build_policy, run_policy_case

    seen = set()
    orig = _C.Context.gemm

    def gemm(self, **kw):
        glu = int(kw.get("glu", 0))
        bn = kw.get("block_n") or block_n_for(kw["N"], glu)
        if kw.get("a_lo8") is not None:
            mode = "f16f8"
        else:
            mode = ("bf16" if kw.get("dtype", 0) == 1 else "f16") + ("x3" if kw.get("a_lo") is not None else "")
        seen.add((mode, f"glu{bn}" if glu else str(bn), int(kw["K"])))
        return orig(self, **kw)

    prev = engine.get_precision()
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(_C.Context, "gemm", gemm)
        try:
            for name in ("cfg1", "cfg3_small"):
                case = synth.CASES[name]
                pol = build_policy(case.model)
                for prec in ("f16x3", "f16f8"):
                    vima_b200.set_precision(prec)
                    run_policy_case(pol, case)
        finally:
            vima_b200.set_precision(prev)
    torch.cuda.synchronize()
    return seen


@pytest.mark.gpu
def test_sweep_covers_the_policy_gemms(policy_gemm_shapes):
    """Every K the policy runs is in the sweep's K list and every (mode, tile width) it runs is a swept pair: a new layer width fails
    here instead of running an untested schedule."""
    ks = sorted({k for _, _, k in policy_gemm_shapes})
    pairs = sorted({(m, b) for m, b, _ in policy_gemm_shapes})
    print(f"\npolicy GEMMs: K {ks}; (mode, block_n) {pairs}")
    assert {m for m, _ in pairs} >= {"f16x3", "f16f8"}, pairs
    assert set(ks) <= set(SWEEP_KS), f"K not in the sweep: {sorted(set(ks) - set(SWEEP_KS))}"
    assert set(pairs) <= {(m, b) for m in MODES for b in BN_KEYS}, pairs
