"""GPU: every C-ABI kernel against a plain torch fp32 statement of the same op (called through the C ABI)."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DT = {"f16": (0, torch.float16), "bf16": (1, torch.bfloat16)}


@pytest.fixture(scope="module")
def ctx():
    from vima_b200 import _C

    return _C.Context.get(torch.device("cuda", 0))


def dev(t):
    return t.to("cuda")


def split_ops(ctx, x, dt, split, pad_to=8):
    """fp32 [rows, cols] -> (hi, lo|None) 16-bit [rows, ld] with ld padded to a multiple of 8."""
    rows, cols = x.shape
    ld = (cols + pad_to - 1) // pad_to * pad_to
    hi = torch.empty(rows, ld, dtype=torch.int16, device="cuda")
    lo = torch.empty_like(hi) if split else None
    ctx.split(x.contiguous(), hi, lo, cols=cols, pad_cols=ld, dtype=dt)
    return hi, lo, ld


def merge(hi, lo, tdt, cols):
    a = hi.view(tdt)[:, :cols].float()
    if lo is not None:
        a = a + lo.view(tdt)[:, :cols].float()
    return a


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize("dtname", ["f16", "bf16"])
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (300, 320, 776), (1000, 768, 768), (257, 2304, 768), (4100, 96, 3072)])
def test_gemm_plain(ctx, dtname, split, M, N, K):
    dt, tdt = DT[dtname]
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
    bias = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g)
    a_hi, a_lo, lda = split_ops(ctx, A, dt, split)
    b_hi, b_lo, ldb = split_ops(ctx, W, dt, split)
    out = torch.full((M, N), float("nan"), device="cuda")
    ctx.gemm(M=M, N=N, K=K, a_hi=a_hi, a_lo=a_lo, lda=lda, b_hi=b_hi, b_lo=b_lo, ldb=ldb, dtype=dt, bias=bias, residual=res, out_f32=out)
    torch.cuda.synchronize()
    if split:
        ref = A.double() @ W.double().t() + bias.double() + res.double()
        tol = 2e-5 if dtname == "f16" else 1e-4
    else:
        ref = merge(a_hi, None, tdt, K).double() @ merge(b_hi, None, tdt, K).double().t() + bias.double() + res.double()
        tol = 5e-6
    assert torch.isfinite(out).all()
    assert rel(out, ref) < tol, rel(out, ref)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("M,N,K", [(4736, 2304, 768), (4741, 768, 3072), (20000, 768, 768)])
def test_gemm_cluster_multicast(ctx, split, M, N, K):
    """Shapes with more tiles than SMs (every persistent CTA walks several tiles), incl. an odd number of m-blocks and a ragged
    last block.  (Named after the 2-CTA multicast launch mode these shapes were first written for.)"""
    dt, tdt = DT["f16"]
    g = torch.Generator(device="cuda").manual_seed(M + N)
    A = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
    bias = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g)
    a_hi, a_lo, lda = split_ops(ctx, A, dt, split)
    b_hi, b_lo, ldb = split_ops(ctx, W * 256.0, dt, split)
    out = torch.full((M, N), float("nan"), device="cuda")
    ctx.gemm(M=M, N=N, K=K, a_hi=a_hi, a_lo=a_lo, lda=lda, b_hi=b_hi, b_lo=b_lo, ldb=ldb, dtype=dt, bias=bias, residual=res, out_f32=out,
             acc_scale=1 / 256.0)
    torch.cuda.synchronize()
    Ar = A if split else merge(a_hi, None, tdt, K)
    Wr = W if split else merge(b_hi, None, tdt, K) / 256.0
    ref = Ar.double() @ Wr.double().t() + bias.double() + res.double()
    assert torch.isfinite(out).all()
    assert rel(out, ref) < 1e-5, rel(out, ref)


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (1000, 768, 768), (515, 2304, 768), (300, 768, 3072), (9472, 2304, 768)])
def test_gemm_f16f8(ctx, M, N, K):
    """fp16 hi*hi + two e4m3 cross terms: per-GEMM error ~1e-5 (vs 3e-4 for single-pass fp16); also checks the e4m3 views the
    epilogue emits for the next GEMM."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
    bias = torch.randn(N, device="cuda", generator=g)
    ws = 2.0 ** math.floor(math.log2(1024.0 / W.abs().max().item()))
    a_hi, _, lda = split_ops(ctx, A, 0, False)
    ld8 = (K + 15) // 16 * 16
    a_lo8 = torch.zeros(M, ld8, dtype=torch.uint8, device="cuda"); a_hi8 = torch.zeros_like(a_lo8)
    ctx.split_f8(A, a_lo8, a_hi8)
    b_hi = torch.empty(N, lda, dtype=torch.int16, device="cuda")
    ctx.pack_weight(W, b_hi, None, transposed=False, scale=ws, dtype=0)
    b_hi8 = torch.zeros(N, ld8, dtype=torch.uint8, device="cuda"); b_lo8 = torch.zeros_like(b_hi8)
    ctx.pack_weight_f8(W, b_hi8, b_lo8, transposed=False, scale=ws)
    out = torch.empty(M, N, device="cuda")
    o_hi = torch.zeros(M, N, dtype=torch.int16, device="cuda")
    n8 = (N + 15) // 16 * 16
    o_lo8 = torch.zeros(M, n8, dtype=torch.uint8, device="cuda"); o_hi8 = torch.zeros_like(o_lo8)
    ctx.gemm(M=M, N=N, K=K, a_hi=a_hi, a_lo=None, lda=lda, b_hi=b_hi, b_lo=None, ldb=lda, dtype=0, bias=bias, acc_scale=1.0 / ws, out_f32=out,
             out_hi=o_hi, a_lo8=a_lo8, a_hi8=a_hi8, b_hi8=b_hi8, b_lo8=b_lo8, out_lo8=o_lo8, out_hi8=o_hi8)
    torch.cuda.synchronize()
    ref = A.double() @ W.double().t() + bias.double()
    e = rel(out, ref)
    single = rel(merge(a_hi, None, torch.float16, K).double() @ (merge(b_hi, None, torch.float16, K).double() / ws).t() + bias.double(), ref)
    assert e < 4e-5 and e < single / 5, (e, single)
    # emitted views reconstruct the output: hi16 + lo8/2^10 ~ out (lo8 has 4 bits), hi8*8 ~ out (4 bits)
    hi16 = o_hi.view(torch.float16).float()
    rec = hi16 + o_lo8[:, :N].view(torch.float8_e4m3fn).float() / 1024.0
    assert rel(rec, out) < 2e-5
    assert rel(o_hi8[:, :N].view(torch.float8_e4m3fn).float() * 8.0, out) < 4e-2


@pytest.mark.parametrize("split", [False, True])
def test_gemm_epilogues(ctx, split):
    dt, tdt = DT["f16"]
    M, N, K = 515, 384, 392
    g = torch.Generator(device="cuda").manual_seed(7)
    A = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
    bias = torch.randn(N, device="cuda", generator=g)
    mul = torch.randn(M, N, device="cuda", generator=g)
    a_hi, a_lo, lda = split_ops(ctx, A, dt, split)
    scale = 64.0  # packed weights may be pre-scaled by a power of two
    b_hi, b_lo, ldb = split_ops(ctx, W * scale, dt, split)
    Ar = A if split else merge(a_hi, None, tdt, K)
    Wr = W if split else merge(b_hi, None, tdt, K) / scale
    base = Ar.double() @ Wr.double().t() + bias.double()
    for act, fn in [(1, torch.relu), (2, lambda x: x * torch.sigmoid(1.702 * x)), (3, lambda x: torch.nn.functional.gelu(x))]:
        out = torch.empty(M, N, device="cuda")
        o_hi = torch.zeros(M, N + 8, dtype=torch.int16, device="cuda")
        o_lo = torch.zeros_like(o_hi)
        ctx.gemm(M=M, N=N, K=K, a_hi=a_hi, a_lo=a_lo, lda=lda, b_hi=b_hi, b_lo=b_lo, ldb=ldb, dtype=dt, bias=bias, act=act, mul=mul,
                 acc_scale=1.0 / scale, out_f32=out, out_hi=o_hi, out_lo=o_lo)
        torch.cuda.synchronize()
        ref = fn(base) * mul.double()
        assert rel(out, ref) < 5e-6, (act, rel(out, ref))
        assert rel(merge(o_hi, o_lo, tdt, N), out) < 2e-6
        assert rel(merge(o_hi, None, tdt, N), out) < 1e-3
        assert (o_hi[:, N:] == 0).all()


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("n_out", [384, 1024, 3072])
def test_gemm_glu(ctx, split, n_out):
    """GEGLU: out = gelu(A Wv^T + bv) * (A Wg^T) with value/gate rows interleaved per accumulator tile."""
    dt, tdt = DT["f16"]
    M, K = 333, 256
    g = torch.Generator(device="cuda").manual_seed(9)
    A = torch.randn(M, K, device="cuda", generator=g)
    Wv = torch.randn(n_out, K, device="cuda", generator=g) / math.sqrt(K)
    Wg = torch.randn(n_out, K, device="cuda", generator=g) / math.sqrt(K)
    bv = torch.randn(n_out, device="cuda", generator=g)
    bn = ctx.glu_block_n(n_out)
    half = bn // 2
    tiles = (n_out + half - 1) // half
    Wp = torch.zeros(tiles * bn, K, device="cuda")
    bp = torch.zeros(tiles * bn, device="cuda")
    for t in range(tiles):
        n = min(half, n_out - t * half)
        Wp[t * bn : t * bn + n] = Wv[t * half : t * half + n]
        Wp[t * bn + half : t * bn + half + n] = Wg[t * half : t * half + n]
        bp[t * bn : t * bn + n] = bv[t * half : t * half + n]
    a_hi, a_lo, lda = split_ops(ctx, A, dt, split)
    b_hi, b_lo, ldb = split_ops(ctx, Wp, dt, split)
    o_hi = torch.zeros(M, n_out, dtype=torch.int16, device="cuda")
    o_lo = torch.zeros_like(o_hi)
    ctx.gemm(M=M, N=tiles * bn, K=K, a_hi=a_hi, a_lo=a_lo, lda=lda, b_hi=b_hi, b_lo=b_lo, ldb=ldb, dtype=dt, bias=bp, act=3, glu=1,
             out_hi=o_hi, out_lo=o_lo, block_n=bn)
    torch.cuda.synchronize()
    Ar = A if split else merge(a_hi, None, tdt, K)
    if split:
        ref = torch.nn.functional.gelu(Ar.double() @ Wv.double().t() + bv.double()) * (Ar.double() @ Wg.double().t())
    else:
        Wr = merge(b_hi, None, tdt, K)
        full = Ar.double() @ Wr.double().t() + bp.double()
        ref = torch.cat([torch.nn.functional.gelu(full[:, t * bn : t * bn + half]) * full[:, t * bn + half : (t + 1) * bn] for t in range(tiles)], 1)[:, :n_out]
    assert rel(merge(o_hi, o_lo, tdt, n_out), ref) < 5e-6


@pytest.mark.parametrize("cols", [256, 320, 768, 1024])
def test_norm(ctx, cols):
    rows = 1037
    g = torch.Generator(device="cuda").manual_seed(cols)
    x = torch.randn(rows, cols, device="cuda", generator=g) * 3 + 0.5
    add = torch.randn(rows, cols, device="cuda", generator=g)
    w = torch.randn(cols, device="cuda", generator=g)
    b = torch.randn(cols, device="cuda", generator=g)
    w2 = torch.randn(cols, device="cuda", generator=g)
    b2 = torch.randn(cols, device="cuda", generator=g)
    F = torch.nn.functional
    # LayerNorm(x + add) -> fp32 + hi/lo
    o = torch.empty_like(x)
    hi = torch.empty(rows, cols, dtype=torch.int16, device="cuda")
    lo = torch.empty_like(hi)
    ctx.norm(x, rows=rows, cols=cols, ldx=cols, add=add, w=w, b=b, out_f32=o, out_hi=hi, out_lo=lo)
    ref = F.layer_norm((x + add).double(), (cols,), w.double(), b.double(), 1e-5)
    assert rel(o, ref) < 2e-6
    assert rel(merge(hi, lo, torch.float16, cols), o) < 2e-6
    # chained: y1 = LN(x) fp32, y2 = LN2(y1) as operands + fp32
    o2 = torch.empty_like(x)
    ctx.norm(x, rows=rows, cols=cols, ldx=cols, w=w, b=b, w2=w2, b2=b2, out_f32=o, out2_f32=o2, out_hi=hi, out_lo=lo)
    ref1 = F.layer_norm(x.double(), (cols,), w.double(), b.double(), 1e-5)
    ref2 = F.layer_norm(ref1, (cols,), w2.double(), b2.double(), 1e-5)
    assert rel(o, ref1) < 2e-6 and rel(o2, ref2) < 5e-6
    assert rel(merge(hi, lo, torch.float16, cols), o2) < 2e-6
    # T5 RMSNorm
    ctx.norm(x, rows=rows, cols=cols, ldx=cols, w=w, eps=1e-6, rms=1, out_f32=o)
    xd = x.double()
    ref = w.double() * xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-6)
    assert rel(o, ref) < 2e-6
    # pure convert (no norm): x + add -> operands
    ctx.norm(x, rows=rows, cols=cols, ldx=cols, add=add, out_hi=hi, out_lo=lo)
    assert rel(merge(hi, lo, torch.float16, cols), x + add) < 2e-6


def ref_attention(q, k, v, scale, causal, key_mask, bias):
    """q (B,H,Lq,D) etc. in float64; reference mask semantics."""
    s = torch.matmul(q, k.transpose(-1, -2)) * scale
    if bias is not None:
        s = s + bias
    Lq, Lk = s.shape[-2:]
    if causal:
        tril = torch.tril(torch.ones(Lq, Lk, dtype=s.dtype, device=s.device))
        s = s * tril + -1e4 * (1 - tril)
    if key_mask is not None:
        s = s + (1.0 - key_mask[:, None, None, :].to(s.dtype)) * torch.finfo(torch.float32).min
    return torch.matmul(torch.softmax(s, -1), v)


@pytest.fixture(params=["mma", "tc", "tc+tail_off"])
def attn_impl(request, ctx):
    """Both attention kernels: mma.sync (attention.cu) and wgmma (attention_tc.cu; shapes it does not take fall back), the latter
    with its two treatments of the <= 8 rows past the last full 128-row tile: the SIMT tail kernel (default) or one more wgmma tile."""
    impl, _, tail = request.param.partition("+tail_")
    ctx.set_option("attn", impl)
    ctx.set_option("attn_tail", tail or "kernel")
    yield request.param
    ctx.set_option("attn", "tc")
    ctx.set_option("attn_tail", "kernel")


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("case", ["self32", "cross32", "t5_64", "tiny", "gato392", "cross512"])
def test_attention(ctx, split, case, attn_impl):
    dt, tdt = DT["f16"]
    g = torch.Generator(device="cuda").manual_seed(3)
    if case == "self32":
        B, H, Lq, Lk, D, causal, scale = 3, 5, 263, 263, 32, True, 1 / math.sqrt(32)
    elif case == "cross32":
        B, H, Lq, Lk, D, causal, scale = 2, 4, 263, 250, 32, False, 1 / math.sqrt(32)
    elif case == "t5_64":
        B, H, Lq, Lk, D, causal, scale = 2, 3, 200, 200, 64, False, 1.0
    elif case == "gato392":  # BASELINE.json configs[4]: one causal sequence prompt | sep | history
        B, H, Lq, Lk, D, causal, scale = 2, 3, 392, 392, 32, True, 1 / math.sqrt(32)
    elif case == "cross512":  # survey row #3x: 512 prompt tokens
        B, H, Lq, Lk, D, causal, scale = 2, 2, 263, 512, 32, False, 1 / math.sqrt(32)
    else:
        B, H, Lq, Lk, D, causal, scale = 1, 8, 6, 10, 32, False, 1 / math.sqrt(32)
    E = H * D
    if case in ("self32", "gato392"):
        qkv = torch.randn(B * Lq, 3 * E, device="cuda", generator=g)
        hi, lo, ld = split_ops(ctx, qkv, dt, split)
        q = (hi, lo, ld, 0); k = (hi, lo, ld, E); v = (hi, lo, ld, 2 * E)
        Q, K, V = qkv[:, :E], qkv[:, E : 2 * E], qkv[:, 2 * E :]
    else:
        Qm = torch.randn(B * Lq, E, device="cuda", generator=g) * (0.35 if case == "t5_64" else 1.0)
        KV = torch.randn(B * Lk, 2 * E, device="cuda", generator=g)
        qh, ql, ldq = split_ops(ctx, Qm, dt, split)
        kh, kl, ldk = split_ops(ctx, KV, dt, split)
        q = (qh, ql, ldq, 0); k = (kh, kl, ldk, 0); v = (kh, kl, ldk, E)
        Q, K, V = Qm, KV[:, :E], KV[:, E:]
    key_mask = (torch.rand(B, Lk, device="cuda", generator=g) > 0.2)
    key_mask[:, 0] = True
    bias = None
    rel_bias = None
    if case == "t5_64":
        rel_bias = torch.randn(H, 2 * Lk - 1, device="cuda", generator=g)
        ii = torch.arange(Lq, device="cuda")[:, None]
        jj = torch.arange(Lk, device="cuda")[None, :]
        bias = rel_bias[:, (jj - ii + Lk - 1)].unsqueeze(0).double()
    o_hi = torch.zeros(B * Lq, E, dtype=torch.int16, device="cuda")
    o_lo = torch.zeros_like(o_hi)
    ctx.attention(q=q, k=k, v=v, o=(o_hi, o_lo, E, 0), B=B, H=H, Lq=Lq, Lk=Lk, D=D, scale=scale, causal=causal,
                  key_mask=key_mask.to(torch.uint8), rel_bias=rel_bias, dtype=dt)
    torch.cuda.synchronize()

    def heads(x, L):
        return x.reshape(B, L, H, D).permute(0, 2, 1, 3).double()

    if not split:  # compare against the same rounded operands
        rnd = lambda x: x.to(tdt).float()
        Q, K, V = rnd(Q), rnd(K), rnd(V)
    ref = ref_attention(heads(Q, Lq), heads(K, Lk), heads(V, Lk), scale, causal, key_mask, bias)
    ref = ref.permute(0, 2, 1, 3).reshape(B * Lq, E)
    got = merge(o_hi, o_lo, tdt, E)
    tol = 1e-5 if split else 2e-3  # single pass also rounds P to 11 bits
    assert torch.isfinite(got).all()
    assert rel(got, ref) < tol, rel(got, ref)


def test_attention_fully_masked_prefix(ctx, attn_impl):
    """Rows whose causally visible keys are all padded follow the reference's -1e4 soft mask exactly."""
    dt, tdt = DT["f16"]
    B, H, L, D = 1, 2, 70, 32
    E = H * D
    g = torch.Generator(device="cuda").manual_seed(5)
    qkv = torch.randn(B * L, 3 * E, device="cuda", generator=g)
    key_mask = torch.ones(B, L, dtype=torch.bool, device="cuda")
    key_mask[:, :3] = False  # queries 0..2 see only padded keys
    hi, lo, ld = split_ops(ctx, qkv, dt, True)
    o_hi = torch.zeros(B * L, E, dtype=torch.int16, device="cuda"); o_lo = torch.zeros_like(o_hi)
    ctx.attention(q=(hi, lo, ld, 0), k=(hi, lo, ld, E), v=(hi, lo, ld, 2 * E), o=(o_hi, o_lo, E, 0), B=B, H=H, Lq=L, Lk=L, D=D,
                  scale=1 / math.sqrt(D), causal=True, key_mask=key_mask.to(torch.uint8), dtype=dt)
    hd = lambda x: x.reshape(B, L, H, D).permute(0, 2, 1, 3).double()
    ref = ref_attention(hd(qkv[:, :E]), hd(qkv[:, E:2 * E]), hd(qkv[:, 2 * E:]), 1 / math.sqrt(D), True, key_mask, None)
    ref = ref.permute(0, 2, 1, 3).reshape(B * L, E)
    assert rel(merge(o_hi, o_lo, tdt, E), ref) < 1e-5


@pytest.mark.parametrize("L0,Ln", [(0, 33), (66, 33), (230, 33), (131, 1)])
def test_attention_kv_cache_addressing(ctx, L0, Ln, attn_impl):
    """Incremental decode: Ln new queries at positions L0.. attend causally over a cache with row pitch Lmax per episode
    (kv_batch_rows / mask_ld / q_pos0); equals the matching rows of the full-history causal attention."""
    dt, tdt = DT["f16"]
    B, H, D, Lmax = 3, 4, 32, 263
    E = H * D
    L = L0 + Ln
    g = torch.Generator(device="cuda").manual_seed(11)
    qkv_full = torch.randn(B, Lmax, 3 * E, device="cuda", generator=g)
    key_mask = torch.rand(B, Lmax, device="cuda", generator=g) > 0.2
    key_mask[:, 0] = True
    # cache layout: [B*Lmax, 2E] (K | V); rows >= L hold junk that must not be read as valid keys
    cache = qkv_full[:, :, E:].clone()
    cache[:, L:] = 1e4
    ch, cl, ldc = split_ops(ctx, cache.reshape(B * Lmax, 2 * E), dt, True)
    qn = qkv_full[:, L0:L, :E].reshape(B * Ln, E).contiguous()
    qh, ql, ldq = split_ops(ctx, qn, dt, True)
    o_hi = torch.zeros(B * Ln, E, dtype=torch.int16, device="cuda"); o_lo = torch.zeros_like(o_hi)
    ctx.attention(q=(qh, ql, ldq, 0), k=(ch, cl, ldc, 0), v=(ch, cl, ldc, E), o=(o_hi, o_lo, E, 0), B=B, H=H, Lq=Ln, Lk=L, D=D,
                  scale=1 / math.sqrt(D), causal=True, key_mask=key_mask.to(torch.uint8), dtype=dt, kv_batch_rows=Lmax, mask_ld=Lmax, q_pos0=L0)
    hd = lambda x, n: x.reshape(B, n, H, D).permute(0, 2, 1, 3).double()
    full = qkv_full[:, :L]
    ref = ref_attention(hd(full[..., :E], L), hd(full[..., E:2 * E], L), hd(full[..., 2 * E:], L), 1 / math.sqrt(D), True, key_mask[:, :L], None)
    ref = ref[:, :, L0:L].permute(0, 2, 1, 3).reshape(B * Ln, E)
    assert rel(merge(o_hi, o_lo, tdt, E), ref) < 1e-5
    with pytest.raises(RuntimeError):
        ctx.attention(q=(qh, ql, ldq, 0), k=(ch, cl, ldc, 0), v=(ch, cl, ldc, E), o=(o_hi, o_lo, E, 0), B=B, H=H, Lq=Ln, Lk=L, D=D,
                      scale=1 / math.sqrt(D), causal=True, dtype=dt, kv_batch_rows=Lmax, q_pos0=-1)


def test_small_attention(ctx):
    N, S, H, W = 37, 5, 24, 768
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv = torch.randn(N * S, 3 * W, device="cuda", generator=g)
    o = torch.empty(N * S, W, device="cuda")
    hi = torch.empty(N * S, W, dtype=torch.int16, device="cuda"); lo = torch.empty_like(hi)
    ctx.small_attention(qkv, N=N, S=S, H=H, W=W, scale=1 / math.sqrt(32), o_hi=hi, o_lo=lo, o_f32=o)
    q, k, v = [t.reshape(N, S, H, 32).transpose(1, 2).double() for t in qkv.split(W, dim=1)]
    ref = (torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(32), -1) @ v).transpose(1, 2).reshape(N * S, W)
    assert rel(o, ref) < 2e-6 and rel(merge(hi, lo, torch.float16, W), o) < 2e-6


def test_gemm_f32_grouped(ctx):
    import ctypes as C
    from vima_b200 import _C

    M = 77
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(M, 260, device="cuda", generator=g)
    specs = [(50, 260), (100, 260), (512, 4)]
    groups = (_C.F32GemmGroup * len(specs))()
    keep, refs = [], []
    for i, (n, k) in enumerate(specs):
        w = torch.randn(n, k, device="cuda", generator=g); b = torch.randn(n, device="cuda", generator=g)
        y = torch.zeros(M, n + 3, device="cuda")
        keep += [w, b, y]
        groups[i] = _C.F32GemmGroup(x.data_ptr(), x.stride(0), w.data_ptr(), k, b.data_ptr(), y.data_ptr(), y.stride(0), n, k)
        refs.append((y, torch.relu(x[:, :k].double() @ w.double().t() + b.double()), n))
    gd = torch.frombuffer(bytearray(bytes(groups)), dtype=torch.uint8).cuda()
    ctx.gemm_f32_grouped(gd, len(specs), M, 512, 1)
    for y, ref, n in refs:
        assert rel(y[:, :n], ref) < 2e-6 and (y[:, n:] == 0).all()
        y.zero_()
    # same launch with the descriptors travelling by value (host array; the CUDA-graph-safe form the modules use)
    ctx.gemm_f32_grouped_host(groups, len(specs), M, 512, 1)
    for y, ref, n in refs:
        assert rel(y[:, :n], ref) < 2e-6 and (y[:, n:] == 0).all()


def test_token_assembly(ctx):
    """Bit-exact interleave / masks / position ids against the oracle restatement of vima_policy.py:124-147."""
    from oracle import vima_oracle as O

    T, B, Q, E = 3, 4, 5, 64
    g = torch.Generator().manual_seed(0)
    obs = torch.randn(T, B, Q, E, generator=g)
    mask = torch.rand(T, B, Q, generator=g) > 0.3
    mask[0, :, 0] = True
    for La in (T - 1, T):
        act = torch.randn(La, B, E, generator=g)
        toks, masks, ids = O.assemble_history(obs, mask, act)
        L = T * Q + La
        tokens = torch.empty(L, B, E, device="cuda"); m_bl = torch.empty(B, L, dtype=torch.uint8, device="cuda")
        p_bl = torch.empty(B, L, dtype=torch.int64, device="cuda")
        ctx.assemble_history(dev(obs), dev(mask).to(torch.uint8), dev(act), tokens, m_bl, p_bl)
        assert torch.equal(tokens.cpu(), toks) and torch.equal(m_bl.cpu().bool(), masks.t()) and torch.equal(p_bl.cpu(), ids.t())
    pm = torch.tensor([[1, 1, 1, 1, 0, 0], [1, 0, 1, 1, 0, 1]], dtype=torch.uint8, device="cuda")
    pos = torch.empty(2, 6, dtype=torch.int64, device="cuda")
    ctx.mask_cumsum(pm, pos)
    assert pos.tolist() == [[0, 1, 2, 3, 3, 3], [0, 0, 1, 2, 2, 3]]
    # long sequence crossing the block size
    big = (torch.rand(3, 700, generator=g) > 0.4).to(torch.uint8)
    pos = torch.empty(3, 700, dtype=torch.int64, device="cuda")
    ctx.mask_cumsum(dev(big), pos)
    assert torch.equal(pos.cpu(), torch.cumsum(big.long(), 1) - 1)


def test_add_pos_embed_and_gather(ctx):
    B, L, E = 3, 11, 64
    g = torch.Generator().manual_seed(4)
    tok = torch.randn(L, B, E, generator=g)  # seq-first, read with strides
    ids = torch.randint(0, 20, (B, L), generator=g)
    table = torch.randn(20, E, generator=g)
    out = torch.empty(B, L, E, device="cuda")
    hi = torch.empty(B * L, E, dtype=torch.int16, device="cuda"); lo = torch.empty_like(hi)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    ctx.add_pos_embed(dev(tok), E, B * E, dev(ids), dev(table), B, L, E, out_f32=out, hi=hi, lo=lo, err_flag=err)
    ref = tok.transpose(0, 1) + table[ids]
    assert torch.equal(out.cpu(), ref) and err.item() == 0
    assert rel(merge(hi, lo, torch.float16, E).cpu(), ref.reshape(B * L, E)) < 2e-6
    bad = ids.clone(); bad[0, 0] = -1
    ctx.add_pos_embed(dev(tok), E, B * E, dev(bad), dev(table), B, L, E, out_f32=out, err_flag=err)
    assert err.item() == 1
    # prompt gather
    D, Lp = 32, 6
    word_table = torch.randn(50, D, generator=g); word_ids = torch.tensor([7, 3, 9, 1])
    img_emb = torch.randn(4, D, generator=g); img_mask = torch.tensor([1, 0, 1, 1], dtype=torch.uint8)
    kind = torch.tensor([[1, 2, 2, 1, 0, 0], [1, 1, 2, 2, 0, 0]], dtype=torch.int32)
    index = torch.tensor([[0, 0, 1, 1, 0, 0], [2, 3, 2, 3, 0, 0]], dtype=torch.int32)
    o = torch.empty(2, Lp, D, device="cuda"); mo = torch.empty(2, Lp, dtype=torch.uint8, device="cuda")
    ctx.gather_prompt(dev(kind), dev(index), dev(word_ids), dev(word_table), dev(img_emb), dev(img_mask), 2, Lp, D, o, mo)
    exp = torch.zeros(2, Lp, D); expm = torch.zeros(2, Lp, dtype=torch.uint8)
    for b in range(2):
        for p in range(Lp):
            if kind[b, p] == 1:
                exp[b, p] = word_table[word_ids[index[b, p]]]; expm[b, p] = 1
            elif kind[b, p] == 2:
                exp[b, p] = img_emb[index[b, p]]; expm[b, p] = img_mask[index[b, p]]
    assert torch.equal(o.cpu(), exp) and torch.equal(mo.cpu(), expm)


def test_patchify_and_small_preps(ctx):
    from oracle import vima_oracle as O

    N = 9
    g = torch.Generator().manual_seed(6)
    img = torch.randint(0, 256, (N, 3, 32, 32), generator=g, dtype=torch.uint8)
    hi = torch.empty(N * 4, 768, dtype=torch.int16, device="cuda"); lo = torch.empty_like(hi)
    ctx.patchify(dev(img), N, 32, 32, 16, hi, lo)
    ref = torch.nn.functional.unfold(O.image_preprocess(img), kernel_size=16, stride=16).transpose(1, 2).reshape(N * 4, 768)
    got = merge(hi, lo, torch.float16, 768).cpu()
    assert rel(got, ref) < 1e-6
    bbox = torch.randint(0, 128, (13, 4), generator=g)
    o = torch.empty(13, 4, device="cuda")
    ctx.bbox_norm(dev(bbox), 13, o)
    assert torch.equal(o.cpu(), bbox.float() / torch.tensor([256.0, 128.0, 128.0, 256.0]))
    idx = torch.randint(0, 50, (21, 2), generator=g)
    bins = torch.tensor([50.0, 100.0])
    o = torch.empty(21, 2, device="cuda")
    ctx.action_scale(dev(idx), 21, 2, dev(bins), o)
    assert torch.equal(o.cpu(), idx.float() / bins)
    mx = torch.zeros(1, dtype=torch.int32, device="cuda")
    ctx.max_u8(dev(img), mx)
    assert mx.item() == int(img.max())


def test_head_select(ctx):
    from oracle import vima_oracle as O

    B = 33
    g = torch.Generator().manual_seed(8)
    logits = torch.randn(1, B, 700, generator=g)
    dims = [n for d in O.ACTION_DIMS.values() for n in d]
    off = torch.tensor(np.concatenate([[0], np.cumsum(dims)]), dtype=torch.int32)
    norm = torch.empty(B, 700, device="cuda"); modes = torch.empty(B, 12, dtype=torch.int64, device="cuda")
    ctx.head_select(dev(logits[0]), B, 12, dev(off), norm, modes)
    exp = torch.cat([v for v in O.action_modes(logits).values()], dim=-1)[0]
    assert torch.equal(modes.cpu(), exp)
    refn = torch.cat([torch.log_softmax(x, -1) for x in torch.split(logits[0], dims, -1)], -1)
    assert rel(norm.cpu(), refn) < 1e-6


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm folded into the GEMMs (DESIGN.md "LN folding"): row statistics out of one epilogue, applied in the next
# ------------------------------------------------------------------------------------------------------------------
def _ln(x, w, b, eps=1e-5):
    return torch.nn.functional.layer_norm(x.double(), (x.shape[-1],), w.double(), b.double(), eps)


@pytest.mark.parametrize("mode", ["f16x3", "f16f8", "bf16x3"])
@pytest.mark.parametrize("M,E", [(263 * 9, 768), (130, 256), (1000, 384), (40000, 768)])
def test_gemm_row_stats_and_folded_layernorm(ctx, mode, M, E):
    """s = A Wo^T + res with row statistics from the epilogue  ->  GEGLU over the un-normalised s with LN folded into the weights
    (both halves: the GPT block; value half only: XAttention)  ->  projection whose residual is LN(s) rebuilt in the epilogue.
    Checked against fp64 torch statements of the reference modules (components.py:23-37,97-102,218-226)."""
    import vima_b200
    from vima_b200 import engine as eng

    vima_b200.set_precision(mode)
    try:
        p = eng.prec()
        g = torch.Generator(device="cuda").manual_seed(M + E)
        rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
        A = rn(M, E)
        Wo = rn(E, E) / math.sqrt(E)
        res = rn(M, E) * 2.0 + 0.7  # non-zero row means
        gam, bet = 1.0 + 0.1 * rn(E), 0.1 * rn(E)
        W1, Wg = rn(4 * E, E) / math.sqrt(E), rn(4 * E, E) / math.sqrt(E)
        b1 = 0.1 * rn(4 * E)
        W2 = rn(E, 4 * E) / math.sqrt(4 * E)
        b2 = 0.1 * rn(E)
        a16 = eng.to_operand(ctx, A, p)
        if p.f8:
            a16 = eng.Opnd(M, E, "cuda", True, f8=True)
            ctx.split(A, a16.hi, None, dtype=p.dtype)
            ctx.split_f8(A, a16.lo8, a16.hi8)
        pwo = eng.pack_linear(ctx, Wo, None, transposed=False, p=p, f8=True)
        part = eng.stats_buffer(ctx, M, pwo, "cuda")
        s32, s16 = eng.gemm(ctx, a16, pwo, p, residual=res, want_f32=True, want16=True, out_f8=True, stats_out=part)
        st = eng.row_stats_of(ctx, part, M, E, 1e-5)
        s_ref = A.double() @ Wo.double().t() + res.double()
        assert rel(s32, s_ref) < 3e-5
        mean_ref = s_ref.mean(dim=1)
        rstd_ref = 1.0 / torch.sqrt(s_ref.var(dim=1, unbiased=False) + 1e-5)
        assert (st[:, 0].double() - mean_ref).abs().max().item() < 2e-5 * (1 + mean_ref.abs().max().item())
        assert ((st[:, 1].double() - rstd_ref) / rstd_ref).abs().max().item() < 2e-5
        n_ref = _ln(s_ref, gam, bet)
        for ln_gate in (True, False):
            pw = eng.pack_glu(ctx, W1, b1, Wg, val_transposed=False, gate_transposed=False, p=p, f8=True, ln=(gam, bet), ln_gate=ln_gate)
            _, h16 = eng.gemm(ctx, s16, pw, p, act=3, want16=True, out_f8=True, row_stats=st)
            gate_in = n_ref if ln_gate else s_ref
            h_ref = torch.nn.functional.gelu(n_ref @ W1.double().t() + b1.double()) * (gate_in @ Wg.double().t())
            h = h16.hi.view(torch.float16 if p.dtype == 0 else torch.bfloat16)[:, : 4 * E].double()
            if h16.lo is not None:
                h = h + h16.lo.view(torch.float16 if p.dtype == 0 else torch.bfloat16)[:, : 4 * E].double()
            else:
                h = h + h16.lo8[:, : 4 * E].view(torch.float8_e4m3fn).double() / 1024.0
            tol = 2e-4 if mode == "bf16x3" else 6e-5
            assert rel(h, h_ref) < tol, (ln_gate, rel(h, h_ref))
            if ln_gate:  # the block's projection: residual = LN(s), rebuilt from s32 + (mean, rstd) in the epilogue
                pw2 = eng.pack_linear(ctx, W2, b2, transposed=False, p=p, f8=True)
                t32, _ = eng.gemm(ctx, h16, pw2, p, residual=s32, res_ln=(st, gam, bet), want_f32=True)
                t_ref = h_ref @ W2.double().t() + b2.double() + n_ref
                assert rel(t32, t_ref) < tol, rel(t32, t_ref)
        # a plain (non-GLU) Linear with a folded LayerNorm in front of it
        pwl = eng.pack_linear(ctx, Wo, b2, transposed=False, p=p, f8=True, ln=(gam, bet))
        y32, _ = eng.gemm(ctx, s16, pwl, p, want_f32=True, row_stats=st)
        assert rel(y32, n_ref @ Wo.double().t() + b2.double()) < (2e-4 if mode == "bf16x3" else 6e-5)
    finally:
        vima_b200.set_precision("f16x3")


def test_row_statistics_are_batch_slice_deterministic(ctx):
    """The partial sums are reduced in a fixed order: the first rows of a big GEMM get the same statistics, bit for bit, as the
    same rows run alone (different tile counts / cluster pairing)."""
    import vima_b200
    from vima_b200 import engine as eng

    vima_b200.set_precision("f16f8")
    try:
        p = eng.prec()
        g = torch.Generator(device="cuda").manual_seed(5)
        M, E, n = 50000, 768, 263 * 3
        A = torch.randn(M, E, device="cuda", generator=g)
        Wo = torch.randn(E, E, device="cuda", generator=g) / math.sqrt(E)
        res = torch.randn(M, E, device="cuda", generator=g)
        pwo = eng.pack_linear(ctx, Wo, None, transposed=False, p=p, f8=True)
        outs = []
        for rows in (M, n):
            a16 = eng.Opnd(rows, E, "cuda", True, f8=True)
            ctx.split(A[:rows].contiguous(), a16.hi, None, dtype=p.dtype)
            ctx.split_f8(A[:rows].contiguous(), a16.lo8, a16.hi8)
            part = eng.stats_buffer(ctx, rows, pwo, "cuda")
            eng.gemm(ctx, a16, pwo, p, residual=res[:rows].contiguous(), want_f32=True, stats_out=part)
            outs.append(eng.row_stats_of(ctx, part, rows, E, 1e-5)[:n].clone())
        assert torch.equal(outs[0], outs[1])
    finally:
        vima_b200.set_precision("f16x3")


def test_gemm_desc_v4_size_is_still_accepted(ctx):
    """Descriptor growth: a caller compiled against the ABI-v4 struct (no folded-LN fields) passes the v4 size and is served."""
    import ctypes as C

    from vima_b200 import _C

    M, N, K = 256, 256, 64
    A = torch.randn(M, K, device="cuda")
    W = torch.randn(N, K, device="cuda") / 8
    a_hi, _, lda = split_ops(ctx, A, 0, False)
    b_hi, _, ldb = split_ops(ctx, W, 0, False)
    out = torch.empty(M, N, device="cuda")
    d = _C.GemmDesc()
    d.struct_size = _C.GemmDesc.row_stats.offset  # = VIMA_GEMM_DESC_V4_SIZE
    d.M, d.N, d.K = M, N, K
    d.a_hi, d.lda, d.b_hi, d.ldb = a_hi.data_ptr(), lda, b_hi.data_ptr(), ldb
    d.dtype, d.acc_scale = 0, 1.0
    d.out_f32, d.ld_o32 = out.data_ptr(), N
    d.row_stats = 0xDEAD0  # beyond struct_size: must never be read
    assert ctx.lib.vima_gemm(ctx.h, C.byref(d), C.c_void_p(ctx._s())) == 0, ctx.lib.vima_last_error(ctx.h)
    torch.cuda.synchronize()
    ref = merge(a_hi, None, torch.float16, K).double() @ merge(b_hi, None, torch.float16, K).double().t()
    assert rel(out, ref) < 5e-6
