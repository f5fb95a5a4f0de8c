"""GPU probe: do wgmma f16 and mma.sync flush fp16 subnormal inputs?"""
import math, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vima_b200 import _C
ctx = _C.Context.get(torch.device("cuda", 0))
M, N, K = 128, 32, 64
tiny = 2.0 ** -20
A = torch.full((M, K), tiny, device="cuda")
W = torch.ones(N, K, device="cuda")
a_hi = torch.empty(M, K, dtype=torch.int16, device="cuda"); b_hi = torch.empty(N, K, dtype=torch.int16, device="cuda")
ctx.split(A, a_hi, None, dtype=0); ctx.split(W, b_hi, None, dtype=0)
print("A as fp16 (subnormal) value:", a_hi.view(torch.float16)[0, 0].item())
out = torch.empty(M, N, device="cuda")
ctx.gemm(M=M, N=N, K=K, a_hi=a_hi, a_lo=None, lda=K, b_hi=b_hi, b_lo=None, ldb=K, dtype=0, out_f32=out)
torch.cuda.synchronize()
print("wgmma: sum of 64 subnormal*1 =", out[0, 0].item(), "expected", K * tiny, "->", "subnormals HONOURED" if out[0, 0].item() > 0 else "FLUSHED")
# B subnormal
ctx.split(W, a_hi, None, dtype=0); A2 = torch.full((N, K), tiny, device="cuda"); ctx.split(A2, b_hi, None, dtype=0)
ctx.gemm(M=M, N=N, K=K, a_hi=a_hi, a_lo=None, lda=K, b_hi=b_hi, b_lo=None, ldb=K, dtype=0, out_f32=out)
torch.cuda.synchronize()
print("wgmma (B subnormal):", out[0, 0].item())
# mma.sync through the attention kernel: V subnormal constant -> O should equal it
B, H, L, D = 1, 1, 64, 32
q = torch.zeros(L, D, device="cuda"); kv = torch.cat([torch.zeros(L, D, device="cuda"), torch.full((L, D), tiny, device="cuda")], 1)
qh = torch.empty(L, D, dtype=torch.int16, device="cuda"); kh = torch.empty(L, 2 * D, dtype=torch.int16, device="cuda")
ctx.split(q, qh, None, dtype=0); ctx.split(kv.contiguous(), kh, None, dtype=0)
oh = torch.zeros(L, D, dtype=torch.int16, device="cuda"); ol = torch.zeros_like(oh)
ctx.attention(q=(qh, None, D, 0), k=(kh, None, 2 * D, 0), v=(kh, None, 2 * D, D), o=(oh, ol, D, 0), B=B, H=H, Lq=L, Lk=L, D=D, scale=1.0, dtype=0)
torch.cuda.synchronize()
o = oh.view(torch.float16).float() + ol.view(torch.float16).float()
print("mma.sync: P(=1/64 each, normal) x V(subnormal) ->", o[0, 0].item(), "expected", tiny)
