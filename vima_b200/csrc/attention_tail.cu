// Tail rows of the decoder attentions (head_dim 32), companion of attention_tc.cu.
//
// The wgmma kernel works on 128-query tiles.  The decoder's sequence lengths are T*(Q+1)-1 (263 for the 200M benchmark
// configuration, 392 = prompt | sep | history for VIMA-Gato): a handful of rows (7 / 8) spill into one more tile per (batch, head)
// that occupies a CTA slot for its whole key range while one warp of eight has work.  Those rows are taken here instead: a warp per
// (batch, head), up to 8 query rows, plain fp32 FMAs on the (hi + lo) operands -- about 2 MFLOP per unit, no tensor
// cores, no shared-memory staging of K / V (each element is read exactly once, straight from L2).
//
//   phase 1  lane = key:    y[j][i] = (q_i * scale*log2e) . k_j  + mask terms      -> shared [Lk][8], running row maxima
//   phase 2  lane = key:    p = exp2(y - max_i), row sums
//   phase 3  lane = (key mod 4, 4-dim group):  o_i += p[j][i] * v_j                -> xor-shuffle reduce over the 4 key groups
//
// Same mask semantics as attention.cu / attention_tc.cu (reference components.py:51-80, modeling_openai.py:86-115): causal
// replaces a hidden score by the soft -1e4, key padding adds finfo.min, keys beyond Lk are excluded, softmax over the full key
// range in fp32 (so a row whose visible keys are all padded gets the reference's degenerate weights without any special case).
#include "kernels.h"

namespace vima {

namespace {

constexpr int TAIL_NT = ATTN_TAIL_MAX_ROWS;
constexpr int TAIL_WARPS = 8;
constexpr int TAIL_D = 32;

template <int DT>
__device__ __forceinline__ float2 unpack2(uint32_t w) {
  if constexpr (DT == DT_F16) return __half22float2(*reinterpret_cast<const __half2*>(&w));
  else return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
}
__device__ __forceinline__ unsigned long long pack2(float x, float y) {
  unsigned long long r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(x), "f"(y));
  return r;
}
__device__ __forceinline__ float2 unpack64(unsigned long long v) {
  float2 r;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v));
  return r;
}
// acc += a * b on two packed fp32 lanes (two scalar FFMAs: sm_90 has no packed fp32 FMA)
__device__ __forceinline__ void ffma2(unsigned long long& acc, unsigned long long a, unsigned long long b) {
  const float2 x = unpack64(acc), y = unpack64(a), z = unpack64(b);
  acc = pack2(fmaf(y.x, z.x, x.x), fmaf(y.y, z.y, x.y));
}

template <int DT, bool PAGED>  // PAGED: k / v rows through the page table (attn_kv_row)
__global__ void __launch_bounds__(TAIL_WARPS * 32) attention_tail_kernel(const AttnParams p, int row0, int nt, int lk_pad) {
  extern __shared__ __align__(16) float smt[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // (batch ascending, like the wgmma kernel before it)
  const long long unit = (long long)blockIdx.x * TAIL_WARPS + warp;
  if (unit >= (long long)p.B * p.H) return;  // whole warps leave; nothing below synchronises across warps
  const int b = (int)(unit / p.H), h = (int)(unit % p.H);
  const int mld = p.mask_ld ? p.mask_ld : p.Lk;
  const int qbr = p.q_batch_rows ? p.q_batch_rows : p.Lq;
  int qp0, Lk;  // this batch element's (per-batch with q_pos)
  attn_batch_keys(p, b, qbr, qp0, Lk);
  float* qs = smt + (size_t)warp * (TAIL_NT * TAIL_D + (size_t)lk_pad * TAIL_NT);  // [8][32] queries, pre-scaled
  float* sc = qs + TAIL_NT * TAIL_D;                                                 // [lk_pad][8] scores -> weights
  lk_pad = (Lk + 31) & ~31;  // keys this batch element walks (the shared-memory carve above keeps the launch's capacity)

  // ---- queries: lane = dim ----
  const float c_l2 = p.scale * LOG2E;
#pragma unroll
  for (int i = 0; i < TAIL_NT; ++i) {
    float q = 0.f;
    if (i < nt) {
      const size_t off = ((size_t)b * qbr + row0 + i) * p.ldq + h * TAIL_D + lane;
      q = Op16<DT>::back(p.q_hi[off]);
      if (p.q_lo) q += Op16<DT>::back(p.q_lo[off]);
    }
    qs[i * TAIL_D + lane] = q * c_l2;
  }
  __syncwarp();

  // ---- phase 1: scores, lane = key ----
  float mx[TAIL_NT];
#pragma unroll
  for (int i = 0; i < TAIL_NT; ++i) mx[i] = -INFINITY;
  const int pos0 = row0 + qp0;  // key position of tail row 0 (causal)
  // raw (hi, lo) words of this lane's key row; the NEXT batch's rows are requested as soon as the current ones are converted, so the
  // L2 round trip overlaps the 128 packed FMAs of the batch in hand
  uint4 kh[4], kl[4];
  auto load_k = [&](int j) {
#pragma unroll
    for (int c = 0; c < 4; ++c) { kh[c] = make_uint4(0u, 0u, 0u, 0u); kl[c] = kh[c]; }
    if (j < Lk) {
      const size_t rk = (size_t)attn_kv_row<PAGED>(p, b, j) * p.ldk + h * TAIL_D;
      const uint4* ph = reinterpret_cast<const uint4*>(p.k_hi + rk);
#pragma unroll
      for (int c = 0; c < 4; ++c) kh[c] = __ldg(ph + c);
      if (p.k_lo) {
        const uint4* pl = reinterpret_cast<const uint4*>(p.k_lo + rk);
#pragma unroll
        for (int c = 0; c < 4; ++c) kl[c] = __ldg(pl + c);
      }
    }
  };
  load_k(lane);
  for (int j0 = 0; j0 < lk_pad; j0 += 32) {
    const int j = j0 + lane;
    const bool valid = j < Lk;
    unsigned long long kf[TAIL_D / 2];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const uint32_t aw[4] = {kh[c].x, kh[c].y, kh[c].z, kh[c].w};
      const uint32_t lw[4] = {kl[c].x, kl[c].y, kl[c].z, kl[c].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 x = unpack2<DT>(aw[e]), y = unpack2<DT>(lw[e]);
        kf[c * 4 + e] = pack2(x.x + y.x, x.y + y.y);
      }
    }
    if (j0 + 32 < lk_pad) load_k(j + 32);
    // attn_key_mask_term(p, b, mld, j, Lk) written out: through the helper, ptxas gives this kernel 3 to 5 more registers
    float madd = -INFINITY;
    if (valid) madd = (p.key_mask == nullptr || p.key_mask[(size_t)b * mld + j]) ? 0.f : FP32_MIN;
    float y[TAIL_NT];
#pragma unroll
    for (int i = 0; i < TAIL_NT; ++i) {
      const ulonglong2* q2 = reinterpret_cast<const ulonglong2*>(qs + i * TAIL_D);
      unsigned long long a0 = 0ull, a1 = 0ull;
#pragma unroll
      for (int c = 0; c < TAIL_D / 4; ++c) {
        const ulonglong2 q = q2[c];  // broadcast: every lane reads the same 16 bytes
        ffma2(a0, q.x, kf[2 * c]);
        ffma2(a1, q.y, kf[2 * c + 1]);
      }
      const float2 s0 = unpack64(a0), s1 = unpack64(a1);
      float v = ((s0.x + s0.y) + (s1.x + s1.y)) + madd;
      if (p.causal && j > pos0 + i) v = CAUSAL_L2 + madd;
      y[i] = v;
      mx[i] = fmaxf(mx[i], v);
    }
    float4* dst = reinterpret_cast<float4*>(sc + (size_t)j * TAIL_NT);
    dst[0] = make_float4(y[0], y[1], y[2], y[3]);
    dst[1] = make_float4(y[4], y[5], y[6], y[7]);
  }
#pragma unroll
  for (int i = 0; i < TAIL_NT; ++i) mx[i] = warp_max(mx[i]);

  // ---- phase 2: weights and row sums (every lane re-reads what it wrote itself) ----
  float ls[TAIL_NT];
#pragma unroll
  for (int i = 0; i < TAIL_NT; ++i) ls[i] = 0.f;
  for (int j0 = 0; j0 < lk_pad; j0 += 32) {
    float4* cell = reinterpret_cast<float4*>(sc + (size_t)(j0 + lane) * TAIL_NT);
    const float4 a = cell[0], c = cell[1];
    float w[TAIL_NT] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
#pragma unroll
    for (int i = 0; i < TAIL_NT; ++i) {
      w[i] = ex2_approx(w[i] - mx[i]);
      ls[i] += w[i];
    }
    cell[0] = make_float4(w[0], w[1], w[2], w[3]);
    cell[1] = make_float4(w[4], w[5], w[6], w[7]);
  }
#pragma unroll
  for (int i = 0; i < TAIL_NT; ++i) ls[i] = warp_sum(ls[i]);
  __syncwarp();

  // ---- phase 3: O = P V, lane = (key group kg of 4, 4-dim group dg of 8) ----
  const int kg = lane >> 3, dg = lane & 7;
  unsigned long long acc[TAIL_NT][2];
#pragma unroll
  for (int i = 0; i < TAIL_NT; ++i) { acc[i][0] = 0ull; acc[i][1] = 0ull; }
  for (int j = kg; j < Lk; j += 16) {  // 4 keys per lane group per trip: their loads are all in flight before the first FMA
    uint2 vh[4], vl[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int jj = j + 4 * u;
      vh[u] = make_uint2(0u, 0u); vl[u] = vh[u];
      if (jj < Lk) {
        const size_t rv = (size_t)attn_kv_row<PAGED>(p, b, jj) * p.ldv + h * TAIL_D + dg * 4;
        vh[u] = __ldg(reinterpret_cast<const uint2*>(p.v_hi + rv));
        if (p.v_lo) vl[u] = __ldg(reinterpret_cast<const uint2*>(p.v_lo + rv));
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int jj = j + 4 * u;
      if (jj >= Lk) break;
      const float2 h0 = unpack2<DT>(vh[u].x), l0 = unpack2<DT>(vl[u].x), h1 = unpack2<DT>(vh[u].y), l1 = unpack2<DT>(vl[u].y);
      const unsigned long long v01 = pack2(h0.x + l0.x, h0.y + l0.y), v23 = pack2(h1.x + l1.x, h1.y + l1.y);
      const float4* cell = reinterpret_cast<const float4*>(sc + (size_t)jj * TAIL_NT);
      const float4 a = cell[0], c = cell[1];
      const float w[TAIL_NT] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
#pragma unroll
      for (int i = 0; i < TAIL_NT; ++i) {
        const unsigned long long ww = pack2(w[i], w[i]);
        ffma2(acc[i][0], ww, v01);
        ffma2(acc[i][1], ww, v23);
      }
    }
  }
  // fold the 4 key groups (lanes differing in bits 3 and 4); afterwards every lane holds the full sums of its 4 dims
#pragma unroll
  for (int i = 0; i < TAIL_NT; ++i) {
    const float2 a01 = unpack64(acc[i][0]), a23 = unpack64(acc[i][1]);
    float4 o = make_float4(a01.x, a01.y, a23.x, a23.y);
    o.x += __shfl_xor_sync(0xffffffffu, o.x, 8); o.y += __shfl_xor_sync(0xffffffffu, o.y, 8);
    o.z += __shfl_xor_sync(0xffffffffu, o.z, 8); o.w += __shfl_xor_sync(0xffffffffu, o.w, 8);
    o.x += __shfl_xor_sync(0xffffffffu, o.x, 16); o.y += __shfl_xor_sync(0xffffffffu, o.y, 16);
    o.z += __shfl_xor_sync(0xffffffffu, o.z, 16); o.w += __shfl_xor_sync(0xffffffffu, o.w, 16);
    if ((i & 3) != kg || i >= nt) continue;  // key group kg stores rows kg and kg + 4
    const float inv = 1.0f / ls[i];
    o.x *= inv; o.y *= inv; o.z *= inv; o.w *= inv;
    const size_t row = (size_t)b * qbr + row0 + i;
    const size_t off = row * p.ldo + h * TAIL_D + dg * 4;
    if (p.o_lo8) {  // fp16 hi + e4m3 cross-term views (an "f16f8" consumer GEMM); the 16-bit lo part only if asked for
      uint2 h16;
      uint32_t l8, h8;
      split4_f8(o, F8_ACT_LO_SCALE, F8_ACT_HI_SCALE, h16, l8, h8);
      *reinterpret_cast<uint2*>(p.o_hi + off) = h16;
      const size_t off8 = row * p.ldo8 + h * TAIL_D + dg * 4;
      *reinterpret_cast<uint32_t*>(p.o_lo8 + off8) = l8;
      *reinterpret_cast<uint32_t*>(p.o_hi8 + off8) = h8;
      if (p.o_lo) {
        uint2 hi, lo;
        split4v<DT>(o, hi, lo);
        *reinterpret_cast<uint2*>(p.o_lo + off) = lo;
      }
    } else {
      uint2 hi, lo;
      split4v<DT>(o, hi, lo);
      *reinterpret_cast<uint2*>(p.o_hi + off) = hi;
      if (p.o_lo) *reinterpret_cast<uint2*>(p.o_lo + off) = lo;
    }
  }
}

constexpr size_t TAIL_SMEM_MAX = (size_t)TAIL_WARPS * (TAIL_NT * TAIL_D + (size_t)ATTN_TAIL_MAX_LK * TAIL_NT) * sizeof(float);

template <int DT, bool PAGED>
cudaError_t launch_tail_t(const AttnParams& p, int row0, int nt, int lk_pad, unsigned grid, size_t smem, cudaStream_t stream) {
  // the ceiling is the capacity's, so it is set once, whatever Lk the first call has
  const cudaError_t e = raise_smem_ceiling<attention_tail_kernel<DT, PAGED>>((int)TAIL_SMEM_MAX);
  if (e != cudaSuccess) return e;
  attention_tail_kernel<DT, PAGED><<<grid, TAIL_WARPS * 32, smem, stream>>>(p, row0, nt, lk_pad);
  return cudaGetLastError();
}

}  // namespace

// rows [row0, row0 + nt) of every (batch, head) of p (nt <= ATTN_TAIL_MAX_ROWS); p.Lq / p.q_batch_rows give the row pitch
cudaError_t launch_attention_tail(const AttnParams& p, int row0, int nt, cudaStream_t stream) {
  if (p.B == 0 || nt <= 0) return cudaSuccess;
  if (nt > TAIL_NT || p.D != TAIL_D) return cudaErrorInvalidValue;
  const int lk_pad = (p.Lk + 31) & ~31;
  const size_t smem = (size_t)TAIL_WARPS * (TAIL_NT * TAIL_D + (size_t)lk_pad * TAIL_NT) * sizeof(float);
  if (smem > TAIL_SMEM_MAX) return cudaErrorInvalidValue;
  const long long units = (long long)p.B * p.H;
  const unsigned grid = (unsigned)((units + TAIL_WARPS - 1) / TAIL_WARPS);
  const bool bf = p.dtype == DT_BF16;
  if (p.kv_pages) return bf ? launch_tail_t<DT_BF16, true>(p, row0, nt, lk_pad, grid, smem, stream) : launch_tail_t<DT_F16, true>(p, row0, nt, lk_pad, grid, smem, stream);
  return bf ? launch_tail_t<DT_BF16, false>(p, row0, nt, lk_pad, grid, smem, stream) : launch_tail_t<DT_F16, false>(p, row0, nt, lk_pad, grid, smem, stream);
}

}  // namespace vima
