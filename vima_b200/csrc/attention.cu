// Fused masked attention, K and V^T resident in shared memory (head_dim 32 or 64; Lk up to what the device's shared memory holds,
// attention_max_lk).  It runs what the streaming wgmma kernels do not take: single-pass f16 / bf16 operands, the decoder at
// head_dim 64, and the T5 encoder's prompts that fit.
//
//   S = scale * Q K^T (+ T5 relative bias) ; causal: S[i][j>i] = -1e4 (the reference's soft mask,
//   components.py:61-63) ; S += (key_mask ? 0 : finfo(fp32).min) ; P = softmax(S) ; O = P V
//
// One CTA per (batch, head): K and V^T of that head stay in shared memory, each warp streams 16-query-row
// blocks with an online fp32 softmax (warp-shuffle row reductions) and mma.sync m16n8k16 tensor-core products.
// In split mode Q,K,V,P are (hi,lo) 16-bit pairs and every product is hi*hi + lo*hi + hi*lo, which keeps the
// logits and the PV sum at ~fp32 accuracy (the reference computes both in fp32).  Scores never touch HBM:
// the reference materialises a 1.7 GB fp32 score tensor per layer at B=256.
#include "kernels.h"

namespace vima {

template <int DT>
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (DT == DT_F16) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}

template <int DT>
__device__ __forceinline__ void pack_split(float x0, float x1, uint32_t& hi, uint32_t& lo) { split2<DT>(x0, x1, hi, lo); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem_row_ptr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(smem_row_ptr)));
}

// Scores are kept in the log2 domain (kernels.h: FP32_MIN, CAUSAL_L2, EXIT_L2).
template <int D, int DT, bool SPLIT>
__global__ void __launch_bounds__(256, (D == 32) ? 2 : 1) attention_kernel(const AttnParams p) {
  constexpr int KS = D / 16;   // k-steps over head_dim for Q K^T
  constexpr int ND = D / 8;    // n-tiles over head_dim for P V
  constexpr int KROW = D + 8;  // padded smem row (halfs) -> conflict-free ldmatrix
  extern __shared__ __align__(16) unsigned char smem[];
  const int h = blockIdx.x, b = blockIdx.y;
  const int Lq = p.Lq;
  const int qbr = p.q_batch_rows ? p.q_batch_rows : Lq;
  int qp0, Lk;  // this batch element's (per-batch with q_pos; shared memory is sized for the capacity p.Lk)
  attn_batch_keys(p, b, qbr, qp0, Lk);
  const int Lk_pad = (Lk + 63) & ~63;
  const int VROW = Lk_pad + 8;
  const int n_kt = Lk_pad / 64;
  unsigned short* Ks_hi = reinterpret_cast<unsigned short*>(smem);
  unsigned short* Ks_lo = Ks_hi + (SPLIT ? Lk_pad * KROW : 0);
  unsigned short* Vt_hi = Ks_lo + Lk_pad * KROW;
  unsigned short* Vt_lo = Vt_hi + (SPLIT ? D * VROW : 0);
  float* maskadd = reinterpret_cast<float*>(Vt_lo + D * VROW);
  int* tile_plain = reinterpret_cast<int*>(maskadd + Lk_pad);  // [n_kt] 1 = every key of the tile is real and unmasked
  int* qb_counter = tile_plain + n_kt;
  float* sbias = reinterpret_cast<float*>(qb_counter + 1);     // [2*Lk-1] (log2 domain) when rel_bias

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int mld = p.mask_ld ? p.mask_ld : p.Lk;
  // ---- stage K (row-major) and V (transposed) of this (b, h) in shared memory ----
  constexpr int CH = D / 8;  // 16-byte chunks per row
  for (int idx = tid; idx < Lk_pad * CH; idx += 256) {
    const int j = idx / CH, c = idx % CH;
    uint4 kh = make_uint4(0, 0, 0, 0), kl = kh, vh = kh, vl = kh;
    if (j < Lk) {
      const size_t row = (size_t)attn_kv_row(p, b, j);
      const size_t rk = row * p.ldk + h * D + c * 8;
      const size_t rv = row * p.ldv + h * D + c * 8;
      kh = __ldg(reinterpret_cast<const uint4*>(p.k_hi + rk));
      vh = __ldg(reinterpret_cast<const uint4*>(p.v_hi + rv));
      if (SPLIT) {
        kl = __ldg(reinterpret_cast<const uint4*>(p.k_lo + rk));
        vl = __ldg(reinterpret_cast<const uint4*>(p.v_lo + rv));
      }
    }
    *reinterpret_cast<uint4*>(Ks_hi + j * KROW + c * 8) = kh;
    if (SPLIT) *reinterpret_cast<uint4*>(Ks_lo + j * KROW + c * 8) = kl;
    const unsigned short* vhs = reinterpret_cast<const unsigned short*>(&vh);
    const unsigned short* vls = reinterpret_cast<const unsigned short*>(&vl);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      Vt_hi[(c * 8 + e) * VROW + j] = vhs[e];
      if (SPLIT) Vt_lo[(c * 8 + e) * VROW + j] = vls[e];
    }
  }
  for (int j = tid; j < Lk_pad; j += 256) maskadd[j] = attn_key_mask_term(p, b, mld, j, Lk);
  if (p.rel_bias)
    for (int j = tid; j < 2 * Lk - 1; j += 256) sbias[j] = __ldg(p.rel_bias + (size_t)h * (2 * Lk - 1) + j) * LOG2E;
  if (tid == 0) *qb_counter = 0;
  __syncthreads();
  for (int kt = warp; kt < n_kt; kt += 8) {
    const bool ok = (maskadd[kt * 64 + lane] == 0.f) && (maskadd[kt * 64 + 32 + lane] == 0.f);
    const bool all_ok = __all_sync(0xffffffffu, ok);
    if (lane == 0) tile_plain[kt] = all_ok ? 1 : 0;
  }
  __syncthreads();

  const int g = lane >> 2, t = lane & 3;
  const int n_qb = (Lq + 15) / 16;
  const float c_l2 = p.scale * LOG2E;
  const int lm_row = lane & 7, lm_chunk = (lane >> 3) * 8;  // ldmatrix: row within the 8x8 matrix, which of the 4 matrices
  for (;;) {
    // dynamic work distribution over 16-row query blocks, longest (latest, under the causal mask) first
    int ticket = 0;
    if (lane == 0) ticket = atomicAdd(qb_counter, 1);
    ticket = __shfl_sync(0xffffffffu, ticket, 0);
    if (ticket >= n_qb) break;
    const int qb = n_qb - 1 - ticket;
    const int r0 = qb * 16 + g, r1 = r0 + 8;
    uint32_t qh[KS][4], ql[KS][4];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = (e & 1) ? r1 : r0;
        const int c = ks * 16 + 2 * t + ((e & 2) ? 8 : 0);
        uint32_t vh = 0, vl = 0;
        if (r < Lq) {
          const size_t off = ((size_t)b * qbr + r) * p.ldq + h * D + c;
          vh = __ldg(reinterpret_cast<const uint32_t*>(p.q_hi + off));
          if (SPLIT) vl = __ldg(reinterpret_cast<const uint32_t*>(p.q_lo + off));
        }
        qh[ks][e] = vh;
        ql[ks][e] = vl;
      }
    }
    float o[ND][4];
#pragma unroll
    for (int n = 0; n < ND; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};

    for (int kt = 0; kt < n_kt; ++kt) {
      float s[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      // MMAs are issued round-robin over 4 independent accumulators so that back-to-back HMMAs never depend on each
      // other (a chain of 6 dependent HMMAs per accumulator leaves the pipe waiting on each result)
#pragma unroll
      for (int half = 0; half < 2; ++half) {
#pragma unroll
        for (int kk = 0; kk < KS; kk += 2) {  // one ldmatrix.x4 = B fragments of two k-steps (32 head-dim columns)
          uint32_t bh[4][4], bl[4][4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int key = kt * 64 + (half * 4 + q) * 8 + lm_row;
            ldmatrix_x4(bh[q], Ks_hi + key * KROW + kk * 16 + lm_chunk);
            if (SPLIT) ldmatrix_x4(bl[q], Ks_lo + key * KROW + kk * 16 + lm_chunk);
          }
#pragma unroll
          for (int k2 = 0; k2 < 2; ++k2) {
#pragma unroll
            for (int q = 0; q < 4; ++q) mma16816<DT>(s[half * 4 + q], qh[kk + k2], bh[q][2 * k2], bh[q][2 * k2 + 1]);
            if (SPLIT) {
#pragma unroll
              for (int q = 0; q < 4; ++q) mma16816<DT>(s[half * 4 + q], ql[kk + k2], bh[q][2 * k2], bh[q][2 * k2 + 1]);
#pragma unroll
              for (int q = 0; q < 4; ++q) mma16816<DT>(s[half * 4 + q], qh[kk + k2], bl[q][2 * k2], bl[q][2 * k2 + 1]);
            }
          }
        }
      }
      // ---- log2-domain scores; bias / soft causal mask / key mask only where the tile needs them ----
      const bool needs_mask = !tile_plain[kt];
      const bool needs_causal = p.causal && (kt * 64 + 63 > qb * 16 + qp0);
      float mx[2] = {-INFINITY, -INFINITY};
      if (!needs_mask && !needs_causal && p.rel_bias == nullptr) {
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float y = s[nt][e] * c_l2;
            s[nt][e] = y;
            mx[e >> 1] = fmaxf(mx[e >> 1], y);
          }
        }
      } else {
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int j = kt * 64 + nt * 8 + 2 * t + (e & 1);
            const int i = (e & 2) ? r1 : r0;
            float y = s[nt][e] * c_l2;
            if (p.rel_bias && j < Lk) y += sbias[j - min(i, Lq - 1) + Lk - 1];
            if (needs_causal && j > i + qp0) y = CAUSAL_L2;
            if (needs_mask) y += maskadd[j];
            s[nt][e] = y;
            mx[e >> 1] = fmaxf(mx[e >> 1], y);
          }
        }
      }
      float corr[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float m_new = fmaxf(mrow[r], mx[r]);
        corr[r] = ex2_approx(mrow[r] - m_new);
        mrow[r] = m_new;
        lrow[r] *= corr[r];
      }
      float ps[2] = {0.f, 0.f};
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float pv = ex2_approx(s[nt][e] - mrow[e >> 1]);
          s[nt][e] = pv;
          ps[e >> 1] += pv;
        }
      }
      lrow[0] += ps[0];
      lrow[1] += ps[1];
#pragma unroll
      for (int n = 0; n < ND; ++n) {
        o[n][0] *= corr[0]; o[n][1] *= corr[0];
        o[n][2] *= corr[1]; o[n][3] *= corr[1];
      }
      // ---- O += P V ----
      uint32_t ph[4][4], pl[4][4];
#pragma unroll
      for (int k2 = 0; k2 < 4; ++k2) {
        pack_split<DT>(s[2 * k2][0], s[2 * k2][1], ph[k2][0], pl[k2][0]);
        pack_split<DT>(s[2 * k2][2], s[2 * k2][3], ph[k2][1], pl[k2][1]);
        pack_split<DT>(s[2 * k2 + 1][0], s[2 * k2 + 1][1], ph[k2][2], pl[k2][2]);
        pack_split<DT>(s[2 * k2 + 1][2], s[2 * k2 + 1][3], ph[k2][3], pl[k2][3]);
      }
#pragma unroll
      for (int ng = 0; ng < ND; ng += 4) {  // 4 independent output accumulators per round
#pragma unroll
        for (int kp = 0; kp < 2; ++kp) {  // one ldmatrix.x4 = V^T fragments of two 16-key steps
          uint32_t vh4[4][4], vl4[4][4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int drow = (ng + q) * 8 + lm_row;
            ldmatrix_x4(vh4[q], Vt_hi + drow * VROW + kt * 64 + kp * 32 + lm_chunk);
            if (SPLIT) ldmatrix_x4(vl4[q], Vt_lo + drow * VROW + kt * 64 + kp * 32 + lm_chunk);
          }
#pragma unroll
          for (int k2 = 0; k2 < 2; ++k2) {
#pragma unroll
            for (int q = 0; q < 4; ++q) mma16816<DT>(o[ng + q], ph[2 * kp + k2], vh4[q][2 * k2], vh4[q][2 * k2 + 1]);
            if (SPLIT) {
#pragma unroll
              for (int q = 0; q < 4; ++q) mma16816<DT>(o[ng + q], pl[2 * kp + k2], vh4[q][2 * k2], vh4[q][2 * k2 + 1]);
#pragma unroll
              for (int q = 0; q < 4; ++q) mma16816<DT>(o[ng + q], ph[2 * kp + k2], vl4[q][2 * k2], vl4[q][2 * k2 + 1]);
            }
          }
        }
      }
      // Every later key tile is causally masked for all 16 rows: its weights are exp(-1e4 - m), exactly 0 in
      // fp32 once m > -1e4 + 104, so stopping here is bit-identical to the reference's full-width softmax.
      if (p.causal && (kt + 1) * 64 > qb * 16 + 15 + qp0) {
        const bool done = (mrow[0] > EXIT_L2) && (mrow[1] > EXIT_L2);
        if (__all_sync(0xffffffffu, done)) break;
      }
    }
    // row sums live in the 4 lanes of a quad
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 1);
      lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 2);
    }
    const float inv0 = 1.0f / lrow[0], inv1 = 1.0f / lrow[1];
#pragma unroll
    for (int n = 0; n < ND; ++n) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int r = half ? r1 : r0;
        if (r >= Lq) continue;
        const float inv = half ? inv1 : inv0;
        attn_store_pair<DT>(p, (size_t)b * qbr + r, h * D + n * 8 + 2 * t, o[n][2 * half] * inv, o[n][2 * half + 1] * inv);
      }
    }
  }
}

// dynamic shared memory of attention_kernel: K [Lk_pad, D+8] and V^T [D, Lk_pad+8] per operand part, mask row, tile flags, bias row
size_t attention_smem_bytes(const AttnParams& p) {
  const int D = p.D;
  const int Lk_pad = (p.Lk + 63) & ~63;
  const size_t parts = p.split ? 2 : 1;
  size_t smem = parts * (size_t)Lk_pad * (D + 8) * 2 + parts * (size_t)D * (Lk_pad + 8) * 2 + (size_t)Lk_pad * 4 + (size_t)(Lk_pad / 64 + 1) * 4;
  if (p.rel_bias) smem += (size_t)(2 * p.Lk) * 4;
  return smem;
}

int attention_max_lk(const AttnParams& p, size_t smem_limit) {
  AttnParams q = p;
  int best = 0;
  for (int lk = 64; lk <= 4096; lk += 64) {
    q.Lk = lk;
    if (attention_smem_bytes(q) <= smem_limit) best = lk; else break;
  }
  return best;
}

template <int D, int DT, bool SPLIT>
static cudaError_t launch_attn_t(const AttnParams& p, cudaStream_t stream) {
  const size_t smem = attention_smem_bytes(p);
  const cudaError_t e = raise_smem_ceiling<attention_kernel<D, DT, SPLIT>>((int)smem);  // raised to the largest Lk seen so far
  if (e != cudaSuccess) return e;
  dim3 grid(p.H, p.B);
  attention_kernel<D, DT, SPLIT><<<grid, 256, smem, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_attention(const AttnParams& p, cudaStream_t stream) {
  if (p.B == 0 || p.Lq == 0) return cudaSuccess;
  const bool sp = p.split != 0;
  if (p.D == 32) {
    if (p.dtype == DT_F16) return sp ? launch_attn_t<32, DT_F16, true>(p, stream) : launch_attn_t<32, DT_F16, false>(p, stream);
    return sp ? launch_attn_t<32, DT_BF16, true>(p, stream) : launch_attn_t<32, DT_BF16, false>(p, stream);
  }
  if (p.D == 64) {
    if (p.dtype == DT_F16) return sp ? launch_attn_t<64, DT_F16, true>(p, stream) : launch_attn_t<64, DT_F16, false>(p, stream);
    return sp ? launch_attn_t<64, DT_BF16, true>(p, stream) : launch_attn_t<64, DT_BF16, false>(p, stream);
  }
  return cudaErrorInvalidValue;
}

// ---------------------------------------------------------------------------------------------------------
// Tiny-sequence attention in fp32 (ViT: 5 tokens per crop).  One THREAD per (crop, head, query token): the query row, the
// S scores and the 32-wide output stay in registers, K / V head slices are read as float4 (the S query threads of one
// (crop, head) are adjacent lanes, so their K / V loads coalesce into the same sectors).  head_dim must be 32.  qkv carries
// the in_proj bias already.  ~6x fewer instructions than the round-1 warp-per-(crop, head) shuffle-reduction form.
// ---------------------------------------------------------------------------------------------------------
constexpr int SMALL_S_MAX = 16;

template <int DT>
__global__ void __launch_bounds__(128) small_attention_kernel(const SmallAttnParams p) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int S = p.S;
  if (t >= p.N * p.H * S) return;
  const int i = (int)(t % S);
  const long long nh = t / S;
  const int h = (int)(nh % p.H);
  const long long n = nh / p.H;
  const float* base = p.qkv + (size_t)(n * S) * p.ld + h * 32;
  float4 q[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) q[c] = __ldg(reinterpret_cast<const float4*>(base + (size_t)i * p.ld) + c);
  float sc[SMALL_S_MAX];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < SMALL_S_MAX; ++j) {
    if (j < S) {
      const float4* kr = reinterpret_cast<const float4*>(base + (size_t)j * p.ld + p.W);
      float a0 = 0.f, a1 = 0.f;
#pragma unroll
      for (int c = 0; c < 8; c += 2) {
        const float4 k0 = __ldg(kr + c), k1 = __ldg(kr + c + 1);
        a0 = fmaf(q[c].x, k0.x, a0); a0 = fmaf(q[c].y, k0.y, a0); a0 = fmaf(q[c].z, k0.z, a0); a0 = fmaf(q[c].w, k0.w, a0);
        a1 = fmaf(q[c + 1].x, k1.x, a1); a1 = fmaf(q[c + 1].y, k1.y, a1); a1 = fmaf(q[c + 1].z, k1.z, a1); a1 = fmaf(q[c + 1].w, k1.w, a1);
      }
      sc[j] = (a0 + a1) * p.scale;
      mx = fmaxf(mx, sc[j]);
    }
  }
  float den = 0.f;
#pragma unroll
  for (int j = 0; j < SMALL_S_MAX; ++j) {
    if (j < S) {
      sc[j] = expf(sc[j] - mx);
      den += sc[j];
    }
  }
  const float inv = 1.0f / den;
  float4 o[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) o[c] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int j = 0; j < SMALL_S_MAX; ++j) {
    if (j < S) {
      const float4* vr = reinterpret_cast<const float4*>(base + (size_t)j * p.ld + 2 * p.W);
      const float w = sc[j] * inv;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float4 v = __ldg(vr + c);
        o[c].x = fmaf(w, v.x, o[c].x); o[c].y = fmaf(w, v.y, o[c].y); o[c].z = fmaf(w, v.z, o[c].z); o[c].w = fmaf(w, v.w, o[c].w);
      }
    }
  }
  const size_t off = (size_t)(n * S + i) * p.ldo + h * 32;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    if (p.o_f32) *reinterpret_cast<float4*>(p.o_f32 + off + c * 4) = o[c];
    if (p.o_hi) {
      uint2 hi, lo;
      split4v<DT>(o[c], hi, lo);
      *reinterpret_cast<uint2*>(p.o_hi + off + c * 4) = hi;
      if (p.o_lo) *reinterpret_cast<uint2*>(p.o_lo + off + c * 4) = lo;
    }
  }
}

cudaError_t launch_small_attention(const SmallAttnParams& p, cudaStream_t stream) {
  if (p.N == 0) return cudaSuccess;
  if (p.S > SMALL_S_MAX || p.S < 1 || p.W != p.H * 32 || (p.ld & 3) || (p.ldo & 3)) return cudaErrorInvalidValue;
  const long long threads = p.N * p.H * p.S;
  const long long blocks = (threads + 127) / 128;
  if (p.dtype == DT_BF16)
    small_attention_kernel<DT_BF16><<<(unsigned)blocks, 128, 0, stream>>>(p);
  else
    small_attention_kernel<DT_F16><<<(unsigned)blocks, 128, 0, stream>>>(p);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------
// Latent attention in fp32 (HF Perceiver resampler of the VIMA-Flamingo baseline, modeling_perceiver.py PerceiverSelfAttention):
// a handful of latent queries against <= 16 keys, head_dim <= 128.  One warp per (image, head); lane l owns head
// dimensions l, l+32, l+64, l+96.  q may be shared by all images (q_batch_stride 0: the cross-attention queries are the
// learned latents).
// ---------------------------------------------------------------------------------------------------------
constexpr int LAT_LK_MAX = 16, LAT_DV = 4;

__global__ void __launch_bounds__(256) latent_attention_kernel(const LatentAttnParams p) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= p.N * p.H) return;
  const long long n = w / p.H;
  const int h = (int)(w % p.H);
  const int d = p.d;
  const float* qb = p.q + (size_t)n * p.q_batch_stride + h * d;
  const float* kb = p.k + (size_t)n * p.Lk * p.ldk + h * d;
  const float* vb = p.v + (size_t)n * p.Lk * p.ldv + h * d;
  for (int i = 0; i < p.Lq; ++i) {
    float qv[LAT_DV];
#pragma unroll
    for (int e = 0; e < LAT_DV; ++e) qv[e] = (lane + 32 * e < d) ? __ldg(qb + (size_t)i * p.ldq + lane + 32 * e) : 0.f;
    float sc[LAT_LK_MAX];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < LAT_LK_MAX; ++j) {
      if (j < p.Lk) {
        float part = 0.f;
#pragma unroll
        for (int e = 0; e < LAT_DV; ++e)
          if (lane + 32 * e < d) part = fmaf(qv[e], __ldg(kb + (size_t)j * p.ldk + lane + 32 * e), part);
        sc[j] = warp_sum(part) * p.scale;
        mx = fmaxf(mx, sc[j]);
      }
    }
    float den = 0.f, acc[LAT_DV] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < LAT_LK_MAX; ++j) {
      if (j < p.Lk) {
        const float e_ = expf(sc[j] - mx);
        den += e_;
#pragma unroll
        for (int e = 0; e < LAT_DV; ++e)
          if (lane + 32 * e < d) acc[e] = fmaf(e_, __ldg(vb + (size_t)j * p.ldv + lane + 32 * e), acc[e]);
      }
    }
    const float inv = 1.0f / den;
#pragma unroll
    for (int e = 0; e < LAT_DV; ++e)
      if (lane + 32 * e < d) p.o[((size_t)n * p.Lq + i) * p.ldo + h * d + lane + 32 * e] = acc[e] * inv;
  }
}

cudaError_t launch_latent_attention(const LatentAttnParams& p, cudaStream_t stream) {
  if (p.N == 0 || p.Lq == 0) return cudaSuccess;
  if (p.Lk > LAT_LK_MAX || p.Lk < 1 || p.d > 32 * LAT_DV || p.d < 1) return cudaErrorInvalidValue;
  const long long warps = p.N * p.H;
  latent_attention_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace vima
