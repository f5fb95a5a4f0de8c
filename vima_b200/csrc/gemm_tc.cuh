// wgmma GEMM for sm_90a:  C[M,N] = epilogue( A[M,K] * B[N,K]^T )
//
//  * A (activations) and B (packed weights) are K-major 16-bit operands (fp16 or bf16), optionally as (hi, lo)
//    pairs: in split mode the kernel accumulates A_hi*B_hi + A_lo*B_hi + A_hi*B_lo in the SAME fp32 register
//    accumulator, which restores ~fp32 products (see DESIGN.md "operand precision").
//  * Persistent, warp-specialised: warps 0-7 = two consumer warpgroups (rows [0,64) and [64,128) of the 128-row tile; each
//    issues one wgmma M64 N{BN} instruction per k step and operand pair and runs the epilogue of its rows), warps 8-11 = the
//    producer warpgroup (one lane issues the TMA loads).  The producer warpgroup hands its registers to the consumers
//    (setmaxnreg), which hold up to two 64 x 128 fp32 accumulators per warpgroup in f16f8 mode.
//  * The split mode (SPLIT) and the tile width (BN) are template parameters, so every wgmma of the main loop is issued
//    unconditionally: a wgmma under a run-time branch makes ptxas serialise the whole pipeline.
//  * smem ring of `n_stages` stages {A_hi,[A_lo],B_hi,[B_lo]} in the 128-byte swizzled K-major layout that TMA
//    writes and the wgmma descriptors read; the producer fills the next tile's stages while the consumers run the epilogue.
//  * Epilogue: acc*scale + bias -> activation -> (GLU pair product) -> *mul -> +residual -> fp32 and/or (hi,lo).
//    The epilogue is specialised at compile time (EpiCfg) for the combinations the VIMA path uses; a generic
//    runtime-flag variant covers everything else.
#pragma once
#include "common.cuh"

namespace vima {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;                       // 64 x 2 B = 128 B = one swizzle row
constexpr int GEMM_A_TILE_BYTES = GEMM_BM * 128;  // 16 KB
constexpr int GEMM_CONSUMERS = 256;               // two warpgroups
constexpr int GEMM_THREADS = GEMM_CONSUMERS + 128;  // + the producer warpgroup
constexpr int GEMM_PRODUCER_REGS = 40;              // setmaxnreg split of the 64K-register file: 128 x 40 + 256 x 232 <= 65536
constexpr int GEMM_CONSUMER_REGS = 232;
constexpr int GEMM_MAX_BN = 128;                    // 64 fp32 accumulator registers per thread and accumulator
constexpr int GEMM_MAX_STAGES = 8;
constexpr int GEMM_STAGING_BYTES = 8 * 16 * 32 * 4;  // per-consumer-warp 16x32 fp32 transpose buffers (XOR-swizzled)

struct alignas(64) GemmParams {
  CUtensorMap tm_a_hi, tm_a_lo, tm_b_hi, tm_b_lo;  // in mode 2: tm_a_lo = A_lo8, tm_b_lo = B_lo8
  CUtensorMap tm_a_hi8, tm_b_hi8;                    // mode 2 only
  int M, N, K;      // N = accumulator columns (2x the output columns in GLU mode)
  int n_stages;
  int dtype;        // DT_F16 / DT_BF16 (operand and 16-bit output format)
  int epi_prefetch; // 1: consumer warps pull the next tile's residual / multiplier rows into L2 one tile ahead
  int glu;          // 1: out[:, t*bn/2 + c] = act(acc[c]+bias[c]) * (acc[bn/2+c]+bias[bn/2+c]) per tile t
  int act;
  float acc_scale;  // un-scale of pre-scaled packed weights (power of two)
  const float* bias;      // [N] in accumulator-column order, or null
  const float* mul;       // fp32 [M, Nout] multiplier, or null
  int ld_mul;
  const float* residual;  // fp32 [M, Nout], or null
  int ld_res;
  float* out_f32;         // or null
  int ld_o32;
  unsigned short* out_hi; // 16-bit outputs (operand format), or null
  unsigned short* out_lo;
  int ld_o16;
  unsigned char* out_lo8; // fp8 cross-term views of the output (mode-2 consumers), or null
  unsigned char* out_hi8;
  int ld_o8;
  // LayerNorm folded into the GEMM: A holds the un-normalised rows, B holds W*gamma, and the epilogue applies
  //   v = rstd[row] * (acc*acc_scale - mean[row]*ln_c1[col]) + bias[col]        (bias already contains W*beta)
  const float* row_stats;  // fp32 [M, 2] = (mean, rstd), or null
  const float* ln_c1;      // fp32 [N] in accumulator-column order: sum_k (W*gamma)[col, k]
  int ln_cols;             // 1: every accumulator column, 2: only the value half of each GLU tile
  // residual rows LayerNorm'd on the fly: r = (residual - mean[row]) * rstd[row] * res_gamma[col] + res_beta[col]
  const float* res_stats;  // fp32 [M, 2], or null
  const float* res_gamma;  // fp32 [Nout]
  const float* res_beta;
  // per-row partial sums (sum, sum of squares) of the stored output over this (n-tile, epilogue-half)'s columns
  float* stats_out;        // fp32 [M, stats_parts, 2], or null
  int stats_parts;         // = 2 * tiles_n
};

// Compile-time epilogue description. GENERIC: every flag is read from GemmParams at run time instead.
// The kernel's other template parameters: SPLIT (0: hi*hi only, 1: three-term fp16 split product, 2: fp16 hi*hi + two fp8 cross
// terms) and BN (tile width: 32, 64, 96 or 128; 64 or 128 in GLU mode).
template <bool GENERIC_, int ACT_, bool GLU_, bool MUL_, bool RES_, bool O32_, bool O16_, int DT_, bool LNA_ = false, bool LNR_ = false,
          bool STATS_ = false>
struct EpiCfg {
  static constexpr bool GENERIC = GENERIC_;
  static constexpr int ACT = ACT_;
  static constexpr bool GLU = GLU_, MUL = MUL_, RES = RES_, O32 = O32_, O16 = O16_;
  static constexpr int DT = DT_;
  static constexpr bool LNA = LNA_;      // LayerNorm of the A operand folded in (row_stats, ln_c1)
  static constexpr bool LNR = LNR_;      // residual rows LayerNorm'd on the fly (res_stats, res_gamma, res_beta)
  static constexpr bool STATS = STATS_;  // emit per-row partial (sum, sum of squares) of the output
};

constexpr int GEMM_COLVEC_PLANES = 4;  // per buffer: bias | ln_c1 | res_gamma | res_beta, 256 floats each

template <int ACT>
__device__ __forceinline__ float act_ct(float x) {
  if constexpr (ACT == ACT_RELU) return fmaxf(x, 0.f);
  else if constexpr (ACT == ACT_QUICKGELU) return quick_gelu(x);
  else if constexpr (ACT == ACT_GELU) return gelu_erf(x);
  else if constexpr (ACT == ACT_GELU_TANH) return gelu_tanh(x);
  else return x;
}

template <int DT>
__device__ __forceinline__ void split4(const float4& y, uint2& hi, uint2& lo) { split4v<DT>(y, hi, lo); }

// the 8 accumulator values of 16-column group s (columns 16s .. 16s+15) of this thread: in the generic variant the gate half of
// a GLU tile sits at a run-time offset (BN / 2 or not at all), so its group index is only known at run time
template <int BN>
__device__ __forceinline__ void acc_group16(const float (&acc)[BN / 2], int s, float (&v)[8]) {
#pragma unroll
  for (int t = 0; t < BN / 16; ++t)
    if (t == s) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = acc[t * 8 + i];
    }
}

// One accumulator tile, this warp's share: rows [row_base, +16) x every column, in 32-column chunks.  Per chunk: fragment registers
// -> bias/act/GLU -> smem transpose (16 x 32 floats, 16-byte chunks XOR-swizzled by 2 * (row & 3)) -> [4 rows x 8 lanes x float4]
// -> mul / residual / stores.  Each store instruction covers 4 rows of whole 32-byte sectors: a 128-byte line per row of fp32,
// 64 bytes of fp16 and 32 bytes of each e4m3 view.  The multiplier / residual rows of every chunk (NB chunks in the generic variant)
// are requested together before the first chunk is processed, so the tile waits out one L2 round trip instead of one per chunk.
// Row statistics keep the two column halves of the original layout: part 2*tn + ((column / 32) & 1), i.e. the chunk's parity.  The
// even chunks run first, then the odd ones, so each half's sums are complete before the other's start.  The summation tree is that of
// 16-column sub-chunks: per row and 4-column group kc, the sub-chunks of the half in ascending order (columns 4kc.. of a chunk are
// lane c8 = kc, columns 16 + 4kc.. lane kc + 4), then the xor-1 / xor-2 fold over kc.
// acc is the m64nNk16 fragment: element 4*g + e holds column 8*g + 2*(lane % 4) + (e & 1), row 8*(e >> 1) + lane / 4.
template <class E, int BN>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const float (&acc)[BN / 2], const float* __restrict__ sb,
                                              float* __restrict__ st, int lane, int row_base, int tn, int bn_out, int n_out) {
  constexpr int NCH = BN / 32;                                // 32-column chunks (bn_out is a multiple of 32 too)
  constexpr int NEV = (NCH + 1) / 2;                          // even chunks: statistics half 0
  constexpr int NB = E::GENERIC ? (NCH < 2 ? NCH : 2) : NCH;  // chunks whose mul / residual rows are in registers together
  const bool glu = E::GENERIC ? (p.glu != 0) : E::GLU;
  const bool has_mul = E::GENERIC ? (p.mul != nullptr) : E::MUL;
  const bool has_res = E::GENERIC ? (p.residual != nullptr) : E::RES;
  const bool o32 = E::GENERIC ? (p.out_f32 != nullptr) : E::O32;
  const bool o16 = E::GENERIC ? (p.out_hi != nullptr) : E::O16;
  const bool lna = E::GENERIC ? (p.row_stats != nullptr) : E::LNA;
  const bool lnr = E::GENERIC ? (p.res_stats != nullptr) : E::LNR;
  const bool stats = E::GENERIC ? (p.stats_out != nullptr) : E::STATS;
  const float scale = p.acc_scale;
  const int sub = lane >> 2;        // fragment row within a group of 8
  const int kc = lane & 3;          // fragment column pair
  const int rq = lane >> 3;         // transposed layout: row within a group of 4 (rows 4*it + rq)
  const int c8 = lane & 7;          // transposed layout: 4-column group of the chunk
  const float* sc1 = sb + 256;      // ln_c1 tile (accumulator-column order, like the bias tile)
  const float* sgam = sb + 512;     // res_gamma / res_beta tiles (output-column order)
  const float* sbet = sb + 768;
  // folded LayerNorm of the A rows: this thread's fragment rows are row_base + sub + 8*h
  float a_mean[2] = {0.f, 0.f}, a_rstd[2] = {1.f, 1.f};
  if (lna) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row_base + sub + 8 * h;
      if (row < p.M) {
        const float2 ms = __ldg(reinterpret_cast<const float2*>(p.row_stats) + row);
        a_mean[h] = ms.x; a_rstd[h] = ms.y;
      }
    }
  }
  const bool ln_gate = lna && p.ln_cols == 1;
  // on-the-fly LayerNorm of the residual rows / running output statistics of the current half: rows 4*it + rq
  float r_mean[4], r_rstd[4], st1[4], st2[4];
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    r_mean[it] = 0.f; r_rstd[it] = 1.f;
    st1[it] = st2[it] = 0.f;
    if (lnr) {
      const int row = row_base + it * 4 + rq;
      if (row < p.M) {
        const float2 ms = __ldg(reinterpret_cast<const float2*>(p.res_stats) + row);
        r_mean[it] = ms.x; r_rstd[it] = ms.y;
      }
    }
  }
  // fold the (sum, sum of squares) of statistics half hf over the row's four column groups and let lane c8 == 0 write them
  auto flush_stats = [&](int hf) {
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      float s1 = st1[it], s2 = st2[it];
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1); s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 2); s2 += __shfl_xor_sync(0xffffffffu, s2, 2);
      const int row = row_base + it * 4 + rq;
      if (c8 == 0 && row < p.M) reinterpret_cast<float2*>(p.stats_out)[(size_t)row * p.stats_parts + tn * 2 + hf] = make_float2(s1, s2);
      st1[it] = st2[it] = 0.f;
    }
  };
  auto load_mr = [&](int j, float4 (&mm_)[4], float4 (&rr_)[4]) {
    const int col = tn * bn_out + j + c8 * 4;
    const bool col_ok = j < bn_out && col < n_out;
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int row = row_base + it * 4 + rq;
      const bool ok = col_ok && row < p.M;
      if (has_mul) mm_[it] = ok ? __ldg(reinterpret_cast<const float4*>(p.mul + (size_t)row * p.ld_mul + col)) : make_float4(1.f, 1.f, 1.f, 1.f);
      if (has_res) rr_[it] = ok ? __ldg(reinterpret_cast<const float4*>(p.residual + (size_t)row * p.ld_res + col)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto chunk_of = [](int k) { return k < NEV ? 2 * k : 2 * (k - NEV) + 1; };  // processing order: even chunks, then odd ones
  float4 mm[NB][4], rr[NB][4];
  const int wsw = (sub & 3) << 1;  // transpose swizzle of this thread's fragment rows (sub and sub + 8 share it)
  const int rsw = rq << 1;         // and of its transposed rows 4*it + rq
#pragma unroll
  for (int k = 0; k < NCH; ++k) {
    const int c = chunk_of(k);
    const int j = c * 32;
    if (k % NB == 0) {
#pragma unroll
      for (int b = 0; b < NB; ++b)
        if (k + b < NCH) load_mr(chunk_of(k + b) * 32, mm[b], rr[b]);
    }
    if (j < bn_out) {
#pragma unroll
      for (int u = 0; u < 2; ++u) {  // the chunk's two 16-column fragment groups
        const int s = 2 * c + u;
        float v[8], g[8], x[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = acc[s * 8 + i];
        if (glu) acc_group16<BN>(acc, s + bn_out / 16, g);
        // fragment element i: row sub + 8*((i>>1)&1), column 16s + 8*(i>>2) + 2*kc + (i&1)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int cc = s * 16 + 8 * (i >> 2) + 2 * kc + (i & 1);
          const int h = (i >> 1) & 1;
          float a;
          if (lna) a = fmaf(fmaf(-a_mean[h], sc1[cc], v[i] * scale), a_rstd[h], sb[cc]);
          else a = fmaf(v[i], scale, sb[cc]);
          if (glu) {
            float gt;
            if (ln_gate) gt = fmaf(fmaf(-a_mean[h], sc1[bn_out + cc], g[i] * scale), a_rstd[h], sb[bn_out + cc]);
            else gt = fmaf(g[i], scale, sb[bn_out + cc]);
            a = E::GENERIC ? apply_act(p.act, a) : act_ct<E::ACT>(a);
            x[i] = a * gt;
          } else {
            x[i] = E::GENERIC ? apply_act(p.act, a) : act_ct<E::ACT>(a);
          }
        }
#pragma unroll
        for (int q = 0; q < 2; ++q)     // chunk columns 16u + 8q .. +7: 16-byte chunk 4u + 2q + kc/2, float2 at (2*kc) % 4
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = sub + 8 * h;
            const int ch = (4 * u + 2 * q + (kc >> 1)) ^ wsw;
            *reinterpret_cast<float2*>(st + r * 32 + ch * 4 + (2 * kc & 3)) = make_float2(x[4 * q + 2 * h], x[4 * q + 2 * h + 1]);
          }
      }
      __syncwarp();
      float4 y[4];
#pragma unroll
      for (int it = 0; it < 4; ++it) y[it] = *reinterpret_cast<const float4*>(st + (it * 4 + rq) * 32 + ((c8 ^ rsw) << 2));
      const int col = tn * bn_out + j + c8 * 4;
      const bool col_ok = col < n_out;  // n_out % 4 == 0 (checked on the host)
      float4 gm, bt;
      if (lnr) {
        gm = *reinterpret_cast<const float4*>(sgam + j + c8 * 4);
        bt = *reinterpret_cast<const float4*>(sbet + j + c8 * 4);
      }
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int row = row_base + it * 4 + rq;
        float q1 = 0.f, q2 = 0.f;
        if (col_ok && row < p.M) {
          float4 o = y[it];
          if (has_mul) { const float4 m = mm[k % NB][it]; o.x *= m.x; o.y *= m.y; o.z *= m.z; o.w *= m.w; }
          if (has_res) {
            float4 r = rr[k % NB][it];
            if (lnr) {
              const float m_ = r_mean[it], s_ = r_rstd[it];
              r.x = fmaf((r.x - m_) * s_, gm.x, bt.x); r.y = fmaf((r.y - m_) * s_, gm.y, bt.y);
              r.z = fmaf((r.z - m_) * s_, gm.z, bt.z); r.w = fmaf((r.w - m_) * s_, gm.w, bt.w);
            }
            o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
          }
          if (stats) {
            q1 = (o.x + o.y) + (o.z + o.w);
            q2 = fmaf(o.x, o.x, o.y * o.y) + fmaf(o.z, o.z, o.w * o.w);
          }
          if (o32) *reinterpret_cast<float4*>(p.out_f32 + (size_t)row * p.ld_o32 + col) = o;
          if (o16) {
            if (p.out_lo8) {  // fp16 hi + e4m3 cross-term views for an "f16f8" consumer
              uint2 h16;
              uint32_t l8, h8;
              split4_f8(o, F8_ACT_LO_SCALE, F8_ACT_HI_SCALE, h16, l8, h8);
              *reinterpret_cast<uint2*>(p.out_hi + (size_t)row * p.ld_o16 + col) = h16;
              *reinterpret_cast<uint32_t*>(p.out_lo8 + (size_t)row * p.ld_o8 + col) = l8;
              *reinterpret_cast<uint32_t*>(p.out_hi8 + (size_t)row * p.ld_o8 + col) = h8;
            } else {
              uint2 hi, lo;
              if (E::GENERIC) {
                if (p.dtype == DT_F16) split4<DT_F16>(o, hi, lo); else split4<DT_BF16>(o, hi, lo);
              } else {
                split4<E::DT>(o, hi, lo);
              }
              *reinterpret_cast<uint2*>(p.out_hi + (size_t)row * p.ld_o16 + col) = hi;
              if (p.out_lo) *reinterpret_cast<uint2*>(p.out_lo + (size_t)row * p.ld_o16 + col) = lo;
            }
          }
        }
        if (stats) {
          // lanes c8 and c8 ^ 4 hold the two 16-column sub-chunks of this 4-column group; both add them in sub-chunk order.  A
          // column past n_out adds +0, which leaves the sum unchanged (it starts at +0 and so is never -0)
          const float p1 = __shfl_xor_sync(0xffffffffu, q1, 4), p2 = __shfl_xor_sync(0xffffffffu, q2, 4);
          const bool first = c8 < 4;
          st1[it] = (st1[it] + (first ? q1 : p1)) + (first ? p1 : q1);
          st2[it] = (st2[it] + (first ? q2 : p2)) + (first ? p2 : q2);
        }
      }
      __syncwarp();
    }
    if (stats && k == NEV - 1) flush_stats(0);
  }
  if (stats) flush_stats(1);
}

template <class E, int SPLIT, int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
  static_assert(SPLIT >= 0 && SPLIT <= 2 && BN % 32 == 0 && BN <= GEMM_MAX_BN, "gemm_tc_kernel: bad SPLIT / BN");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stages][staging][column vectors 2 x 4 x 256 f32][barriers]
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr int b_tile_bytes = BN * 128;
  constexpr int n_parts = SPLIT ? 2 : 1;  // mode 2: the second "part" holds the two half-size fp8 tiles of each operand
  constexpr int stage_bytes = (GEMM_A_TILE_BYTES + b_tile_bytes) * n_parts;
  uint8_t* stages = smem;
  float* staging = (float*)(smem + (size_t)p.n_stages * stage_bytes);
  float* sbias = staging + GEMM_STAGING_BYTES / 4;  // [2 buffers][GEMM_COLVEC_PLANES][256]
  uint64_t* bars = (uint64_t*)(sbias + 2 * GEMM_COLVEC_PLANES * 256);
  uint64_t* full_bar = bars;                     // [n_stages]
  uint64_t* empty_bar = bars + GEMM_MAX_STAGES;  // [n_stages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int tiles_m = (p.M + GEMM_BM - 1) / GEMM_BM;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int num_kb = (p.K + GEMM_BK - 1) / GEMM_BK;
  const int num_tiles = tiles_m * tiles_n;

  if (threadIdx.x == GEMM_CONSUMERS) {
    tma_prefetch_desc(&p.tm_a_hi);
    tma_prefetch_desc(&p.tm_b_hi);
    if (SPLIT) {
      tma_prefetch_desc(&p.tm_a_lo);
      tma_prefetch_desc(&p.tm_b_lo);
    }
    if (SPLIT == 2) {
      tma_prefetch_desc(&p.tm_a_hi8);
      tma_prefetch_desc(&p.tm_b_hi8);
    }
    for (int s = 0; s < p.n_stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], GEMM_CONSUMERS / 32);  // one arrive per consumer warp once its wgmma reads of the slot retired
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= GEMM_CONSUMERS / 32) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<GEMM_PRODUCER_REGS>();
    if (threadIdx.x == GEMM_CONSUMERS) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / tiles_n) * GEMM_BM;
        const int n0 = (tile % tiles_n) * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* st = stages + (size_t)stage * stage_bytes;
          const int k0 = kb * GEMM_BK;
          uint8_t* sb = st + GEMM_A_TILE_BYTES * n_parts;
          mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)stage_bytes);
          tma_load_2d(st, &p.tm_a_hi, &full_bar[stage], k0, m0);
          tma_load_2d(sb, &p.tm_b_hi, &full_bar[stage], k0, n0);
          if (SPLIT == 1) {
            tma_load_2d(st + GEMM_A_TILE_BYTES, &p.tm_a_lo, &full_bar[stage], k0, m0);
            tma_load_2d(sb + b_tile_bytes, &p.tm_b_lo, &full_bar[stage], k0, n0);
          } else if (SPLIT == 2) {  // [A_lo8 | A_hi8] and [B_hi8 | B_lo8]: 64-byte rows, half the fp16 tile each
            tma_load_2d(st + GEMM_A_TILE_BYTES, &p.tm_a_lo, &full_bar[stage], k0, m0);
            tma_load_2d(st + GEMM_A_TILE_BYTES + GEMM_A_TILE_BYTES / 2, &p.tm_a_hi8, &full_bar[stage], k0, m0);
            tma_load_2d(sb + b_tile_bytes, &p.tm_b_hi8, &full_bar[stage], k0, n0);
            tma_load_2d(sb + b_tile_bytes + b_tile_bytes / 2, &p.tm_b_lo, &full_bar[stage], k0, n0);
          }
          if (++stage == p.n_stages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers: wgmma main loop + epilogue of rows [64*wg, +64) =====================
  setmaxnreg_inc<GEMM_CONSUMER_REGS>();
  const int wg = warp >> 2;
  const int et = threadIdx.x;  // 0..255
  float* st = staging + warp * (16 * 32);
  const bool glu = E::GENERIC ? (p.glu != 0) : E::GLU;
  const int n_out = glu ? p.N / 2 : p.N;
  const int bn_out = glu ? BN / 2 : BN;
  const bool has_mul = E::GENERIC ? (p.mul != nullptr) : E::MUL;
  const bool has_res = E::GENERIC ? (p.residual != nullptr) : E::RES;
  // Pull a tile's multiplier / residual rows into L2 one tile ahead of its epilogue, so the epilogue's 128-bit
  // loads are L2 hits instead of DRAM round trips.
  auto prefetch_tile = [&](int t) {
    if (!p.epi_prefetch || !(has_mul || has_res) || t >= num_tiles) return;
    if (et >= GEMM_BM) return;
    const int row = (t / tiles_n) * GEMM_BM + et;
    if (row >= p.M) return;
    const int c0 = (t % tiles_n) * bn_out;
    for (int c = 0; c < bn_out && c0 + c < n_out; c += 32) {
      if (has_mul) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.mul + (size_t)row * p.ld_mul + c0 + c));
      if (has_res) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.residual + (size_t)row * p.ld_res + c0 + c));
    }
  };
  prefetch_tile(blockIdx.x);
  int stage = 0;
  uint32_t phase = 0;
  int ab = 0;
  const uint32_t a_off = (uint32_t)wg * 64 * 128;  // this warpgroup's 64 rows of the 128-byte-row A tile
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    prefetch_tile(tile + gridDim.x);
    const int m0 = (tile / tiles_n) * GEMM_BM;
    const int tn = tile % tiles_n;
    const int n0 = tn * BN;
    // the e4m3 cross terms get an accumulator of their own: fp8 wgmma adds its products into the accumulator with ~14 bits
    // kept, which would truncate these 2^-11-sized terms against the fp16 sum; their own sum is added in fp32 after the tile
    float acc[BN / 2], acc8[SPLIT == 2 ? BN / 2 : 1];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    if constexpr (SPLIT == 2) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc8[i] = 0.f;
    }
    int prev_stage = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_hi = smem_u32(stages + (size_t)stage * stage_bytes);
      const uint32_t b_hi = a_hi + GEMM_A_TILE_BYTES * n_parts;
      const uint64_t da_hi = wgmma_desc_sw128(a_hi + a_off);
      const uint64_t db_hi = wgmma_desc_sw128(b_hi);
      wgmma_fence();
      // per accumulator element: every hi*hi step of the k block, then lo*hi and hi*lo per k step
#pragma unroll
      for (int k = 0; k < GEMM_BK / 16; ++k)  // +32 B per K=16 step inside the 128 B swizzle row
        wgmma_m64nNk16_ss<E::DT, BN>(acc, da_hi + 2 * k, db_hi + 2 * k, 1u);
      if constexpr (SPLIT == 1) {
        const uint64_t da_lo = wgmma_desc_sw128(a_hi + GEMM_A_TILE_BYTES + a_off);
        const uint64_t db_lo = wgmma_desc_sw128(b_hi + b_tile_bytes);
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k) {
          wgmma_m64nNk16_ss<E::DT, BN>(acc, da_lo + 2 * k, db_hi + 2 * k, 1u);
          wgmma_m64nNk16_ss<E::DT, BN>(acc, da_hi + 2 * k, db_lo + 2 * k, 1u);
        }
      } else if constexpr (SPLIT == 2) {
        // cross terms at the fp8 rate: A_lo8 * B_hi8 and A_hi8 * B_lo8 (e4m3, K = 32 per instruction, 64-byte rows)
        const uint64_t da_lo8 = wgmma_desc_sw64(a_hi + GEMM_A_TILE_BYTES + a_off / 2);
        const uint64_t da_hi8 = wgmma_desc_sw64(a_hi + GEMM_A_TILE_BYTES + GEMM_A_TILE_BYTES / 2 + a_off / 2);
        const uint64_t db_hi8 = wgmma_desc_sw64(b_hi + b_tile_bytes);
        const uint64_t db_lo8 = wgmma_desc_sw64(b_hi + b_tile_bytes + b_tile_bytes / 2);
#pragma unroll
        for (int k = 0; k < GEMM_BK / 32; ++k) {
          wgmma_m64nNk32_e4m3_ss<BN>(acc8, da_lo8 + 2 * k, db_hi8 + 2 * k);
          wgmma_m64nNk32_e4m3_ss<BN>(acc8, da_hi8 + 2 * k, db_lo8 + 2 * k);
        }
      }
      wgmma_commit();
      // keep this k block in flight; the previous one has retired -> its smem slot goes back to the producer
      wgmma_wait<1>();
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == p.n_stages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    if constexpr (SPLIT == 2) {
      wgmma_fence_acc(acc8);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] += acc8[i];
    }
    if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
    // per-column vectors of this tile -> smem (double-buffered: the other buffer may still be read by the slower warpgroup)
    float* sb = sbias + ab * (GEMM_COLVEC_PLANES * 256);
    for (int c = et; c < BN; c += GEMM_CONSUMERS) {
      sb[c] = (p.bias != nullptr && n0 + c < p.N) ? __ldg(p.bias + n0 + c) : 0.f;
      if (E::GENERIC ? (p.row_stats != nullptr) : E::LNA) sb[256 + c] = (n0 + c < p.N) ? __ldg(p.ln_c1 + n0 + c) : 0.f;
      if (E::GENERIC ? (p.res_stats != nullptr) : E::LNR) {
        const int oc = tn * bn_out + c;  // output column (no GLU with a LayerNorm'd residual)
        const bool okc = c < bn_out && oc < n_out;
        sb[512 + c] = okc ? __ldg(p.res_gamma + oc) : 0.f;
        sb[768 + c] = okc ? __ldg(p.res_beta + oc) : 0.f;
      }
    }
    named_bar_sync(1, GEMM_CONSUMERS);
    epilogue_tile<E, BN>(p, acc, sb, st, lane, m0 + wg * 64 + (warp & 3) * 16, tn, bn_out, n_out);
    ab ^= 1;
  }
}

inline size_t gemm_smem_bytes(int block_n, int split, int n_stages) {
  const size_t stage = (size_t)(GEMM_A_TILE_BYTES + block_n * 128) * (split ? 2 : 1);
  return 1024 /*align slack*/ + n_stages * stage + GEMM_STAGING_BYTES + 2 * GEMM_COLVEC_PLANES * 256 * 4 + 2 * GEMM_MAX_STAGES * 8 + 16;
}

}  // namespace vima
