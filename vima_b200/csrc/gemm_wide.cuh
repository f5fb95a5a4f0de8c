// Wide-tile wgmma GEMM for the "f16f8" split mode on sm_90a:  C[M,N] = epilogue( A[M,K] * B[N,K]^T ), 128 x 256 tiles.
//
// gemm_tc_kernel's f16f8 tile (128 x 128 x 64) loads 64 KB of operands per 1 M multiply-adds; this kernel's 128 x 256 x 64 tile
// loads 96 KB per 2 M, a quarter less operand traffic from L2, in the same row formats (128-byte fp16 rows, 64-byte e4m3 rows).
//
//  * Registers.  Each consumer warpgroup holds the fp32 hi*hi accumulator of its 64 x 256 block (128 registers) and the e4m3
//    cross terms in an fp16 accumulator (m64n256k32.f16.e4m3.e4m3: 64 f16x2 registers): 192 of the 232 that setmaxnreg gives.
//    A second fp32 accumulator would need 256.  The cross terms are ~2^-11 of the product and their e4m3 views already limit
//    them to ~2^-4 relative, so an fp16 sum (~2^-11 relative to them) adds ~2^-22 of the result.  The hi*hi sum is the fp32
//    accumulation of gemm_tc_kernel, in the same ascending K16 order.  acc8 is folded into acc in fp32 at the end of the tile.
//  * Shared memory.  A whole 128 x 256 x 64 k block is 96 KB: only two would fit, the consumers would hold both (one computing,
//    one in flight), and one load at a time cannot cover the L2 latency (measured at 0.98-1.26x the 128-wide kernel's time).
//    So each k block travels as two 48 KB half-blocks in a ring of four: the fp16 half in the even slots, the e4m3 half in the
//    odd ones, up to three loads in flight while one half-block computes.
//      even slot: A hi16 [128 x 128 B, 128-byte swizzle] | B hi16 [256 x 128 B]
//      odd slot:  A lo8 [128 x 64 B, 64-byte swizzle] | A hi8 [128 x 64 B] | B hi8 [256 x 64 B] | B lo8 [256 x 64 B]
//    (gemm_tc_kernel's layouts; the tensor maps differ only in the B box height).  Per k block each consumer warpgroup issues
//    4 x m64n256k16 (fp16) on the even slot and 4 x m64n256k32 (e4m3, two per cross term) on the odd one, each half-block its own
//    commit group, so the slot of the half-block before it is released one half-block later.
//  * Producer / consumer protocol, persistent n-fastest tile order and the epilogue are gemm_tc_kernel's: a 256-wide tile is two
//    adjacent 128-wide tiles of the 128-wide kernel (same GLU value | gate pairing, row-statistics parts and packed weights), so
//    the epilogue runs epilogue_tile<E, 128> on each half.
#pragma once
#include "gemm_tc_variants.cuh"

namespace vima {

constexpr int GEMM_WIDE_BN = 256;
constexpr int GEMM_WIDE_A16 = GEMM_BM * GEMM_BK * 2;       // 16 KB
constexpr int GEMM_WIDE_A8 = GEMM_BM * GEMM_BK;            // 8 KB per e4m3 view
constexpr int GEMM_WIDE_B16 = GEMM_WIDE_BN * GEMM_BK * 2;  // 32 KB
constexpr int GEMM_WIDE_B8 = GEMM_WIDE_BN * GEMM_BK;       // 16 KB per e4m3 view
constexpr int GEMM_WIDE_STAGE_BYTES = GEMM_WIDE_A16 + GEMM_WIDE_B16;  // 48 KB = 2 x A8 + 2 x B8
static_assert(GEMM_WIDE_STAGE_BYTES == 2 * GEMM_WIDE_A8 + 2 * GEMM_WIDE_B8, "the fp16 and the e4m3 half-blocks fill a slot each");
constexpr int GEMM_WIDE_STAGES = 4;  // two k blocks

#define VIMA_R128                                                                                                                  \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, "  \
  "%27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, "   \
  "%52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, "   \
  "%77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, " \
  "%102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, "  \
  "%123, %124, %125, %126, %127}"
#define VIMA_U8(d, o)                                                                                                           \
  "+r"(d[(o) + 0]), "+r"(d[(o) + 1]), "+r"(d[(o) + 2]), "+r"(d[(o) + 3]), "+r"(d[(o) + 4]), "+r"(d[(o) + 5]), "+r"(d[(o) + 6]), \
      "+r"(d[(o) + 7])
#define VIMA_U64(d) VIMA_U8(d, 0), VIMA_U8(d, 8), VIMA_U8(d, 16), VIMA_U8(d, 24), VIMA_U8(d, 32), VIMA_U8(d, 40), VIMA_U8(d, 48), VIMA_U8(d, 56)

// fp16 operands, K-major in shared memory: M64 N256 K16 into fp32.  d0 holds accumulator columns 0-127 (the m64n128 fragment of
// those columns), d1 columns 128-255.
__device__ __forceinline__ void wgmma_m64n256k16_f16(float (&d0)[64], float (&d1)[64], uint64_t da, uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " VIMA_R128 ", %128, %129, 1, 1, 1, 0, 0;"
               : VIMA_ACC64(d0), VIMA_ACC64(d1)
               : "l"(da), "l"(db));
}
// e4m3 operands, K-major in shared memory: M64 N256 K32 into fp16.  Register r holds the (low, high) f16 pair of fp32-fragment
// elements 2r and 2r + 1.
__device__ __forceinline__ void wgmma_m64n256k32_e4m3_f16(uint32_t (&d)[64], uint64_t da, uint64_t db) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n256k32.f16.e4m3.e4m3 " VIMA_R64 ", %64, %65, 1, 1, 1;"
               : VIMA_U64(d)
               : "l"(da), "l"(db));
}
#undef VIMA_U64
#undef VIMA_U8
#undef VIMA_R128

template <int N>
__device__ __forceinline__ void wgmma_fence_acc(uint32_t (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

template <class E>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_wide_kernel(const __grid_constant__ GemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stages][staging][column vectors 2 x 4 x 256 f32][barriers]
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr int BN = GEMM_WIDE_BN;
  constexpr int off_b16 = GEMM_WIDE_A16;  // even slot
  constexpr int off_a_hi8 = GEMM_WIDE_A8, off_b_hi8 = 2 * GEMM_WIDE_A8, off_b_lo8 = off_b_hi8 + GEMM_WIDE_B8;  // odd slot (A lo8 at 0)
  uint8_t* stages = smem;
  float* staging = (float*)(smem + GEMM_WIDE_STAGES * GEMM_WIDE_STAGE_BYTES);
  float* sbias = staging + GEMM_STAGING_BYTES / 4;  // [2 buffers][GEMM_COLVEC_PLANES][256]
  uint64_t* bars = (uint64_t*)(sbias + 2 * GEMM_COLVEC_PLANES * 256);
  uint64_t* full_bar = bars;                      // [GEMM_WIDE_STAGES]
  uint64_t* empty_bar = bars + GEMM_WIDE_STAGES;  // [GEMM_WIDE_STAGES]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int tiles_m = (p.M + GEMM_BM - 1) / GEMM_BM;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int num_kb = (p.K + GEMM_BK - 1) / GEMM_BK;
  const int num_tiles = tiles_m * tiles_n;

  if (threadIdx.x == GEMM_CONSUMERS) {
    tma_prefetch_desc(&p.tm_a_hi);
    tma_prefetch_desc(&p.tm_b_hi);
    tma_prefetch_desc(&p.tm_a_lo);
    tma_prefetch_desc(&p.tm_b_lo);
    tma_prefetch_desc(&p.tm_a_hi8);
    tma_prefetch_desc(&p.tm_b_hi8);
    for (int s = 0; s < GEMM_WIDE_STAGES; ++s) {
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
      int pair = 0;  // slots 2 * pair (fp16) and 2 * pair + 1 (e4m3)
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / tiles_n) * GEMM_BM;
        const int n0 = (tile % tiles_n) * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          const int k0 = kb * GEMM_BK;
          const int s16 = 2 * pair, s8 = 2 * pair + 1;
          uint8_t* st16 = stages + (size_t)s16 * GEMM_WIDE_STAGE_BYTES;
          uint8_t* st8 = stages + (size_t)s8 * GEMM_WIDE_STAGE_BYTES;
          mbar_wait(&empty_bar[s16], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[s16], (uint32_t)GEMM_WIDE_STAGE_BYTES);
          tma_load_2d(st16, &p.tm_a_hi, &full_bar[s16], k0, m0);
          tma_load_2d(st16 + off_b16, &p.tm_b_hi, &full_bar[s16], k0, n0);
          mbar_wait(&empty_bar[s8], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[s8], (uint32_t)GEMM_WIDE_STAGE_BYTES);
          tma_load_2d(st8, &p.tm_a_lo, &full_bar[s8], k0, m0);
          tma_load_2d(st8 + off_a_hi8, &p.tm_a_hi8, &full_bar[s8], k0, m0);
          tma_load_2d(st8 + off_b_hi8, &p.tm_b_hi8, &full_bar[s8], k0, n0);
          tma_load_2d(st8 + off_b_lo8, &p.tm_b_lo, &full_bar[s8], k0, n0);
          pair ^= 1;
          if (pair == 0) phase ^= 1;
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
  auto prefetch_tile = [&](int t) {  // gemm_tc_kernel's L2 prefetch of the next tile's multiplier / residual rows
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
  int pair = 0;
  uint32_t phase = 0;
  int ab = 0;
  const uint32_t a16_off = (uint32_t)wg * 64 * (GEMM_BK * 2);  // this warpgroup's 64 rows of the A tiles
  const uint32_t a8_off = (uint32_t)wg * 64 * GEMM_BK;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    prefetch_tile(tile + gridDim.x);
    const int m0 = (tile / tiles_n) * GEMM_BM;
    const int tn = tile % tiles_n;
    const int n0 = tn * BN;
    float acc0[64], acc1[64];  // columns [0, 128) and [128, 256) of the tile
    uint32_t acc8[64];         // e4m3 cross terms, f16x2
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; acc8[i] = 0u; }
    int prev_stage = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      const int s16 = 2 * pair, s8 = 2 * pair + 1;
      // fp16 half-block: every hi*hi step of the k block
      mbar_wait(&full_bar[s16], phase);
      const uint32_t b16 = smem_u32(stages + (size_t)s16 * GEMM_WIDE_STAGE_BYTES);
      const uint64_t da_hi = wgmma_desc_sw128(b16 + a16_off);
      const uint64_t db_hi = wgmma_desc_sw128(b16 + off_b16);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < GEMM_BK / 16; ++k)  // +32 B per K=16 step inside the 128 B swizzle row
        wgmma_m64n256k16_f16(acc0, acc1, da_hi + 2 * k, db_hi + 2 * k);
      wgmma_commit();
      // keep this half-block in flight; the previous one has retired -> its slot goes back to the producer
      wgmma_wait<1>();
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      // e4m3 half-block: the cross terms A_lo8 * B_hi8 and A_hi8 * B_lo8 (K = 32 per instruction, 64-byte rows)
      mbar_wait(&full_bar[s8], phase);
      const uint32_t b8 = smem_u32(stages + (size_t)s8 * GEMM_WIDE_STAGE_BYTES);
      const uint64_t da_lo8 = wgmma_desc_sw64(b8 + a8_off), db_hi8 = wgmma_desc_sw64(b8 + off_b_hi8);
      const uint64_t da_hi8 = wgmma_desc_sw64(b8 + off_a_hi8 + a8_off), db_lo8 = wgmma_desc_sw64(b8 + off_b_lo8);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < GEMM_BK / 32; ++k) {
        wgmma_m64n256k32_e4m3_f16(acc8, da_lo8 + 2 * k, db_hi8 + 2 * k);
        wgmma_m64n256k32_e4m3_f16(acc8, da_hi8 + 2 * k, db_lo8 + 2 * k);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (lane == 0) mbar_arrive(&empty_bar[s16]);
      prev_stage = s8;
      pair ^= 1;
      if (pair == 0) phase ^= 1;
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc0);
    wgmma_fence_acc(acc1);
    wgmma_fence_acc(acc8);
#pragma unroll
    for (int r = 0; r < 32; ++r) {
      const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&acc8[r]));
      const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&acc8[32 + r]));
      acc0[2 * r] += lo.x; acc0[2 * r + 1] += lo.y;
      acc1[2 * r] += hi.x; acc1[2 * r + 1] += hi.y;
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
    // the two 128-wide halves: every column-vector plane is 256 wide, so the second half's planes start 128 further on
    const int row_base = m0 + wg * 64 + (warp & 3) * 16;
    epilogue_tile<E, 128>(p, acc0, sb, st, lane, row_base, 2 * tn, bn_out / 2, n_out);
    epilogue_tile<E, 128>(p, acc1, sb + 128, st, lane, row_base, 2 * tn + 1, bn_out / 2, n_out);
    ab ^= 1;
  }
}

constexpr size_t gemm_wide_smem_bytes() {
  return 1024 /*align slack*/ + (size_t)GEMM_WIDE_STAGES * GEMM_WIDE_STAGE_BYTES + GEMM_STAGING_BYTES + 2 * GEMM_COLVEC_PLANES * 256 * 4 +
         2 * GEMM_WIDE_STAGES * 8 + 16;
}

// Whether l's epilogue is one of VIMA_GEMM_VARIANTS, the ones gemm_wide_kernel is instantiated for.
bool gemm_wide_has_epilogue(const GemmLaunch& l);
// Launches gemm_wide_kernel with the epilogue specialisation of l (cudaErrorInvalidValue if it has none).
cudaError_t launch_gemm_wide(const GemmParams& p, const GemmLaunch& l, int grid, size_t smem, int max_smem, cudaStream_t stream);

}  // namespace vima
