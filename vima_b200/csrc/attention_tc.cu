// wgmma attention for the decoder's hot shapes (head_dim 32, (hi, lo) operand pairs, no relative bias):
//
//   one CTA per (batch, head, 128-query-row tile), two warpgroups of 64 query rows each; keys stream through in chunks of 64.
//   per chunk c, every warpgroup:
//     S[64x64] = Q K^T     6 x wgmma M64 N64 K16 (hi*hi, lo*hi, hi*lo), Q and K(c) from shared memory (TMA, 64-byte swizzle);
//                          K(c+2) is loaded by TMA into the slot K(c) leaves
//     V(c) -> V^T          while S is computed, every thread loads 8 values of V(c) (hi and lo) and writes them transposed into
//                          a 128-byte-swizzled K-major tile, the B operand layout wgmma reads; it also stages chunk c+1's 64
//                          key-mask terms in a double buffer, so no shared memory is sized by Lk (no length cap)
//     softmax              in registers on the accumulator fragment (4 lanes share a row), online maximum, exp2 with the scale
//                          folded into the FMA; P as (hi, lo) 16-bit pairs stays in registers
//     O[64x32] += P V      12 x wgmma M64 N32 K16 with A = P from registers, B = V^T from shared memory
//
// Same mask semantics as attention.cu (reference components.py:51-80): the causal constant is the reference's soft -1e4, key
// padding adds finfo.min, keys beyond Lk are excluded.  A causal tile first runs the chunks up to its diagonal; hidden keys have
// weight exp(-1e4 - m) == 0 exactly in fp32 once m > -1e4 + 104, so stopping there is bit-compatible with the reference's
// full-width softmax.  If some row has only seen padded keys by then (m still <= -9000), the tile is re-run over every chunk
// (rare: the first history slot is always valid in VIMA's data).
#include "kernels.h"

namespace vima {

namespace {

constexpr float FP32_MIN_TC = -3.4028234663852886e38f;
constexpr float LOG2E_TC = 1.4426950408889634f;
constexpr float CAUSAL_L2_TC = -1e4f * LOG2E_TC;
constexpr float EXIT_L2_TC = -9000.f * LOG2E_TC;

constexpr int ATC_THREADS = 256;
constexpr int ATC_BM = 128, ATC_KC = 64, ATC_D = 32;
// shared memory carve (bytes; swizzled tiles 1024-aligned)
constexpr int OFF_QH = 0, OFF_QL = 8192;     // 128 rows x 64 B each
constexpr int OFF_K = 16384;                 // 2 stages x {hi 4096, lo 4096}: 64 keys x 64 B
constexpr int OFF_VT = 32768;                // 2 buffers x {hi 4096, lo 4096}: V^T, 32 dims x 128 B
constexpr int OFF_MASK = 49152;              // float[2][64]: key-mask terms of a chunk
constexpr int OFF_BAR = OFF_MASK + 2 * ATC_KC * 4;  // 3 mbarriers
constexpr int ATC_SMEM = OFF_BAR + 32;

struct AttnTcParams {
  AttnParams a;
  CUtensorMap tm_q_hi, tm_q_lo, tm_k_hi, tm_k_lo;
};

template <int DT>
__global__ void __launch_bounds__(ATC_THREADS, 2) attention_tc_kernel(const __grid_constant__ AttnTcParams P) {
  const AttnParams& p = P.a;
  extern __shared__ __align__(1024) uint8_t sm[];
  float* maskadd = reinterpret_cast<float*>(sm + OFF_MASK);  // [2][64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + OFF_BAR);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;  // [2]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  const int q0 = blockIdx.x * ATC_BM, h = blockIdx.y, b = blockIdx.z;
  const int Lq = p.Lq;
  const int kvb = p.kv_batch_rows ? p.kv_batch_rows : p.Lk;
  const int mld = p.mask_ld ? p.mask_ld : p.Lk;
  const int qbr = p.q_batch_rows ? p.q_batch_rows : Lq;
  int qp0, Lk;  // this batch element's (per-batch with q_pos)
  attn_batch_keys(p, b, qbr, qp0, Lk);
  const uint32_t sbase = smem_u32(sm);
  const int rows_here = min(ATC_BM, Lq - q0);
  const int n_all = (Lk + ATC_KC - 1) / ATC_KC;
  int n_plan = n_all;  // causal: chunks up to the tile's diagonal
  if (p.causal) {
    const int last_key = min(Lk - 1, q0 + rows_here - 1 + qp0);
    n_plan = last_key / ATC_KC + 1;
  }
  const bool may_rerun = p.causal && n_plan < n_all;

  if ((sbase & 1023u) != 0u) {  // the swizzled tiles assume a 1024-byte aligned window (no static shared memory in this kernel)
    if (tid == 0) printf("vima_b200: attention_tc shared memory window is not 1024-byte aligned\n");
    __trap();
  }
  const int x_col = h * ATC_D;  // element column of this head inside the q / k / v row
  const int kv_row0 = b * kvb;
  if (tid == 0) {
    mbar_init(q_full, 1);
    mbar_init(&k_full[0], 1);
    mbar_init(&k_full[1], 1);
    fence_barrier_init();
    tma_prefetch_desc(&P.tm_q_hi); tma_prefetch_desc(&P.tm_q_lo);
    tma_prefetch_desc(&P.tm_k_hi); tma_prefetch_desc(&P.tm_k_lo);
  }
  // chunk c's key-mask terms of this batch element into buffer c & 1 (threads 192..255, one key each)
  auto stage_mask = [&](int c) {
    if (tid >= ATC_THREADS - ATC_KC) {
      const int j = c * ATC_KC + tid - (ATC_THREADS - ATC_KC);
      float mk = -INFINITY;  // beyond the sequence: excluded
      if (j < Lk) mk = (p.key_mask == nullptr || p.key_mask[(size_t)b * mld + j]) ? 0.f : FP32_MIN_TC;
      maskadd[(c & 1) * ATC_KC + tid - (ATC_THREADS - ATC_KC)] = mk;
    }
  };
  stage_mask(0);
  __syncthreads();

  auto load_k = [&](int c, int stage) {  // thread 0 only
    uint8_t* dst = sm + OFF_K + stage * 8192;
    mbar_arrive_expect_tx(&k_full[stage], 8192u);
    tma_load_2d(dst, &P.tm_k_hi, &k_full[stage], x_col, kv_row0 + c * ATC_KC);
    tma_load_2d(dst + 4096, &P.tm_k_lo, &k_full[stage], x_col, kv_row0 + c * ATC_KC);
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(q_full, 16384u);
    tma_load_2d(sm + OFF_QH, &P.tm_q_hi, q_full, x_col, b * qbr + q0);
    tma_load_2d(sm + OFF_QL, &P.tm_q_lo, q_full, x_col, b * qbr + q0);
  }

  // accumulator fragment rows of this thread: r_loc + 8*hh (hh = 0, 1) inside the tile; columns 8*g + 2*qd + (0, 1)
  const int r_loc = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int qd = lane & 3;
  const float c_l2 = p.scale * LOG2E_TC;
  const uint64_t dqh = wgmma_desc_sw64(sbase + OFF_QH + wg * 4096), dql = wgmma_desc_sw64(sbase + OFF_QL + wg * 4096);
  // this thread's share of a V chunk: key vj, dims 8*vd .. 8*vd+7 (hi and lo)
  const int vj = tid >> 2, vd = tid & 3;
  uint32_t k_use[2] = {0u, 0u};  // completed fills of each K stage
  float o[16], m_run[2], l_run[2];
  int n = n_plan;
  for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
    for (int i = 0; i < 16; ++i) o[i] = 0.f;
    m_run[0] = m_run[1] = -INFINITY;
    l_run[0] = l_run[1] = 0.f;
    if (tid == 0) {
      load_k(0, 0);
      if (n > 1) load_k(1, 1);
    }
    if (pass == 0) mbar_wait(q_full, 0);
    for (int c = 0; c < n; ++c) {
      const int stage = c & 1;
      const int k0 = c * ATC_KC;
      mbar_wait(&k_full[stage], k_use[stage] & 1u);
      k_use[stage]++;
      float s[32];
      {
        const uint64_t dkh = wgmma_desc_sw64(sbase + OFF_K + stage * 8192), dkl = wgmma_desc_sw64(sbase + OFF_K + stage * 8192 + 4096);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < ATC_D / 16; ++k) wgmma_m64nNk16_ss<DT, 64>(s, dqh + 2 * k, dkh + 2 * k, (uint32_t)(k != 0));
#pragma unroll
        for (int k = 0; k < ATC_D / 16; ++k) wgmma_m64nNk16_ss<DT, 64>(s, dql + 2 * k, dkh + 2 * k, 1u);
#pragma unroll
        for (int k = 0; k < ATC_D / 16; ++k) wgmma_m64nNk16_ss<DT, 64>(s, dqh + 2 * k, dkl + 2 * k, 1u);
        wgmma_commit();
      }
      // V(c) -> V^T tile (dim n, key k at n*128 + (((k>>3) ^ (n&7)) << 4) + (k&7)*2), while the tensor cores work on S
      {
        uint4 vh = make_uint4(0u, 0u, 0u, 0u), vl = vh;
        if (k0 + vj < Lk) {
          const size_t off = (size_t)(kv_row0 + k0 + vj) * p.ldv + x_col + vd * 8;
          vh = __ldg(reinterpret_cast<const uint4*>(p.v_hi + off));
          vl = __ldg(reinterpret_cast<const uint4*>(p.v_lo + off));
        }
        if (c + 1 < n) stage_mask(c + 1);  // read after the barrier below; buffer (c+1)&1 was last read before the previous one
        uint8_t* vt = sm + OFF_VT + stage * 8192;
        const uint32_t wh[4] = {vh.x, vh.y, vh.z, vh.w}, wl[4] = {vl.x, vl.y, vl.z, vl.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int nn = vd * 8 + e;
          const int off = nn * 128 + ((((vj >> 3) ^ (nn & 7))) << 4) + (vj & 7) * 2;
          *reinterpret_cast<unsigned short*>(vt + off) = (unsigned short)(wh[e >> 1] >> (16 * (e & 1)));
          *reinterpret_cast<unsigned short*>(vt + 4096 + off) = (unsigned short)(wl[e >> 1] >> (16 * (e & 1)));
        }
        fence_proxy_async();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
      }
      wgmma_wait<0>();
      wgmma_fence_acc(s);
      // ---- softmax on the fragment: element 4g+e is row r_loc + 8*(e>>1), key k0 + 8g + 2qd + (e&1) ----
      const float* mk = maskadd + stage * ATC_KC;
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int g = 0; g < 8; ++g)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int jj = 8 * g + 2 * qd + (e & 1), key = k0 + jj;
          const float mm = mk[jj];
          float y = fmaf(s[4 * g + e], c_l2, mm);
          if (p.causal && key > q0 + r_loc + 8 * (e >> 1) + qp0) y = CAUSAL_L2_TC + mm;
          s[4 * g + e] = y;
          mx[e >> 1] = fmaxf(mx[e >> 1], y);
        }
      float f[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
        const float m_new = fmaxf(m_run[hh], mx[hh]);
        f[hh] = ex2_approx(m_run[hh] - m_new);  // 0 on the first chunk (m_run = -inf)
        m_run[hh] = m_new;
      }
      uint32_t ph[16], pl[16];
      float ps[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 16; ++i) {  // pair i = elements 2i, 2i+1: row half (i & 1)
        const int hh = i & 1;
        const float p0 = ex2_approx(s[2 * i] - m_run[hh]), p1 = ex2_approx(s[2 * i + 1] - m_run[hh]);
        ps[hh] += p0 + p1;
        split2<DT>(p0, p1, ph[i], pl[i]);
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) l_run[hh] = l_run[hh] * f[hh] + ps[hh];
#pragma unroll
      for (int i = 0; i < 16; ++i) o[i] *= f[(i >> 1) & 1];
      // V^T(c) and chunk c+1's mask terms are complete, and both warpgroups are done reading K(c): its slot takes K(c+2)
      named_bar_sync(1, ATC_THREADS);
      if (tid == 0 && c + 2 < n) load_k(c + 2, stage);
      {
        const uint64_t dvh = wgmma_desc_sw128(sbase + OFF_VT + stage * 8192), dvl = wgmma_desc_sw128(sbase + OFF_VT + stage * 8192 + 4096);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < ATC_KC / 16; ++kk) {  // A fragment of keys [16kk, +16): pairs 4kk .. 4kk+3
          const uint32_t ah[4] = {ph[4 * kk], ph[4 * kk + 1], ph[4 * kk + 2], ph[4 * kk + 3]};
          const uint32_t al[4] = {pl[4 * kk], pl[4 * kk + 1], pl[4 * kk + 2], pl[4 * kk + 3]};
          wgmma_m64n32k16_rs<DT>(o, ah, dvh + 2 * kk, 1u);
          wgmma_m64n32k16_rs<DT>(o, al, dvh + 2 * kk, 1u);
          wgmma_m64n32k16_rs<DT>(o, ah, dvl + 2 * kk, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(o);
      }
    }
    // every row past the causal range must have seen a valid key; otherwise the whole tile is redone over all chunks
    if (pass == 1 || !may_rerun) break;
    const int undone = (r_loc < rows_here && !(m_run[0] > EXIT_L2_TC)) || (r_loc + 8 < rows_here && !(m_run[1] > EXIT_L2_TC));
    if (!__syncthreads_or(undone)) break;
    n = n_all;
    stage_mask(0);  // every read of pass 0's mask buffers precedes the barrier above
    __syncthreads();
  }
  // ---- normalise and store (hi, lo) [+ e4m3 views] ----
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float l = l_run[hh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int row = q0 + r_loc + 8 * hh;
    if (row < Lq) {
      const float inv = 1.0f / l;
      const size_t brow = (size_t)b * qbr + row;
#pragma unroll
      for (int g = 0; g < 4; ++g) attn_store_pair<DT>(p, brow, x_col + 8 * g + 2 * qd, o[4 * g + 2 * hh] * inv, o[4 * g + 2 * hh + 1] * inv);
    }
  }
}

typedef CUresult (*PFN_encodeTiled_attn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                         const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                         CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// [rows, H*32] 16-bit view of one operand (row pitch ld elements), boxes of box_rows x 32 elements (64 bytes), 64B swizzle
static bool make_map(void* encode, CUtensorMap* tm, const void* base, int dtype, long long rows, int cols, int ld, int box_rows) {
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {(cuuint32_t)ATC_D, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = dtype == DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  return ((PFN_encodeTiled_attn)encode)(tm, dt, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                        CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

// Shapes this kernel takes (everything else stays on the mma.sync kernel of attention.cu).
bool attention_tc_supported(const AttnParams& p) {
  const int kvb = p.kv_batch_rows ? p.kv_batch_rows : p.Lk;  // TMA row coordinates of K and Q are 32-bit
  const int qbr = p.q_batch_rows ? p.q_batch_rows : p.Lq;
  auto al = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
  if (!(al(p.q_hi) && al(p.q_lo) && al(p.k_hi) && al(p.k_lo) && al(p.v_hi) && al(p.v_lo) && al(p.o_hi) && al(p.o_lo) && al(p.o_lo8) && al(p.o_hi8)))
    return false;
  return p.D == 32 && p.split != 0 && p.rel_bias == nullptr && p.q_lo && p.k_lo && p.v_lo && (p.ldq % 8 == 0) && (p.ldk % 8 == 0) &&
         (p.ldv % 8 == 0) && (p.ldo % 8 == 0) && (p.o_lo8 == nullptr || p.ldo8 % 8 == 0) && p.H <= 65535 && p.B <= 65535 && p.Lk >= 1 &&
         (long long)p.B * kvb <= 0x7fffffffll && (long long)p.B * qbr <= 0x7fffffffll;
}

cudaError_t launch_attention_tc(const AttnParams& p, void* encode_fn, cudaStream_t stream) {
  if (p.B == 0 || p.Lq == 0) return cudaSuccess;
  AttnTcParams P;
  P.a = p;
  const int kvb = p.kv_batch_rows ? p.kv_batch_rows : p.Lk;
  const int qbr = p.q_batch_rows ? p.q_batch_rows : p.Lq;
  const int cols = p.H * ATC_D;
  bool ok = make_map(encode_fn, &P.tm_q_hi, p.q_hi, p.dtype, (long long)p.B * qbr, cols, p.ldq, ATC_BM) &&
            make_map(encode_fn, &P.tm_q_lo, p.q_lo, p.dtype, (long long)p.B * qbr, cols, p.ldq, ATC_BM) &&
            make_map(encode_fn, &P.tm_k_hi, p.k_hi, p.dtype, (long long)p.B * kvb, cols, p.ldk, ATC_KC) &&
            make_map(encode_fn, &P.tm_k_lo, p.k_lo, p.dtype, (long long)p.B * kvb, cols, p.ldk, ATC_KC);
  if (!ok) return cudaErrorInvalidValue;
  dim3 grid((p.Lq + ATC_BM - 1) / ATC_BM, p.H, p.B);
  const size_t smem = ATC_SMEM;
  static bool attr_set[2][64] = {};  // once per (format, device): not legal inside a CUDA-graph capture
  int dev = 0;
  cudaGetDevice(&dev);
  const int fi = p.dtype == DT_BF16 ? 1 : 0;
  if (!attr_set[fi][dev & 63]) {
    cudaError_t e = fi ? cudaFuncSetAttribute(attention_tc_kernel<DT_BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                       : cudaFuncSetAttribute(attention_tc_kernel<DT_F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr_set[fi][dev & 63] = true;
  }
  if (fi) attention_tc_kernel<DT_BF16><<<grid, ATC_THREADS, smem, stream>>>(P);
  else attention_tc_kernel<DT_F16><<<grid, ATC_THREADS, smem, stream>>>(P);
  return cudaGetLastError();
}

}  // namespace vima
