// wgmma attention for the T5 prompt encoder (head_dim 64, T5 relative-position bias, key padding mask, non-causal, Lq == Lk):
//
//   one CTA per (batch, head, 128-query-row tile), two warpgroups of 64 query rows each; keys stream through in chunks of 64, so the
//   sequence length has no cap (attention.cu keeps K and V^T of a whole (batch, head) in shared memory: Lk <= 384 with split operands).
//   per chunk c, every warpgroup:
//     S[64x64] = Q K^T     wgmma M64 N64 K16 (hi*hi, lo*hi, hi*lo with split operands, hi*hi alone without), Q and K(c) from shared
//                          memory (TMA, 128-byte swizzle); K(c+2) is loaded by TMA into the slot K(c) leaves
//     V(c) -> V^T          while S is computed, every thread loads 16 values of V(c) (hi and lo) and writes them transposed into a
//                          128-byte-swizzled K-major tile, the B operand layout wgmma reads; it also stages chunk c+1's key-mask terms
//                          and the 191 bias values that (tile, chunk c+1) can index
//     softmax              in registers on the accumulator fragment (4 lanes share a row), online maximum, exp2; P as 16-bit
//                          (hi, lo) pairs stays in registers
//     O[64x64] += P V      wgmma M64 N64 K16 with A = P from registers, B = V^T from shared memory
//
// Scores follow attention.cu's formula in the log2 domain: y = s * scale*log2e + bias[h][j - i + Lk - 1]*log2e, then + finfo(fp32).min
// for a padded key (a row whose keys are all padded gets the reference's uniform average) and -inf for a key past Lk.
#include "kernels.h"

namespace vima {

namespace {

constexpr float FP32_MIN_BT = -3.4028234663852886e38f;
constexpr float LOG2E_BT = 1.4426950408889634f;

constexpr int ABT_THREADS = 256;
constexpr int ABT_BM = 128, ABT_KC = 64, ABT_D = 64;
constexpr int ABT_WIN = ABT_BM + ABT_KC - 1;  // offsets j - i one (tile, chunk) pair can see: [k0 - q0 - 127, k0 - q0 + 63]
// shared memory carve (bytes; swizzled tiles 1024-aligned).  The lo halves stay reserved in single-pass mode: one carve for both.
constexpr int OFF_QH = 0, OFF_QL = 16384;   // 128 rows x 128 B each
constexpr int OFF_K = 32768;                // 2 stages x {hi 8192, lo 8192}: 64 keys x 128 B
constexpr int OFF_VT = 65536;               // 2 buffers x {hi 8192, lo 8192}: V^T, 64 dims x 128 B
constexpr int OFF_MASK = 98304;             // float[2][64]: key-mask terms of a chunk
constexpr int OFF_BIAS = OFF_MASK + 2 * ABT_KC * 4;  // float[2][192]: bias window of a (tile, chunk) pair, log2 domain
constexpr int OFF_BAR = OFF_BIAS + 2 * 192 * 4;      // 3 mbarriers
constexpr int ABT_SMEM = OFF_BAR + 32;

struct AttnBiasTcParams {
  AttnParams a;
  CUtensorMap tm_q_hi, tm_q_lo, tm_k_hi, tm_k_lo;
};

template <int DT, bool SPLIT>
__global__ void __launch_bounds__(ABT_THREADS, 2) attention_bias_tc_kernel(const __grid_constant__ AttnBiasTcParams P) {
  constexpr int PARTS = SPLIT ? 2 : 1;
  const AttnParams& p = P.a;
  extern __shared__ __align__(1024) uint8_t sm[];
  float* maskadd = reinterpret_cast<float*>(sm + OFF_MASK);  // [2][64]
  float* sbias = reinterpret_cast<float*>(sm + OFF_BIAS);    // [2][192]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + OFF_BAR);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;  // [2]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  const int q0 = blockIdx.x * ABT_BM, h = blockIdx.y, b = blockIdx.z;
  const int Lq = p.Lq, Lk = p.Lk;
  const uint32_t sbase = smem_u32(sm);
  const int n = (Lk + ABT_KC - 1) / ABT_KC;

  if ((sbase & 1023u) != 0u) __trap();  // the swizzled tiles assume a 1024-byte aligned window (no static shared memory here)
  const int x_col = h * ABT_D;  // element column of this head inside the q / k / v row
  const int kv_row0 = b * Lk;
  const float* bias_row = p.rel_bias + (size_t)h * (2 * Lk - 1);
  if (tid == 0) {
    mbar_init(q_full, 1);
    mbar_init(&k_full[0], 1);
    mbar_init(&k_full[1], 1);
    fence_barrier_init();
    tma_prefetch_desc(&P.tm_q_hi); tma_prefetch_desc(&P.tm_k_hi);
    if (SPLIT) { tma_prefetch_desc(&P.tm_q_lo); tma_prefetch_desc(&P.tm_k_lo); }
  }
  // chunk c's key-mask terms (threads 192..255) and bias window (threads 0..190) into buffer c & 1; one value per thread
  auto stage_chunk = [&](int c) {
    const int k0 = c * ABT_KC;
    if (tid >= 192) {
      const int j = k0 + tid - 192;
      float mk = -INFINITY;  // beyond the sequence: excluded
      if (j < Lk) mk = (p.key_mask == nullptr || p.key_mask[(size_t)b * Lk + j]) ? 0.f : FP32_MIN_BT;
      maskadd[(c & 1) * ABT_KC + tid - 192] = mk;
    } else if (tid < ABT_WIN) {
      const long long t = (long long)k0 - q0 - (ABT_BM - 1) + tid + Lk - 1;  // table index of offset j - i = k0 - q0 - 127 + tid
      sbias[(c & 1) * 192 + tid] = (t >= 0 && t < 2ll * Lk - 1) ? __ldg(bias_row + t) * LOG2E_BT : 0.f;
    }
  };
  stage_chunk(0);
  __syncthreads();

  auto load_k = [&](int c, int stage) {  // thread 0 only
    uint8_t* dst = sm + OFF_K + stage * 16384;
    mbar_arrive_expect_tx(&k_full[stage], 8192u * PARTS);
    tma_load_2d(dst, &P.tm_k_hi, &k_full[stage], x_col, kv_row0 + c * ABT_KC);
    if (SPLIT) tma_load_2d(dst + 8192, &P.tm_k_lo, &k_full[stage], x_col, kv_row0 + c * ABT_KC);
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(q_full, 16384u * PARTS);
    tma_load_2d(sm + OFF_QH, &P.tm_q_hi, q_full, x_col, b * Lq + q0);
    if (SPLIT) tma_load_2d(sm + OFF_QL, &P.tm_q_lo, q_full, x_col, b * Lq + q0);
    load_k(0, 0);
    if (n > 1) load_k(1, 1);
  }

  // accumulator fragment rows of this thread: r_loc + 8*hh (hh = 0, 1) inside the tile; columns 8*g + 2*qd + (0, 1)
  const int r_loc = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int qd = lane & 3;
  const float c_l2 = p.scale * LOG2E_BT;
  const uint64_t dqh = wgmma_desc_sw128(sbase + OFF_QH + wg * 8192), dql = wgmma_desc_sw128(sbase + OFF_QL + wg * 8192);
  // this thread's share of a V chunk: key vj, dims 16*vd .. 16*vd+15 (hi and lo)
  const int vj = tid >> 2, vd = tid & 3;
  float o[32], m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  mbar_wait(q_full, 0);
  for (int c = 0; c < n; ++c) {
    const int stage = c & 1;
    const int k0 = c * ABT_KC;
    mbar_wait(&k_full[stage], (c >> 1) & 1);
    float s[32];
    {
      const uint64_t dkh = wgmma_desc_sw128(sbase + OFF_K + stage * 16384), dkl = wgmma_desc_sw128(sbase + OFF_K + stage * 16384 + 8192);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < ABT_D / 16; ++k) wgmma_m64nNk16_ss<DT, 64>(s, dqh + 2 * k, dkh + 2 * k, (uint32_t)(k != 0));
      if constexpr (SPLIT) {
#pragma unroll
        for (int k = 0; k < ABT_D / 16; ++k) wgmma_m64nNk16_ss<DT, 64>(s, dql + 2 * k, dkh + 2 * k, 1u);
#pragma unroll
        for (int k = 0; k < ABT_D / 16; ++k) wgmma_m64nNk16_ss<DT, 64>(s, dqh + 2 * k, dkl + 2 * k, 1u);
      }
      wgmma_commit();
    }
    // V(c) -> V^T tile (dim nn, key k at nn*128 + (((k>>3) ^ (nn&7)) << 4) + (k&7)*2), while the tensor cores work on S
    {
      uint4 v[2 * PARTS];
#pragma unroll
      for (int i = 0; i < 2 * PARTS; ++i) v[i] = make_uint4(0u, 0u, 0u, 0u);
      if (k0 + vj < Lk) {
        const size_t off = (size_t)(kv_row0 + k0 + vj) * p.ldv + x_col + vd * 16;
        v[0] = __ldg(reinterpret_cast<const uint4*>(p.v_hi + off));
        v[1] = __ldg(reinterpret_cast<const uint4*>(p.v_hi + off + 8));
        if constexpr (SPLIT) {
          v[2] = __ldg(reinterpret_cast<const uint4*>(p.v_lo + off));
          v[3] = __ldg(reinterpret_cast<const uint4*>(p.v_lo + off + 8));
        }
      }
      if (c + 1 < n) stage_chunk(c + 1);  // read after the barrier below; buffer (c+1)&1 was last read before the previous one
      uint8_t* vt = sm + OFF_VT + stage * 16384;
#pragma unroll
      for (int part = 0; part < PARTS; ++part) {
        const uint32_t w[8] = {v[2 * part].x, v[2 * part].y, v[2 * part].z, v[2 * part].w,
                               v[2 * part + 1].x, v[2 * part + 1].y, v[2 * part + 1].z, v[2 * part + 1].w};
#pragma unroll
        for (int e = 0; e < 16; ++e) {
          const int nn = vd * 16 + e;
          const int off = nn * 128 + ((((vj >> 3) ^ (nn & 7))) << 4) + (vj & 7) * 2;
          *reinterpret_cast<unsigned short*>(vt + part * 8192 + off) = (unsigned short)(w[e >> 1] >> (16 * (e & 1)));
        }
      }
      fence_proxy_async();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
    }
    wgmma_wait<0>();
    wgmma_fence_acc(s);
    // ---- softmax on the fragment: element 4g+e is row r_loc + 8*(e>>1), key k0 + 8g + 2qd + (e&1) ----
    const float* mk = maskadd + stage * ABT_KC;
    const float* bw = sbias + stage * 192 + (ABT_BM - 1) - r_loc;  // bw[jj - 8*hh] = bias of (row r_loc + 8*hh, key k0 + jj)
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int g = 0; g < 8; ++g)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int jj = 8 * g + 2 * qd + (e & 1);
        float y = s[4 * g + e] * c_l2;
        y += bw[jj - 8 * (e >> 1)];
        y += mk[jj];
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
    for (int i = 0; i < 32; ++i) o[i] *= f[(i >> 1) & 1];
    // V^T(c) and chunk c+1's mask / bias are complete, and both warpgroups are done reading K(c): its slot takes K(c+2)
    named_bar_sync(1, ABT_THREADS);
    if (tid == 0 && c + 2 < n) load_k(c + 2, stage);
    {
      const uint64_t dvh = wgmma_desc_sw128(sbase + OFF_VT + stage * 16384), dvl = wgmma_desc_sw128(sbase + OFF_VT + stage * 16384 + 8192);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < ABT_KC / 16; ++kk) {  // A fragment of keys [16kk, +16): pairs 4kk .. 4kk+3
        const uint32_t ah[4] = {ph[4 * kk], ph[4 * kk + 1], ph[4 * kk + 2], ph[4 * kk + 3]};
        wgmma_m64n64k16_rs<DT>(o, ah, dvh + 2 * kk, 1u);
        if constexpr (SPLIT) {
          const uint32_t al[4] = {pl[4 * kk], pl[4 * kk + 1], pl[4 * kk + 2], pl[4 * kk + 3]};
          wgmma_m64n64k16_rs<DT>(o, al, dvh + 2 * kk, 1u);
          wgmma_m64n64k16_rs<DT>(o, ah, dvl + 2 * kk, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(o);
    }
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
      const size_t brow = (size_t)b * Lq + row;
#pragma unroll
      for (int g = 0; g < 8; ++g) attn_store_pair<DT>(p, brow, x_col + 8 * g + 2 * qd, o[4 * g + 2 * hh] * inv, o[4 * g + 2 * hh + 1] * inv);
    }
  }
}

typedef CUresult (*PFN_encodeTiled_attn_bias)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// [rows, H*64] 16-bit view of one operand (row pitch ld elements), boxes of box_rows x 64 elements (128 bytes), 128B swizzle
static bool make_map(void* encode, CUtensorMap* tm, const void* base, int dtype, long long rows, int cols, int ld, int box_rows) {
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {(cuuint32_t)ABT_D, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = dtype == DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  return ((PFN_encodeTiled_attn_bias)encode)(tm, dt, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int DT, bool SPLIT>
cudaError_t launch_t(const AttnBiasTcParams& P, dim3 grid, cudaStream_t stream) {
  auto kern = attention_bias_tc_kernel<DT, SPLIT>;
  static bool attr_set[64] = {};  // once per device: not legal inside a CUDA-graph capture
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_set[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, ABT_SMEM);
    if (e != cudaSuccess) return e;
    attr_set[dev & 63] = true;
  }
  kern<<<grid, ABT_THREADS, ABT_SMEM, stream>>>(P);
  return cudaGetLastError();
}

}  // namespace

// Shapes this kernel takes: the T5 encoder's self-attention.  Operand rows and the per-batch key count are the plain [B*L, ld] layout.
bool attention_bias_tc_supported(const AttnParams& p) {
  auto al = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
  if (!(al(p.q_hi) && al(p.q_lo) && al(p.k_hi) && al(p.k_lo) && al(p.v_hi) && al(p.v_lo) && al(p.o_hi) && al(p.o_lo) && al(p.o_lo8) && al(p.o_hi8)))
    return false;
  const bool split_ok = p.split ? (p.q_lo && p.k_lo && p.v_lo) : (!p.q_lo && !p.k_lo && !p.v_lo);
  return p.D == 64 && p.rel_bias != nullptr && !p.causal && p.q_pos == nullptr && p.q_pos0 == 0 && p.q_batch_rows == 0 && p.Lq == p.Lk &&
         (p.kv_batch_rows == 0 || p.kv_batch_rows == p.Lk) && (p.mask_ld == 0 || p.mask_ld == p.Lk) && split_ok && (p.ldq % 8 == 0) &&
         (p.ldk % 8 == 0) && (p.ldv % 8 == 0) && (p.ldo % 2 == 0) && (p.o_lo8 == nullptr || p.ldo8 % 2 == 0) && p.H <= 65535 &&
         p.B <= 65535 && p.Lk >= 1 && (long long)p.B * p.Lk <= 0x7fffffffll;
}

cudaError_t launch_attention_bias_tc(const AttnParams& p, void* encode_fn, cudaStream_t stream) {
  if (p.B == 0 || p.Lq == 0) return cudaSuccess;
  AttnBiasTcParams P;
  memset(&P, 0, sizeof(P));
  P.a = p;
  const long long rows = (long long)p.B * p.Lk;
  const int cols = p.H * ABT_D;
  bool ok = make_map(encode_fn, &P.tm_q_hi, p.q_hi, p.dtype, rows, cols, p.ldq, ABT_BM) &&
            make_map(encode_fn, &P.tm_k_hi, p.k_hi, p.dtype, rows, cols, p.ldk, ABT_KC);
  if (p.split)
    ok = ok && make_map(encode_fn, &P.tm_q_lo, p.q_lo, p.dtype, rows, cols, p.ldq, ABT_BM) &&
         make_map(encode_fn, &P.tm_k_lo, p.k_lo, p.dtype, rows, cols, p.ldk, ABT_KC);
  if (!ok) return cudaErrorInvalidValue;
  dim3 grid((p.Lq + ABT_BM - 1) / ABT_BM, p.H, p.B);
  if (p.dtype == DT_BF16) return p.split ? launch_t<DT_BF16, true>(P, grid, stream) : launch_t<DT_BF16, false>(P, grid, stream);
  return p.split ? launch_t<DT_F16, true>(P, grid, stream) : launch_t<DT_F16, false>(P, grid, stream);
}

}  // namespace vima
