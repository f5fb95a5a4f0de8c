// K/V-streaming wgmma attention: one kernel body, three entry points.
//
//   attention_tc_kernel<DT>             the decoders: head_dim 32, (hi, lo) operand pairs, causal or not, KV caches (per-batch keys)
//   attention_tc_paged_kernel<DT>       the same over a K/V page pool (slot decode; attention_tc_paged.cu): rows through attn_kv_row
//   attention_bias_tc_kernel<DT, SPLIT> the T5 prompt encoder: head_dim 64, T5 relative-position bias, non-causal, Lq == Lk, split or
//                                       single-pass operands
//
//   one CTA per (batch, head, 128-query-row tile), two warpgroups of 64 query rows each; keys stream through in chunks of 64, so no
//   shared memory is sized by Lk (no length cap).  per chunk c, every warpgroup:
//     S[64x64] = Q K^T     wgmma M64 N64 K16 (hi*hi, lo*hi, hi*lo with split operands, hi*hi alone without), Q and K(c) from shared
//                          memory (TMA; 64-byte swizzle at D = 32, 128-byte at D = 64); K(c+2) is loaded by TMA into the slot K(c) leaves
//     V(c) -> V^T          while S is computed, every thread loads D/4 values of V(c) (hi and lo) and writes them transposed into a
//                          128-byte-swizzled K-major tile, the B operand layout wgmma reads; it also stages chunk c+1's 64 key-mask
//                          terms in a double buffer (with the bias: also the 191 bias values that (tile, chunk c+1) can index)
//     softmax              in registers on the accumulator fragment (4 lanes share a row), online maximum, exp2 with the scale
//                          folded in; P as (hi, lo) 16-bit pairs stays in registers
//     O[64xD] += P V       wgmma M64 N{D} K16 with A = P from registers, B = V^T from shared memory
//
// Same mask semantics as attention.cu (reference components.py:51-80): the causal constant is the reference's soft -1e4, key
// padding adds finfo.min, keys beyond Lk are excluded.  A causal tile first runs the chunks up to its diagonal; hidden keys have
// weight exp(-1e4 - m) == 0 exactly in fp32 once m > -1e4 + 104, so stopping there is bit-compatible with the reference's
// full-width softmax.  If some row has only seen padded keys by then (m still <= -9000), the tile is re-run over every chunk
// (rare: the first history slot is always valid in VIMA's data).
// With the bias, scores follow attention.cu's formula in the log2 domain: y = s * scale*log2e + bias[h][j - i + Lk - 1]*log2e, then
// + finfo(fp32).min for a padded key (a row whose keys are all padded gets the reference's uniform average) and -inf past Lk.
//
// The body is shared by two translation units: attention_tc.cu (the unpaged entry points) and attention_tc_paged.cu (the decoder
// entry point over a K/V page pool, slot decode), so each compiles to its own code with no run-time test of the layout.
#pragma once
#include "kernels.h"

namespace vima {

struct AttnTcParams {
  AttnParams a;
  CUtensorMap tm_q_hi, tm_q_lo, tm_k_hi, tm_k_lo;
};
// the decoder entry point over a page pool (attention_tc_paged.cu)
cudaError_t launch_attention_tc_paged(const AttnTcParams& P, dim3 grid, cudaStream_t stream);

namespace {

constexpr int ATC_THREADS = 256;
constexpr int ATC_BM = 128, ATC_KC = 64;
constexpr int ATC_WIN = ATC_BM + ATC_KC - 1;  // bias offsets j - i one (tile, chunk) pair can see: [k0 - q0 - 127, k0 - q0 + 63]

// shared memory carve (bytes; swizzled tiles 1024-aligned).  The lo halves stay reserved in single-pass mode: one carve for both.
template <int D, bool BIAS>
struct AtcSmem {
  static constexpr int Q_PART = ATC_BM * D * 2;   // 128 rows x 2D bytes
  static constexpr int K_PART = ATC_KC * D * 2;   // 64 keys x 2D bytes; V^T: D dims x 128 bytes, the same size
  static constexpr int QH = 0, QL = Q_PART;
  static constexpr int K = 2 * Q_PART;            // 2 stages x {hi, lo}
  static constexpr int VT = K + 4 * K_PART;       // 2 buffers x {hi, lo}
  static constexpr int MASK = VT + 4 * K_PART;    // float[2][64]: key-mask terms of a chunk
  static constexpr int BIAS_W = MASK + 2 * ATC_KC * 4;               // float[2][192]: bias window of a (tile, chunk) pair, log2 domain
  static constexpr int BAR = BIAS_W + (BIAS ? 2 * 192 * 4 : 0);      // 3 mbarriers
  static constexpr int BYTES = BAR + 32;
};

template <int DT, int D, bool SPLIT, bool BIAS, bool PAGED>
__device__ __forceinline__ void attention_tc_body(const AttnTcParams& P) {
  using S = AtcSmem<D, BIAS>;
  constexpr int PARTS = SPLIT ? 2 : 1;
  constexpr int VN = D / 4;  // V values each thread transposes per part
  const AttnParams& p = P.a;
  extern __shared__ __align__(1024) uint8_t sm[];
  float* maskadd = reinterpret_cast<float*>(sm + S::MASK);  // [2][64]
  float* sbias = reinterpret_cast<float*>(sm + S::BIAS_W);  // [2][192]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + S::BAR);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;  // [2]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  const int q0 = blockIdx.x * ATC_BM, h = blockIdx.y, b = blockIdx.z;
  const int Lq = p.Lq;
  // row pitches of key_mask and q / o, this batch element's causal position and key count (per-batch with q_pos); the T5 encoder's
  // operands are the plain [B*L, ld] layout (attention_bias_tc_supported).  k / v rows: attn_kv_row.
  const int mld = !BIAS && p.mask_ld ? p.mask_ld : p.Lk;
  const int qbr = !BIAS && p.q_batch_rows ? p.q_batch_rows : Lq;
  int qp0 = 0, Lk = p.Lk;
  if constexpr (!BIAS) attn_batch_keys(p, b, qbr, qp0, Lk);
  const uint32_t sbase = smem_u32(sm);
  const int rows_here = min(ATC_BM, Lq - q0);
  const int n_all = (Lk + ATC_KC - 1) / ATC_KC;
  int n_plan = n_all;  // causal: chunks up to the tile's diagonal
  if (!BIAS && p.causal) {
    const int last_key = min(Lk - 1, q0 + rows_here - 1 + qp0);
    n_plan = last_key / ATC_KC + 1;
  }
  const bool may_rerun = !BIAS && p.causal && n_plan < n_all;

  if ((sbase & 1023u) != 0u) {  // the swizzled tiles assume a 1024-byte aligned window (no static shared memory in this kernel)
    if (tid == 0) printf("vima_b200: attention_tc shared memory window is not 1024-byte aligned\n");
    __trap();
  }
  const int x_col = h * D;  // element column of this head inside the q / k / v row
  // k / v row of chunk c's first key; a chunk is one page, so key k0 + vj of the chunk is row chunk_row(c) + vj either way
  // (PAGED is a template parameter: a run-time test in the chunk loop cost the unpaged kernel 3 % at the cfg3 shapes)
  const int kv_row0 = PAGED ? 0 : (int)attn_kv_row<false>(p, b, 0);
  auto chunk_row = [&](int c) { return PAGED ? (int)attn_kv_row(p, b, c * ATC_KC) : kv_row0 + c * ATC_KC; };
  const float* bias_row = p.rel_bias + (size_t)h * (2 * Lk - 1);
  if (tid == 0) {
    mbar_init(q_full, 1);
    mbar_init(&k_full[0], 1);
    mbar_init(&k_full[1], 1);
    fence_barrier_init();
    tma_prefetch_desc(&P.tm_q_hi);
    if (SPLIT) tma_prefetch_desc(&P.tm_q_lo);
    tma_prefetch_desc(&P.tm_k_hi);
    if (SPLIT) tma_prefetch_desc(&P.tm_k_lo);
  }
  // chunk c's key-mask terms of this batch element (threads 192..255, one key each) and bias window (threads 0..190) into buffer c & 1
  auto stage_chunk = [&](int c) {
    if (tid >= ATC_THREADS - ATC_KC) {
      const int j = c * ATC_KC + tid - (ATC_THREADS - ATC_KC);
      const float mk = attn_key_mask_term(p, b, mld, j, Lk);
      maskadd[(c & 1) * ATC_KC + tid - (ATC_THREADS - ATC_KC)] = mk;
    } else if constexpr (BIAS) {
      if (tid < ATC_WIN) {
        const long long t = (long long)c * ATC_KC - q0 - (ATC_BM - 1) + tid + Lk - 1;  // table index of offset j - i = k0 - q0 - 127 + tid
        sbias[(c & 1) * 192 + tid] = (t >= 0 && t < 2ll * Lk - 1) ? __ldg(bias_row + t) * LOG2E : 0.f;
      }
    }
  };
  stage_chunk(0);
  __syncthreads();

  auto load_k = [&](int c, int stage) {  // thread 0 only
    uint8_t* dst = sm + S::K + stage * 2 * S::K_PART;
    mbar_arrive_expect_tx(&k_full[stage], (uint32_t)(S::K_PART * PARTS));
    const int row = chunk_row(c);
    tma_load_2d(dst, &P.tm_k_hi, &k_full[stage], x_col, row);
    if (SPLIT) tma_load_2d(dst + S::K_PART, &P.tm_k_lo, &k_full[stage], x_col, row);
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(q_full, (uint32_t)(S::Q_PART * PARTS));
    tma_load_2d(sm + S::QH, &P.tm_q_hi, q_full, x_col, b * qbr + q0);
    if (SPLIT) tma_load_2d(sm + S::QL, &P.tm_q_lo, q_full, x_col, b * qbr + q0);
  }

  // accumulator fragment rows of this thread: r_loc + 8*hh (hh = 0, 1) inside the tile; columns 8*g + 2*qd + (0, 1)
  const int r_loc = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int qd = lane & 3;
  const float c_l2 = p.scale * LOG2E;
  auto desc_qk = [](uint32_t addr) { return D == 32 ? wgmma_desc_sw64(addr) : wgmma_desc_sw128(addr); };
  const uint64_t dqh = desc_qk(sbase + S::QH + wg * (S::Q_PART / 2)), dql = desc_qk(sbase + S::QL + wg * (S::Q_PART / 2));
  // this thread's share of a V chunk: key vj, dims VN*vd .. VN*vd + VN-1 (hi and lo)
  const int vj = tid >> 2, vd = tid & 3;
  uint32_t k_use[2] = {0u, 0u};  // completed fills of each K stage
  float o[D / 2], m_run[2], l_run[2];
  int n = n_plan;
  for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
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
        const uint32_t k_addr = sbase + S::K + stage * 2 * S::K_PART;
        const uint64_t dkh = desc_qk(k_addr), dkl = desc_qk(k_addr + S::K_PART);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < D / 16; ++k) wgmma_m64nNk16_ss<DT, 64>(s, dqh + 2 * k, dkh + 2 * k, (uint32_t)(k != 0));
        if constexpr (SPLIT) {
#pragma unroll
          for (int k = 0; k < D / 16; ++k) wgmma_m64nNk16_ss<DT, 64>(s, dql + 2 * k, dkh + 2 * k, 1u);
#pragma unroll
          for (int k = 0; k < D / 16; ++k) wgmma_m64nNk16_ss<DT, 64>(s, dqh + 2 * k, dkl + 2 * k, 1u);
        }
        wgmma_commit();
      }
      // V(c) -> V^T tile (dim nn, key k at nn*128 + (((k>>3) ^ (nn&7)) << 4) + (k&7)*2), while the tensor cores work on S
      {
        uint4 vh[VN / 8], vl[VN / 8];
#pragma unroll
        for (int i = 0; i < VN / 8; ++i) vh[i] = vl[i] = make_uint4(0u, 0u, 0u, 0u);
        if (k0 + vj < Lk) {
          const size_t off = (size_t)(chunk_row(c) + vj) * p.ldv + x_col + vd * VN;
#pragma unroll
          for (int i = 0; i < VN / 8; ++i) {
            vh[i] = __ldg(reinterpret_cast<const uint4*>(p.v_hi + off + 8 * i));
            if constexpr (SPLIT) vl[i] = __ldg(reinterpret_cast<const uint4*>(p.v_lo + off + 8 * i));
          }
        }
        if (c + 1 < n) stage_chunk(c + 1);  // read after the barrier below; buffer (c+1)&1 was last read before the previous one
        uint8_t* vt = sm + S::VT + stage * 2 * S::K_PART;
        uint32_t wh[VN / 2], wl[VN / 2];
#pragma unroll
        for (int i = 0; i < VN / 8; ++i) {
          wh[4 * i] = vh[i].x; wh[4 * i + 1] = vh[i].y; wh[4 * i + 2] = vh[i].z; wh[4 * i + 3] = vh[i].w;
          wl[4 * i] = vl[i].x; wl[4 * i + 1] = vl[i].y; wl[4 * i + 2] = vl[i].z; wl[4 * i + 3] = vl[i].w;
        }
#pragma unroll
        for (int e = 0; e < VN; ++e) {
          const int nn = vd * VN + e;
          const int off = nn * 128 + ((((vj >> 3) ^ (nn & 7))) << 4) + (vj & 7) * 2;
          *reinterpret_cast<unsigned short*>(vt + off) = (unsigned short)(wh[e >> 1] >> (16 * (e & 1)));
          if constexpr (SPLIT) *reinterpret_cast<unsigned short*>(vt + S::K_PART + off) = (unsigned short)(wl[e >> 1] >> (16 * (e & 1)));
        }
        fence_proxy_async();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
      }
      wgmma_wait<0>();
      wgmma_fence_acc(s);
      // ---- softmax on the fragment: element 4g+e is row r_loc + 8*(e>>1), key k0 + 8g + 2qd + (e&1) ----
      const float* mk = maskadd + stage * ATC_KC;
      const float* bw = sbias + stage * 192 + (ATC_BM - 1) - r_loc;  // bw[jj - 8*hh] = bias of (row r_loc + 8*hh, key k0 + jj)
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int g = 0; g < 8; ++g)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int jj = 8 * g + 2 * qd + (e & 1), key = k0 + jj;
          const float mm = mk[jj];
          float y;
          if constexpr (BIAS) {  // three roundings, in this order
            y = s[4 * g + e] * c_l2;
            y += bw[jj - 8 * (e >> 1)];
            y += mm;
          } else {
            y = fmaf(s[4 * g + e], c_l2, mm);
            if (p.causal && key > q0 + r_loc + 8 * (e >> 1) + qp0) y = CAUSAL_L2 + mm;
          }
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
      for (int i = 0; i < D / 2; ++i) o[i] *= f[(i >> 1) & 1];
      // V^T(c) and chunk c+1's mask terms (and bias) are complete, and both warpgroups are done reading K(c): its slot takes K(c+2)
      named_bar_sync(1, ATC_THREADS);
      if (tid == 0 && c + 2 < n) load_k(c + 2, stage);
      {
        const uint32_t vt_addr = sbase + S::VT + stage * 2 * S::K_PART;
        const uint64_t dvh = wgmma_desc_sw128(vt_addr), dvl = wgmma_desc_sw128(vt_addr + S::K_PART);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < ATC_KC / 16; ++kk) {  // A fragment of keys [16kk, +16): pairs 4kk .. 4kk+3
          const uint32_t ah[4] = {ph[4 * kk], ph[4 * kk + 1], ph[4 * kk + 2], ph[4 * kk + 3]};
          const uint32_t al[4] = {pl[4 * kk], pl[4 * kk + 1], pl[4 * kk + 2], pl[4 * kk + 3]};
          wgmma_m64nNk16_rs<DT, D>(o, ah, dvh + 2 * kk, 1u);
          if constexpr (SPLIT) {
            wgmma_m64nNk16_rs<DT, D>(o, al, dvh + 2 * kk, 1u);
            wgmma_m64nNk16_rs<DT, D>(o, ah, dvl + 2 * kk, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(o);
      }
    }
    // every row past the causal range must have seen a valid key; otherwise the whole tile is redone over all chunks
    if (pass == 1 || !may_rerun) break;
    if constexpr (!BIAS) {
      const int undone = (r_loc < rows_here && !(m_run[0] > EXIT_L2)) || (r_loc + 8 < rows_here && !(m_run[1] > EXIT_L2));
      if (!__syncthreads_or(undone)) break;
      n = n_all;
      stage_chunk(0);  // every read of pass 0's mask buffers precedes the barrier above
      __syncthreads();
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
      const size_t brow = (size_t)b * qbr + row;
#pragma unroll
      for (int g = 0; g < D / 8; ++g) attn_store_pair<DT>(p, brow, x_col + 8 * g + 2 * qd, o[4 * g + 2 * hh] * inv, o[4 * g + 2 * hh + 1] * inv);
    }
  }
}

template <auto KERNEL, int D, bool BIAS>
cudaError_t launch_t(const AttnTcParams& P, dim3 grid, cudaStream_t stream) {
  constexpr int smem = AtcSmem<D, BIAS>::BYTES;
  const cudaError_t e = raise_smem_ceiling<KERNEL>(smem);
  if (e != cudaSuccess) return e;
  KERNEL<<<grid, ATC_THREADS, smem, stream>>>(P);
  return cudaGetLastError();
}

}  // namespace

}  // namespace vima
