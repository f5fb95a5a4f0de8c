// K/V-streaming wgmma attention (attention_tc.cuh): the unpaged entry points and the launcher of all three.
#include "attention_tc.cuh"

namespace vima {

namespace {

template <int DT>
__global__ void __launch_bounds__(ATC_THREADS, 2) attention_tc_kernel(const __grid_constant__ AttnTcParams P) {
  attention_tc_body<DT, 32, true, false, false>(P);
}
template <int DT, bool SPLIT>
__global__ void __launch_bounds__(ATC_THREADS, 2) attention_bias_tc_kernel(const __grid_constant__ AttnTcParams P) {
  attention_tc_body<DT, 64, SPLIT, true, false>(P);
}

// 16-byte alignment of every operand and output base (vectorised loads / stores, TMA)
bool aligned_operands(const AttnParams& p) {
  auto al = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
  return al(p.q_hi) && al(p.q_lo) && al(p.k_hi) && al(p.k_lo) && al(p.v_hi) && al(p.v_lo) && al(p.o_hi) && al(p.o_lo) && al(p.o_lo8) &&
         al(p.o_hi8);
}

}  // namespace

// rows of the k / v operands: the page pool's, or B batch elements of kv_batch_rows (0 = Lk)
long long attention_kv_rows(const AttnParams& p) {
  if (p.kv_pages) return (long long)p.kv_pool_pages * KV_PAGE_TOKENS;
  return (long long)p.B * (p.kv_batch_rows ? p.kv_batch_rows : p.Lk);
}

// Shapes the decoder entry point takes (everything else stays on the mma.sync kernel of attention.cu).
bool attention_tc_supported(const AttnParams& p) {
  const int qbr = p.q_batch_rows ? p.q_batch_rows : p.Lq;  // TMA row coordinates of K and Q are 32-bit
  if (!aligned_operands(p)) return false;
  return p.D == 32 && p.split != 0 && p.rel_bias == nullptr && p.q_lo && p.k_lo && p.v_lo && (p.ldq % 8 == 0) && (p.ldk % 8 == 0) &&
         (p.ldv % 8 == 0) && (p.ldo % 8 == 0) && (p.o_lo8 == nullptr || p.ldo8 % 8 == 0) && p.H <= 65535 && p.B <= 65535 && p.Lk >= 1 &&
         attention_kv_rows(p) <= 0x7fffffffll && (long long)p.B * qbr <= 0x7fffffffll;
}

// Shapes the T5 entry point takes: the T5 encoder's self-attention.  Operand rows and the per-batch key count are the plain [B*L, ld]
// layout.
bool attention_bias_tc_supported(const AttnParams& p) {
  if (!aligned_operands(p)) return false;
  const bool split_ok = p.split ? (p.q_lo && p.k_lo && p.v_lo) : (!p.q_lo && !p.k_lo && !p.v_lo);
  return p.D == 64 && p.rel_bias != nullptr && !p.causal && p.q_pos == nullptr && p.q_pos0 == 0 && p.q_batch_rows == 0 && p.Lq == p.Lk &&
         (p.kv_batch_rows == 0 || p.kv_batch_rows == p.Lk) && (p.mask_ld == 0 || p.mask_ld == p.Lk) && split_ok && (p.ldq % 8 == 0) &&
         (p.ldk % 8 == 0) && (p.ldv % 8 == 0) && (p.ldo % 2 == 0) && (p.o_lo8 == nullptr || p.ldo8 % 2 == 0) && p.H <= 65535 &&
         p.B <= 65535 && p.Lk >= 1 && (long long)p.B * p.Lk <= 0x7fffffffll;
}

cudaError_t launch_attention_tc(const AttnParams& p, void* encode_fn, cudaStream_t stream) {
  if (p.B == 0 || p.Lq == 0) return cudaSuccess;
  const bool bias = p.rel_bias != nullptr;
  const int D = bias ? 64 : 32;
  AttnTcParams P;
  memset(&P, 0, sizeof(P));
  P.a = p;
  const long long kv_rows = attention_kv_rows(p);
  const long long q_rows = (long long)p.B * (p.q_batch_rows ? p.q_batch_rows : p.Lq);
  // [rows, H*D] 16-bit view of one operand (row pitch ld elements), boxes of box_rows x D elements (2D bytes, swizzled to match)
  auto map = [&](CUtensorMap* tm, const void* base, long long rows, int ld, int box_rows) {
    return encode_tmap_2d(encode_fn, tm, p.dtype == DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, base,
                          (uint64_t)rows, (uint64_t)p.H * D, (uint64_t)ld * 2, (uint32_t)D, (uint32_t)box_rows,
                          D == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B) == CUDA_SUCCESS;
  };
  bool ok = map(&P.tm_q_hi, p.q_hi, q_rows, p.ldq, ATC_BM) && map(&P.tm_k_hi, p.k_hi, kv_rows, p.ldk, ATC_KC);
  if (p.split) ok = ok && map(&P.tm_q_lo, p.q_lo, q_rows, p.ldq, ATC_BM) && map(&P.tm_k_lo, p.k_lo, kv_rows, p.ldk, ATC_KC);
  if (!ok) return cudaErrorInvalidValue;
  dim3 grid((p.Lq + ATC_BM - 1) / ATC_BM, p.H, p.B);
  const bool bf = p.dtype == DT_BF16;
  if (!bias && p.kv_pages) return launch_attention_tc_paged(P, grid, stream);
  if (!bias) return bf ? launch_t<attention_tc_kernel<DT_BF16>, 32, false>(P, grid, stream) : launch_t<attention_tc_kernel<DT_F16>, 32, false>(P, grid, stream);
  if (bf) return p.split ? launch_t<attention_bias_tc_kernel<DT_BF16, true>, 64, true>(P, grid, stream)
                         : launch_t<attention_bias_tc_kernel<DT_BF16, false>, 64, true>(P, grid, stream);
  return p.split ? launch_t<attention_bias_tc_kernel<DT_F16, true>, 64, true>(P, grid, stream)
                 : launch_t<attention_bias_tc_kernel<DT_F16, false>, 64, true>(P, grid, stream);
}

}  // namespace vima
