// The decoder entry point of the streaming wgmma attention (attention_tc.cuh) over a K/V page pool (slot decode): the same body with
// every chunk's K box and V rows at its page (attn_kv_row).
#include "attention_tc.cuh"

namespace vima {

namespace {

template <int DT>
__global__ void __launch_bounds__(ATC_THREADS, 2) attention_tc_paged_kernel(const __grid_constant__ AttnTcParams P) {
  attention_tc_body<DT, 32, true, false, true>(P);
}

}  // namespace

cudaError_t launch_attention_tc_paged(const AttnTcParams& P, dim3 grid, cudaStream_t stream) {
  return P.a.dtype == DT_BF16 ? launch_t<attention_tc_paged_kernel<DT_BF16>, 32, false>(P, grid, stream)
                              : launch_t<attention_tc_paged_kernel<DT_F16>, 32, false>(P, grid, stream);
}

}  // namespace vima
