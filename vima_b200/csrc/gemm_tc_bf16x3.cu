// gemm_tc_kernel instantiations of the "bf16x3" mode: bf16 (hi, lo) pairs, three-term products
#include "gemm_tc_variants.cuh"
namespace vima {
template cudaError_t launch_gemm_tc<DT_BF16, 1>(const GemmParams&, const GemmLaunch&, int, size_t, int, cudaStream_t);
}  // namespace vima
