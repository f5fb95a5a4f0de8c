// gemm_tc_kernel instantiations of the "bf16" mode: bf16 operands, hi*hi only
#include "gemm_tc_variants.cuh"
namespace vima {
template cudaError_t launch_gemm_tc<DT_BF16, 0>(const GemmParams&, const GemmLaunch&, int, size_t, int, cudaStream_t);
}  // namespace vima
