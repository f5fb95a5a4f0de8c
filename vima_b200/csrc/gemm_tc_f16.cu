// gemm_tc_kernel instantiations of the "f16" mode: fp16 operands, hi*hi only
#include "gemm_tc_variants.cuh"
namespace vima {
template cudaError_t launch_gemm_tc<DT_F16, 0>(const GemmParams&, const GemmLaunch&, int, size_t, int, cudaStream_t);
}  // namespace vima
