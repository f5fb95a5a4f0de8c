// gemm_tc_kernel instantiations of the "f16f8" mode: fp16 hi*hi + two e4m3 cross terms
#include "gemm_tc_variants.cuh"
namespace vima {
template cudaError_t launch_gemm_tc<DT_F16, 2>(const GemmParams&, const GemmLaunch&, int, size_t, int, cudaStream_t);
}  // namespace vima
