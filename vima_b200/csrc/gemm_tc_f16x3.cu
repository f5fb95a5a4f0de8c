// gemm_tc_kernel instantiations of the "f16x3" mode: fp16 (hi, lo) pairs, three-term products
#include "gemm_tc_variants.cuh"
namespace vima {
template cudaError_t launch_gemm_tc<DT_F16, 1>(const GemmParams&, const GemmLaunch&, int, size_t, int, cudaStream_t);
}  // namespace vima
