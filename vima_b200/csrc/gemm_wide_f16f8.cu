// gemm_wide_kernel instantiations: the epilogues of VIMA_GEMM_VARIANTS in f16f8 mode.  No generic runtime-flag variant: its
// 256-wide tile spills, so other epilogues stay on gemm_tc_kernel.
#include "gemm_wide.cuh"
namespace vima {

template <class E>
static cudaError_t launch_wide_one(const GemmParams& p, int grid, size_t smem, int max_smem, cudaStream_t stream) {
  const cudaError_t e = raise_smem_ceiling<gemm_wide_kernel<E>>(max_smem);  // the device's opt-in limit: set once
  if (e != cudaSuccess) return e;
  gemm_wide_kernel<E><<<grid, GEMM_THREADS, smem, stream>>>(p);
  return cudaGetLastError();
}

#define VIMA_MATCH(ACT, GLU, MUL, RES, O32, O16, LNA, LNR, STATS)                                                        \
  (l.act == ACT && l.glu == (int)GLU && l.mul == (int)MUL && l.res == (int)RES && l.o32 == (int)O32 && l.o16 == (int)O16 && \
   l.lna == (int)LNA && l.lnr == (int)LNR && l.stats == (int)STATS)

bool gemm_wide_has_epilogue(const GemmLaunch& l) {
#define VIMA_TRY(ACT, GLU, MUL, RES, O32, O16, DTT, LNA, LNR, STATS) \
  if (VIMA_MATCH(ACT, GLU, MUL, RES, O32, O16, LNA, LNR, STATS)) return true;
  VIMA_GEMM_VARIANTS(VIMA_TRY, DT_F16)
#undef VIMA_TRY
  return false;
}

cudaError_t launch_gemm_wide(const GemmParams& p, const GemmLaunch& l, int grid, size_t smem, int max_smem, cudaStream_t stream) {
#define VIMA_TRY(ACT, GLU, MUL, RES, O32, O16, DTT, LNA, LNR, STATS) \
  if (VIMA_MATCH(ACT, GLU, MUL, RES, O32, O16, LNA, LNR, STATS))      \
    return launch_wide_one<EpiCfg<false, ACT, GLU, MUL, RES, O32, O16, DTT, LNA, LNR, STATS>>(p, grid, smem, max_smem, stream);
  VIMA_GEMM_VARIANTS(VIMA_TRY, DT_F16)
#undef VIMA_TRY
  return cudaErrorInvalidValue;
}
#undef VIMA_MATCH

}  // namespace vima
