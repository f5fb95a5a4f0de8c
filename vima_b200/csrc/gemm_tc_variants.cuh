// Epilogue specialisations of gemm_tc_kernel that the VIMA path uses (ACT, GLU, MUL, RES, O32, O16); everything else
// runs the generic runtime-flag variant.  Each epilogue is instantiated for every tile width a descriptor can ask for, once
// per (16-bit format, split mode) in gemm_tc_{f16,bf16}*.cu, so the library's GEMM sources compile in parallel.
#pragma once
#include "gemm_tc.cuh"

namespace vima {

struct GemmLaunch {
  int act, glu, mul, res, o32, o16, dtype;
  int lna, lnr, stats;  // folded A-side LayerNorm, LayerNorm'd residual, partial row statistics of the output
  int split, block_n;   // kernel template parameters: split mode (0 / 1 / 2) and tile width (32, 64, 96, 128)
};

// (ACT, GLU, MUL, RES, O32, O16, DT, LNA, LNR, STATS)
#define VIMA_GEMM_VARIANTS(X, DT)                                                   \
  X(ACT_NONE, false, false, false, false, true, DT, false, false, false)      /* q / kv / c_attn / T5 qkv */ \
  X(ACT_NONE, false, false, true, true, true, DT, false, false, false)        /* linear2 (+ residual -> fp32 + operands) */  \
  X(ACT_NONE, false, false, true, true, true, DT, false, false, true)         /* xattn out-proj, c_proj: + row statistics for the folded LN */ \
  X(ACT_NONE, false, false, false, true, false, DT, false, false, false)      /* conv1, in_proj -> fp32 */ \
  X(ACT_GELU, false, true, false, false, true, DT, false, false, false)       /* linear1: gelu(.) * gate (unfused form) */   \
  X(ACT_NONE, false, false, true, true, false, DT, false, false, false)       /* T5 o, wo + residual */ \
  X(ACT_NONE, false, false, true, true, false, DT, false, true, false)        /* mlp c_proj + LayerNorm'd residual */ \
  X(ACT_GELU, true, false, false, false, true, DT, false, false, false)       /* GEGLU (pre-normalised operand) */ \
  X(ACT_GELU, true, false, false, false, true, DT, true, false, false)        /* GEGLU with the LayerNorm folded in (linear1||gate, c_fc||gate) */ \
  X(ACT_RELU, false, false, false, false, true, DT, false, false, false)      /* MLP hidden layers, T5 wi */  \
  X(ACT_QUICKGELU, false, false, false, false, true, DT, false, false, false) /* ViT c_fc (pre-normalised operand) */ \
  X(ACT_QUICKGELU, false, false, false, false, true, DT, true, false, false)  /* ViT c_fc with ln_2 folded in */ \
  X(ACT_NONE, false, false, false, true, false, DT, true, false, false)       /* ViT in_proj with ln_1 folded in -> fp32 */

template <class E, int SPLIT, int BN>
inline cudaError_t launch_one(const GemmParams& p, int grid, size_t smem, int max_smem, cudaStream_t stream) {
  const cudaError_t e = raise_smem_ceiling<gemm_tc_kernel<E, SPLIT, BN>>(max_smem);  // the device's opt-in limit: set once
  if (e != cudaSuccess) return e;
  gemm_tc_kernel<E, SPLIT, BN><<<grid, GEMM_THREADS, smem, stream>>>(p);
  return cudaGetLastError();
}

// GLU tiles are 64 or 128 columns wide (a value and a gate half of 32-column multiples); other tiles 32, 64, 96 or 128
template <class E, int SPLIT>
inline cudaError_t launch_bn(const GemmParams& p, const GemmLaunch& l, int grid, size_t smem, int max_smem, cudaStream_t stream) {
  if (l.block_n == 64) return launch_one<E, SPLIT, 64>(p, grid, smem, max_smem, stream);
  if (l.block_n == 128) return launch_one<E, SPLIT, 128>(p, grid, smem, max_smem, stream);
  if constexpr (E::GENERIC || !E::GLU) {
    if (l.block_n == 32) return launch_one<E, SPLIT, 32>(p, grid, smem, max_smem, stream);
    if (l.block_n == 96) return launch_one<E, SPLIT, 96>(p, grid, smem, max_smem, stream);
  }
  return cudaErrorInvalidValue;
}

template <int DT, int SPLIT>
cudaError_t launch_gemm_tc(const GemmParams& p, const GemmLaunch& l, int grid, size_t smem, int max_smem, cudaStream_t stream) {
#define VIMA_TRY(ACT, GLU, MUL, RES, O32, O16, DTT, LNA, LNR, STATS)                                                     \
  if (l.act == ACT && l.glu == (int)GLU && l.mul == (int)MUL && l.res == (int)RES && l.o32 == (int)O32 && l.o16 == (int)O16 && \
      l.lna == (int)LNA && l.lnr == (int)LNR && l.stats == (int)STATS)                                                  \
    return launch_bn<EpiCfg<false, ACT, GLU, MUL, RES, O32, O16, DTT, LNA, LNR, STATS>, SPLIT>(p, l, grid, smem, max_smem, stream);
  VIMA_GEMM_VARIANTS(VIMA_TRY, DT)
#undef VIMA_TRY
  return launch_bn<EpiCfg<true, 0, false, false, false, false, false, DT>, SPLIT>(p, l, grid, smem, max_smem, stream);
}

#define VIMA_GEMM_INSTANCES(X) X(DT_F16, 0) X(DT_F16, 1) X(DT_F16, 2) X(DT_BF16, 0) X(DT_BF16, 1)
#define VIMA_EXTERN(DT, SPLIT) \
  extern template cudaError_t launch_gemm_tc<DT, SPLIT>(const GemmParams&, const GemmLaunch&, int, size_t, int, cudaStream_t);
VIMA_GEMM_INSTANCES(VIMA_EXTERN)
#undef VIMA_EXTERN

}  // namespace vima
