// Shared device helpers for the vima_b200 kernels (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#ifndef VIMA_WAIT_CYCLES
#define VIMA_WAIT_CYCLES (3000000000ll)  // an mbarrier wait longer than ~2 s of SM clock is a protocol bug: trap instead of hanging the box
#endif

namespace vima {

enum : int { DT_F16 = 0, DT_BF16 = 1 };
enum : int { ACT_NONE = 0, ACT_RELU = 1, ACT_QUICKGELU = 2, ACT_GELU = 3, ACT_GELU_TANH = 4 };

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------------------------------------
// reduced-precision operand pairs: x ~= hi + lo, both in the 16-bit operand format.
// ---------------------------------------------------------------------------------------------
template <int DT>
struct Op16;
template <>
struct Op16<DT_F16> {
  using T = __half;
  static __device__ __forceinline__ unsigned short bits(float x) { return __half_as_ushort(__float2half_rn(x)); }
  static __device__ __forceinline__ float back(unsigned short b) { return __half2float(__ushort_as_half(b)); }
};
template <>
struct Op16<DT_BF16> {
  using T = __nv_bfloat16;
  static __device__ __forceinline__ unsigned short bits(float x) { return __bfloat16_as_ushort(__float2bfloat16_rn(x)); }
  static __device__ __forceinline__ float back(unsigned short b) { return __bfloat162float(__ushort_as_bfloat16(b)); }
};

// Packed pair split: two F2FP (saturating, so |x| > 65504 degrades instead of producing inf/NaN) + one unpack.
// Low 16 bits = first element.  3 instructions per element instead of 7 for the scalar form.
// Both halves saturate: +-inf -> +-MAX_NORM in hi and lo, NaN -> NaN in hi and lo.
template <int DT>
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  if constexpr (DT == DT_F16) {
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
    const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(x1 - hf.y), "f"(x0 - hf.x));
  } else {
    asm("cvt.rn.satfinite.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
    const float2 hf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hi));
    asm("cvt.rn.satfinite.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(x1 - hf.y), "f"(x0 - hf.x));
  }
}

// Scalar split (module inputs, weight packing): the packed form on (x, 0), so every producer of an operand pair gives the
// same bits for the same value, including |x| > 65504, +-inf and NaN.
template <int DT>
__device__ __forceinline__ void split16(float x, unsigned short& hi, unsigned short& lo) {
  uint32_t h2, l2;
  split2<DT>(x, 0.f, h2, l2);
  hi = (unsigned short)(h2 & 0xFFFFu);
  lo = (unsigned short)(l2 & 0xFFFFu);
}
// ---- fp8 (e4m3) cross-term operands ("f16f8" mode, DESIGN.md section 3) --------------------------------------------
// a*b ~= a_hi16*b_hi16 + a_lo8*b_hi8 + a_hi8*b_lo8 with   a_lo8 = e4m3((a - a_hi16) * 2^10),  a_hi8 = e4m3(a * 2^-3),
//                                                        b_hi8 = e4m3(b * 2^-10),           b_lo8 = e4m3((b - b_hi16) * 2^3)
// (b already carries the pack-time power-of-two scale), so all three products land in the same accumulator units.
constexpr float F8_ACT_LO_SCALE = 1024.0f, F8_ACT_HI_SCALE = 0.125f;
constexpr float F8_W_HI_SCALE = 1.0f / 1024.0f, F8_W_LO_SCALE = 8.0f;

__device__ __forceinline__ uint32_t e4m3x4(float x0, float x1, float x2, float x3) {  // byte 0 = x0
  unsigned short a, b;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(a) : "f"(x1), "f"(x0));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(b) : "f"(x3), "f"(x2));
  return (uint32_t)a | ((uint32_t)b << 16);
}
// fp16 hi + the two fp8 views of 4 consecutive values (lo_scale / hi_scale differ for activations and weights)
__device__ __forceinline__ void split4_f8(const float4& y, float lo_scale, float hi_scale, uint2& hi16, uint32_t& lo8, uint32_t& hi8) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi16.x) : "f"(y.y), "f"(y.x));
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi16.y) : "f"(y.w), "f"(y.z));
  const float2 h01 = __half22float2(*reinterpret_cast<const __half2*>(&hi16.x));
  const float2 h23 = __half22float2(*reinterpret_cast<const __half2*>(&hi16.y));
  lo8 = e4m3x4((y.x - h01.x) * lo_scale, (y.y - h01.y) * lo_scale, (y.z - h23.x) * lo_scale, (y.w - h23.y) * lo_scale);
  hi8 = e4m3x4(y.x * hi_scale, y.y * hi_scale, y.z * hi_scale, y.w * hi_scale);
}

template <int DT>
__device__ __forceinline__ void split4v(const float4& y, uint2& hi, uint2& lo) {
  split2<DT>(y.x, y.y, hi.x, lo.x);
  split2<DT>(y.z, y.w, hi.y, lo.y);
}

// ---------------------------------------------------------------------------------------------
// activations
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// exact-erf GELU (nn.GELU()): erf by Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, i.e. fp32 round-off level) --
// branch-free, 2 MUFU + ~12 FMA-class instructions; libdevice erff costs ~3x as much and made the GELU epilogues
// instruction-bound.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float e = ex2_approx(-z * z * 1.4426950408889634f);
  const float erf_abs = fmaf(-poly * t, e, 1.0f);
  return 0.5f * x * (1.0f + copysignf(erf_abs, x));
}
__device__ __forceinline__ float quick_gelu(float x) { return x / (1.0f + __expf(-1.702f * x)); }
// HF NewGELUActivation ("gelu_new", OpenAIGPTConfig.afn = "gelu"): 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))), with
// tanh(u) = 1 - 2 / (1 + e^{2u}) on ex2.approx / rcp.approx (absolute error ~2e-7; saturates correctly at both ends)
__device__ __forceinline__ float gelu_tanh(float x) {
  const float u = 0.7978845608028654f * fmaf(0.044715f * x * x, x, x);
  const float e = ex2_approx(u * 2.8853900817779268f);  // e^{2u}
  const float th = 1.0f - __fdividef(2.0f, 1.0f + e);
  return 0.5f * x * (1.0f + th);
}
__device__ __forceinline__ float apply_act(int act, float x) {
  switch (act) {
    case ACT_RELU: return fmaxf(x, 0.f);
    case ACT_QUICKGELU: return quick_gelu(x);
    case ACT_GELU: return gelu_erf(x);
    case ACT_GELU_TANH: return gelu_tanh(x);
    default: return x;
  }
}

// ---------------------------------------------------------------------------------------------
// warp reductions
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------------------------------------
// mbarrier / TMA / cluster PTX wrappers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (the launch fails with an error) instead of hanging the GPU.  No printf on the timeout
// path: a function call inside a wgmma loop makes ptxas serialise every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 1023u) == 0u && clock64() - t0 > VIMA_WAIT_CYCLES) __trap();
  }
}

__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// 2-D tiled load: c0 = innermost (element) coordinate, c1 = row coordinate.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma (sm_90a): D[64 x N] (+)= A[64 x K] * B[N x K]^T, fp32 accumulators in registers of the issuing warpgroup.
// Accumulator fragment of thread t (warp w = (t / 32) % 4, lane l): element 4*g + e holds row 16*w + l/4 + 8*(e >> 1),
// column 8*g + 2*(l % 4) + (e & 1).
// ---------------------------------------------------------------------------------------------
// shared-memory matrix descriptor: start address [0,14) (>>4) | LBO [16,30) (unused by swizzled K-major tiles; 1)
// | SBO [32,46) = 8 rows * row bytes | layout [62,64): 1 = 128-byte swizzle, 2 = 64-byte swizzle.
// A K step inside the swizzle row advances the start address by its byte offset (>> 4).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ uint64_t wgmma_desc_sw64(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(512 >> 4) << 32) | (2ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[N]) {  // keeps the compiler from moving accumulator accesses across wgmma
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define VIMA_ACC8(d, o)                                                                                                  \
  "+f"(d[(o) + 0]), "+f"(d[(o) + 1]), "+f"(d[(o) + 2]), "+f"(d[(o) + 3]), "+f"(d[(o) + 4]), "+f"(d[(o) + 5]), "+f"(d[(o) + 6]), \
      "+f"(d[(o) + 7])
#define VIMA_ACC16(d) VIMA_ACC8(d, 0), VIMA_ACC8(d, 8)
#define VIMA_ACC32(d) VIMA_ACC16(d), VIMA_ACC8(d, 16), VIMA_ACC8(d, 24)
#define VIMA_ACC48(d) VIMA_ACC32(d), VIMA_ACC8(d, 32), VIMA_ACC8(d, 40)
#define VIMA_ACC64(d) VIMA_ACC48(d), VIMA_ACC8(d, 48), VIMA_ACC8(d, 56)
#define VIMA_R16 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}"
#define VIMA_R32 \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define VIMA_R48 \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}"
#define VIMA_R64 \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"

// 16-bit operands (DT_F16 / DT_BF16), both K-major in shared memory: M64 N{N} K16.  IA / IB / IP: operand numbers of the A and
// B descriptors and of the scale-d flag (they follow the N/2 accumulator operands).
#define VIMA_WGMMA_K16(N, R, ACC, IA, IB, IP)                                                                                      \
  if constexpr (DT == DT_F16)                                                                                                      \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " IP ", 0;\n\t"                                                             \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 " R ", " IA ", " IB ", p, 1, 1, 0, 0;\n\t}"              \
                 : ACC(d) : "l"(da), "l"(db), "r"(accumulate));                                                                    \
  else                                                                                                                             \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " IP ", 0;\n\t"                                                             \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 " R ", " IA ", " IB ", p, 1, 1, 0, 0;\n\t}"            \
                 : ACC(d) : "l"(da), "l"(db), "r"(accumulate))
template <int DT, int N>
__device__ __forceinline__ void wgmma_m64nNk16_ss(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  static_assert(N == 32 || N == 64 || N == 96 || N == 128, "wgmma_m64nNk16_ss: N is 32, 64, 96 or 128");
  if constexpr (N == 32) { VIMA_WGMMA_K16(32, VIMA_R16, VIMA_ACC16, "%16", "%17", "%18"); }
  else if constexpr (N == 64) { VIMA_WGMMA_K16(64, VIMA_R32, VIMA_ACC32, "%32", "%33", "%34"); }
  else if constexpr (N == 96) { VIMA_WGMMA_K16(96, VIMA_R48, VIMA_ACC48, "%48", "%49", "%50"); }
  else { VIMA_WGMMA_K16(128, VIMA_R64, VIMA_ACC64, "%64", "%65", "%66"); }
}
#undef VIMA_WGMMA_K16
// e4m3 operands, both K-major in shared memory: M64 N{N} K32, always accumulating
#define VIMA_WGMMA_E4M3(N, R, ACC, IA, IB)                                                                     \
  asm volatile("wgmma.mma_async.sync.aligned.m64n" #N "k32.f32.e4m3.e4m3 " R ", " IA ", " IB ", 1, 1, 1;" \
               : ACC(d) : "l"(da), "l"(db))
template <int N>
__device__ __forceinline__ void wgmma_m64nNk32_e4m3_ss(float (&d)[N / 2], uint64_t da, uint64_t db) {
  static_assert(N == 32 || N == 64 || N == 96 || N == 128, "wgmma_m64nNk32_e4m3_ss: N is 32, 64, 96 or 128");
  if constexpr (N == 32) { VIMA_WGMMA_E4M3(32, VIMA_R16, VIMA_ACC16, "%16", "%17"); }
  else if constexpr (N == 64) { VIMA_WGMMA_E4M3(64, VIMA_R32, VIMA_ACC32, "%32", "%33"); }
  else if constexpr (N == 96) { VIMA_WGMMA_E4M3(96, VIMA_R48, VIMA_ACC48, "%48", "%49"); }
  else { VIMA_WGMMA_E4M3(128, VIMA_R64, VIMA_ACC64, "%64", "%65"); }
}
#undef VIMA_WGMMA_E4M3
// warp-specialised register split: the producer warpgroup gives registers back, the consumer warpgroups take them
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// A from registers (the 16-bit fragment of a previous accumulator), B K-major in shared memory: M64 N{N} K16 (attention's
// O[64 x D] += P V).  IA / IB / IP as above.
#define VIMA_WGMMA_K16_RS(N, R, ACC, IA, IB, IP)                                                                                   \
  if constexpr (DT == DT_F16)                                                                                                      \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " IP ", 0;\n\t"                                                             \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 " R ", " IA ", " IB ", p, 1, 1, 0;\n\t}"                 \
                 : ACC(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));                               \
  else                                                                                                                             \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " IP ", 0;\n\t"                                                             \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 " R ", " IA ", " IB ", p, 1, 1, 0;\n\t}"               \
                 : ACC(d) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate))
template <int DT, int N>
__device__ __forceinline__ void wgmma_m64nNk16_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
  static_assert(N == 32 || N == 64, "wgmma_m64nNk16_rs: N is 32 or 64");
  if constexpr (N == 32) { VIMA_WGMMA_K16_RS(32, VIMA_R16, VIMA_ACC16, "{%16, %17, %18, %19}", "%20", "%21"); }
  else { VIMA_WGMMA_K16_RS(64, VIMA_R32, VIMA_ACC32, "{%32, %33, %34, %35}", "%36", "%37"); }
}
#undef VIMA_WGMMA_K16_RS

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------------------------------------
// host-side launch helpers
// ---------------------------------------------------------------------------------------------
// 2-D tiled TMA map of a row-major [rows, cols] matrix (row pitch ld_bytes), boxes of box_cols x box_rows elements.
// encode_fn is the driver's cuTensorMapEncodeTiled (cudaGetDriverEntryPoint; the runtime links no libcuda).
inline CUresult encode_tmap_2d(void* encode_fn, CUtensorMap* tm, CUtensorMapDataType dtype, const void* base, uint64_t rows, uint64_t cols,
                               uint64_t ld_bytes, uint32_t box_cols, uint32_t box_rows, CUtensorMapSwizzle swizzle,
                               CUtensorMapL2promotion l2_promotion) {
  typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  const cuuint64_t gdim[2] = {cols, rows};
  const cuuint64_t gstride[1] = {ld_bytes};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return ((PFN_encodeTiled)encode_fn)(tm, dtype, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                                      l2_promotion, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

// Raises KERNEL's dynamic shared-memory ceiling on the current device to at least `bytes`.  cudaFuncSetAttribute is no stream
// operation and is not legal inside a CUDA-graph capture, so the ceiling only ever grows and is set once per (instantiation,
// device) for a fixed size: after the first launch a capture never sees the call.
template <auto KERNEL>
inline cudaError_t raise_smem_ceiling(int bytes) {
  static int ceiling[64] = {};  // per device (function attributes are per device)
  int dev = 0;
  cudaGetDevice(&dev);
  if (bytes <= ceiling[dev & 63]) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) ceiling[dev & 63] = bytes;
  return e;
}

}  // namespace vima
