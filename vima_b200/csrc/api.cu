// C ABI of libvima_b200.so (see include/vima_b200.h).  Thin: validates arguments, builds TMA tensor maps and
// launch configurations, and forwards to the kernels.  No host synchronisation anywhere.
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <cstdlib>

#include "../../include/vima_b200.h"
#include "gemm_wide.cuh"
#include "kernels.h"

using namespace vima;
static_assert(VIMA_KV_PAGE_TOKENS == KV_PAGE_TOKENS, "page size of the C ABI and of the kernels");

struct vima_ctx {
  int device;
  int sm_count;
  int max_smem_optin;
  long long launches;
  char err[512];
  void* encode_tiled;  // cuTensorMapEncodeTiled
  // environment, read once in vima_create
  int attn_tc;       // VIMA_B200_ATTN: tc (1, default) | mma (0)
  int attn_tail;     // VIMA_B200_ATTN_TAIL: the <= 8 rows past the last full 128-row tile: 1 = "kernel" (default; SIMT tail kernel),
                     // 0 = "off" (one more tensor-core tile)
  int epi_prefetch;  // VIMA_B200_EPI_PREFETCH: L2 prefetch of the next tile's residual / multiplier rows (default 0)
  int attn_bias_tc;  // VIMA_B200_ATTN_BIAS: relative-bias attention (T5) on the streaming wgmma kernel: 0 = "auto" (default; only past the
                     // resident-K/V kernel's shared memory), 1 = "tc" (at every length)
  int gemm_wide;     // VIMA_B200_GEMM_WIDE: f16f8 GEMMs of 128-wide tiles and N % 256 == 0 on gemm_wide_kernel (1, default) | gemm_tc_kernel (0)
};

// Restores the calling thread's CUDA device when an entry point returns (the library switches to the context's device).
struct DeviceGuard {
  int prev = -1;
  bool armed = false;
  cudaError_t enter(int dev) {
    cudaError_t e = cudaGetDevice(&prev);
    if (e != cudaSuccess) return e;
    if (prev == dev) return cudaSuccess;
    armed = true;
    return cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    if (armed) cudaSetDevice(prev);
  }
};

static int fail(vima_ctx* c, int code, const char* fmt, ...) {
  if (c) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(c->err, sizeof(c->err), fmt, ap);
    va_end(ap);
  }
  return code;
}
static int cuda_fail(vima_ctx* c, cudaError_t e, const char* what) {
  return fail(c, VIMA_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
}
#define CHECK_CTX(c)                  \
  if (!(c)) return VIMA_E_INVALID;    \
  DeviceGuard dev_guard_;             \
  {                                   \
    cudaError_t e_ = dev_guard_.enter((c)->device); \
    if (e_ != cudaSuccess) return cuda_fail((c), e_, "cudaSetDevice"); \
  }

// Descriptor versioning: the caller states the size of the struct it was compiled against; anything between the ABI-v4 size and
// this library's own size is accepted (unknown tail fields read as zero), everything else is rejected before a field is touched.
template <class D>
static int load_desc(vima_ctx* c, const D* in, D* out, size_t min_size, const char* what) {
  if (!in) return fail(c, VIMA_E_INVALID, "%s: null descriptor", what);
  const uint32_t sz = in->struct_size;
  if (sz < min_size || sz > sizeof(D))
    return fail(c, VIMA_E_INVALID, "%s: descriptor struct_size %u outside [%zu, %zu] (C-ABI v%d): the caller was built against another vima_b200.h",
                what, sz, min_size, sizeof(D), VIMA_B200_ABI_VERSION);
  memset(out, 0, sizeof(D));
  memcpy(out, in, sz);
  return VIMA_OK;
}
#define LAUNCHED(c, expr, name)                          \
  {                                                      \
    cudaError_t e_ = (expr);                             \
    if (e_ != cudaSuccess) return cuda_fail((c), e_, name); \
    (c)->launches++;                                     \
    return VIMA_OK;                                      \
  }

extern "C" {

int vima_abi_version(void) { return VIMA_B200_ABI_VERSION; }

int vima_set_option(vima_ctx* c, const char* key, const char* value) {
  if (!c) return VIMA_E_INVALID;
  if (!key || !value) return fail(c, VIMA_E_INVALID, "set_option: null key or value");
  if (!strcmp(key, "attn")) {
    if (!strcmp(value, "tc")) { c->attn_tc = 1; return VIMA_OK; }
    if (!strcmp(value, "mma")) { c->attn_tc = 0; return VIMA_OK; }
  } else if (!strcmp(key, "attn_tail")) {
    if (!strcmp(value, "kernel")) { c->attn_tail = 1; return VIMA_OK; }
    if (!strcmp(value, "off")) { c->attn_tail = 0; return VIMA_OK; }
  } else if (!strcmp(key, "attn_bias")) {
    if (!strcmp(value, "auto")) { c->attn_bias_tc = 0; return VIMA_OK; }
    if (!strcmp(value, "tc")) { c->attn_bias_tc = 1; return VIMA_OK; }
  } else if (!strcmp(key, "epi_prefetch")) {
    if (!strcmp(value, "0") || !strcmp(value, "1")) { c->epi_prefetch = value[0] == '1'; return VIMA_OK; }
  } else if (!strcmp(key, "gemm_wide")) {
    if (!strcmp(value, "0") || !strcmp(value, "1")) { c->gemm_wide = value[0] == '1'; return VIMA_OK; }
  }
  return fail(c, VIMA_E_INVALID, "set_option: unknown option %s=%s", key, value);
}

int vima_create(vima_ctx** out, int device) {
  if (!out) return VIMA_E_INVALID;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) return VIMA_E_CUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return VIMA_E_CUDA;
  if (prop.major != 9 || prop.minor != 0) return VIMA_E_UNSUPPORTED;  // sm_90a code only; there is no fallback path
  vima_ctx* c = new vima_ctx();
  memset(c, 0, sizeof(*c));
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  c->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
  DeviceGuard guard;  // the calling thread's current device is restored on every return path below
  if (guard.enter(device) != cudaSuccess) { delete c; return VIMA_E_CUDA; }
  cudaFree(0);
  cudaDriverEntryPointQueryResult q;
  void* fn = nullptr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || fn == nullptr) {
    delete c;
    return VIMA_E_CUDA;
  }
  c->encode_tiled = fn;
  c->attn_tc = 1; c->attn_tail = 1; c->epi_prefetch = 0; c->attn_bias_tc = 0; c->gemm_wide = 1;
  if (const char* e = getenv("VIMA_B200_ATTN")) vima_set_option(c, "attn", e);  // unknown values keep the default
  if (const char* e = getenv("VIMA_B200_ATTN_TAIL")) vima_set_option(c, "attn_tail", e);
  if (const char* e = getenv("VIMA_B200_EPI_PREFETCH")) vima_set_option(c, "epi_prefetch", e);
  if (const char* e = getenv("VIMA_B200_ATTN_BIAS")) vima_set_option(c, "attn_bias", e);
  if (const char* e = getenv("VIMA_B200_GEMM_WIDE")) vima_set_option(c, "gemm_wide", e);
  c->err[0] = 0;
  *out = c;
  return VIMA_OK;
}

void vima_destroy(vima_ctx* c) { delete c; }
const char* vima_last_error(vima_ctx* c) { return c ? c->err : "null context"; }
int vima_sm_count(vima_ctx* c) { return c ? c->sm_count : 0; }
int vima_sizeof_gemm_desc(void) { return (int)sizeof(vima_gemm_desc); }
int vima_sizeof_norm_desc(void) { return (int)sizeof(vima_norm_desc); }
int vima_sizeof_attn_desc(void) { return (int)sizeof(vima_attn_desc); }
int vima_sizeof_f32_gemm_group(void) { return (int)sizeof(vima_f32_gemm_group); }
int64_t vima_launch_count(vima_ctx* c) { return c ? c->launches : 0; }

int vima_split_f32(vima_ctx* c, const float* x, int64_t rows, int cols, int ldx, void* hi, void* lo, int ld16, int pad_cols, float scale,
                   int dtype, void* stream) {
  CHECK_CTX(c);
  if (!x || !hi || pad_cols < cols || pad_cols > ld16) return fail(c, VIMA_E_INVALID, "split_f32: bad arguments");
  LAUNCHED(c, launch_split(x, rows, cols, ldx, (unsigned short*)hi, (unsigned short*)lo, ld16, pad_cols, scale, dtype, (cudaStream_t)stream),
           "split_f32");
}

int vima_pack_weight(vima_ctx* c, const float* w, int n, int k, int transposed, int ldw, void* hi, void* lo, int ld16, float scale, int dtype,
                     void* stream) {
  CHECK_CTX(c);
  if (!w || !hi || ld16 < k || (ld16 & 7)) return fail(c, VIMA_E_INVALID, "pack_weight: ld16 must be >= k and a multiple of 8");
  LAUNCHED(c, launch_pack_weight(w, n, k, transposed, ldw, (unsigned short*)hi, (unsigned short*)lo, ld16, scale, dtype, (cudaStream_t)stream),
           "pack_weight");
}

int vima_pack_weight_f8(vima_ctx* c, const float* w, int n, int k, int transposed, int ldw, void* hi8, void* lo8, int ld8, float scale, void* stream) {
  CHECK_CTX(c);
  if (!w || !hi8 || !lo8 || ld8 < k || (ld8 & 15)) return fail(c, VIMA_E_INVALID, "pack_weight_f8: ld8 must be >= k and a multiple of 16");
  LAUNCHED(c, launch_pack_weight_f8(w, n, k, transposed, ldw, (unsigned char*)hi8, (unsigned char*)lo8, ld8, scale, (cudaStream_t)stream),
           "pack_weight_f8");
}

int vima_split_f8(vima_ctx* c, const float* x, int64_t rows, int cols, int ldx, void* lo8, void* hi8, int ld8, void* stream) {
  CHECK_CTX(c);
  if (!x || !lo8 || !hi8 || (cols & 3) || (ldx & 3) || (ld8 & 3) || ld8 < cols) return fail(c, VIMA_E_INVALID, "split_f8: bad arguments");
  LAUNCHED(c, launch_split_f8(x, rows, cols, ldx, (unsigned char*)lo8, (unsigned char*)hi8, ld8, (cudaStream_t)stream), "split_f8");
}

static int choose_block_n(int N, int glu) {
  const int step = glu ? 64 : 32;
  int best = step, best_pad = 1 << 30;
  for (int bn = step; bn <= GEMM_MAX_BN; bn += step) {
    const int padded = ((N + bn - 1) / bn) * bn;
    if (padded < best_pad || (padded == best_pad && bn > best)) { best = bn; best_pad = padded; }
  }
  return best;
}
int vima_glu_block_n(int n_out) { return choose_block_n(2 * n_out, 1); }
int vima_gemm_stats_parts(int N, int glu, int block_n) {
  const int bn = block_n > 0 ? block_n : choose_block_n(N, glu);
  return 2 * ((N + bn - 1) / bn);
}

int vima_row_stats_finalize(vima_ctx* c, const float* partial, int64_t rows, int parts, int cols, float eps, int rms, float* stats, void* stream) {
  CHECK_CTX(c);
  if (!partial || !stats || rows < 0 || parts <= 0 || cols <= 0 || ((uintptr_t)partial & 7) || ((uintptr_t)stats & 7))
    return fail(c, VIMA_E_INVALID, "row_stats_finalize: bad arguments");
  LAUNCHED(c, launch_row_stats_finalize(partial, rows, parts, cols, eps, rms, stats, (cudaStream_t)stream), "row_stats_finalize");
}

// fp8 operand tile: rows of 64 bytes (64 K-elements), 64-byte swizzle
static int make_tmap_f8(vima_ctx* c, CUtensorMap* tm, const void* base, int rows, int cols, int ld, int box_rows) {
  CUresult r = encode_tmap_2d(c->encode_tiled, tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, base, (uint64_t)rows, (uint64_t)cols, (uint64_t)ld, GEMM_BK,
                              (uint32_t)box_rows, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (r != CUDA_SUCCESS) return fail(c, VIMA_E_CUDA, "cuTensorMapEncodeTiled(fp8) failed (%d): rows %d cols %d ld %d box %d", (int)r, rows, cols, ld, box_rows);
  return VIMA_OK;
}

// 16-bit operand tile: rows of 128 bytes (64 K-elements), 128-byte swizzle
static int make_tmap(vima_ctx* c, CUtensorMap* tm, const void* base, int dtype, int rows, int cols, int ld, int box_rows) {
  const CUtensorMapDataType dt = dtype == DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUresult r = encode_tmap_2d(c->encode_tiled, tm, dt, base, (uint64_t)rows, (uint64_t)cols, (uint64_t)ld * 2, GEMM_BK, (uint32_t)box_rows,
                              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (r != CUDA_SUCCESS) return fail(c, VIMA_E_CUDA, "cuTensorMapEncodeTiled failed (%d): rows %d cols %d ld %d box %d", (int)r, rows, cols, ld, box_rows);
  return VIMA_OK;
}

int vima_gemm(vima_ctx* c, const vima_gemm_desc* d_in, void* stream) {
  CHECK_CTX(c);
  vima_gemm_desc d_local;
  if (int rc_ = load_desc(c, d_in, &d_local, VIMA_GEMM_DESC_V4_SIZE, "gemm")) return rc_;
  const vima_gemm_desc* d = &d_local;
  if (!d->a_hi || !d->b_hi) return fail(c, VIMA_E_INVALID, "gemm: null operand");
  if (d->M <= 0 || d->N <= 0 || d->K <= 0) return fail(c, VIMA_E_INVALID, "gemm: empty problem");
  if ((d->lda & 7) || (d->ldb & 7) || ((uintptr_t)d->a_hi & 15) || ((uintptr_t)d->b_hi & 15))
    return fail(c, VIMA_E_INVALID, "gemm: operands need 16-byte aligned bases and ld %% 8 == 0 (lda %d ldb %d)", d->lda, d->ldb);
  if ((d->a_lo == nullptr) != (d->b_lo == nullptr)) return fail(c, VIMA_E_INVALID, "gemm: a_lo and b_lo must both be set or both be null");
  const bool f8 = d->a_lo8 || d->a_hi8 || d->b_hi8 || d->b_lo8;
  if (f8) {
    if (!(d->a_lo8 && d->a_hi8 && d->b_hi8 && d->b_lo8) || d->a_lo || d->dtype != DT_F16)
      return fail(c, VIMA_E_INVALID, "gemm: f16f8 mode needs all four e4m3 operands, fp16 hi operands and no 16-bit lo operands");
    if ((d->lda8 & 15) || (d->ldb8 & 15) || ((uintptr_t)d->a_lo8 & 15) || ((uintptr_t)d->a_hi8 & 15) || ((uintptr_t)d->b_hi8 & 15) ||
        ((uintptr_t)d->b_lo8 & 15) || d->lda8 < d->K || d->ldb8 < d->K)
      return fail(c, VIMA_E_INVALID, "gemm: e4m3 operands need 16-byte aligned bases and ld %% 16 == 0");
  }
  if ((d->out_lo8 == nullptr) != (d->out_hi8 == nullptr) || (d->out_lo8 && (!d->out_hi || d->dtype != DT_F16 || (d->ld_o8 & 3))))
    return fail(c, VIMA_E_INVALID, "gemm: out_lo8/out_hi8 come together, with an fp16 out_hi, ld_o8 %% 4 == 0");
  if (d->lda < d->K || d->ldb < d->K) return fail(c, VIMA_E_INVALID, "gemm: leading dimension smaller than K");
  int bn = d->block_n > 0 ? d->block_n : choose_block_n(d->N, d->glu);
  if (bn > GEMM_MAX_BN || (bn % (d->glu ? 64 : 32))) return fail(c, VIMA_E_INVALID, "gemm: bad block_n %d (multiple of 32, 64 with GLU, <= %d)", bn, GEMM_MAX_BN);
  if (d->glu && (d->N % bn)) return fail(c, VIMA_E_INVALID, "gemm: GLU needs N %% block_n == 0");
  {
    const int n_out = d->glu ? d->N / 2 : d->N;
    const bool bad = (n_out & 3) || (d->out_f32 && ((d->ld_o32 & 3) || ((uintptr_t)d->out_f32 & 15))) ||
                     (d->out_hi && ((d->ld_o16 & 3) || ((uintptr_t)d->out_hi & 7) || (d->out_lo && ((uintptr_t)d->out_lo & 7)))) ||
                     (d->mul && ((d->ld_mul & 3) || ((uintptr_t)d->mul & 15))) || (d->residual && ((d->ld_res & 3) || ((uintptr_t)d->residual & 15)));
    if (bad) return fail(c, VIMA_E_INVALID, "gemm: epilogue tensors need N %% 4 == 0, ld %% 4 == 0 and 16-byte (fp32) / 8-byte (16-bit) aligned bases");
  }

  if (d->row_stats) {
    if (!d->ln_c1 || (d->ln_cols != 1 && d->ln_cols != 2) || (d->ln_cols == 2 && !d->glu) || ((uintptr_t)d->row_stats & 7))
      return fail(c, VIMA_E_INVALID, "gemm: folded LayerNorm needs row_stats (8-byte aligned), ln_c1 and ln_cols 1 (all columns) or 2 (GLU value half)");
  }
  if (d->res_stats) {
    if (!d->residual || !d->res_gamma || !d->res_beta || d->glu || ((uintptr_t)d->res_stats & 7))
      return fail(c, VIMA_E_INVALID, "gemm: a LayerNorm'd residual needs residual, res_stats (8-byte aligned), res_gamma, res_beta and no GLU");
  }
  if (d->stats_out) {
    if (d->stats_parts != 2 * ((d->N + bn - 1) / bn) || ((uintptr_t)d->stats_out & 7))
      return fail(c, VIMA_E_INVALID, "gemm: stats_parts must be vima_gemm_stats_parts(N, glu, block_n) = %d (got %d)", 2 * ((d->N + bn - 1) / bn), d->stats_parts);
  }

  GemmParams p;
  memset(&p, 0, sizeof(p));
  const int split = f8 ? 2 : (d->a_lo != nullptr ? 1 : 0);
  GemmLaunch l;
  l.act = d->act; l.glu = d->glu != 0; l.mul = d->mul != nullptr; l.res = d->residual != nullptr;
  l.o32 = d->out_f32 != nullptr; l.o16 = d->out_hi != nullptr; l.dtype = d->dtype;
  l.lna = d->row_stats != nullptr; l.lnr = d->res_stats != nullptr; l.stats = d->stats_out != nullptr;
  l.split = split; l.block_n = bn;
  // f16f8 GEMMs of 128-wide tiles run as pairs of adjacent tiles on the 128 x 256 kernel (a quarter less operand traffic from L2
  // per multiply-add); the epilogue, the GLU pairing and the row-statistics parts are those of the 128-wide tiles
  const bool wide = c->gemm_wide && split == 2 && bn == 128 && d->N % GEMM_WIDE_BN == 0 && gemm_wide_has_epilogue(l) &&
                    gemm_wide_smem_bytes() <= (size_t)c->max_smem_optin;
  const int tile_n = wide ? GEMM_WIDE_BN : bn;
  int rc;
  const int tiles_m_ = (d->M + GEMM_BM - 1) / GEMM_BM, tiles_n_ = (d->N + tile_n - 1) / tile_n;
  if ((rc = make_tmap(c, &p.tm_a_hi, d->a_hi, d->dtype, d->M, d->K, d->lda, GEMM_BM))) return rc;
  if ((rc = make_tmap(c, &p.tm_b_hi, d->b_hi, d->dtype, d->N, d->K, d->ldb, tile_n))) return rc;
  if (split == 1) {
    if ((rc = make_tmap(c, &p.tm_a_lo, d->a_lo, d->dtype, d->M, d->K, d->lda, GEMM_BM))) return rc;
    if ((rc = make_tmap(c, &p.tm_b_lo, d->b_lo, d->dtype, d->N, d->K, d->ldb, bn))) return rc;
  } else if (split == 2) {
    if ((rc = make_tmap_f8(c, &p.tm_a_lo, d->a_lo8, d->M, d->K, d->lda8, GEMM_BM))) return rc;
    if ((rc = make_tmap_f8(c, &p.tm_a_hi8, d->a_hi8, d->M, d->K, d->lda8, GEMM_BM))) return rc;
    if ((rc = make_tmap_f8(c, &p.tm_b_hi8, d->b_hi8, d->N, d->K, d->ldb8, tile_n))) return rc;
    if ((rc = make_tmap_f8(c, &p.tm_b_lo, d->b_lo8, d->N, d->K, d->ldb8, tile_n))) return rc;
  }
  p.M = d->M; p.N = d->N; p.K = d->K;
  p.dtype = d->dtype;
  p.glu = d->glu;
  p.epi_prefetch = c->epi_prefetch;
  p.act = d->act;
  p.acc_scale = d->acc_scale == 0.f ? 1.f : d->acc_scale;
  p.bias = d->bias;
  p.mul = d->mul; p.ld_mul = d->ld_mul;
  p.residual = d->residual; p.ld_res = d->ld_res;
  p.out_f32 = d->out_f32; p.ld_o32 = d->ld_o32;
  p.out_hi = (unsigned short*)d->out_hi; p.out_lo = (unsigned short*)d->out_lo; p.ld_o16 = d->ld_o16;
  p.out_lo8 = (unsigned char*)d->out_lo8; p.out_hi8 = (unsigned char*)d->out_hi8; p.ld_o8 = d->ld_o8;
  p.row_stats = d->row_stats; p.ln_c1 = d->ln_c1; p.ln_cols = d->ln_cols;
  p.res_stats = d->res_stats; p.res_gamma = d->res_gamma; p.res_beta = d->res_beta;
  p.stats_out = d->stats_out; p.stats_parts = d->stats_parts;

  const int tiles = tiles_m_ * tiles_n_;
  const int grid = tiles < c->sm_count ? tiles : c->sm_count;  // persistent: one CTA per SM walks the tiles
  if (wide) LAUNCHED(c, launch_gemm_wide(p, l, grid, gemm_wide_smem_bytes(), c->max_smem_optin, (cudaStream_t)stream), "gemm_wide_kernel");
  const size_t stage = (size_t)(GEMM_A_TILE_BYTES + bn * 128) * (split ? 2 : 1);
  const size_t fixed = gemm_smem_bytes(bn, split, 0);
  int n_stages = (int)(((size_t)c->max_smem_optin - fixed) / stage);
  if (n_stages > GEMM_MAX_STAGES) n_stages = GEMM_MAX_STAGES;
  if (n_stages < 2) return fail(c, VIMA_E_UNSUPPORTED, "gemm: not enough shared memory for 2 stages");
  p.n_stages = n_stages;
  const size_t smem = gemm_smem_bytes(bn, split, n_stages);
  // f16f8 (split 2) is fp16-only (checked above)
  auto launch = d->dtype == DT_BF16 ? (split ? launch_gemm_tc<DT_BF16, 1> : launch_gemm_tc<DT_BF16, 0>)
                                    : (split == 2 ? launch_gemm_tc<DT_F16, 2> : split ? launch_gemm_tc<DT_F16, 1> : launch_gemm_tc<DT_F16, 0>);
  LAUNCHED(c, launch(p, l, grid, smem, c->max_smem_optin, (cudaStream_t)stream), "gemm_tc_kernel");
}

int vima_gemm_f32_grouped(vima_ctx* c, const vima_f32_gemm_group* groups_dev, int n_groups, int M, int max_n, int act, void* stream) {
  CHECK_CTX(c);
  static_assert(sizeof(vima_f32_gemm_group) == sizeof(SimtGemmGroup), "group layout");
  if (!groups_dev) return fail(c, VIMA_E_INVALID, "gemm_f32_grouped: null groups");
  LAUNCHED(c, launch_simt_gemm_grouped(reinterpret_cast<const SimtGemmGroup*>(groups_dev), n_groups, M, max_n, act, (cudaStream_t)stream),
           "simt_gemm");
}

int vima_gemm_f32_grouped_host(vima_ctx* c, const vima_f32_gemm_group* groups_host, int n_groups, int M, int max_n, int act, void* stream) {
  CHECK_CTX(c);
  if (!groups_host || n_groups < 0) return fail(c, VIMA_E_INVALID, "gemm_f32_grouped_host: null groups");
  if (M < 0) return fail(c, VIMA_E_INVALID, "gemm_f32_grouped_host: M = %d < 0", M);
  // max_n sizes the grid's column tiles: a group with more columns would have its last ones silently never written
  for (int i = 0; i < n_groups; ++i)
    if (groups_host[i].n > max_n)
      return fail(c, VIMA_E_INVALID, "gemm_f32_grouped_host: group %d has n = %d columns, more than max_n = %d", i, groups_host[i].n, max_n);
  cudaError_t e = launch_simt_gemm_grouped_host(reinterpret_cast<const SimtGemmGroup*>(groups_host), n_groups, M, max_n, act, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(c, e, "simt_gemm");
  c->launches += (n_groups + SIMT_MAX_HOST_GROUPS - 1) / SIMT_MAX_HOST_GROUPS;
  return VIMA_OK;
}

int vima_norm(vima_ctx* c, const vima_norm_desc* d_in, void* stream) {
  CHECK_CTX(c);
  vima_norm_desc d_local;
  if (int rc_ = load_desc(c, d_in, &d_local, VIMA_NORM_DESC_V4_SIZE, "norm")) return rc_;
  const vima_norm_desc* d = &d_local;
  if (!d->x) return fail(c, VIMA_E_INVALID, "norm: null input");
  if ((d->cols & 3) || d->cols > 1024 || d->cols <= 0) return fail(c, VIMA_E_INVALID, "norm: cols must be a multiple of 4, <= 1024 (got %d)", d->cols);
  if ((d->ldx & 3) || (d->add && (d->ld_add & 3)) || (d->out_f32 && (d->ld_o32 & 3)) || (d->out2_f32 && (d->ld_o2 & 3)) || (d->out_hi && (d->ld_o16 & 3)))
    return fail(c, VIMA_E_INVALID, "norm: leading dimensions must be multiples of 4");
  NormParams p;
  p.x = d->x; p.rows = d->rows; p.cols = d->cols; p.ldx = d->ldx;
  p.add = d->add; p.ld_add = d->ld_add;
  p.w = d->w; p.b = d->b; p.eps = d->eps; p.rms = d->rms;
  p.w2 = d->w2; p.b2 = d->b2; p.eps2 = d->eps2;
  p.out_f32 = d->out_f32; p.ld_o32 = d->ld_o32;
  p.out2_f32 = d->out2_f32; p.ld_o2 = d->ld_o2;
  p.out_hi = (unsigned short*)d->out_hi; p.out_lo = (unsigned short*)d->out_lo; p.ld_o16 = d->ld_o16;
  p.dtype = d->dtype;
  p.out_lo8 = (unsigned char*)d->out_lo8; p.out_hi8 = (unsigned char*)d->out_hi8; p.ld_o8 = d->ld_o8;
  p.stats_out = d->stats_out; p.stats_eps = d->stats_eps;
  if (p.stats_out && ((uintptr_t)p.stats_out & 7)) return fail(c, VIMA_E_INVALID, "norm: stats_out must be 8-byte aligned");
  if ((p.out_lo8 == nullptr) != (p.out_hi8 == nullptr) || (p.out_lo8 && (p.ld_o8 & 3)))
    return fail(c, VIMA_E_INVALID, "norm: out_lo8/out_hi8 come together with ld_o8 %% 4 == 0");
  LAUNCHED(c, launch_norm(p, (cudaStream_t)stream), "norm");
}

int vima_attention(vima_ctx* c, const vima_attn_desc* d_in, void* stream) {
  CHECK_CTX(c);
  vima_attn_desc d_local;
  if (int rc_ = load_desc(c, d_in, &d_local, VIMA_ATTN_DESC_V4_SIZE, "attention")) return rc_;
  const vima_attn_desc* d = &d_local;
  if (!d->q_hi || !d->k_hi || !d->v_hi || !d->o_hi) return fail(c, VIMA_E_INVALID, "attention: null operand");
  if (d->D != 32 && d->D != 64) return fail(c, VIMA_E_UNSUPPORTED, "attention: head_dim %d (32 and 64 are built)", d->D);
  if ((d->ldq & 7) || (d->ldk & 7) || (d->ldv & 7) || (d->ldo & 1)) return fail(c, VIMA_E_INVALID, "attention: leading dimensions must be multiples of 8");
  const bool split = d->q_lo != nullptr;
  if (split != (d->k_lo != nullptr) || split != (d->v_lo != nullptr)) return fail(c, VIMA_E_INVALID, "attention: q/k/v lo parts must be all set or all null");
  if (d->rel_bias && d->Lq != d->Lk) return fail(c, VIMA_E_INVALID, "attention: relative bias needs Lq == Lk");
  if (!(d->scale > 0.f)) return fail(c, VIMA_E_INVALID, "attention: scale must be positive");
  AttnParams p;
  p.q_hi = (const unsigned short*)d->q_hi; p.q_lo = (const unsigned short*)d->q_lo; p.ldq = d->ldq;
  p.k_hi = (const unsigned short*)d->k_hi; p.k_lo = (const unsigned short*)d->k_lo; p.ldk = d->ldk;
  p.v_hi = (const unsigned short*)d->v_hi; p.v_lo = (const unsigned short*)d->v_lo; p.ldv = d->ldv;
  p.key_mask = d->key_mask; p.rel_bias = d->rel_bias;
  p.o_hi = (unsigned short*)d->o_hi; p.o_lo = (unsigned short*)d->o_lo; p.ldo = d->ldo;
  p.B = d->B; p.H = d->H; p.Lq = d->Lq; p.Lk = d->Lk; p.D = d->D;
  p.scale = d->scale; p.causal = d->causal; p.split = split; p.dtype = d->dtype;
  p.o_lo8 = (unsigned char*)d->o_lo8; p.o_hi8 = (unsigned char*)d->o_hi8; p.ldo8 = d->ldo8;
  p.kv_batch_rows = d->kv_batch_rows; p.mask_ld = d->mask_ld; p.q_pos0 = d->q_pos0; p.q_batch_rows = 0;
  p.q_pos = d->q_pos;
  p.kv_pages = d->kv_pages; p.kv_page_ld = d->kv_page_ld; p.kv_pool_pages = d->kv_pool_pages;
  p.kv_len = d->kv_len;
  if (d->kv_pages && ((d->causal && !d->q_pos) || d->rel_bias || d->kv_page_ld < 1 || d->kv_pool_pages < 1 ||
                      d->Lk > (long long)d->kv_page_ld * VIMA_KV_PAGE_TOKENS || (long long)d->kv_pool_pages * VIMA_KV_PAGE_TOKENS > 0x7fffffffll))
    return fail(c, VIMA_E_INVALID, "attention: paged k / v need q_pos (or non-causal attention), no relative bias, Lk <= kv_page_ld*%d (Lk %d, "
                "kv_page_ld %d) and 1 <= kv_pool_pages with kv_pool_pages*%d rows inside the 32-bit row range (kv_pool_pages %d)",
                VIMA_KV_PAGE_TOKENS, d->Lk, d->kv_page_ld, VIMA_KV_PAGE_TOKENS, d->kv_pool_pages);
  if (d->kv_len && (d->causal || d->q_pos || d->rel_bias))
    return fail(c, VIMA_E_INVALID, "attention: per-batch kv_len needs non-causal attention without q_pos or relative bias");
  if ((d->kv_batch_rows && d->kv_batch_rows < d->Lk) || (d->mask_ld && d->mask_ld < d->Lk) || d->q_pos0 < 0)
    return fail(c, VIMA_E_INVALID, "attention: kv_batch_rows / mask_ld must cover Lk, q_pos0 >= 0");
  if (d->q_pos && (!d->causal || d->rel_bias || d->Lq > d->Lk))
    return fail(c, VIMA_E_INVALID, "attention: per-batch q_pos needs causal attention, no relative bias and Lq <= Lk");
  if ((p.o_lo8 == nullptr) != (p.o_hi8 == nullptr) || (p.o_lo8 && ((p.ldo8 & 1) || d->dtype != DT_F16)))
    return fail(c, VIMA_E_INVALID, "attention: o_lo8/o_hi8 come together (fp16 format, even ldo8)");
  // wgmma kernel for the shapes it takes (head_dim 32, split operands, no relative bias), mma.sync kernel otherwise;
  // VIMA_B200_ATTN=mma (read once in vima_create) forces the latter.  Both are covered by the kernel tests.
  if (c->attn_tc && attention_tc_supported(p)) {
    // the wgmma kernel works on 128-row query tiles: a few rows past the last full tile (7 of 263, 8 of 392) would hold a CTA slot
    // for the whole key range with one warp of eight at work -- they go to the SIMT tail kernel instead (attention_tail.cu), as
    // long as its shared memory holds the key range; past that they run in the wgmma kernel's last tile.
    const int tail = p.Lq % 128;
    if (c->attn_tail && p.Lq > 128 && tail >= 1 && tail <= ATTN_TAIL_MAX_ROWS && p.Lk <= ATTN_TAIL_MAX_LK) {
      AttnParams body = p;
      body.Lq = p.Lq - tail;
      body.q_batch_rows = p.Lq;
      cudaError_t e_ = launch_attention_tc(body, c->encode_tiled, (cudaStream_t)stream);
      if (e_ != cudaSuccess) return cuda_fail(c, e_, "attention_tc");
      c->launches++;
      LAUNCHED(c, launch_attention_tail(p, p.Lq - tail, tail, (cudaStream_t)stream), "attention_tail");
    }
    LAUNCHED(c, launch_attention_tc(p, c->encode_tiled, (cudaStream_t)stream), "attention_tc");
  }
  // T5's relative-bias attention (head_dim 64, non-causal): the streaming wgmma kernel takes every length the resident-K/V kernel
  // cannot hold, and every length with attn_bias=tc.  Everything that fits stays on the mma.sync kernel below by default.
  if (c->attn_tc && attention_bias_tc_supported(p) && (c->attn_bias_tc || attention_smem_bytes(p) > (size_t)c->max_smem_optin))
    LAUNCHED(c, launch_attention_tc(p, c->encode_tiled, (cudaStream_t)stream), "attention_bias_tc");
  {
    // the mma.sync kernel keeps K and V^T (hi + lo) of one (batch, head) resident in shared memory
    const size_t need = attention_smem_bytes(p);
    if (need > (size_t)c->max_smem_optin)
      return fail(c, VIMA_E_UNSUPPORTED,
                  "attention: Lk = %d keys of head_dim %d (%s operands%s) need %zu bytes of shared memory, the device offers %d: the "
                  "resident-K/V kernel takes Lk <= %d at this head_dim", d->Lk, d->D, split ? "split" : "single", d->rel_bias ? ", relative bias" : "",
                  need, c->max_smem_optin, attention_max_lk(p, (size_t)c->max_smem_optin));
  }
  LAUNCHED(c, launch_attention(p, (cudaStream_t)stream), "attention");
}

int vima_latent_attention(vima_ctx* c, const float* q, int ldq, int64_t q_batch_stride, const float* k, int ldk, const float* v, int ldv, float* o,
                          int ldo, int64_t N, int Lq, int Lk, int H, int d, float scale, void* stream) {
  CHECK_CTX(c);
  if (!q || !k || !v || !o) return fail(c, VIMA_E_INVALID, "latent_attention: null pointer");
  if (Lk < 1 || Lk > 16 || d < 1 || d > 128 || Lq < 0 || N < 0 || H < 1)
    return fail(c, VIMA_E_UNSUPPORTED, "latent_attention: 1..16 keys, head_dim <= 128 (Lk %d, d %d)", Lk, d);
  LatentAttnParams p;
  p.q = q; p.ldq = ldq; p.q_batch_stride = q_batch_stride; p.k = k; p.ldk = ldk; p.v = v; p.ldv = ldv; p.o = o; p.ldo = ldo;
  p.N = N; p.Lq = Lq; p.Lk = Lk; p.H = H; p.d = d; p.scale = scale;
  LAUNCHED(c, launch_latent_attention(p, (cudaStream_t)stream), "latent_attention");
}

int vima_small_attention(vima_ctx* c, const float* qkv, int ld, int64_t N, int S, int H, int W, float scale, void* o_hi, void* o_lo, int ldo,
                         float* o_f32, int dtype, void* stream) {
  CHECK_CTX(c);
  if (!qkv) return fail(c, VIMA_E_INVALID, "small_attention: null input");
  SmallAttnParams p;
  p.qkv = qkv; p.ld = ld; p.o_hi = (unsigned short*)o_hi; p.o_lo = (unsigned short*)o_lo; p.ldo = ldo; p.o_f32 = o_f32;
  p.N = N; p.S = S; p.H = H; p.W = W; p.scale = scale; p.dtype = dtype;
  LAUNCHED(c, launch_small_attention(p, (cudaStream_t)stream), "small_attention");
}

int vima_assemble_history(vima_ctx* c, const float* obs, const uint8_t* obs_mask, const float* action, int T, int B, int Q, int E, int La,
                          float* tokens, uint8_t* masks_bl, int64_t* pos_bl, void* stream) {
  CHECK_CTX(c);
  if (!obs || !obs_mask || !tokens || !masks_bl || !pos_bl || (La > 0 && !action) || (E & 3))
    return fail(c, VIMA_E_INVALID, "assemble_history: bad arguments");
  if (La != T && La != T - 1) return fail(c, VIMA_E_INVALID, "assemble_history: need T-1 or T action tokens");
  cudaError_t e = launch_assemble_history(obs, obs_mask, action, T, B, Q, E, La, tokens, masks_bl, (long long*)pos_bl, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(c, e, "assemble_history");
  c->launches += 2;
  return VIMA_OK;
}

int vima_mask_cumsum(vima_ctx* c, const uint8_t* mask, int B, int L, int64_t* pos, void* stream) {
  CHECK_CTX(c);
  LAUNCHED(c, launch_mask_cumsum(mask, B, L, (long long*)pos, (cudaStream_t)stream), "mask_cumsum");
}

int vima_slot_step_begin(vima_ctx* c, const float* obs, const uint8_t* obs_mask, const float* action, int S, int Q, int E, int Lmax,
                         const int32_t* len, const int32_t* n_valid, const int32_t* has_action, const int32_t* active, float* tokens,
                         uint8_t* step_mask, int64_t* pos, int32_t* q_pos, uint8_t* slot_mask, void* stream) {
  CHECK_CTX(c);
  if (!obs || !obs_mask || !action || !len || !n_valid || !has_action || !active || !tokens || !step_mask || !pos || !q_pos || !slot_mask)
    return fail(c, VIMA_E_INVALID, "slot_step_begin: null pointer");
  if (S < 0 || Q < 1 || (E & 3) || E <= 0 || Q + 1 > Lmax || ((uintptr_t)obs & 15) || ((uintptr_t)action & 15) || ((uintptr_t)tokens & 15))
    return fail(c, VIMA_E_INVALID, "slot_step_begin: S >= 0, 1 <= Q < Lmax, E %% 4 == 0, 16-byte aligned fp32 rows");
  LAUNCHED(c, launch_slot_step_begin(obs, obs_mask, action, S, Q, E, Lmax, len, n_valid, has_action, active, tokens, step_mask,
                                     (long long*)pos, q_pos, slot_mask, (cudaStream_t)stream),
           "slot_step_begin");
}

int vima_slot_kv_append(vima_ctx* c, const void* qkv_hi, const void* qkv_lo, int ld_qkv, int col0, int width, int S, int Lq, const int32_t* q_pos,
                        void* kv_hi, void* kv_lo, int ld_kv, int Lmax, void* stream) {
  CHECK_CTX(c);
  if (!qkv_hi || !kv_hi || !q_pos || (qkv_lo == nullptr) != (kv_lo == nullptr)) return fail(c, VIMA_E_INVALID, "slot_kv_append: null pointer");
  auto al = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
  if ((ld_qkv & 7) || (col0 & 7) || (width & 7) || (ld_kv & 7) || width <= 0 || col0 + width > ld_qkv || width > ld_kv || Lq < 1 || Lq > Lmax ||
      !al(qkv_hi) || !al(qkv_lo) || !al(kv_hi) || !al(kv_lo))
    return fail(c, VIMA_E_INVALID, "slot_kv_append: ld / col0 / width multiples of 8 inside the rows, 16-byte aligned bases, Lq <= Lmax");
  LAUNCHED(c, launch_slot_kv_append((const unsigned short*)qkv_hi, (const unsigned short*)qkv_lo, ld_qkv, col0, width, S, Lq, q_pos,
                                    (unsigned short*)kv_hi, (unsigned short*)kv_lo, ld_kv, Lmax, nullptr, 0, (cudaStream_t)stream),
           "slot_kv_append");
}

int vima_slot_kv_append_paged(vima_ctx* c, const void* qkv_hi, const void* qkv_lo, int ld_qkv, int col0, int width, int S, int Lq,
                              const int32_t* q_pos, void* kv_hi, void* kv_lo, int ld_kv, const int32_t* pages, int page_ld, int pool_pages,
                              void* stream) {
  CHECK_CTX(c);
  if (!qkv_hi || !kv_hi || !q_pos || !pages || (qkv_lo == nullptr) != (kv_lo == nullptr))
    return fail(c, VIMA_E_INVALID, "slot_kv_append_paged: null pointer");
  auto al = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
  if ((ld_qkv & 7) || (col0 & 7) || (width & 7) || (ld_kv & 7) || width <= 0 || col0 < 0 || col0 + width > ld_qkv || width > ld_kv || Lq < 1 ||
      page_ld < 1 || (long long)page_ld * VIMA_KV_PAGE_TOKENS > 0x7fffffffll || Lq > page_ld * VIMA_KV_PAGE_TOKENS || pool_pages < 1 ||
      !al(qkv_hi) || !al(qkv_lo) || !al(kv_hi) || !al(kv_lo))
    return fail(c, VIMA_E_INVALID, "slot_kv_append_paged: ld / col0 / width multiples of 8 inside the rows, 16-byte aligned bases, "
                                   "page_ld >= 1, Lq <= page_ld*%d, pool_pages >= 1", VIMA_KV_PAGE_TOKENS);
  LAUNCHED(c, launch_slot_kv_append((const unsigned short*)qkv_hi, (const unsigned short*)qkv_lo, ld_qkv, col0, width, S, Lq, q_pos,
                                    (unsigned short*)kv_hi, (unsigned short*)kv_lo, ld_kv, page_ld * VIMA_KV_PAGE_TOKENS, pages, pool_pages,
                                    (cudaStream_t)stream),
           "slot_kv_append_paged");
}

int vima_slot_step_end(vima_ctx* c, const float* x, int ldx, int S, int Q, int E, const uint8_t* step_mask, int32_t* len, int32_t* n_valid,
                       int32_t* has_action, const int32_t* active, float* out, void* stream) {
  CHECK_CTX(c);
  if (!x || !step_mask || !len || !n_valid || !has_action || !active || !out) return fail(c, VIMA_E_INVALID, "slot_step_end: null pointer");
  if (S < 0 || Q < 1 || (E & 3) || E <= 0 || (ldx & 3) || ldx < E || ((uintptr_t)x & 15) || ((uintptr_t)out & 15))
    return fail(c, VIMA_E_INVALID, "slot_step_end: Q >= 1, E and ldx multiples of 4, 16-byte aligned fp32 rows");
  LAUNCHED(c, launch_slot_step_end(x, ldx, S, Q, E, step_mask, len, n_valid, has_action, active, out, (cudaStream_t)stream), "slot_step_end");
}

int vima_slot_kv_scatter(vima_ctx* c, const void* qkv_hi, const void* qkv_lo, int ld_qkv, int col0, int width, int n, int Lq, const int32_t* slots,
                         void* kv_hi, void* kv_lo, int ld_kv, int Lmax, void* stream) {
  CHECK_CTX(c);
  if (!qkv_hi || !kv_hi || !slots || (qkv_lo == nullptr) != (kv_lo == nullptr)) return fail(c, VIMA_E_INVALID, "slot_kv_scatter: null pointer");
  auto al = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
  if ((ld_qkv & 7) || (col0 & 7) || (width & 7) || (ld_kv & 7) || width <= 0 || col0 < 0 || col0 + width > ld_qkv || width > ld_kv || n < 0 ||
      Lq < 1 || Lq > Lmax || !al(qkv_hi) || !al(qkv_lo) || !al(kv_hi) || !al(kv_lo))
    return fail(c, VIMA_E_INVALID, "slot_kv_scatter: ld / col0 / width multiples of 8 inside the rows, 16-byte aligned bases, 1 <= Lq <= Lmax");
  LAUNCHED(c, launch_slot_kv_scatter((const unsigned short*)qkv_hi, (const unsigned short*)qkv_lo, ld_qkv, col0, width, n, Lq, slots,
                                     (unsigned short*)kv_hi, (unsigned short*)kv_lo, ld_kv, Lmax, nullptr, 0, (cudaStream_t)stream),
           "slot_kv_scatter");
}

int vima_slot_kv_scatter_paged(vima_ctx* c, const void* qkv_hi, const void* qkv_lo, int ld_qkv, int col0, int width, int n, int Lq,
                               const int32_t* slots, void* kv_hi, void* kv_lo, int ld_kv, const int32_t* pages, int page_ld, int pool_pages,
                               void* stream) {
  CHECK_CTX(c);
  if (!qkv_hi || !kv_hi || !slots || !pages || (qkv_lo == nullptr) != (kv_lo == nullptr))
    return fail(c, VIMA_E_INVALID, "slot_kv_scatter_paged: null pointer");
  auto al = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
  if ((ld_qkv & 7) || (col0 & 7) || (width & 7) || (ld_kv & 7) || width <= 0 || col0 < 0 || col0 + width > ld_qkv || width > ld_kv || n < 0 ||
      Lq < 1 || page_ld < 1 || (long long)page_ld * VIMA_KV_PAGE_TOKENS > 0x7fffffffll || Lq > page_ld * VIMA_KV_PAGE_TOKENS ||
      pool_pages < 1 || !al(qkv_hi) || !al(qkv_lo) || !al(kv_hi) || !al(kv_lo))
    return fail(c, VIMA_E_INVALID, "slot_kv_scatter_paged: ld / col0 / width multiples of 8 inside the rows, 16-byte aligned bases, "
                                   "page_ld >= 1, 1 <= Lq <= page_ld*%d, pool_pages >= 1", VIMA_KV_PAGE_TOKENS);
  LAUNCHED(c, launch_slot_kv_scatter((const unsigned short*)qkv_hi, (const unsigned short*)qkv_lo, ld_qkv, col0, width, n, Lq, slots,
                                     (unsigned short*)kv_hi, (unsigned short*)kv_lo, ld_kv, page_ld * VIMA_KV_PAGE_TOKENS, pages, pool_pages,
                                     (cudaStream_t)stream),
           "slot_kv_scatter_paged");
}

int vima_slot_admit_prefix(vima_ctx* c, const int32_t* slots, int n, const uint8_t* prompt_mask, int Lp, int Lmax, uint8_t* slot_mask,
                           int32_t* len, int32_t* n_valid, int32_t* has_action, int32_t* active, void* stream) {
  CHECK_CTX(c);
  if (!slots || !prompt_mask || !slot_mask || !len || !n_valid || !has_action || !active)
    return fail(c, VIMA_E_INVALID, "slot_admit_prefix: null pointer");
  if (n < 0 || Lp < 0 || Lp + 1 > Lmax) return fail(c, VIMA_E_INVALID, "slot_admit_prefix: n >= 0, 0 <= Lp, Lp + 1 <= Lmax");
  LAUNCHED(c, launch_slot_admit_prefix(slots, n, prompt_mask, Lp, Lmax, slot_mask, len, n_valid, has_action, active, (cudaStream_t)stream),
           "slot_admit_prefix");
}

int vima_slot_assemble_history(vima_ctx* c, const float* obs, const uint8_t* obs_mask, const float* action, const int32_t* steps, int T, int n,
                               int Q, int E, int P, int L, float* tokens, uint8_t* mask, int64_t* pos, void* stream) {
  CHECK_CTX(c);
  if (!steps || !tokens || !mask || !pos || (T > 0 && (!obs || !action)))
    return fail(c, VIMA_E_INVALID, "slot_assemble_history: null pointer");
  auto al = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
  if (T < 0 || n < 0 || Q < 1 || E < 4 || (E & 3) || P < 0 || L < P || !al(obs) || !al(action) || !al(tokens))
    return fail(c, VIMA_E_INVALID, "slot_assemble_history: T >= 0, n >= 0, Q >= 1, E a positive multiple of 4, 0 <= P <= L, 16-byte aligned "
                                   "obs / action / tokens");
  LAUNCHED(c, launch_slot_assemble_history(obs, obs_mask, action, steps, T, n, Q, E, P, L, tokens, mask, (long long*)pos, (cudaStream_t)stream),
           "slot_assemble_history");
}

int vima_slot_admit_history(vima_ctx* c, const int32_t* slots, const int32_t* steps, int n, int S, int T, int Q, int P, int L,
                            const uint8_t* mask, const float* action, int E, int Lmax, uint8_t* slot_mask, int32_t* len, int32_t* n_valid,
                            int32_t* has_action, int32_t* active, float* action_token, void* stream) {
  CHECK_CTX(c);
  if (!slots || !steps || (L > 0 && !mask) || (T > 0 && !action) || !slot_mask || !len || !n_valid || !has_action || !active || !action_token)
    return fail(c, VIMA_E_INVALID, "slot_admit_history: null pointer");
  auto al = [](const void* q) { return ((uintptr_t)q & 15) == 0; };
  if (n < 0 || S < 1 || T < 0 || Q < 1 || P < 0 || L < P || L > Lmax || E < 4 || (E & 3) || !al(action) || !al(action_token))
    return fail(c, VIMA_E_INVALID, "slot_admit_history: n >= 0, S >= 1, T >= 0, Q >= 1, 0 <= P <= L <= Lmax, E a positive multiple of 4, "
                                   "16-byte aligned action / action_token");
  LAUNCHED(c, launch_slot_admit_history(slots, steps, n, S, T, Q, P, L, mask, action, E, Lmax, slot_mask, len, n_valid, has_action, active,
                                        action_token, (cudaStream_t)stream),
           "slot_admit_history");
}

int vima_kv_copy_blocks(vima_ctx* c, void* const* bufs, int n_buf, int64_t row_bytes, const int64_t* src_row0, const int64_t* dst_row0,
                        int n_blocks, int block_rows, int64_t buf_rows, void* stream) {
  CHECK_CTX(c);
  if (!bufs || !src_row0 || !dst_row0) return fail(c, VIMA_E_INVALID, "kv_copy_blocks: null pointer");
  if (((uintptr_t)bufs & 7) || ((uintptr_t)src_row0 & 7) || ((uintptr_t)dst_row0 & 7) || n_buf < 1 || n_buf > 65535 || row_bytes < 16 ||
      (row_bytes & 15) || block_rows < 1 || n_blocks < 0 || buf_rows < 0)
    return fail(c, VIMA_E_INVALID, "kv_copy_blocks: 1 <= n_buf <= 65535, row_bytes a positive multiple of 16, block_rows >= 1, "
                                   "n_blocks >= 0, buf_rows >= 0, 8-byte aligned device arrays");
  LAUNCHED(c, launch_kv_copy_blocks(bufs, n_buf, (long long)row_bytes, (const long long*)src_row0, (const long long*)dst_row0, n_blocks,
                                    block_rows, (long long)buf_rows, (cudaStream_t)stream),
           "kv_copy_blocks");
}

int vima_kv_pack_blocks(vima_ctx* c, void* const* bufs, int n_buf, int64_t row_bytes, const int64_t* row0, int n_blocks, int block_rows,
                        int64_t buf_rows, void* packed, int unpack, void* stream) {
  CHECK_CTX(c);
  if (!bufs || !row0 || !packed) return fail(c, VIMA_E_INVALID, "kv_pack_blocks: null pointer");
  if (((uintptr_t)bufs & 7) || ((uintptr_t)row0 & 7) || ((uintptr_t)packed & 15) || n_buf < 1 || n_buf > 65535 || row_bytes < 16 ||
      (row_bytes & 15) || block_rows < 1 || n_blocks < 0 || buf_rows < 0 || (unpack != 0 && unpack != 1))
    return fail(c, VIMA_E_INVALID, "kv_pack_blocks: 1 <= n_buf <= 65535, row_bytes a positive multiple of 16, block_rows >= 1, "
                                   "n_blocks >= 0, buf_rows >= 0, unpack 0 or 1, 8-byte aligned device arrays, 16-byte aligned packed");
  LAUNCHED(c, launch_kv_pack_blocks(bufs, n_buf, (long long)row_bytes, (const long long*)row0, n_blocks, block_rows, (long long)buf_rows,
                                    packed, unpack, (cudaStream_t)stream),
           "kv_pack_blocks");
}

int vima_add_pos_embed(vima_ctx* c, const float* tok, int64_t stride_b, int64_t stride_l, const int64_t* ids, const float* table, int n_pos, int B,
                       int L, int E, float* out_f32, void* hi, void* lo, int ld16, int dtype, int* err_flag, void* stream) {
  CHECK_CTX(c);
  if ((E & 3) || (stride_b & 3) || (stride_l & 3) || (hi && (ld16 & 3))) return fail(c, VIMA_E_INVALID, "add_pos_embed: alignment");
  LAUNCHED(c, launch_add_pos_embed(tok, stride_b, stride_l, (const long long*)ids, table, n_pos, B, L, E, out_f32, (unsigned short*)hi,
                                   (unsigned short*)lo, ld16, dtype, err_flag, (cudaStream_t)stream),
           "add_pos_embed");
}

int vima_gather_prompt(vima_ctx* c, const int32_t* kind, const int32_t* index, const int64_t* word_ids, const float* word_table,
                       const float* img_emb, const uint8_t* img_mask, int B, int Lp, int D, float* out, uint8_t* mask_out, void* stream) {
  CHECK_CTX(c);
  if (D & 3) return fail(c, VIMA_E_INVALID, "gather_prompt: D %% 4");
  LAUNCHED(c, launch_gather_prompt(kind, index, (const long long*)word_ids, word_table, img_emb, img_mask, B, Lp, D, out, mask_out,
                                   (cudaStream_t)stream),
           "gather_prompt");
}

int vima_patchify(vima_ctx* c, const uint8_t* img, int64_t N, int H, int W, int P, void* hi, void* lo, int ld16, int dtype, void* stream) {
  CHECK_CTX(c);
  if ((P & 3) || (H % P) || (W % P) || (ld16 & 3) || ld16 < 3 * P * P) return fail(c, VIMA_E_INVALID, "patchify: bad geometry");
  LAUNCHED(c, launch_patchify(img, N, H, W, P, (unsigned short*)hi, (unsigned short*)lo, ld16, dtype, (cudaStream_t)stream), "patchify");
}

int vima_vit_tokens(vima_ctx* c, const float* patch_out, const float* cls, const float* pos, int64_t N, int S, int W, float* out, void* stream) {
  CHECK_CTX(c);
  if (W & 3) return fail(c, VIMA_E_INVALID, "vit_tokens: W %% 4");
  LAUNCHED(c, launch_vit_tokens(patch_out, cls, pos, N, S, W, out, (cudaStream_t)stream), "vit_tokens");
}

int vima_bbox_norm(vima_ctx* c, const int64_t* bbox, int64_t n, float* out, void* stream) {
  CHECK_CTX(c);
  LAUNCHED(c, launch_bbox_norm((const long long*)bbox, n, out, (cudaStream_t)stream), "bbox_norm");
}

int vima_fill_ee(vima_ctx* c, const int64_t* ee, const float* table, int64_t n_te, int Q, void* hi, void* lo, int ld16, int col0, int n_pad,
                 int dtype, void* stream) {
  CHECK_CTX(c);
  LAUNCHED(c, launch_fill_ee((const long long*)ee, table, n_te, Q, (unsigned short*)hi, (unsigned short*)lo, ld16, col0, n_pad, dtype,
                             (cudaStream_t)stream),
           "fill_ee");
}

int vima_gato_positions(vima_ctx* c, const uint8_t* prompt_mask, int B, int Lp, int L, uint8_t* mask_out, int64_t* pos_out, void* stream) {
  CHECK_CTX(c);
  if (!prompt_mask || !mask_out || !pos_out || L < Lp) return fail(c, VIMA_E_INVALID, "gato_positions: bad arguments");
  LAUNCHED(c, launch_gato_positions(prompt_mask, B, Lp, L, mask_out, (long long*)pos_out, (cudaStream_t)stream), "gato_positions");
}

int vima_max_u8(vima_ctx* c, const uint8_t* x, int64_t n, int* out_max, void* stream) {
  CHECK_CTX(c);
  LAUNCHED(c, launch_max_u8(x, n, out_max, (cudaStream_t)stream), "max_u8");
}

int vima_action_scale(vima_ctx* c, const int64_t* idx, int64_t n, int width, const float* bins_dev, float* out, void* stream) {
  CHECK_CTX(c);
  LAUNCHED(c, launch_action_scale((const long long*)idx, n, width, bins_dev, out, (cudaStream_t)stream), "action_scale");
}

int vima_object_stats(vima_ctx* c, const void* segm, int segm_elem_bytes, int n_img, int H, int W, const int64_t* obj_ids_dev, int n_obj,
                      int ids_per_image, int32_t* stats, void* stream) {
  CHECK_CTX(c);
  if ((segm_elem_bytes != 1 && segm_elem_bytes != 4 && segm_elem_bytes != 8) || n_obj < 0 || n_obj > 64 || n_img < 0 || H <= 0 || W <= 0)
    return fail(c, VIMA_E_INVALID, "object_stats: segm elements of 1/4/8 bytes, at most 64 object ids per image");
  LAUNCHED(c, launch_object_stats(segm, segm_elem_bytes, n_img, H, W, (const long long*)obj_ids_dev, n_obj, ids_per_image, stats,
                                  (cudaStream_t)stream), "object_stats");
}

int vima_crop_resize(vima_ctx* c, const uint8_t* rgb, int n_img, int H, int W, const int32_t* stats, int n_obj, uint8_t* crops,
                     int64_t* bbox, uint8_t* mask, int32_t* n_valid, void* stream) {
  CHECK_CTX(c);
  if (n_obj < 0 || n_obj > 64 || n_img < 0 || n_img > 65535 || H <= 0 || W <= 0)
    return fail(c, VIMA_E_INVALID, "crop_resize: at most 64 object ids per image and 65535 images per call");
  LAUNCHED(c, launch_crop_resize(rgb, n_img, H, W, stats, n_obj, crops, (long long*)bbox, mask, n_valid, (cudaStream_t)stream),
           "crop_resize");
}

int vima_action_postprocess(vima_ctx* c, const int64_t* idx, int64_t n, int width, const float* bins_dev, const float* lo_dev,
                            const float* hi_dev, int bound_stride, float* out, void* stream) {
  CHECK_CTX(c);
  if (width <= 0 || n < 0 || (bound_stride != 0 && bound_stride < width))
    return fail(c, VIMA_E_INVALID, "action_postprocess: width > 0, n >= 0, bound_stride 0 (broadcast) or >= width");
  LAUNCHED(c, launch_action_post((const long long*)idx, n, width, bins_dev, lo_dev, hi_dev, bound_stride, out, (cudaStream_t)stream),
           "action_postprocess");
}

int vima_head_select(vima_ctx* c, const float* logits, int B, int n_heads, const int32_t* head_off_dev, float* logits_norm, int64_t* modes,
                     void* stream) {
  CHECK_CTX(c);
  LAUNCHED(c, launch_head_select(logits, B, n_heads, head_off_dev, logits_norm, (long long*)modes, (cudaStream_t)stream), "head_select");
}

int vima_head_sample(vima_ctx* c, const vima_head_sample_desc* desc, void* stream) {
  CHECK_CTX(c);
  vima_head_sample_desc d;
  if (int rc = load_desc(c, desc, &d, sizeof(vima_head_sample_desc), "head_sample")) return rc;
  const bool draw = !d.actions_in && !d.greedy;
  if (d.B < 0 || d.n_heads <= 0 || (d.B > 0 && (!d.logits || !d.head_off_dev || (!d.actions_in && !d.actions_out))) ||
      (draw && !d.counter_dev))
    return fail(c, VIMA_E_INVALID, "head_sample: needs n_heads > 0, B >= 0, counter_dev when drawing, and for B > 0 logits, head_off "
                                   "and actions_out unless actions_in is given");
  HeadParams p = {};
  p.logits = d.logits; p.B = d.B; p.n_heads = d.n_heads; p.head_off = d.head_off_dev;
  p.mode = d.actions_in ? HEAD_SCORE : (d.greedy ? HEAD_SELECT : HEAD_SAMPLE);
  p.actions_in = (const long long*)d.actions_in;
  p.seed = d.seed;
  p.counter = (const unsigned long long*)d.counter_dev;
  p.actions_out = (long long*)d.actions_out;
  p.log_prob = d.log_prob; p.entropy = d.entropy; p.logits_norm = d.logits_norm;
  const cudaError_t e = launch_head_kernel(p, (cudaStream_t)stream);
  if (e != cudaSuccess) return cuda_fail(c, e, "head_sample");
  c->launches += head_kernel_launches(p);
  return VIMA_OK;
}
int vima_sizeof_head_sample_desc(void) { return (int)sizeof(vima_head_sample_desc); }

}  // extern "C"
