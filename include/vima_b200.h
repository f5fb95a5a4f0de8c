/*
 * vima_b200 -- C ABI of the H100 (sm_90a) kernels behind the VIMA policy forward pass.
 *
 * The reference (vimalabs/VIMA) is pure Python/PyTorch and has no FFI of its own (SURVEY.md 8(b)); its
 * operator surface is the `vima.nn` module tree.  Every entry point below replaces the arithmetic of one
 * reference module `forward` (cited per function, paths relative to the reference root; `HF:` = the
 * `transformers` package it subclasses) and is what a maintainer would bind from those modules -- see
 * INTEGRATION.md for the ctypes stub.
 *
 * Conventions
 *   - plain C: raw DEVICE pointers, explicit sizes / leading dimensions (in elements), a `cudaStream_t` passed
 *     as `void*`.  No torch types.  The caller owns every buffer; the library owns only the context.
 *   - every call is asynchronous on the given stream and performs no host synchronisation.
 *   - return value: 0 = ok, otherwise a VIMA_E_* code; `vima_last_error(ctx)` gives the message.  Never throws.
 *   - one context per (device, host thread); not thread-safe.
 *   - 16-bit GEMM operands: activations and packed weights are K-major arrays of fp16 (VIMA_DT_F16) or bf16
 *     (VIMA_DT_BF16).  In split mode every operand is a (hi, lo) PAIR of such arrays with x ~= hi + lo and the
 *     kernels accumulate hi*hi + lo*hi + hi*lo in fp32, which reproduces the reference's fp32 products to
 *     ~1e-5 rel end to end (DESIGN.md "operand precision").  `lo == NULL` selects single-pass mode.
 *   - `ld*` of 16-bit operand arrays must be multiples of 8 elements and base pointers 16-byte aligned (TMA).
 *   - descriptor structs (`vima_*_desc`) start with `uint32_t struct_size` = sizeof(the struct the CALLER was compiled
 *     against).  The library accepts any size between the struct's ABI-v4 size (the fields up to the `v4 end` comment) and its own
 *     sizeof -- fields the caller does not know about read as zero / NULL -- and rejects everything else with
 *     VIMA_E_INVALID, so growing a descriptor never makes an old binding read or write through garbage.
 *     `vima_sizeof_*()` report the library's own sizes (bindings assert equality at load time).
 *   - the calling thread's current CUDA device is saved and restored around every call.
 *   - environment (read ONCE, in vima_create): VIMA_B200_ATTN = tc (default) | mma;  VIMA_B200_ATTN_TAIL = kernel (default) | off;
 *     VIMA_B200_EPI_PREFETCH = 0 (default) | 1;  VIMA_B200_ATTN_BIAS = auto (default) | tc;  VIMA_B200_GEMM_WIDE = 1 (default) | 0.
 */
#ifndef VIMA_B200_H
#define VIMA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#pragma GCC visibility push(default)

#define VIMA_B200_ABI_VERSION 5

enum { VIMA_OK = 0, VIMA_E_INVALID = 1, VIMA_E_CUDA = 2, VIMA_E_UNSUPPORTED = 3 };
enum { VIMA_DT_F16 = 0, VIMA_DT_BF16 = 1 };
enum { VIMA_ACT_NONE = 0, VIMA_ACT_RELU = 1, VIMA_ACT_QUICKGELU = 2, VIMA_ACT_GELU = 3 /* erf, nn.GELU() */,
       VIMA_ACT_GELU_TANH = 4 /* HF NewGELUActivation, OpenAIGPTConfig.afn = "gelu" */ };

typedef struct vima_ctx vima_ctx;

int vima_abi_version(void);
/* Creates a context on `device` (cudaSetDevice is applied inside every call). Fails if the device is not sm_90. */
int vima_create(vima_ctx** out, int device);
void vima_destroy(vima_ctx* ctx);
const char* vima_last_error(vima_ctx* ctx);
int vima_sm_count(vima_ctx* ctx);
/* Kernel-selection options, initialised from the environment in vima_create (see "environment" above) and switchable per context:
 * key "attn" = "tc" | "mma";  "attn_tail" = "kernel" | "off" (the <= 8 query rows past the last full 128-row tile: SIMT tail
 * kernel, or one more wgmma tile);
 * "epi_prefetch" = "1" | "0";
 * "gemm_wide" = "1" | "0" (f16f8 GEMMs whose tiles are 128 wide and N % 256 == 0, with an epilogue of the specialised list: "1" runs
 * each pair of adjacent tiles as one 128 x 256 tile, a quarter less operand traffic from L2 per multiply-add; results, the GLU
 * pairing and stats_parts are those of the 128-wide tiles, up to the rounding of the e4m3 cross terms' fp16 sum);
 * "attn_bias" = "auto" | "tc" (relative-bias attention, head_dim 64, non-causal -- the T5 encoder: "auto" runs the K/V-streaming
 * wgmma kernel only where the resident-K/V kernel's shared memory does not fit, "tc" at every length; needs "attn" = "tc").
 * Unknown key/value: VIMA_E_INVALID. */
int vima_set_option(vima_ctx* ctx, const char* key, const char* value);
/* sizeof() of the descriptor structs as THIS library was compiled (bindings check their mirror structs against these). */
int vima_sizeof_gemm_desc(void);
int vima_sizeof_norm_desc(void);
int vima_sizeof_attn_desc(void);
int vima_sizeof_f32_gemm_group(void);
/* Number of kernels this context has launched so far (bench.py's `gpu_launches`). */
int64_t vima_launch_count(vima_ctx* ctx);

/* ---- operand preparation ------------------------------------------------------------------------------- */
/* fp32 [rows, cols] (ldx) -> 16-bit operands (hi, lo|NULL) [rows, ld16]; columns [cols, pad_cols) are zeroed. */
int vima_split_f32(vima_ctx*, const float* x, int64_t rows, int cols, int ldx, void* hi, void* lo, int ld16, int pad_cols,
                   float scale, int dtype, void* stream);
/* Weight packing: w is [n, k] (nn.Linear.weight) or, if transposed != 0, [k, n] (HF Conv1D.weight,
 * HF:pytorch_utils.py:97-123).  Output: K-major (hi, lo|NULL) [n, ld16], zero padded, multiplied by `scale`. */
int vima_pack_weight(vima_ctx*, const float* w, int n, int k, int transposed, int ldw, void* hi, void* lo, int ld16, float scale,
                     int dtype, void* stream);
/* Same source, e4m3 cross-term views for the "f16f8" GEMM mode: hi8 = e4m3(w*scale*2^-10), lo8 = e4m3((w*scale - f16(w*scale))*2^3). */
int vima_pack_weight_f8(vima_ctx*, const float* w, int n, int k, int transposed, int ldw, void* hi8, void* lo8, int ld8, float scale,
                        void* stream);

/* ---- wgmma GEMM: out = epilogue(A[M,K] * B[N,K]^T) ------------------------------------------------------
 * Replaces every large Linear / Conv1D on the path: components.py:87-88,130-142 (c_attn, c_proj, c_fc, query,
 * key_value, attention_out, linear1/2, gated_layer), vit.py:151-157,203-213 (conv1, in/out_proj, mlp),
 * obj_encoder.py:86-93, prompt_encoder.py T5 q/k/v/o/wi/wo, vima_policy.py:49,97-108.
 * Epilogue order: v = acc*acc_scale + bias[col]; v = act(v); GLU: v *= (acc2*acc_scale + bias[col2]);
 * v *= mul[row,col]; v += residual[row,col]; store fp32 and/or (hi, lo).
 * GLU mode: B holds, per tile of block_n accumulator columns, block_n/2 "value" rows followed by the matching
 * block_n/2 "gate" rows (see vima_glu_block_n); N = 2 * output columns. */
typedef struct {
  uint32_t struct_size;    /* = sizeof(vima_gemm_desc) of the caller's header */
  int M, N, K;
  const void *a_hi, *a_lo; /* [M, lda] */
  int lda;
  const void *b_hi, *b_lo; /* [N, ldb] packed weights */
  int ldb;
  int dtype;
  int glu;
  int act;
  float acc_scale;
  const float* bias;     /* [N] or NULL */
  const float* mul;      /* fp32 [M, ld_mul] or NULL */
  int ld_mul;
  const float* residual; /* fp32 [M, ld_res] or NULL */
  int ld_res;
  float* out_f32;        /* or NULL */
  int ld_o32;
  void *out_hi, *out_lo; /* 16-bit outputs or NULL */
  int ld_o16;
  int block_n;           /* 0 = choose */
  /* "f16f8" mode (fp16 operands only): fp16 hi*hi plus two e4m3 cross terms at the fp8 rate. a_lo8 = e4m3((a-a_hi)*2^10),
   * a_hi8 = e4m3(a*2^-3), b_hi8 = e4m3(b*2^-10), b_lo8 = e4m3((b-b_hi)*2^3); [rows, ld8] bytes, ld8 % 16 == 0.  Set all four
   * (and leave a_lo / b_lo NULL) to select it.  out_lo8 / out_hi8 make the epilogue emit the same views of its output. */
  const void *a_lo8, *a_hi8;
  int lda8;
  const void *b_hi8, *b_lo8;
  int ldb8;
  void *out_lo8, *out_hi8;
  int ld_o8;
  /* ---- v4 end: later releases append below; callers built against v4 pass the v4 size and the tail reads as zero ---- */
  /* v5: LayerNorm folded into the GEMM (DESIGN.md "LN folding"; components.py:128,135 `ln`, components.py:19-21 `ln_1`).
   * A holds the UN-normalised rows x, the packed weights hold W*gamma and `bias` holds b + W*beta; the epilogue applies
   *     v = rstd[row] * (acc*acc_scale - mean[row] * ln_c1[col]) + bias[col],   ln_c1[col] = sum_k (W*gamma)[col, k]
   * to every accumulator column (ln_cols = 1) or only to the value half of each GLU tile (ln_cols = 2: the gate reads x).
   * row_stats: fp32 [M, 2] = (mean, rstd) per row (vima_row_stats_finalize). */
  const float* row_stats;
  const float* ln_c1;    /* [N], accumulator-column order like `bias` */
  int ln_cols;
  /* v5: the residual rows are LayerNorm'd on the fly (post-LN block, components.py:31-36: the residual of the MLP is ln_1(s)):
   *     r = (residual[row,col] - mean[row]) * rstd[row] * res_gamma[col] + res_beta[col],  res_stats fp32 [M, 2]. Not with GLU. */
  const float* res_stats;
  const float* res_gamma;
  const float* res_beta;
  /* v5: per-row partial (sum, sum of squares) of the stored output, one pair per (n-tile, epilogue half):
   * stats_out fp32 [M, stats_parts, 2] with stats_parts = vima_gemm_stats_parts(N, glu, block_n). */
  float* stats_out;
  int stats_parts;
} vima_gemm_desc;
#define VIMA_GEMM_DESC_V4_SIZE offsetof(vima_gemm_desc, row_stats)
int vima_gemm(vima_ctx*, const vima_gemm_desc* d, void* stream);
/* Accumulator tile width the GLU weight interleave must use for an output width of n_out columns. */
int vima_glu_block_n(int n_out);
/* Number of partial-statistics slots per row a GEMM with N accumulator columns writes (`stats_out`); block_n 0 = the library's choice. */
int vima_gemm_stats_parts(int N, int glu, int block_n);
/* partial [rows, parts, 2] (sum, sum of squares over disjoint column sets covering `cols` columns) -> stats [rows, 2] =
 * (mean, 1/sqrt(var + eps)), biased variance like nn.LayerNorm; rms != 0: (0, 1/sqrt(mean(x^2) + eps)) for a folded T5 RMSNorm
 * (HF:modeling_t5.py:46-68). */
int vima_row_stats_finalize(vima_ctx*, const float* partial, int64_t rows, int parts, int cols, float eps, int rms, float* stats, void* stream);

/* ---- exact fp32 grouped GEMM (CUDA cores) for the tiny layers -------------------------------------------------
 * action_decoder.py:151-166 (12 MLPs E->512->512->{50|100}), action_embd.py:29-56, obj_encoder.py:86 first layer.
 * `groups` is a DEVICE array of n_groups descriptors; y[M, n] = act(x[M, k] * w[n, k]^T + b).  Every output accumulates its
 * products in ascending k with one fused multiply-add each, then adds b in fp32: bit for bit the same at any M or grouping.
 * Precondition: max_n >= every group's n.  max_n sets the launch's column tiles, so the columns of a wider group past max_n are
 * never written; the descriptors live on the device, so this entry point cannot check it. */
typedef struct {
  const float* x; int ldx;
  const float* w; int ldw;
  const float* b;
  float* y; int ldy;
  int n, k;
} vima_f32_gemm_group;
int vima_gemm_f32_grouped(vima_ctx*, const vima_f32_gemm_group* groups_dev, int n_groups, int M, int max_n, int act, void* stream);
/* Same, with the descriptor array in HOST memory: the descriptors travel in the kernel's parameter space (16 per launch), so no
 * device-side array has to stay alive and the call can be captured into a CUDA graph.  Returns VIMA_E_INVALID, and launches
 * nothing, when M < 0 or a group's n exceeds max_n. */
int vima_gemm_f32_grouped_host(vima_ctx*, const vima_f32_gemm_group* groups_host, int n_groups, int M, int max_n, int act, void* stream);

/* ---- LayerNorm / T5 RMSNorm over rows ---------------------------------------------------------------------
 * nn.LayerNorm eps 1e-5 (components.py:19,21,128,135; vit.py:164,168,204,214) and HF T5LayerNorm
 * (HF:modeling_t5.py:46-68).  y1 = norm1(x + add); optional y2 = LayerNorm2(y1).  Outputs: y1 fp32, y2 fp32,
 * and the LAST computed norm as (hi, lo) operands.  w == NULL skips norm1 (pure add / convert). cols % 4 == 0,
 * cols <= 1024. */
typedef struct {
  uint32_t struct_size;    /* = sizeof(vima_norm_desc) of the caller's header */
  const float* x; int64_t rows; int cols; int ldx;
  const float* add; int ld_add;
  const float* w; const float* b; float eps; int rms;
  const float* w2; const float* b2; float eps2;
  float* out_f32; int ld_o32;
  float* out2_f32; int ld_o2;
  void *out_hi, *out_lo; int ld_o16;
  int dtype;
  void *out_lo8, *out_hi8; int ld_o8; /* optional e4m3 cross-term views of the last norm's output (fp16 format) */
  /* ---- v4 end ---- */
  /* v5: (mean, rstd = 1/sqrt(var + stats_eps)) of the rows of y1 (rms != 0: (0, 1/sqrt(mean(y1^2) + stats_eps))), fp32 [rows, 2] -- the row statistics a GEMM with a folded
   * LayerNorm (vima_gemm_desc.row_stats) takes when y1 itself, not its LayerNorm, is what gets written out. */
  float* stats_out; float stats_eps;
} vima_norm_desc;
#define VIMA_NORM_DESC_V4_SIZE offsetof(vima_norm_desc, stats_out)
int vima_norm(vima_ctx*, const vima_norm_desc* d, void* stream);

/* ---- fused masked attention -----------------------------------------------------------------------------------
 * Self-attention of the causal block (components.py:51-80: /sqrt(d), soft causal mask w*b + -1e4*(1-b), additive
 * key mask finfo.min), cross-attention (components.py:179-214) and T5 self-attention (prompt_encoder.py:769-816:
 * no scaling, shared relative-position bias + mask).  q/k/v/o pointers address head 0's first column; head h is
 * at +h*D.  key_mask: uint8 [B, Lk] (1 = attend) or NULL.  rel_bias: fp32 [H, 2*Lk-1] indexed by (j-i+Lk-1). */
typedef struct {
  uint32_t struct_size;    /* = sizeof(vima_attn_desc) of the caller's header */
  const void *q_hi, *q_lo; int ldq;
  const void *k_hi, *k_lo; int ldk;
  const void *v_hi, *v_lo; int ldv;
  const uint8_t* key_mask;
  const float* rel_bias;
  void *o_hi, *o_lo; int ldo;
  int B, H, Lq, Lk, D;
  float scale;
  int causal;
  int dtype;
  void *o_lo8, *o_hi8; int ldo8; /* optional e4m3 cross-term views of the output */
  /* KV-cache addressing (incremental decode, SURVEY.md 8(f)1): k/v rows of batch element b start at b*kv_batch_rows (0 = Lk),
   * key_mask rows have pitch mask_ld (0 = Lk), and under `causal` query row i sits at key position q_pos0 + i. */
  int kv_batch_rows, mask_ld, q_pos0;
  /* ---- v4 end ---- */
  /* v5: per-batch causal positions (slot decode: every episode of the batch at its own history length).  DEVICE int [B] or NULL.
   * When set (causal only, no rel_bias), batch element b has query row i at key position q_pos[b] + i and Lk_b = q_pos[b] + Lq
   * keys; `Lk` then only bounds the capacity (q_pos[b] in [0, Lk - Lq]) and q_pos0 is ignored. */
  const int* q_pos;
  /* ---- v5 end ---- */
  /* v6 tail (an addition; the ABI version stays 5): paged k / v (slot decode).  DEVICE int32 [B, kv_page_ld] or NULL.  When set,
   * key j of batch element b is row kv_pages[b*kv_page_ld + j/64]*64 + j%64 of k / v, a pool of kv_pool_pages 64-row pages
   * (kv_batch_rows is ignored); an entry outside [0, kv_pool_pages) reads page 0.  Needs q_pos or non-causal attention, no
   * rel_bias, Lk <= kv_page_ld*64 and kv_pool_pages*64 < 2^31.  Every kernel reads whole pages: rows of a page past the keys a call
   * attends must hold finite values (a slot cache keeps them zero). */
  const int32_t* kv_pages;
  int kv_page_ld, kv_pool_pages;
  /* v7 tail (an addition; the ABI version stays 5): per-batch key count (slot decode's cross-attention over prompts of different
   * lengths).  DEVICE int32 [B] or NULL.  When set, batch element b attends keys [0, clamp(kv_len[b], 1, Lk)); keys past that count
   * are excluded like keys past Lk (and whole 64-key chunks past it are never read).  Non-causal only, without q_pos or rel_bias. */
  const int32_t* kv_len;
} vima_attn_desc;
#define VIMA_ATTN_DESC_V4_SIZE offsetof(vima_attn_desc, q_pos)
#define VIMA_ATTN_DESC_V5_SIZE offsetof(vima_attn_desc, kv_pages)
#define VIMA_ATTN_DESC_V6_SIZE offsetof(vima_attn_desc, kv_len)
#define VIMA_ATTN_DESC_V7_SIZE sizeof(vima_attn_desc)
#define VIMA_KV_PAGE_TOKENS 64 /* rows of one K/V page: the streaming attention kernel's key chunk */
int vima_attention(vima_ctx*, const vima_attn_desc* d, void* stream);

/* HF modeling_perceiver.py PerceiverSelfAttention (the resampler of vima/nn/obj_encoder/perceiver/perceiver.py:11-41), fp32:
 * o[n,i,h*d:(h+1)*d] = softmax_j(q[n,i,h] . k[n,j,h] * scale) v[n,j,h]; Lk <= 16, d <= 128; q_batch_stride 0 shares the queries
 * (the learned latents of the cross-attention layer) between all N images. */
int vima_latent_attention(vima_ctx*, const float* q, int ldq, int64_t q_batch_stride, const float* k, int ldk, const float* v, int ldv, float* o,
                          int ldo, int64_t N, int Lq, int Lk, int H, int d, float scale, void* stream);
/* nn.MultiheadAttention core on tiny sequences (ViT, vit.py:203,224-230): fp32 qkv [N*S, ld] (q|k|v, W wide each,
 * bias included) -> (hi, lo) [N*S, ldo].  head_dim must be 32, S <= 16. */
int vima_small_attention(vima_ctx*, const float* qkv, int ld, int64_t N, int S, int H, int W, float scale, void* o_hi, void* o_lo,
                         int ldo, float* o_f32, int dtype, void* stream);

/* ---- token assembly ------------------------------------------------------------------------------------------
 * vima_policy.py:124-147: interleave obs (T,B,Q,E) / action (La,B,E) tokens into (L,B,E), L = T*Q + La; masks
 * (B,L) uint8 (action slots 1); position ids (B,L) int64 = cumsum(mask)-1. */
int vima_assemble_history(vima_ctx*, const float* obs, const uint8_t* obs_mask, const float* action, int T, int B, int Q, int E, int La,
                          float* tokens, uint8_t* masks_bl, int64_t* pos_bl, void* stream);
/* pos[b, l] = cumsum(mask[b, :l+1]) - 1   (vima_policy.py:147) */
int vima_mask_cumsum(vima_ctx*, const uint8_t* mask, int B, int L, int64_t* pos, void* stream);

/* ---- slot decode: every row of the batch is a slot holding one episode at its own history length (DESIGN.md 7 (f)1) ----------
 * Per-slot DEVICE state, int32 [S] each: len (cache columns used), n_valid (next position id), has_action (0 before the slot's
 * first step), active.  A step block has Q+1 rows per slot: [action, obs_1..obs_Q] once the slot has an action, else
 * [obs_1..obs_Q, dummy] with a zero, masked dummy row that no real row sees (causality) and the next step overwrites.
 * step_begin: obs fp32 [S, Q, E], obs_mask uint8 [S, Q], action fp32 [S, E] -> tokens fp32 [S*(Q+1), E], step_mask uint8 [S, Q+1],
 * pos int64 [S, Q+1] (n_valid + running count of valid tokens - 1; 0 on inactive slots), q_pos int32 [S] (len, 0 on inactive slots),
 * and step_mask into columns q_pos .. q_pos+Q of slot_mask uint8 [S, Lmax]. */
int vima_slot_step_begin(vima_ctx*, const float* obs, const uint8_t* obs_mask, const float* action, int S, int Q, int E, int Lmax,
                         const int32_t* len, const int32_t* n_valid, const int32_t* has_action, const int32_t* active, float* tokens,
                         uint8_t* step_mask, int64_t* pos, int32_t* q_pos, uint8_t* slot_mask, void* stream);
/* Per layer: columns [col0, col0 + width) of the step's rows qkv [S*Lq, ld_qkv] (hi, lo|NULL 16-bit) -> cache rows
 * b*Lmax + q_pos[b] + r of kv [S*Lmax, ld_kv].  width, col0, ld_* multiples of 8 elements, 16-byte aligned bases. */
int vima_slot_kv_append(vima_ctx*, const void* qkv_hi, const void* qkv_lo, int ld_qkv, int col0, int width, int S, int Lq, const int32_t* q_pos,
                        void* kv_hi, void* kv_lo, int ld_kv, int Lmax, void* stream);
/* vima_slot_kv_append into a paged cache: cache column col of slot b is row pages[b*page_ld + col/64]*64 + col%64 of kv, a pool of
 * pool_pages 64-row pages ([pool_pages*64, ld_kv]); pages: DEVICE int32 [S, page_ld].  Columns past page_ld*64 and writes to page 0
 * (the zero page) or to an entry outside [1, pool_pages) are skipped. */
int vima_slot_kv_append_paged(vima_ctx*, const void* qkv_hi, const void* qkv_lo, int ld_qkv, int col0, int width, int S, int Lq,
                              const int32_t* q_pos, void* kv_hi, void* kv_lo, int ld_kv, const int32_t* pages, int page_ld, int pool_pages,
                              void* stream);
/* out[b] = x[b*(Q+1) + Q-1+has_action[b]] (fp32 rows of E, pitch ldx); then, for active slots, len += Q + has_action,
 * n_valid += sum(step_mask[b]), has_action = 1. */
int vima_slot_step_end(vima_ctx*, const float* x, int ldx, int S, int Q, int E, const uint8_t* step_mask, int32_t* len, int32_t* n_valid,
                       int32_t* has_action, const int32_t* active, float* out, void* stream);
/* Decoder-only admission (VIMA-Gato / VIMA-GPT: prompt + separator live in the self-attention cache).  Per layer: columns
 * [col0, col0 + width) of the prefill rows qkv [n*Lq, ld_qkv] (hi, lo|NULL 16-bit) -> cache rows slots[j]*Lmax + r (r < Lq) of
 * kv [S*Lmax, ld_kv]; slots: DEVICE int32 [n], distinct.  Lq <= Lmax; width, col0, ld_* multiples of 8 elements, 16-byte aligned. */
int vima_slot_kv_scatter(vima_ctx*, const void* qkv_hi, const void* qkv_lo, int ld_qkv, int col0, int width, int n, int Lq, const int32_t* slots,
                         void* kv_hi, void* kv_lo, int ld_kv, int Lmax, void* stream);
/* vima_slot_kv_scatter into a paged cache (page table and pool as vima_slot_kv_append_paged): prefill row (j, r) -> row
 * pages[slots[j]*page_ld + r/64]*64 + r%64 of kv; Lq <= page_ld*64; writes to page 0 or outside the pool are skipped. */
int vima_slot_kv_scatter_paged(vima_ctx*, const void* qkv_hi, const void* qkv_lo, int ld_qkv, int col0, int width, int n, int Lq,
                               const int32_t* slots, void* kv_hi, void* kv_lo, int ld_kv, const int32_t* pages, int page_ld, int pool_pages,
                               void* stream);
/* For each admitted slot b = slots[j] (DEVICE int32 [n]): slot_mask[b, 0:Lp] = prompt_mask[j] (uint8 [n, Lp]), slot_mask[b, Lp] = 1;
 * len[b] = Lp+1, n_valid[b] = sum(prompt_mask[j] != 0) + 1, has_action[b] = 0, active[b] = 1.  Lp + 1 <= Lmax. */
int vima_slot_admit_prefix(vima_ctx*, const int32_t* slots, int n, const uint8_t* prompt_mask, int Lp, int Lmax, uint8_t* slot_mask,
                           int32_t* len, int32_t* n_valid, int32_t* has_action, int32_t* active, void* stream);
/* Slot episodes admitted mid-way from a recorded history (no reference counterpart: it re-runs the whole history every step).  Episode
 * j has completed k_j = steps[j] environment steps (DEVICE int32 [n], clamped to [0, T]); its history columns are forward's
 * [o_0 (Q tokens), a_0, o_1, ..., a_{k-2}, o_{k-1}]: k_j(Q+1) - 1 of them, 0 for k_j = 0.  Rows t >= k_j of obs / obs_mask / action
 * are never read.
 * slot_assemble_history: obs fp32 (T, n, Q, E), obs_mask uint8 (T, n, Q) (NULL = every obs token valid), action fp32 (T, n, E) ->
 * rows [P, L) of tokens fp32 (L, n, E) and columns [P, L) of mask uint8 [n, L] / pos int64 [n, L]: history column c of episode j
 * goes to column P + c; pos = (valid columns of mask[j, 0:P), written by the caller) + cumsum(history mask) - 1.  Columns past
 * the history get a zero token, mask 0 and position id 0.  E % 4 == 0; obs, action, tokens 16-byte aligned.
 * slot_admit_history: for each episode j, slot b = slots[j] (DEVICE int32 [n]; skipped outside [0, S) or when P + its history
 * columns exceed L): slot_mask[b, c] = mask[j, c] for c < len, 0 for len <= c < Lmax, where len = P + history columns;
 * len[b] = len, n_valid[b] = valid columns of mask[j, 0:len], has_action[b] = (k_j > 0), active[b] = 1, and for k_j > 0
 * action_token[b] (fp32 [S, E]) = action[k_j - 1, j].  L <= Lmax. */
int vima_slot_assemble_history(vima_ctx*, const float* obs, const uint8_t* obs_mask, const float* action, const int32_t* steps, int T, int n,
                               int Q, int E, int P, int L, float* tokens, uint8_t* mask, int64_t* pos, void* stream);
int vima_slot_admit_history(vima_ctx*, const int32_t* slots, const int32_t* steps, int n, int S, int T, int Q, int P, int L,
                            const uint8_t* mask, const float* action, int E, int Lmax, uint8_t* slot_mask, int32_t* len, int32_t* n_valid,
                            int32_t* has_action, int32_t* active, float* action_token, void* stream);
/* Forked slots (no reference counterpart: it runs one episode per call): copy block i of block_rows rows from row src_row0[i] to row
 * dst_row0[i] in each of n_buf buffers of the same row width -- the copy on write of a shared K/V page (block_rows = 64, every
 * layer's hi and lo pool) and a fork's prompt K/V rows (block_rows = Lp_cap).  bufs: DEVICE array of n_buf base pointers, each a
 * buffer of buf_rows rows of row_bytes bytes (row_bytes a positive multiple of 16, bases 16-byte aligned; a null or misaligned
 * base is skipped); src_row0 / dst_row0: DEVICE int64 [n_blocks].  A block whose start lies outside [0, buf_rows - block_rows]
 * is skipped, never written.  Destination blocks must not overlap any block's source rows. */
int vima_kv_copy_blocks(vima_ctx*, void* const* bufs, int n_buf, int64_t row_bytes, const int64_t* src_row0, const int64_t* dst_row0,
                        int n_blocks, int block_rows, int64_t buf_rows, void* stream);
/* Swapped slot episodes (no reference counterpart): move block i of block_rows rows at row row0[i] of each of the n_buf buffers
 * (bufs, row_bytes, buf_rows and the skipping rules as vima_kv_copy_blocks) to or from one packed DEVICE buffer laid out
 * [block][buffer][block_rows][row_bytes], so consecutive blocks are one contiguous slice.  unpack = 0: buffers -> packed (pack);
 * unpack = 1: packed -> buffers.  row0: DEVICE int64 [n_blocks]; packed 16-byte aligned.  A skipped block's packed rows are
 * neither read nor written.  Unpacked blocks must not overlap each other. */
int vima_kv_pack_blocks(vima_ctx*, void* const* bufs, int n_buf, int64_t row_bytes, const int64_t* row0, int n_blocks, int block_rows,
                        int64_t buf_rows, void* packed, int unpack, void* stream);
/* out[b,l,:] = tok[b*stride_b + l*stride_l + :] + table[ids[b,l]]  (xattn_gpt.py:103-105,110-114); out-of-range
 * ids set *err_flag (device int) to 1 -- the reference raises IndexError there. */
int vima_add_pos_embed(vima_ctx*, const float* tok, int64_t stride_b, int64_t stride_l, const int64_t* ids, const float* table, int n_pos,
                       int B, int L, int E, float* out_f32, void* hi, void* lo, int ld16, int dtype, int* err_flag, void* stream);
/* fp32 [rows, cols] -> e4m3 cross-term views (lo8 relative to the fp16 hi part, hi8), [rows, ld8] bytes. cols % 4 == 0. */
int vima_split_f8(vima_ctx*, const float* x, int64_t rows, int cols, int ldx, void* lo8, void* hi8, int ld8, void* stream);
/* vima_policy.py:180-233: prompt gather driven by a (kind, index) map per (b, position), see misc.cu. */
int vima_gather_prompt(vima_ctx*, const int32_t* kind, const int32_t* index, const int64_t* word_ids, const float* word_table,
                       const float* img_emb, const uint8_t* img_mask, int B, int Lp, int D, float* out, uint8_t* mask_out, void* stream);

/* vima_gato_policy.py:150-182 (decoder-only baseline): mask [B,L] = [prompt_mask | ones]; position ids: arange over the n
 * valid prompt tokens, n-1 on padded prompt slots, then n, n+1, ... */
int vima_gato_positions(vima_ctx*, const uint8_t* prompt_mask, int B, int Lp, int L, uint8_t* mask_out, int64_t* pos_out, void* stream);

/* ---- object-encoder front end ---------------------------------------------------------------------------------
 * preprocess.py:23-43 + vit.py:151-157,172: uint8 crops (N,3,H,W) -> normalised patch rows (hi, lo) [N*(H/P)*(W/P), ld16]. */
int vima_patchify(vima_ctx*, const uint8_t* img, int64_t N, int H, int W, int P, void* hi, void* lo, int ld16, int dtype, void* stream);
/* vit.py:173-179: tokens[n,0] = cls + pos[0]; tokens[n,1+p] = patch_out[n*(S-1)+p] + pos[1+p].
 * cls == NULL (Gato ViT, vit.py:123-126): tokens[n,s] = patch_out[n*S+s] + pos[s]. */
int vima_vit_tokens(vima_ctx*, const float* patch_out, const float* cls, const float* pos, int64_t N, int S, int W, float* out, void* stream);
/* obj_encoder.py:79-85 */
int vima_bbox_norm(vima_ctx*, const int64_t* bbox, int64_t n, float* out, void* stream);
/* vima_policy.py:253-256: end-effector embedding columns of the obs-fusion operand. */
int vima_fill_ee(vima_ctx*, const int64_t* ee, const float* table, int64_t n_te, int Q, void* hi, void* lo, int ld16, int col0, int n_pad,
                 int dtype, void* stream);
/* preprocess.py:28 range check: *out_max = max(*out_max, max(x)) (device int). */
int vima_max_u8(vima_ctx*, const uint8_t* x, int64_t n, int* out_max, void* stream);

/* ---- observation / prompt-asset preparation: the step before the path (scripts/example.py:243-473) ------------- */
/* example.py:409-416 / 279-286: per (image, object id) pixel count and bounding box of `segm == id`.
 * segm [n_img,H,W] with 1-, 4- or 8-byte integer elements; obj_ids_dev int64 [n_obj] (shared) or [n_img,n_obj] when
 * ids_per_image; stats int32 [n_img,n_obj,5] = {count, xmin, xmax, ymin, ymax}.  n_obj <= 64. */
int vima_object_stats(vima_ctx*, const void* segm, int segm_elem_bytes, int n_img, int H, int W, const int64_t* obj_ids_dev, int n_obj,
                      int ids_per_image, int32_t* stats, void* stream);
/* example.py:412-456: for every object with >= 2 pixels: bbox [int((xmin+xmax)/2), int((ymin+ymax)/2), ymax-ymin, xmax-xmin],
 * crop of rgb [n_img,3,H,W] u8, zero-pad to a square, cv2.resize(.., (32,32), INTER_AREA) (bit-exact with OpenCV's 8-bit
 * code paths); visible objects first, zero-filled slots after.  crops u8 [n_img,n_obj,3,32,32], bbox int64 [n_img,n_obj,4],
 * mask u8 [n_img,n_obj], n_valid int32 [n_img] (optional). */
int vima_crop_resize(vima_ctx*, const uint8_t* rgb, int n_img, int H, int W, const int32_t* stats, int n_obj, uint8_t* crops,
                     int64_t* bbox, uint8_t* mask, int32_t* n_valid, void* stream);

/* ---- action heads -------------------------------------------------------------------------------------------- */
/* vima_policy.py:301-322: out[i,c] = float(idx[i,c]) / bins[c] */
int vima_action_scale(vima_ctx*, const int64_t* idx, int64_t n, int width, const float* bins_dev, float* out, void* stream);
/* scripts/example.py:199-232 (the step after the path): out[i,c] = clamp(idx[i,c]/bins[c] * (hi-lo) + lo, lo, hi), lo/hi
 * [n or 1, width] fp32 on the device (bound_stride 0 = one broadcast row); rotations use lo=-1, hi=1. */
int vima_action_postprocess(vima_ctx*, const int64_t* idx, int64_t n, int width, const float* bins_dev, const float* lo_dev,
                            const float* hi_dev, int bound_stride, float* out, void* stream);
/* dists.py:20-28: per head log-softmax normalised logits and mode (first argmax of probs). head_off: DEVICE int[n_heads+1]. */
int vima_head_select(vima_ctx*, const float* logits, int B, int n_heads, const int32_t* head_off_dev, float* logits_norm, int64_t* modes,
                     void* stream);
/* Acting and scoring on the same heads (torch.distributions.Categorical(logits=...) per head, without torch's host RNG).  logits fp32
 * [B, head_off[n_heads]], head_off DEVICE int[n_heads+1], as vima_head_select.  Per (row, head) the action is
 *   - actions_in[row, head] when actions_in != NULL (scoring; actions_out is not written), else
 *   - the mode, bit-identical to vima_head_select, when greedy != 0, else
 *   - a draw from softmax(logits): u = (word 0 of Philox4x32-10 with key = seed (lo, hi words) and counter = (row, head, draw lo,
 *     draw hi)) >> 8, times 2^-24; the first column with p > 0 whose running sum of exp(logit - max) exceeds u times the total
 *     (lanes of a warp own consecutive 32-column chunks: a fixed summation order), or the last column with p > 0 if rounding
 *     leaves none.  The draw index is the uint64 at counter_dev: every draw of the call reads it, and the call advances it by one
 *     (a one-thread kernel after the sampling kernel; also when B == 0), so the host never passes it and graph replays draw fresh
 *     numbers.
 * Optional fp32 [B, n_heads] outputs: log_prob of the action (NaN for an action outside [0, dim)), entropy = -sum p log p over the
 * p > 0 terms, both accumulated in fp64; logits_norm [B, head_off[n_heads]] as vima_head_select.  A head whose logits are all -inf
 * gives action 0 and NaN log_prob and entropy.  No host synchronisation. */
typedef struct {
  uint32_t struct_size;    /* = sizeof(vima_head_sample_desc) of the caller's header */
  const float* logits; int B; int n_heads; const int32_t* head_off_dev;
  const int64_t* actions_in; /* [B, n_heads] or NULL (choose) */
  int greedy;
  uint64_t seed; uint64_t* counter_dev;
  int64_t* actions_out;    /* [B, n_heads]; required unless actions_in is given */
  float* log_prob; float* entropy; float* logits_norm;
} vima_head_sample_desc;
int vima_sizeof_head_sample_desc(void);
int vima_head_sample(vima_ctx*, const vima_head_sample_desc* d, void* stream);

#pragma GCC visibility pop
#ifdef __cplusplus
}
#endif
#endif /* VIMA_B200_H */
