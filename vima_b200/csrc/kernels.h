// Internal launch interface between the C-ABI layer (api.cu) and the kernel translation units.
#pragma once
#include "common.cuh"

namespace vima {

struct NormParams {
  const float* x; long long rows; int cols; int ldx;
  const float* add; int ld_add;       // optional: normalise (x + add)
  const float* w; const float* b;     // first norm (w == null: no normalisation, passthrough/convert only)
  float eps; int rms;                 // rms=1: T5 RMSNorm (no mean, no bias)
  const float* w2; const float* b2; float eps2;  // optional chained LayerNorm on the first norm's output
  float* out_f32; int ld_o32;         // output of the first norm (fp32), optional
  float* out2_f32; int ld_o2;         // output of the second norm (fp32), optional
  unsigned short* out_hi; unsigned short* out_lo; int ld_o16;  // last norm's output as 16-bit operands, optional
  int dtype;
  unsigned char* out_lo8; unsigned char* out_hi8; int ld_o8;   // e4m3 cross-term views, optional
  float* stats_out; float stats_eps;  // optional [rows, 2] = (mean, rstd) of the FIRST norm's output rows (for a LayerNorm folded downstream)
};
cudaError_t launch_norm(const NormParams& p, cudaStream_t stream);
cudaError_t launch_row_stats_finalize(const float* partial, long long rows, int parts, int cols, float eps, int rms, float* stats,
                                      cudaStream_t stream);

struct AttnParams {
  const unsigned short *q_hi, *q_lo; int ldq;  // [B*Lq, ldq]; pointer already at head 0's first column
  const unsigned short *k_hi, *k_lo; int ldk;  // [B*Lk, ldk]
  const unsigned short *v_hi, *v_lo; int ldv;
  const unsigned char* key_mask;               // [B, Lk] 1 = attend, or null
  const float* rel_bias;                       // [H, 2*Lk-1] additive bias indexed by (j - i + Lk - 1), or null
  unsigned short *o_hi, *o_lo; int ldo;        // [B*Lq, ldo]
  int B, H, Lq, Lk, D;
  float scale; int causal; int split; int dtype;
  unsigned char *o_lo8, *o_hi8; int ldo8;      // e4m3 cross-term views of the output, optional
  int kv_batch_rows;                           // rows between consecutive batch elements in k/v (>= Lk; KV caches), 0 = Lk
  int mask_ld;                                 // row pitch of key_mask, 0 = Lk
  int q_pos0;                                  // causal: query row i sits at key position q_pos0 + i (incremental decode)
  int q_batch_rows;                            // rows between consecutive batch elements in q / o (>= Lq), 0 = Lq
  const int* q_pos;                            // causal, per batch element (device, or null): position q_pos[b], keys q_pos[b] + Lq
  // paged k / v (slot decode): key j of batch element b is row kv_pages[b*kv_page_ld + j/64]*64 + j%64 of a pool of kv_pool_pages
  // pages; null = the contiguous layout above
  const int* kv_pages; int kv_page_ld; int kv_pool_pages;
  const int* kv_len;                           // non-causal, no q_pos (device, or null): batch element b attends keys [0, kv_len[b])
};
constexpr int KV_PAGE_TOKENS = 64;  // = the streaming kernel's key chunk: one chunk is one page
// k / v row of key j of batch element b.  A page entry outside [0, kv_pool_pages) reads as page 0 (the pool's zero page), so no
// table contents can address memory outside the pool.  MAY_PAGE = false: the caller knows p is not paged (no run-time test).
template <bool MAY_PAGE = true>
__device__ __forceinline__ long long attn_kv_row(const AttnParams& p, int b, int j) {
  if (!MAY_PAGE || p.kv_pages == nullptr) return (long long)b * (p.kv_batch_rows ? p.kv_batch_rows : p.Lk) + j;
  int pg = __ldg(p.kv_pages + (size_t)b * p.kv_page_ld + j / KV_PAGE_TOKENS);
  if ((unsigned)pg >= (unsigned)p.kv_pool_pages) pg = 0;
  return (long long)pg * KV_PAGE_TOKENS + j % KV_PAGE_TOKENS;
}
// Attention scores are kept in the log2 domain: y = s * (scale*log2e) [+ bias*log2e]; the soft causal constant becomes
// -1e4*log2e; the key-mask constant stays finfo.min (any value + finfo.min rounds to finfo.min, so "all masked keys are
// equal" -- the reference's degenerate uniform row -- is preserved). softmax is invariant to the common factor.
constexpr float FP32_MIN = -3.4028234663852886e38f;
constexpr float LOG2E = 1.4426950408889634f;
constexpr float CAUSAL_L2 = -1e4f * LOG2E;
constexpr float EXIT_L2 = -9000.f * LOG2E;  // a running row maximum at or below this has only seen hidden or padded keys
// Additive key-mask term of key j in batch element b (mask row pitch mld): 0 = attend, finfo.min = padded, -inf = past Lk.
__device__ __forceinline__ float attn_key_mask_term(const AttnParams& p, int b, int mld, int j, int Lk) {
  float m = -INFINITY;  // beyond the sequence: excluded
  if (j < Lk) m = (p.key_mask == nullptr || p.key_mask[(size_t)b * mld + j]) ? 0.f : FP32_MIN;
  return m;
}
// Causal position of query row 0 and key count of batch element b.  With q_pos the key count is q_pos[b] + (full query count of the
// call; q_batch_rows when a body / tail split gave this launch only part of the rows), clamped to the capacity Lk; with kv_len it is
// kv_len[b] clamped to [1, Lk].  Keys past the count are excluded like keys past Lk, and their chunks are not streamed.
__device__ __forceinline__ void attn_batch_keys(const AttnParams& p, int b, int qbr, int& qp0, int& lk) {
  if (p.q_pos == nullptr) {
    qp0 = p.q_pos0;
    lk = p.kv_len == nullptr ? p.Lk : min(max(__ldg(p.kv_len + b), 1), p.Lk);
  } else {
    qp0 = max(p.q_pos[b], 0);
    lk = max(min(qp0 + qbr, p.Lk), 1);
  }
}
// two adjacent output values of one query row (the tensor-core attention kernels): (hi, lo) 16-bit pairs [+ e4m3 cross-term views for
// an "f16f8" consumer GEMM]
template <int DT>
__device__ __forceinline__ void attn_store_pair(const AttnParams& p, size_t brow, int col, float x0, float x1) {
  uint32_t hi, lo;
  split2<DT>(x0, x1, hi, lo);
  const size_t off = brow * p.ldo + col;
  *reinterpret_cast<uint32_t*>(p.o_hi + off) = hi;
  if (p.o_lo) *reinterpret_cast<uint32_t*>(p.o_lo + off) = lo;
  if (p.o_lo8) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    const size_t off8 = brow * p.ldo8 + col;
    unsigned short l8, h8;  // low byte = x0
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(l8) : "f"((x1 - f.y) * F8_ACT_LO_SCALE), "f"((x0 - f.x) * F8_ACT_LO_SCALE));
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(h8) : "f"(x1 * F8_ACT_HI_SCALE), "f"(x0 * F8_ACT_HI_SCALE));
    *reinterpret_cast<unsigned short*>(p.o_lo8 + off8) = l8;
    *reinterpret_cast<unsigned short*>(p.o_hi8 + off8) = h8;
  }
}
constexpr int ATTN_TAIL_MAX_ROWS = 8;         // attention_tail.cu: query rows per (batch, head) the SIMT tail kernel takes
constexpr int ATTN_TAIL_MAX_LK = 512;         // attention_tail.cu: keys the SIMT tail kernel's shared memory is sized for
cudaError_t launch_attention(const AttnParams& p, cudaStream_t stream);
size_t attention_smem_bytes(const AttnParams& p);             // dynamic shared memory the mma.sync kernel needs for p
int attention_max_lk(const AttnParams& p, size_t smem_limit);  // largest Lk (multiple of 64) that fits smem_limit at p's format
// K/V-streaming wgmma kernel (attention_tc.cu, no length cap), one body with two entry points:
long long attention_kv_rows(const AttnParams& p);      // rows of the k / v operands (the page pool's when paged)
bool attention_tc_supported(const AttnParams& p);       // the decoders: head_dim 32, split operands, no bias
bool attention_bias_tc_supported(const AttnParams& p);  // the T5 encoder: head_dim 64, relative bias, non-causal
// runs p on the entry point its relative bias selects (p must pass one of the two predicates); encode_tiled_fn: cuTensorMapEncodeTiled
cudaError_t launch_attention_tc(const AttnParams& p, void* encode_tiled_fn, cudaStream_t stream);
// query rows [row0, row0 + nt) of every (batch, head) (nt <= ATTN_TAIL_MAX_ROWS, head_dim 32, Lk <= ATTN_TAIL_MAX_LK): the rows that
// would otherwise occupy a nearly empty 128-row tile of the wgmma kernel
cudaError_t launch_attention_tail(const AttnParams& p, int row0, int nt, cudaStream_t stream);

struct SmallAttnParams {  // tiny-sequence fp32 attention (ViT: 5 tokens, 24 heads of 32)
  const float* qkv; int ld;        // [N*S, ld], q | k | v each W wide
  unsigned short *o_hi, *o_lo; int ldo; float* o_f32;  // [N*S, W]
  long long N; int S, H, W; float scale; int dtype;
};
cudaError_t launch_small_attention(const SmallAttnParams& p, cudaStream_t stream);

struct LatentAttnParams {  // fp32 attention of a few latent queries over <= 16 keys (Perceiver resampler)
  const float* q; int ldq; long long q_batch_stride;  // [N or 1][Lq, ldq]; stride 0 = the same queries for every image
  const float* k; int ldk;                            // [N*Lk, ldk]
  const float* v; int ldv;
  float* o; int ldo;                                  // [N*Lq, ldo]
  long long N; int Lq, Lk, H, d; float scale;
};
cudaError_t launch_latent_attention(const LatentAttnParams& p, cudaStream_t stream);

struct SimtGemmGroup {  // one fp32 problem: y[M, n] = act(x[M, k] * w[n, k]^T + b)
  const float* x; int ldx;
  const float* w; int ldw;
  const float* b;
  float* y; int ldy;
  int n, k;
};
cudaError_t launch_simt_gemm_grouped(const SimtGemmGroup* groups_dev, int n_groups, int M, int max_n, int act, cudaStream_t stream);
constexpr int SIMT_MAX_HOST_GROUPS = 16;  // descriptors per launch when they travel by value (kernel parameter space)
cudaError_t launch_simt_gemm_grouped_host(const SimtGemmGroup* groups_host, int n_groups, int M, int max_n, int act, cudaStream_t stream);

// element-wise / gather kernels (misc.cu)
cudaError_t launch_split(const float* x, long long rows, int cols, int ldx, unsigned short* hi, unsigned short* lo, int ld16,
                         int pad_cols, float scale, int dtype, cudaStream_t s);
cudaError_t launch_pack_weight(const float* w, int n, int k, int transposed, int ldw, unsigned short* hi, unsigned short* lo, int ld16,
                               float scale, int dtype, cudaStream_t s);
cudaError_t launch_pack_weight_f8(const float* w, int n, int k, int transposed, int ldw, unsigned char* hi8, unsigned char* lo8, int ld8,
                                  float scale, cudaStream_t s);
cudaError_t launch_split_f8(const float* x, long long rows, int cols, int ldx, unsigned char* lo8, unsigned char* hi8, int ld8, cudaStream_t s);
cudaError_t launch_assemble_history(const float* obs, const unsigned char* obs_mask, const float* act, int T, int B, int Q, int E,
                                    int La, float* tokens, unsigned char* masks_bl, long long* pos_bl, cudaStream_t s);
cudaError_t launch_mask_cumsum(const unsigned char* mask, int B, int L, long long* pos, cudaStream_t s);
cudaError_t launch_add_pos_embed(const float* tok, long long stride_b, long long stride_l, const long long* ids, const float* table,
                                 int n_pos, int B, int L, int E, float* out_f32, unsigned short* hi, unsigned short* lo, int ld16,
                                 int dtype, int* err_flag, cudaStream_t s);
cudaError_t launch_gather_prompt(const int* kind, const int* index, const long long* word_ids, const float* word_table,
                                 const float* img_emb, const unsigned char* img_mask, int B, int Lp, int D, float* out,
                                 unsigned char* mask_out, cudaStream_t s);
cudaError_t launch_patchify(const unsigned char* img, long long N, int H, int W, int P, unsigned short* hi, unsigned short* lo, int ld16,
                            int dtype, cudaStream_t s);
cudaError_t launch_vit_tokens(const float* patch_out, const float* cls, const float* pos, long long N, int S, int W, float* out,
                              cudaStream_t s);
cudaError_t launch_bbox_norm(const long long* bbox, long long n, float* out, cudaStream_t s);
cudaError_t launch_fill_ee(const long long* ee, const float* table, long long n_te, int Q, unsigned short* hi, unsigned short* lo,
                           int ld16, int col0, int n_pad, int dtype, cudaStream_t s);
cudaError_t launch_action_scale(const long long* idx, long long n, int width, const float* inv_bins, float* out, cudaStream_t s);
cudaError_t launch_object_stats(const void* segm, int elem, int n_img, int H, int W, const long long* ids, int n_obj, int ids_per_image,
                                int* stats, cudaStream_t s);
cudaError_t launch_crop_resize(const unsigned char* rgb, int n_img, int H, int W, const int* stats, int n_obj, unsigned char* crops,
                               long long* bbox, unsigned char* mask, int* n_valid, cudaStream_t s);
cudaError_t launch_action_post(const long long* idx, long long n, int width, const float* bins, const float* lo, const float* hi,
                               int bound_stride, float* out, cudaStream_t s);
cudaError_t launch_head_select(const float* logits, int B, int n_heads, const int* head_off, float* logits_norm, long long* modes,
                               cudaStream_t s);
// The action-head kernel (misc.cu): per (row, head) the mode, a Philox draw from softmax(logits), or a given action; optionally the
// log-probability of that action, the entropy and the log-softmax normalised logits.
enum { HEAD_SELECT = 0, HEAD_SAMPLE = 1, HEAD_SCORE = 2 };
struct HeadParams {
  const float* logits; int B; int n_heads; const int* head_off;
  int mode;
  const long long* actions_in;            // HEAD_SCORE: [B, n_heads]
  unsigned long long seed;                // HEAD_SAMPLE: Philox key
  const unsigned long long* counter;      // HEAD_SAMPLE: draw index (device), advanced by launch_head_kernel
  long long* actions_out;                 // HEAD_SELECT / HEAD_SAMPLE: [B, n_heads]
  float* log_prob; float* entropy;        // [B, n_heads], optional
  float* logits_norm;                     // [B, head_off[n_heads]], optional
};
cudaError_t launch_head_kernel(const HeadParams& p, cudaStream_t s);
// kernels the launch enqueued (a sampling launch is followed by the counter's one-thread increment)
inline int head_kernel_launches(const HeadParams& p) { return (p.B > 0) + (p.mode == HEAD_SAMPLE); }
cudaError_t launch_gato_positions(const unsigned char* prompt_mask, int B, int Lp, int L, unsigned char* mask_out, long long* pos_out,
                                  cudaStream_t s);
cudaError_t launch_max_u8(const unsigned char* x, long long n, int* out_max, cudaStream_t s);

// slot decode (slots.cu)
cudaError_t launch_slot_step_begin(const float* obs, const unsigned char* obs_mask, const float* action, int S, int Q, int E, int Lmax,
                                   const int* len, const int* n_valid, const int* has_action, const int* active, float* tokens,
                                   unsigned char* step_mask, long long* pos, int* q_pos, unsigned char* slot_mask, cudaStream_t s);
// The K/V writers take an optional page table (pages: int32 [rows, page_ld] of page indices into a pool of pool_pages pages, null =
// the contiguous [S*Lmax] layout; Lmax is then page_ld*64).  Paged writes to page 0 (the zero page) or past the pool are skipped.
cudaError_t launch_slot_kv_append(const unsigned short* qkv_hi, const unsigned short* qkv_lo, int ld_qkv, int col0, int width, int S, int Lq,
                                  const int* q_pos, unsigned short* kv_hi, unsigned short* kv_lo, int ld_kv, int Lmax, const int* pages,
                                  int pool_pages, cudaStream_t s);
cudaError_t launch_slot_step_end(const float* x, int ldx, int S, int Q, int E, const unsigned char* step_mask, int* len, int* n_valid,
                                 int* has_action, const int* active, float* out, cudaStream_t s);
cudaError_t launch_slot_kv_scatter(const unsigned short* qkv_hi, const unsigned short* qkv_lo, int ld_qkv, int col0, int width, int n, int Lq,
                                   const int* slots, unsigned short* kv_hi, unsigned short* kv_lo, int ld_kv, int Lmax, const int* pages,
                                   int pool_pages, cudaStream_t s);
cudaError_t launch_slot_admit_prefix(const int* slots, int n, const unsigned char* prompt_mask, int Lp, int Lmax, unsigned char* slot_mask,
                                     int* len, int* n_valid, int* has_action, int* active, cudaStream_t s);
// Resumed slot episodes: tokens (L, n, E) rows [P, L), mask / pos [n, L] columns [P, L) of each episode's recorded history
// (steps int32 [n] on the device; obs_mask null = every obs token valid), and the admitted slots' mask rows and state.
cudaError_t launch_slot_assemble_history(const float* obs, const unsigned char* obs_mask, const float* action, const int* steps, int T, int n,
                                         int Q, int E, int P, int L, float* tokens, unsigned char* mask, long long* pos, cudaStream_t s);
cudaError_t launch_slot_admit_history(const int* slots, const int* steps, int n, int S, int T, int Q, int P, int L, const unsigned char* mask,
                                      const float* action, int E, int Lmax, unsigned char* slot_mask, int* len, int* n_valid, int* has_action,
                                      int* active, float* action_token, cudaStream_t s);
// Block i of rows [src_row0[i], +block_rows) -> [dst_row0[i], +block_rows) in each of the n_buf buffers bufs[] (device array),
// rows of row_bytes (a multiple of 16); blocks with a start outside [0, buf_rows - block_rows] are skipped.
cudaError_t launch_kv_copy_blocks(void* const* bufs, int n_buf, long long row_bytes, const long long* src_row0, const long long* dst_row0,
                                  int n_blocks, int block_rows, long long buf_rows, cudaStream_t s);
// Block i of rows [row0[i], +block_rows) of each buffer z <-> packed[i][z] ([block][buffer][block_rows][row_bytes]); unpack = 0 packs
// (buffers -> packed), 1 unpacks.  Blocks with a start outside [0, buf_rows - block_rows] are skipped.
cudaError_t launch_kv_pack_blocks(void* const* bufs, int n_buf, long long row_bytes, const long long* row0, int n_blocks, int block_rows,
                                  long long buf_rows, void* packed, int unpack, cudaStream_t s);

}  // namespace vima
