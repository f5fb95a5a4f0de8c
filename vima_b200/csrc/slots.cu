// Slot decode (DESIGN.md 7 (f)1): every row of the batch is a slot holding one episode at its own history length, so episodes
// are admitted and finish independently.  The per-slot state (len, n_valid, has_action, active: int32 [S]) lives on the device and
// these three kernels read and advance it, so a step takes only by-value arguments and static shapes and captures into one CUDA
// graph.  All three are copies, integer scans and gathers: bit-exact by construction.
#include "kernels.h"

namespace vima {

// One block per slot.  Step block of L = Q+1 rows: [action, obs_1..obs_Q] once the slot has an action, else [obs_1..obs_Q, dummy]
// (zero token, masked: causally hidden from every real row, overwritten by the next step).
__global__ void __launch_bounds__(256) slot_step_begin_kernel(const float4* __restrict__ obs, const unsigned char* __restrict__ obs_mask,
                                                              const float4* __restrict__ action, int Q, int E4, int Lmax,
                                                              const int* __restrict__ len, const int* __restrict__ n_valid,
                                                              const int* __restrict__ has_action, const int* __restrict__ active,
                                                              float4* __restrict__ tokens, unsigned char* __restrict__ step_mask,
                                                              long long* __restrict__ pos, int* __restrict__ q_pos,
                                                              unsigned char* __restrict__ slot_mask) {
  const int b = blockIdx.x, L = Q + 1;
  const bool act = active[b] != 0, ha = has_action[b] != 0;
  const int qp = act ? len[b] : 0;  // an inactive slot computes at column 0 of its own cache and never advances
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int i = threadIdx.x; i < L * E4; i += blockDim.x) {
    const int r = i / E4, e = i % E4;
    float4 v = zero;
    if (ha) v = r == 0 ? __ldg(action + (size_t)b * E4 + e) : __ldg(obs + ((size_t)b * Q + r - 1) * E4 + e);
    else if (r < Q) v = __ldg(obs + ((size_t)b * Q + r) * E4 + e);
    tokens[((size_t)b * L + r) * E4 + e] = v;
  }
  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  const long long base = act ? (long long)n_valid[b] : 0;
  int carry = 0;
  for (int r0 = 0; r0 < L; r0 += 32) {
    const int r = r0 + lane;
    int m = 0;
    if (r < L) m = ha ? (r == 0 ? 1 : obs_mask[(size_t)b * Q + r - 1] != 0) : (r < Q ? obs_mask[(size_t)b * Q + r] != 0 : 0);
    int inc = m;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += y;
    }
    if (r < L) {
      step_mask[(size_t)b * L + r] = (unsigned char)m;
      // position id = cumsum(mask) - 1 over the episode (a masked first token gives -1: the deferred IndexError)
      pos[(size_t)b * L + r] = act ? base + carry + inc - 1 : 0;
      if (qp + r < Lmax) slot_mask[(size_t)b * Lmax + qp + r] = (unsigned char)m;
    }
    carry += __shfl_sync(0xffffffffu, inc, 31);
  }
  if (lane == 0) q_pos[b] = qp;
}

cudaError_t launch_slot_step_begin(const float* obs, const unsigned char* obs_mask, const float* action, int S, int Q, int E, int Lmax,
                                   const int* len, const int* n_valid, const int* has_action, const int* active, float* tokens,
                                   unsigned char* step_mask, long long* pos, int* q_pos, unsigned char* slot_mask, cudaStream_t s) {
  if (S == 0) return cudaSuccess;
  slot_step_begin_kernel<<<S, 256, 0, s>>>(reinterpret_cast<const float4*>(obs), obs_mask, reinterpret_cast<const float4*>(action), Q, E / 4,
                                           Lmax, len, n_valid, has_action, active, reinterpret_cast<float4*>(tokens), step_mask, pos, q_pos,
                                           slot_mask);
  return cudaGetLastError();
}

// Destination row of cache column col (< Lmax) of slot b: b*Lmax + col, or with a page table (pages [*, Lmax/64]) row
// page*64 + col%64 of the pool; -1 = skip (page 0, the zero page no slot owns, or an entry outside the pool).
__device__ __forceinline__ long long slot_kv_row(int b, int col, int Lmax, const int* __restrict__ pages, int pool_pages) {
  if (pages == nullptr) return (long long)b * Lmax + col;
  const int pg = __ldg(pages + (size_t)b * (Lmax / KV_PAGE_TOKENS) + col / KV_PAGE_TOKENS);
  return (pg <= 0 || pg >= pool_pages) ? -1 : (long long)pg * KV_PAGE_TOKENS + col % KV_PAGE_TOKENS;
}

// Step rows (b, r) -> cache column q_pos[b] + r of slot b, 8 16-bit values per thread and trip.
__global__ void slot_kv_append_kernel(const uint4* __restrict__ qkv_hi, const uint4* __restrict__ qkv_lo, int ld_qkv8, int col8, int w8, int S,
                                      int Lq, const int* __restrict__ q_pos, uint4* __restrict__ kv_hi, uint4* __restrict__ kv_lo, int ld_kv8,
                                      int Lmax, const int* __restrict__ pages, int pool_pages) {
  const long long total = (long long)S * Lq * w8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % w8);
    const long long br = i / w8;
    const int r = (int)(br % Lq), b = (int)(br / Lq);
    const int col = q_pos[b] + r;
    if (col < 0 || col >= Lmax) continue;
    const long long row = slot_kv_row(b, col, Lmax, pages, pool_pages);
    if (row < 0) continue;
    const size_t src = (size_t)br * ld_qkv8 + col8 + c;
    const size_t dst = (size_t)row * ld_kv8 + c;
    kv_hi[dst] = __ldg(qkv_hi + src);
    if (kv_lo) kv_lo[dst] = __ldg(qkv_lo + src);
  }
}

cudaError_t launch_slot_kv_append(const unsigned short* qkv_hi, const unsigned short* qkv_lo, int ld_qkv, int col0, int width, int S, int Lq,
                                  const int* q_pos, unsigned short* kv_hi, unsigned short* kv_lo, int ld_kv, int Lmax, const int* pages,
                                  int pool_pages, cudaStream_t s) {
  const long long total = (long long)S * Lq * (width / 8);
  if (total == 0) return cudaSuccess;
  const int blocks = (int)min((total + 255) / 256, (long long)132 * 16);
  slot_kv_append_kernel<<<blocks, 256, 0, s>>>(reinterpret_cast<const uint4*>(qkv_hi), reinterpret_cast<const uint4*>(qkv_lo), ld_qkv / 8,
                                               col0 / 8, width / 8, S, Lq, q_pos, reinterpret_cast<uint4*>(kv_hi),
                                               reinterpret_cast<uint4*>(kv_lo), ld_kv / 8, Lmax, pages, pool_pages);
  return cudaGetLastError();
}

// One block per slot: gather the prediction row (Q-1 + has_action, read before the update), then advance an active slot.
__global__ void __launch_bounds__(128) slot_step_end_kernel(const float4* __restrict__ x, int ldx4, int Q, int E4,
                                                            const unsigned char* __restrict__ step_mask, int* __restrict__ len,
                                                            int* __restrict__ n_valid, int* __restrict__ has_action,
                                                            const int* __restrict__ active, float4* __restrict__ out) {
  const int b = blockIdx.x, L = Q + 1;
  const int ha = has_action[b] != 0;
  const size_t row = (size_t)b * L + Q - 1 + ha;
  for (int e = threadIdx.x; e < E4; e += blockDim.x) out[(size_t)b * E4 + e] = __ldg(x + row * ldx4 + e);
  __syncthreads();  // every thread has read has_action[b]
  if (threadIdx.x >= 32) return;
  int cnt = 0;
  for (int r = threadIdx.x; r < L; r += 32) cnt += step_mask[(size_t)b * L + r] != 0;
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if (threadIdx.x == 0 && active[b]) {
    len[b] += Q + ha;
    n_valid[b] += cnt;
    has_action[b] = 1;
  }
}

cudaError_t launch_slot_step_end(const float* x, int ldx, int S, int Q, int E, const unsigned char* step_mask, int* len, int* n_valid,
                                 int* has_action, const int* active, float* out, cudaStream_t s) {
  if (S == 0) return cudaSuccess;
  slot_step_end_kernel<<<S, 128, 0, s>>>(reinterpret_cast<const float4*>(x), ldx / 4, Q, E / 4, step_mask, len, n_valid, has_action, active,
                                         reinterpret_cast<float4*>(out));
  return cudaGetLastError();
}

// Admission of a decoder-only prompt (the prompt and its separator live in the self-attention cache, columns [0, Lq)).
// Prefill rows (j, r) -> cache column r of slot slots[j], 8 16-bit values per thread and trip: each K/V element is read once and
// written once.
__global__ void slot_kv_scatter_kernel(const uint4* __restrict__ qkv_hi, const uint4* __restrict__ qkv_lo, int ld_qkv8, int col8, int w8, int n,
                                       int Lq, const int* __restrict__ slots, uint4* __restrict__ kv_hi, uint4* __restrict__ kv_lo, int ld_kv8,
                                       int Lmax, const int* __restrict__ pages, int pool_pages) {
  const long long total = (long long)n * Lq * w8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % w8);
    const long long jr = i / w8;
    const int r = (int)(jr % Lq), j = (int)(jr / Lq);
    const long long row = slot_kv_row(__ldg(slots + j), r, Lmax, pages, pool_pages);
    if (row < 0) continue;
    const size_t src = (size_t)jr * ld_qkv8 + col8 + c;
    const size_t dst = (size_t)row * ld_kv8 + c;
    kv_hi[dst] = __ldg(qkv_hi + src);
    if (kv_lo) kv_lo[dst] = __ldg(qkv_lo + src);
  }
}

cudaError_t launch_slot_kv_scatter(const unsigned short* qkv_hi, const unsigned short* qkv_lo, int ld_qkv, int col0, int width, int n, int Lq,
                                   const int* slots, unsigned short* kv_hi, unsigned short* kv_lo, int ld_kv, int Lmax, const int* pages,
                                   int pool_pages, cudaStream_t s) {
  const long long total = (long long)n * Lq * (width / 8);
  if (total == 0) return cudaSuccess;
  const int blocks = (int)min((total + 255) / 256, (long long)132 * 16);
  slot_kv_scatter_kernel<<<blocks, 256, 0, s>>>(reinterpret_cast<const uint4*>(qkv_hi), reinterpret_cast<const uint4*>(qkv_lo), ld_qkv / 8,
                                                col0 / 8, width / 8, n, Lq, slots, reinterpret_cast<uint4*>(kv_hi),
                                                reinterpret_cast<uint4*>(kv_lo), ld_kv / 8, Lmax, pages, pool_pages);
  return cudaGetLastError();
}

// One block per admitted slot b = slots[j]: mask columns [0, Lp) <- prompt_mask[j], column Lp <- 1 (the separator); then
// len = Lp+1, n_valid = valid prompt tokens + 1 (the separator's position id is the valid count), has_action = 0, active = 1.
__global__ void __launch_bounds__(256) slot_admit_prefix_kernel(const int* __restrict__ slots, const unsigned char* __restrict__ prompt_mask,
                                                                int Lp, int Lmax, unsigned char* __restrict__ slot_mask, int* __restrict__ len,
                                                                int* __restrict__ n_valid, int* __restrict__ has_action,
                                                                int* __restrict__ active) {
  __shared__ int warp_cnt[8];
  const int j = blockIdx.x, b = __ldg(slots + j);
  int cnt = 0;
  for (int l = threadIdx.x; l <= Lp; l += blockDim.x) {
    const unsigned char m = l < Lp ? (prompt_mask[(size_t)j * Lp + l] != 0) : 1;
    slot_mask[(size_t)b * Lmax + l] = m;
    cnt += l < Lp ? m : 0;
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) total += warp_cnt[w];
    len[b] = Lp + 1;
    n_valid[b] = total + 1;
    has_action[b] = 0;
    active[b] = 1;
  }
}

cudaError_t launch_slot_admit_prefix(const int* slots, int n, const unsigned char* prompt_mask, int Lp, int Lmax, unsigned char* slot_mask,
                                     int* len, int* n_valid, int* has_action, int* active, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  slot_admit_prefix_kernel<<<n, 256, 0, s>>>(slots, prompt_mask, Lp, Lmax, slot_mask, len, n_valid, has_action, active);
  return cudaGetLastError();
}

// Admission from a recorded history (slot episodes resumed mid-way).  Episode j has completed k = steps[j] environment steps (clamped
// to [0, T]); its history columns are forward's [o_0 (Q), a_0, o_1, ..., a_{k-2}, o_{k-1}], k(Q+1) - 1 of them (0 for k = 0),
// placed after a prefix of P columns (decoder-only: [prompt | separator]).  Rows t >= k of obs / obs_mask / action are never read.
__device__ __forceinline__ int slot_history_cols(const int* __restrict__ steps, int j, int T, int Q) {
  const int k = min(max(__ldg(steps + j), 0), T);
  return k > 0 ? k * (Q + 1) - 1 : 0;
}

// One warp per episode: mask and position ids of columns [P, L) of row j of mask / pos [n, L].  The position ids continue the
// prefix's valid count (columns [0, P) of the same mask row, written by the caller): base + cumsum(history mask) - 1; padding
// columns past the history get mask 0 and position id 0.
__global__ void __launch_bounds__(32) slot_history_mask_kernel(const unsigned char* __restrict__ obs_mask, const int* __restrict__ steps, int T,
                                                               int n, int Q, int P, int L, unsigned char* __restrict__ mask,
                                                               long long* __restrict__ pos) {
  const int j = blockIdx.x, lane = threadIdx.x;
  const int hl = slot_history_cols(steps, j, T, Q);
  unsigned char* mrow = mask + (size_t)j * L;
  int base = 0;
  for (int c = lane; c < P; c += 32) base += mrow[c] != 0;
  base = __reduce_add_sync(0xffffffffu, base);
  __syncwarp();
  int carry = 0;
  for (int c0 = 0; c0 < L - P; c0 += 32) {
    const int c = c0 + lane;
    int m = 0;
    if (c < hl) {
      const int t = c / (Q + 1), q = c % (Q + 1);
      m = (q < Q && obs_mask) ? (obs_mask[((size_t)t * n + j) * Q + q] != 0) : 1;
    }
    int inc = m;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += y;
    }
    if (c < L - P) {
      mrow[P + c] = (unsigned char)m;
      pos[(size_t)j * L + P + c] = c < hl ? (long long)(base + carry + inc - 1) : 0;
    }
    carry += __shfl_sync(0xffffffffu, inc, 31);
  }
}

// Tokens (L, n, E) rows [P, L): history column c of episode j from obs (T, n, Q, E) / action (T, n, E), zero past the history.
__global__ void slot_history_tokens_kernel(const float4* __restrict__ obs, const float4* __restrict__ act, const int* __restrict__ steps, int T,
                                           int n, int Q, int E4, int P, int L, float4* __restrict__ tokens) {
  const long long total = (long long)(L - P) * n * E4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i % E4);
    const long long cj = i / E4;
    const int j = (int)(cj % n), c = (int)(cj / n);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < slot_history_cols(steps, j, T, Q)) {
      const int t = c / (Q + 1), q = c % (Q + 1);
      v = q < Q ? __ldg(obs + (((size_t)t * n + j) * Q + q) * E4 + e) : __ldg(act + ((size_t)t * n + j) * E4 + e);
    }
    tokens[((size_t)(P + c) * n + j) * E4 + e] = v;
  }
}

cudaError_t launch_slot_assemble_history(const float* obs, const unsigned char* obs_mask, const float* action, const int* steps, int T, int n,
                                         int Q, int E, int P, int L, float* tokens, unsigned char* mask, long long* pos, cudaStream_t s) {
  if (n == 0 || L == P) return cudaSuccess;
  slot_history_mask_kernel<<<n, 32, 0, s>>>(obs_mask, steps, T, n, Q, P, L, mask, pos);
  const long long total = (long long)(L - P) * n * (E / 4);
  const int blocks = (int)min((total + 255) / 256, (long long)132 * 16);
  slot_history_tokens_kernel<<<blocks, 256, 0, s>>>(reinterpret_cast<const float4*>(obs), reinterpret_cast<const float4*>(action), steps, T, n,
                                                    Q, E / 4, P, L, reinterpret_cast<float4*>(tokens));
  return cudaGetLastError();
}

// One block per episode j, slot b = slots[j] (skipped outside [0, S), or when its P + history columns exceed L): mask row b of
// slot_mask [S, Lmax] <- columns [0, len) of mask row j, 0 past them; len = P + history columns, n_valid = valid columns of
// [0, len), has_action = (k > 0), active = 1, and for k > 0 the fed-back action row action_token[b] <- action[k-1, j].
__global__ void __launch_bounds__(256) slot_admit_history_kernel(const int* __restrict__ slots, const int* __restrict__ steps, int S, int T,
                                                                 int n, int Q, int P, int L, const unsigned char* __restrict__ mask,
                                                                 const float4* __restrict__ action, int E4, int Lmax,
                                                                 unsigned char* __restrict__ slot_mask, int* __restrict__ len,
                                                                 int* __restrict__ n_valid, int* __restrict__ has_action,
                                                                 int* __restrict__ active, float4* __restrict__ action_token) {
  __shared__ int warp_cnt[8];
  const int j = blockIdx.x, b = __ldg(slots + j);
  const int k = min(max(__ldg(steps + j), 0), T);
  const int ln = P + slot_history_cols(steps, j, T, Q);
  if (b < 0 || b >= S || ln > L) return;
  int cnt = 0;
  for (int c = threadIdx.x; c < Lmax; c += blockDim.x) {
    const unsigned char m = c < ln ? (mask[(size_t)j * L + c] != 0) : 0;
    slot_mask[(size_t)b * Lmax + c] = m;
    cnt += m;
  }
  if (k > 0)
    for (int e = threadIdx.x; e < E4; e += blockDim.x) action_token[(size_t)b * E4 + e] = __ldg(action + ((size_t)(k - 1) * n + j) * E4 + e);
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) total += warp_cnt[w];
    len[b] = ln;
    n_valid[b] = total;
    has_action[b] = k > 0;
    active[b] = 1;
  }
}

cudaError_t launch_slot_admit_history(const int* slots, const int* steps, int n, int S, int T, int Q, int P, int L, const unsigned char* mask,
                                      const float* action, int E, int Lmax, unsigned char* slot_mask, int* len, int* n_valid, int* has_action,
                                      int* active, float* action_token, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  slot_admit_history_kernel<<<n, 256, 0, s>>>(slots, steps, S, T, n, Q, P, L, mask, reinterpret_cast<const float4*>(action), E / 4, Lmax,
                                              slot_mask, len, n_valid, has_action, active, reinterpret_cast<float4*>(action_token));
  return cudaGetLastError();
}

// Block copies between rows of the same buffers (copy on write of shared K/V pages, a fork's prompt K/V rows).  Grid (row chunk,
// block, buffer): block i of buffer z, rows [src_row0[i], +block_rows) -> rows [dst_row0[i], +block_rows), 16 bytes per thread and
// trip.  The block's rows are contiguous (pitch = row_bytes), so each block is one flat copy.  A block with either start outside
// [0, buf_rows - block_rows], or a buffer whose base is null or not 16-byte aligned, is skipped.
__global__ void __launch_bounds__(256) kv_copy_blocks_kernel(void* const* __restrict__ bufs, long long row16,
                                                             const long long* __restrict__ src_row0, const long long* __restrict__ dst_row0,
                                                             int n_blocks, int block_rows, long long buf_rows) {
  uint4* buf = reinterpret_cast<uint4*>(bufs[blockIdx.z]);
  if (buf == nullptr || (reinterpret_cast<uintptr_t>(buf) & 15)) return;
  const long long n16 = (long long)block_rows * row16, last = buf_rows - block_rows;
  for (int i = blockIdx.y; i < n_blocks; i += gridDim.y) {
    const long long s = __ldg(src_row0 + i), d = __ldg(dst_row0 + i);
    if (s < 0 || s > last || d < 0 || d > last) continue;
    const uint4* from = buf + s * row16;
    uint4* to = buf + d * row16;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n16; j += (long long)gridDim.x * blockDim.x) to[j] = from[j];
  }
}

cudaError_t launch_kv_copy_blocks(void* const* bufs, int n_buf, long long row_bytes, const long long* src_row0, const long long* dst_row0,
                                  int n_blocks, int block_rows, long long buf_rows, cudaStream_t s) {
  if (n_blocks == 0) return cudaSuccess;
  const long long n16 = (long long)block_rows * (row_bytes / 16);
  const dim3 grid((unsigned)min((n16 + 255) / 256, 1024ll), (unsigned)min(n_blocks, 65535), (unsigned)n_buf);
  kv_copy_blocks_kernel<<<grid, 256, 0, s>>>(bufs, row_bytes / 16, src_row0, dst_row0, n_blocks, block_rows, buf_rows);
  return cudaGetLastError();
}

// Block moves between the buffers and one packed buffer (swapped slot episodes).  Grid (row chunk, block, buffer): block i of buffer
// z, rows [row0[i], +block_rows), <-> packed[i][z] of the layout [block][buffer][block_rows][row_bytes], 16 bytes per thread and
// trip; `unpack` picks the direction (0: buffers -> packed).  A block whose start lies outside [0, buf_rows - block_rows], or a
// buffer whose base is null or not 16-byte aligned, is skipped (its packed rows are neither read nor written).
__global__ void __launch_bounds__(256) kv_pack_blocks_kernel(void* const* __restrict__ bufs, long long row16,
                                                             const long long* __restrict__ row0, int n_blocks, int block_rows,
                                                             long long buf_rows, uint4* __restrict__ packed, int unpack) {
  uint4* buf = reinterpret_cast<uint4*>(bufs[blockIdx.z]);
  if (buf == nullptr || (reinterpret_cast<uintptr_t>(buf) & 15)) return;
  const long long n16 = (long long)block_rows * row16, last = buf_rows - block_rows;
  for (int i = blockIdx.y; i < n_blocks; i += gridDim.y) {
    const long long r = __ldg(row0 + i);
    if (r < 0 || r > last) continue;
    uint4* rows = buf + r * row16;
    uint4* pk = packed + ((long long)i * gridDim.z + blockIdx.z) * n16;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n16; j += (long long)gridDim.x * blockDim.x) {
      if (unpack)
        rows[j] = pk[j];
      else
        pk[j] = rows[j];
    }
  }
}

cudaError_t launch_kv_pack_blocks(void* const* bufs, int n_buf, long long row_bytes, const long long* row0, int n_blocks, int block_rows,
                                  long long buf_rows, void* packed, int unpack, cudaStream_t s) {
  if (n_blocks == 0) return cudaSuccess;
  const long long n16 = (long long)block_rows * (row_bytes / 16);
  const dim3 grid((unsigned)min((n16 + 255) / 256, 1024ll), (unsigned)min(n_blocks, 65535), (unsigned)n_buf);
  kv_pack_blocks_kernel<<<grid, 256, 0, s>>>(bufs, row_bytes / 16, row0, n_blocks, block_rows, buf_rows, reinterpret_cast<uint4*>(packed),
                                             unpack);
  return cudaGetLastError();
}

}  // namespace vima
