// Memory-bound helper kernels of the VIMA path: operand splitting / weight packing, token assembly (interleave,
// masks, cumsum position ids, position-embedding add), prompt gather, image patchify+normalise, small feature
// prep and the action-head argmax.  Integer / bool / copy outputs are bit-exact by construction.
#include "kernels.h"

namespace vima {

// ---------------------------------------------------------------------------------------------------------
template <int DT>
__global__ void split_kernel(const float* __restrict__ x, long long rows, int cols, int ldx, unsigned short* __restrict__ hi,
                             unsigned short* __restrict__ lo, int ld16, int pad_cols, float scale) {
  const long long total = rows * (long long)pad_cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / pad_cols;
    const int c = (int)(i % pad_cols);
    unsigned short h = 0, l = 0;
    if (c < cols) split16<DT>(__ldg(x + r * ldx + c) * scale, h, l);
    hi[r * ld16 + c] = h;
    if (lo) lo[r * ld16 + c] = l;
  }
}

cudaError_t launch_split(const float* x, long long rows, int cols, int ldx, unsigned short* hi, unsigned short* lo, int ld16,
                         int pad_cols, float scale, int dtype, cudaStream_t s) {
  if (rows == 0) return cudaSuccess;
  const long long total = rows * (long long)pad_cols;
  const int blocks = (int)min((total + 255) / 256, (long long)148 * 16);
  if (dtype == DT_BF16)
    split_kernel<DT_BF16><<<blocks, 256, 0, s>>>(x, rows, cols, ldx, hi, lo, ld16, pad_cols, scale);
  else
    split_kernel<DT_F16><<<blocks, 256, 0, s>>>(x, rows, cols, ldx, hi, lo, ld16, pad_cols, scale);
  return cudaGetLastError();
}

// w is [n][k] (nn.Linear) or, when transposed, [k][n] (HF Conv1D); output is K-major [n][ld16], zero padded.
template <int DT>
__global__ void pack_weight_kernel(const float* __restrict__ w, int n, int k, int transposed, int ldw, unsigned short* __restrict__ hi,
                                   unsigned short* __restrict__ lo, int ld16, float scale) {
  const long long total = (long long)n * ld16;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / ld16), c = (int)(i % ld16);
    unsigned short h = 0, l = 0;
    if (c < k) {
      const float v = transposed ? __ldg(w + (size_t)c * ldw + r) : __ldg(w + (size_t)r * ldw + c);
      split16<DT>(v * scale, h, l);
    }
    hi[i] = h;
    if (lo) lo[i] = l;
  }
}

cudaError_t launch_pack_weight(const float* w, int n, int k, int transposed, int ldw, unsigned short* hi, unsigned short* lo, int ld16,
                               float scale, int dtype, cudaStream_t s) {
  const long long total = (long long)n * ld16;
  if (total == 0) return cudaSuccess;
  const int blocks = (int)min((total + 255) / 256, (long long)148 * 16);
  if (dtype == DT_BF16)
    pack_weight_kernel<DT_BF16><<<blocks, 256, 0, s>>>(w, n, k, transposed, ldw, hi, lo, ld16, scale);
  else
    pack_weight_kernel<DT_F16><<<blocks, 256, 0, s>>>(w, n, k, transposed, ldw, hi, lo, ld16, scale);
  return cudaGetLastError();
}

// e4m3 cross-term views of a packed weight (see common.cuh "f16f8"): hi8 = e4m3(w*scale*2^-10), lo8 = e4m3((w*scale - f16(w*scale))*2^3)
__global__ void pack_weight_f8_kernel(const float* __restrict__ w, int n, int k, int transposed, int ldw, unsigned char* __restrict__ hi8,
                                      unsigned char* __restrict__ lo8, int ld8, float scale) {
  const long long total = (long long)n * (ld8 / 4);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / (ld8 / 4)), c = (int)(i % (ld8 / 4)) * 4;
    float v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int cc = c + q;
      v[q] = (cc < k) ? (transposed ? __ldg(w + (size_t)cc * ldw + r) : __ldg(w + (size_t)r * ldw + cc)) * scale : 0.f;
    }
    uint2 h16;
    uint32_t l8, h8;
    split4_f8(make_float4(v[0], v[1], v[2], v[3]), F8_W_LO_SCALE, F8_W_HI_SCALE, h16, l8, h8);
    *reinterpret_cast<uint32_t*>(hi8 + (size_t)r * ld8 + c) = h8;
    *reinterpret_cast<uint32_t*>(lo8 + (size_t)r * ld8 + c) = l8;
  }
}
cudaError_t launch_pack_weight_f8(const float* w, int n, int k, int transposed, int ldw, unsigned char* hi8, unsigned char* lo8, int ld8,
                                  float scale, cudaStream_t s) {
  const long long total = (long long)n * (ld8 / 4);
  if (total == 0) return cudaSuccess;
  const int blocks = (int)min((total + 255) / 256, (long long)148 * 16);
  pack_weight_f8_kernel<<<blocks, 256, 0, s>>>(w, n, k, transposed, ldw, hi8, lo8, ld8, scale);
  return cudaGetLastError();
}

__global__ void split_f8_kernel(const float* __restrict__ x, long long rows, int cols4, int ldx, unsigned char* __restrict__ lo8,
                                unsigned char* __restrict__ hi8, int ld8) {
  const long long total = rows * cols4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols4;
    const int c = (int)(i % cols4) * 4;
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + r * ldx + c));
    uint2 h16;
    uint32_t l8, h8;
    split4_f8(v, F8_ACT_LO_SCALE, F8_ACT_HI_SCALE, h16, l8, h8);
    *reinterpret_cast<uint32_t*>(lo8 + r * ld8 + c) = l8;
    *reinterpret_cast<uint32_t*>(hi8 + r * ld8 + c) = h8;
  }
}
cudaError_t launch_split_f8(const float* x, long long rows, int cols, int ldx, unsigned char* lo8, unsigned char* hi8, int ld8, cudaStream_t s) {
  const long long total = rows * (cols / 4);
  if (total == 0) return cudaSuccess;
  const int blocks = (int)min((total + 255) / 256, (long long)148 * 16);
  split_f8_kernel<<<blocks, 256, 0, s>>>(x, rows, cols / 4, ldx, lo8, hi8, ld8);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------
// History assembly (vima_policy.py:124-147): token l = t*(Q+1)+q <- obs[t,:,q], l = t*(Q+1)+Q <- action[t];
// masks default True (action slots), position id = cumsum(mask) - 1 along l.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int block_inclusive_scan(int v, int* warp_sums) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int s = (lane < (int)(blockDim.x >> 5)) ? warp_sums[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    warp_sums[lane] = s;
  }
  __syncthreads();
  const int add = warp > 0 ? warp_sums[warp - 1] : 0;
  __syncthreads();
  return x + add;
}

__global__ void __launch_bounds__(1024) history_mask_kernel(const unsigned char* __restrict__ obs_mask, int T, int B, int Q, int La,
                                                            unsigned char* __restrict__ masks_bl, long long* __restrict__ pos_bl) {
  __shared__ int warp_sums[32];
  const int b = blockIdx.x;
  const int L = T * Q + La;
  int carry = 0;
  for (int base = 0; base < L; base += blockDim.x) {
    const int l = base + threadIdx.x;
    int m = 0;
    if (l < L) {
      const int t = l / (Q + 1), q = l % (Q + 1);
      m = (q < Q) ? (obs_mask[((size_t)t * B + b) * Q + q] != 0) : 1;
    }
    const int inc = block_inclusive_scan(m, warp_sums);
    if (l < L) {
      masks_bl[(size_t)b * L + l] = (unsigned char)m;
      pos_bl[(size_t)b * L + l] = (long long)(carry + inc - 1);
    }
    __shared__ int total;
    if (threadIdx.x == blockDim.x - 1) total = inc;
    __syncthreads();
    carry += total;
    __syncthreads();
  }
}

__global__ void history_tokens_kernel(const float4* __restrict__ obs, const float4* __restrict__ act, int T, int B, int Q, int E4, int La,
                                      float4* __restrict__ tokens) {
  const int L = T * Q + La;
  const long long total = (long long)L * B * E4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i % E4);
    const long long lb = i / E4;
    const int b = (int)(lb % B);
    const int l = (int)(lb / B);
    const int t = l / (Q + 1), q = l % (Q + 1);
    float4 v;
    if (q < Q)
      v = __ldg(obs + (((size_t)t * B + b) * Q + q) * E4 + e);
    else
      v = __ldg(act + ((size_t)t * B + b) * E4 + e);
    tokens[i] = v;
  }
}

cudaError_t launch_assemble_history(const float* obs, const unsigned char* obs_mask, const float* act, int T, int B, int Q, int E,
                                    int La, float* tokens, unsigned char* masks_bl, long long* pos_bl, cudaStream_t s) {
  if (B == 0 || T == 0) return cudaSuccess;
  history_mask_kernel<<<B, 512, 0, s>>>(obs_mask, T, B, Q, La, masks_bl, pos_bl);
  const long long total = (long long)(T * Q + La) * B * (E / 4);
  const int blocks = (int)min((total + 255) / 256, (long long)148 * 16);
  history_tokens_kernel<<<blocks, 256, 0, s>>>(reinterpret_cast<const float4*>(obs), reinterpret_cast<const float4*>(act), T, B, Q, E / 4,
                                               La, reinterpret_cast<float4*>(tokens));
  return cudaGetLastError();
}

__global__ void __launch_bounds__(1024) mask_cumsum_kernel(const unsigned char* __restrict__ mask, int L, long long* __restrict__ pos) {
  __shared__ int warp_sums[32];
  __shared__ int total;
  const int b = blockIdx.x;
  int carry = 0;
  for (int base = 0; base < L; base += blockDim.x) {
    const int l = base + threadIdx.x;
    const int m = (l < L) ? (mask[(size_t)b * L + l] != 0) : 0;
    const int inc = block_inclusive_scan(m, warp_sums);
    if (l < L) pos[(size_t)b * L + l] = (long long)(carry + inc - 1);
    if (threadIdx.x == blockDim.x - 1) total = inc;
    __syncthreads();
    carry += total;
    __syncthreads();
  }
}

cudaError_t launch_mask_cumsum(const unsigned char* mask, int B, int L, long long* pos, cudaStream_t s) {
  if (B == 0 || L == 0) return cudaSuccess;
  mask_cumsum_kernel<<<B, 256, 0, s>>>(mask, L, pos);
  return cudaGetLastError();
}

// out[b,l,:] = tok[b*stride_b + l*stride_l + :] + table[ids[b,l]]  (xattn_gpt.py:103-105,110-114)
template <int DT>
__global__ void add_pos_embed_kernel(const float* __restrict__ tok, long long stride_b, long long stride_l, const long long* __restrict__ ids,
                                     const float* __restrict__ table, int n_pos, int B, int L, int E4, float* __restrict__ out_f32,
                                     unsigned short* __restrict__ hi, unsigned short* __restrict__ lo, int ld16, int* err_flag) {
  const long long total = (long long)B * L * E4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i % E4);
    const long long bl = i / E4;
    const int l = (int)(bl % L);
    const int b = (int)(bl / L);
    long long id = __ldg(ids + bl);
    if (id < 0 || id >= n_pos) {  // nn.Embedding would raise IndexError (e.g. first token masked -> id -1)
      if (err_flag) atomicExch(err_flag, 1);
      id = id < 0 ? 0 : n_pos - 1;
    }
    const float4 a = __ldg(reinterpret_cast<const float4*>(tok + b * stride_b + l * stride_l) + e);
    const float4 pz = __ldg(reinterpret_cast<const float4*>(table + id * (long long)(E4 * 4)) + e);
    const float4 v = make_float4(a.x + pz.x, a.y + pz.y, a.z + pz.z, a.w + pz.w);
    if (out_f32) reinterpret_cast<float4*>(out_f32)[i] = v;
    if (hi) {
      uint2 hv, lv;
      split4v<DT>(v, hv, lv);
      const size_t o = (size_t)bl * ld16 + (size_t)e * 4;
      *reinterpret_cast<uint2*>(hi + o) = hv;
      if (lo) *reinterpret_cast<uint2*>(lo + o) = lv;
    }
  }
}

cudaError_t launch_add_pos_embed(const float* tok, long long stride_b, long long stride_l, const long long* ids, const float* table,
                                 int n_pos, int B, int L, int E, float* out_f32, unsigned short* hi, unsigned short* lo, int ld16,
                                 int dtype, int* err_flag, cudaStream_t s) {
  const long long total = (long long)B * L * (E / 4);
  if (total == 0) return cudaSuccess;
  const int blocks = (int)min((total + 255) / 256, (long long)148 * 16);
  if (dtype == DT_BF16)
    add_pos_embed_kernel<DT_BF16><<<blocks, 256, 0, s>>>(tok, stride_b, stride_l, ids, table, n_pos, B, L, E / 4, out_f32, hi, lo, ld16, err_flag);
  else
    add_pos_embed_kernel<DT_F16><<<blocks, 256, 0, s>>>(tok, stride_b, stride_l, ids, table, n_pos, B, L, E / 4, out_f32, hi, lo, ld16, err_flag);
  return cudaGetLastError();
}

// Prompt assembly (vima_policy.py:180-233) driven by a host-built index map: kind 0 = padding (zeros, mask False),
// 1 = word (row word_ids[index] of the T5 table, mask True), 2 = object token (row `index` of the encoded
// prompt objects, mask = that slot's object mask).
__global__ void gather_prompt_kernel(const int* __restrict__ kind, const int* __restrict__ index, const long long* __restrict__ word_ids,
                                     const float* __restrict__ word_table, const float* __restrict__ img_emb,
                                     const unsigned char* __restrict__ img_mask, long long n_tok, int D4, float* __restrict__ out,
                                     unsigned char* __restrict__ mask_out) {
  const long long total = n_tok * D4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i % D4);
    const long long tkn = i / D4;
    const int kd = __ldg(kind + tkn), ix = __ldg(index + tkn);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    unsigned char m = 0;
    if (kd == 1) {
      v = __ldg(reinterpret_cast<const float4*>(word_table + __ldg(word_ids + ix) * (long long)(D4 * 4)) + e);
      m = 1;
    } else if (kd == 2) {
      v = __ldg(reinterpret_cast<const float4*>(img_emb + (long long)ix * (D4 * 4)) + e);
      m = img_mask[ix] != 0;
    }
    reinterpret_cast<float4*>(out)[i] = v;
    if (e == 0) mask_out[tkn] = m;
  }
}

cudaError_t launch_gather_prompt(const int* kind, const int* index, const long long* word_ids, const float* word_table,
                                 const float* img_emb, const unsigned char* img_mask, int B, int Lp, int D, float* out,
                                 unsigned char* mask_out, cudaStream_t s) {
  const long long n_tok = (long long)B * Lp;
  if (n_tok == 0) return cudaSuccess;
  const long long total = n_tok * (D / 4);
  const int blocks = (int)min((total + 255) / 256, (long long)148 * 16);
  gather_prompt_kernel<<<blocks, 256, 0, s>>>(kind, index, word_ids, word_table, img_emb, img_mask, n_tok, D / 4, out, mask_out);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------
// uint8 crops (N,3,H,W) -> normalised patch rows [N*(H/P)*(W/P), 3*P*P] as 16-bit operands: the im2col of the
// k=s=P conv fused with /255, -mean, /std (preprocess.py:23-43, vit.py:9-10).  Column = c*P*P + py*P + px,
// matching conv1.weight.reshape(width, -1).
// ---------------------------------------------------------------------------------------------------------
__constant__ float c_img_mean[3] = {0.3471f, 0.3429f, 0.3383f};
__constant__ float c_img_std[3] = {0.3011f, 0.2961f, 0.2956f};

template <int DT>
__global__ void patchify_kernel(const unsigned char* __restrict__ img, long long N, int H, int W, int P, unsigned short* __restrict__ hi,
                                unsigned short* __restrict__ lo, int ld16) {
  const int gw = W / P, gh = H / P;
  const int K = 3 * P * P;
  const long long total = N * gh * gw * (long long)(K / 4);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k4 = (int)(i % (K / 4));
    const long long prow = i / (K / 4);
    const int gx = (int)(prow % gw);
    const int gy = (int)((prow / gw) % gh);
    const long long n = prow / ((long long)gw * gh);
    const int k = k4 * 4;
    const int c = k / (P * P), py = (k % (P * P)) / P, px = k % P;
    const uchar4 u = *reinterpret_cast<const uchar4*>(img + ((n * 3 + c) * H + gy * P + py) * (long long)W + gx * P + px);
    const float mean = c_img_mean[c], sd = c_img_std[c];
    const float f0 = ((float)u.x / 255.0f - mean) / sd, f1 = ((float)u.y / 255.0f - mean) / sd;
    const float f2 = ((float)u.z / 255.0f - mean) / sd, f3 = ((float)u.w / 255.0f - mean) / sd;
    uint2 hv, lv;
    split4v<DT>(make_float4(f0, f1, f2, f3), hv, lv);
    const size_t o = (size_t)prow * ld16 + k;
    *reinterpret_cast<uint2*>(hi + o) = hv;
    if (lo) *reinterpret_cast<uint2*>(lo + o) = lv;
  }
}

cudaError_t launch_patchify(const unsigned char* img, long long N, int H, int W, int P, unsigned short* hi, unsigned short* lo, int ld16,
                            int dtype, cudaStream_t s) {
  const long long total = N * (H / P) * (W / P) * (long long)(3 * P * P / 4);
  if (total == 0) return cudaSuccess;
  const int blocks = (int)min((total + 255) / 256, (long long)148 * 16);
  if (dtype == DT_BF16)
    patchify_kernel<DT_BF16><<<blocks, 256, 0, s>>>(img, N, H, W, P, hi, lo, ld16);
  else
    patchify_kernel<DT_F16><<<blocks, 256, 0, s>>>(img, N, H, W, P, hi, lo, ld16);
  return cudaGetLastError();
}

// x[n, 0] = cls + pos[0]; x[n, 1+p] = patch_out[n*(S-1)+p] + pos[1+p]   (vit.py:173-179)
// cls == null (Gato ViT, vit.py:123-126): x[n, s] = patch_out[n*S+s] + pos[s]
__global__ void vit_tokens_kernel(const float4* __restrict__ patch_out, const float4* __restrict__ cls, const float4* __restrict__ pos,
                                  long long N, int S, int W4, float4* __restrict__ out) {
  const long long total = N * S * W4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i % W4);
    const long long ns = i / W4;
    const int s = (int)(ns % S);
    const long long n = ns / S;
    const float4 a = (cls == nullptr) ? __ldg(patch_out + ns * W4 + e)
                                      : ((s == 0) ? __ldg(cls + e) : __ldg(patch_out + (n * (S - 1) + (s - 1)) * W4 + e));
    const float4 p = __ldg(pos + (size_t)s * W4 + e);
    out[i] = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
  }
}

cudaError_t launch_vit_tokens(const float* patch_out, const float* cls, const float* pos, long long N, int S, int W, float* out,
                              cudaStream_t s) {
  const long long total = N * S * (W / 4);
  if (total == 0) return cudaSuccess;
  const int blocks = (int)min((total + 255) / 256, (long long)148 * 16);
  vit_tokens_kernel<<<blocks, 256, 0, s>>>(reinterpret_cast<const float4*>(patch_out), reinterpret_cast<const float4*>(cls),
                                           reinterpret_cast<const float4*>(pos), N, S, W / 4, reinterpret_cast<float4*>(out));
  return cudaGetLastError();
}

// bbox int64 [n,4] -> float / [256,128,128,256]   (obj_encoder.py:79-85)
__global__ void bbox_norm_kernel(const long long* __restrict__ bbox, long long n4, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const int c = (int)(i & 3);
  const float d = (c == 0 || c == 3) ? 256.0f : 128.0f;
  out[i] = (float)bbox[i] / d;
}
cudaError_t launch_bbox_norm(const long long* bbox, long long n, float* out, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  bbox_norm_kernel<<<(unsigned)((n * 4 + 255) / 256), 256, 0, s>>>(bbox, n * 4, out);
  return cudaGetLastError();
}

// end-effector embedding columns of the obs-fusion operand (vima_policy.py:253-256): row (te*Q + q), columns
// [col0, col0+2) = table[ee[te]], then n_pad zero columns.
template <int DT>
__global__ void fill_ee_kernel(const long long* __restrict__ ee, const float* __restrict__ table, long long n_rows, int Q,
                               unsigned short* __restrict__ hi, unsigned short* __restrict__ lo, int ld16, int col0, int n_pad) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  const long long id = ee[r / Q];
  for (int c = 0; c < 2 + n_pad; ++c) {
    unsigned short h = 0, l = 0;
    if (c < 2) split16<DT>(__ldg(table + id * 2 + c), h, l);
    hi[r * ld16 + col0 + c] = h;
    if (lo) lo[r * ld16 + col0 + c] = l;
  }
}
cudaError_t launch_fill_ee(const long long* ee, const float* table, long long n_te, int Q, unsigned short* hi, unsigned short* lo,
                           int ld16, int col0, int n_pad, int dtype, cudaStream_t s) {
  const long long n_rows = n_te * Q;
  if (n_rows == 0) return cudaSuccess;
  const unsigned blocks = (unsigned)((n_rows + 255) / 256);
  if (dtype == DT_BF16)
    fill_ee_kernel<DT_BF16><<<blocks, 256, 0, s>>>(ee, table, n_rows, Q, hi, lo, ld16, col0, n_pad);
  else
    fill_ee_kernel<DT_F16><<<blocks, 256, 0, s>>>(ee, table, n_rows, Q, hi, lo, ld16, col0, n_pad);
  return cudaGetLastError();
}

// de-discretise (vima_policy.py:301-322): out[i, c] = float(idx[i, c]) / bins[c]
__global__ void action_scale_kernel(const long long* __restrict__ idx, long long n, int width, const float* __restrict__ bins,
                                    float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * width) return;
  out[i] = (float)idx[i] / __ldg(bins + (i % width));
}
cudaError_t launch_action_scale(const long long* idx, long long n, int width, const float* bins, float* out, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  action_scale_kernel<<<(unsigned)((n * width + 255) / 256), 256, 0, s>>>(idx, n, width, bins, out);
  return cudaGetLastError();
}

// The environment-facing step after the heads (scripts/example.py:199-232): de-discretise, affine to the action bounds,
// clamp: out[i,c] = clamp(idx[i,c]/bins[c] * (hi-lo) + lo, lo, hi) with separately rounded *, + as in torch eager.
// lo/hi: [rows or 1, width] fp32 (bound_stride 0 broadcasts one row); rotations pass lo=-1, hi=1 (x*2-1, clamp to [-1,1]).
__global__ void action_post_kernel(const long long* __restrict__ idx, long long n, int width, const float* __restrict__ bins,
                                   const float* __restrict__ lo, const float* __restrict__ hi, int bound_stride, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * width) return;
  const int c = (int)(i % width);
  const long long r = i / width;
  const float a = (float)idx[i] / __ldg(bins + c);
  const float l = __ldg(lo + r * bound_stride + c), h = __ldg(hi + r * bound_stride + c);
  const float y = __fadd_rn(__fmul_rn(a, __fsub_rn(h, l)), l);
  out[i] = fminf(fmaxf(y, l), h);
}
cudaError_t launch_action_post(const long long* idx, long long n, int width, const float* bins, const float* lo, const float* hi,
                               int bound_stride, float* out, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  action_post_kernel<<<(unsigned)((n * width + 255) / 256), 256, 0, s>>>(idx, n, width, bins, lo, hi, bound_stride, out);
  return cudaGetLastError();
}

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11), the Random123 round function and key schedule.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k.x += 0x9E3779B9u; k.y += 0xBB67AE85u; }
    const unsigned lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const unsigned lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
  }
  return c;
}

// Inverse-CDF draw over columns [o0, o1) of `row` with weights e_c = expf(row[c] - mx): lane l owns the 32 consecutive columns
// [base + 32 l, base + 32 l + 32) of each 1024-column round; its running sum at column c is (carry + exclusive warp scan of the lane
// sums) + the lane's own sequential sum up to c.  Returns the first column with e_c > 0 whose running sum exceeds u * (sum of all
// e_c); when rounding leaves none (u * sum at or past the last partial sum), the last column with e_c > 0.  Offset from o0.
__device__ __forceinline__ float head_lane_sum(const float* row, int c0, int o1, float mx) {
  float s = 0.f;
  for (int c = c0; c < min(c0 + 32, o1); ++c) s += expf(row[c] - mx);
  return s;
}
__device__ __forceinline__ float warp_scan_incl(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}
__device__ int head_draw(const float* row, int o0, int o1, float mx, float u, int lane) {
  float total = 0.f;
  for (int base = o0; base < o1; base += 1024)
    total += __shfl_sync(0xffffffffu, warp_scan_incl(head_lane_sum(row, base + 32 * lane, o1, mx), lane), 31);
  const float t = u * total;
  float carry = 0.f;
  int last_pos = -1;
  for (int base = o0; base < o1; base += 1024) {
    const int c0 = base + 32 * lane;
    const float s = head_lane_sum(row, c0, o1, mx);
    const float incl = warp_scan_incl(s, lane);
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 0.f;
    const float start = carry + excl;
    int hit = -1;
    float run = 0.f;
    for (int c = c0; c < min(c0 + 32, o1); ++c) {
      const float e = expf(row[c] - mx);
      run += e;
      if (e > 0.f) {
        last_pos = c;
        if (hit < 0 && start + run > t) hit = c;
      }
    }
    const unsigned hits = __ballot_sync(0xffffffffu, hit >= 0);
    if (hits) return __shfl_sync(0xffffffffu, hit, __ffs(hits) - 1) - o0;
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
  // each lane's last_pos is its last positive column over every round, so the head's last one is the largest of them
  last_pos = __reduce_max_sync(0xffffffffu, last_pos);
  return last_pos >= 0 ? last_pos - o0 : 0;
}

// One warp per (row b, head).  Every mode computes the log-softmax normalised logits (Categorical(logits=...), dists.py:20-23) and
// the mode = first argmax of the softmax probabilities (dists.py:25-28) exactly as vima_head_select always has; HEAD_SAMPLE then
// draws the action from softmax(logits) with u = (Philox4x32-10(counter = (b, head, draw lo, draw hi), key = seed).x >> 8) * 2^-24,
// HEAD_SCORE takes it from actions_in.  log_prob and entropy are accumulated in fp64 over d_c = logit_c - max.
__global__ void head_kernel(const HeadParams p) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int n_heads = p.n_heads;
  if (w >= p.B * n_heads) return;
  const int b = w / n_heads, hd = w % n_heads;
  const int o0 = p.head_off[hd], o1 = p.head_off[hd + 1];
  const int total = p.head_off[n_heads];
  const float* row = p.logits + (size_t)b * total;
  float mx = -INFINITY;
  for (int c = o0 + lane; c < o1; c += 32) mx = fmaxf(mx, row[c]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = o0 + lane; c < o1; c += 32) sum += expf(row[c] - mx);
  sum = warp_sum(sum);
  const float lse = mx + logf(sum);
  float best = -INFINITY;
  int best_i = 0x7fffffff;
  for (int c = o0 + lane; c < o1; c += 32) {
    const float ln = row[c] - lse;
    if (p.logits_norm) p.logits_norm[(size_t)b * total + c] = ln;
    const float pr = expf(ln);
    if (pr > best) { best = pr; best_i = c - o0; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    if (ob > best || (ob == best && oi < best_i)) { best = ob; best_i = oi; }
  }
  // a head whose logits are all -inf has NaN probabilities (and NaN normalised logits, as log_softmax gives): argmax over
  // them is index 0 in torch, and no lane found a probability to keep
  if (best_i == 0x7fffffff) best_i = 0;
  const size_t oi = (size_t)b * n_heads + hd;
  const bool dead = mx == -INFINITY;  // all -inf: index 0, NaN log-prob and entropy
  long long act = best_i;
  if (p.mode == HEAD_SAMPLE) {
    const unsigned long long draw = *p.counter;
    const uint4 r = philox4x32_10(make_uint4((unsigned)b, (unsigned)hd, (unsigned)draw, (unsigned)(draw >> 32)),
                                  make_uint2((unsigned)p.seed, (unsigned)(p.seed >> 32)));
    act = dead ? 0 : head_draw(row, o0, o1, mx, (float)(r.x >> 8) * 0x1p-24f, lane);
  } else if (p.mode == HEAD_SCORE) {
    act = p.actions_in[oi];
  }
  if (p.mode != HEAD_SCORE && lane == 0) p.actions_out[oi] = act;
  if (!p.log_prob && !p.entropy) return;
  double S = 0.0, T = 0.0;  // sum of exp(d_c), sum of exp(d_c) * d_c over the finite logits (p = 0 terms dropped)
  for (int c = o0 + lane; c < o1; c += 32) {
    const float x = row[c];
    if (x != -INFINITY) {
      const double d = (double)x - (double)mx;
      const double e = exp(d);
      S += e;
      T += e * d;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    S += __shfl_xor_sync(0xffffffffu, S, o);
    T += __shfl_xor_sync(0xffffffffu, T, o);
  }
  if (lane != 0) return;
  const double logS = log(S);
  if (p.log_prob) {
    const bool ok = !dead && act >= 0 && act < o1 - o0;
    p.log_prob[oi] = ok ? (float)(((double)row[o0 + act] - (double)mx) - logS) : __int_as_float(0x7fc00000);
  }
  if (p.entropy) p.entropy[oi] = dead ? __int_as_float(0x7fc00000) : (float)(logS - T / S);
}

__global__ void counter_increment_kernel(unsigned long long* counter) { *counter += 1; }

cudaError_t launch_head_kernel(const HeadParams& p, cudaStream_t s) {
  if (p.B > 0) {
    const int warps = p.B * p.n_heads;
    head_kernel<<<(warps + 7) / 8, 256, 0, s>>>(p);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  // every warp of the launch above reads the draw index; the increment runs once all of them have, so no replay or later launch
  // ever reuses a draw.  A sampling call over no rows advances it too: the counter counts sampling calls.
  if (p.mode == HEAD_SAMPLE) {
    counter_increment_kernel<<<1, 1, 0, s>>>(const_cast<unsigned long long*>(p.counter));
    return cudaGetLastError();
  }
  return cudaSuccess;
}

cudaError_t launch_head_select(const float* logits, int B, int n_heads, const int* head_off, float* logits_norm, long long* modes,
                               cudaStream_t s) {
  HeadParams p = {};
  p.logits = logits; p.B = B; p.n_heads = n_heads; p.head_off = head_off;
  p.mode = HEAD_SELECT;
  p.actions_out = modes;
  p.logits_norm = logits_norm;
  return launch_head_kernel(p, s);
}

// Gato sequence layout (vima_gato_policy.py:150-182): mask = [prompt_mask | ones], position ids = arange over the
// n valid prompt tokens, (n-1) on padded prompt slots, then n, n+1, ... for the separator + history.
__global__ void gato_positions_kernel(const unsigned char* __restrict__ prompt_mask, int Lp, int L, unsigned char* __restrict__ mask_out,
                                      long long* __restrict__ pos_out) {
  __shared__ int n_valid_s;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) n_valid_s = 0;
  __syncthreads();
  int cnt = 0;
  for (int l = threadIdx.x; l < Lp; l += blockDim.x) cnt += prompt_mask[(size_t)b * Lp + l] != 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&n_valid_s, cnt);
  __syncthreads();
  const int n = n_valid_s;
  for (int l = threadIdx.x; l < L; l += blockDim.x) {
    long long id;
    unsigned char m;
    if (l < Lp) {
      id = l < n ? l : n - 1;
      m = prompt_mask[(size_t)b * Lp + l] != 0;
    } else {
      id = n + (l - Lp);
      m = 1;
    }
    pos_out[(size_t)b * L + l] = id;
    mask_out[(size_t)b * L + l] = m;
  }
}
cudaError_t launch_gato_positions(const unsigned char* prompt_mask, int B, int Lp, int L, unsigned char* mask_out, long long* pos_out,
                                  cudaStream_t s) {
  if (B == 0) return cudaSuccess;
  gato_positions_kernel<<<B, 256, 0, s>>>(prompt_mask, Lp, L, mask_out, pos_out);
  return cudaGetLastError();
}

__global__ void max_u8_kernel(const unsigned char* __restrict__ x, long long n, int* out_max) {
  int m = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) m = max(m, (int)x[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out_max, m);
}
cudaError_t launch_max_u8(const unsigned char* x, long long n, int* out_max, cudaStream_t s) {
  if (n == 0) return cudaSuccess;
  const int blocks = (int)min((n + 255) / 256, (long long)148 * 8);
  max_u8_kernel<<<blocks, 256, 0, s>>>(x, n, out_max);
  return cudaGetLastError();
}

}  // namespace vima
