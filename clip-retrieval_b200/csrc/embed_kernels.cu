// Bandwidth-bound kernels of the embed path: im2col, embeddings, LayerNorm, pooled projection +
// L2-normalise + cast (reference mapper.py:58-59,66-67).  All statistics in fp32.
#include "embed_kernels.cuh"
#include <algorithm>

namespace b200 {

// ---- K1: im2col ------------------------------------------------------------------------------------
// One block per (b, patch row py): reads 3*p image rows of S contiguous floats (coalesced), writes
// the g patches of that row.
__global__ void im2col_kernel(const float* __restrict__ px, __nv_bfloat16* __restrict__ cols, int S, int p, int g,
                              int Kp) {
  const int b = blockIdx.y, py = blockIdx.x;
  const int per_c = p * S;
  const int total = 3 * per_c;
  const float* img = px + (size_t)b * 3 * S * S;
  __nv_bfloat16* out = cols + ((size_t)b * g * g + (size_t)py * g) * Kp;
  for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
    const int c = idx / per_c;
    const int rem = idx - c * per_c;
    const int i = rem / S;
    const int xx = rem - i * S;
    const int pxi = xx / p;
    const int j = xx - pxi * p;
    if (pxi < g) {
      const float v = img[((size_t)c * S + (size_t)(py * p + i)) * S + xx];
      out[(size_t)pxi * Kp + c * p * p + i * p + j] = __float2bfloat16_rn(v);
    }
  }
}

int im2col_patches(const float* pixels, __nv_bfloat16* cols, int B, int S, int p, int Kp, cudaStream_t st) {
  const int g = S / p;
  im2col_kernel<<<dim3(g, B), 256, 0, st>>>(pixels, cols, S, p, g, Kp);
  B200_LAUNCH_OK();
  return B200_OK;
}

// ---- K2: cls rows -----------------------------------------------------------------------------------
__global__ void cls_rows_kernel(__nv_bfloat16* __restrict__ x, const float* __restrict__ v, int T, int w) {
  const int b = blockIdx.x;
  __nv_bfloat16* row = x + (size_t)b * T * w;
  for (int j = threadIdx.x; j < w; j += blockDim.x) row[j] = __float2bfloat16_rn(v[j]);
}
int write_cls_rows(__nv_bfloat16* x, const float* cls_plus_pos0, int B, int T, int w, cudaStream_t st) {
  cls_rows_kernel<<<B, 256, 0, st>>>(x, cls_plus_pos0, T, w);
  B200_LAUNCH_OK();
  return B200_OK;
}

// ---- K9: token embedding + positional embedding ---------------------------------------------------
__global__ void text_embed_kernel(const int64_t* __restrict__ tokens, const __nv_bfloat16* __restrict__ tok_emb,
                                  const float* __restrict__ pos_emb, __nv_bfloat16* __restrict__ x, int T, int w,
                                  int vocab, int64_t rows) {
  const int chunks = w / 8;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * chunks) return;
  const int64_t r = i / chunks;
  const int c = (int)(i - r * chunks);
  const int t = (int)(r % T);
  int64_t tok = tokens[r];
  if (tok < 0) tok = 0;
  if (tok >= vocab) tok = vocab - 1;
  const uint4 e = *reinterpret_cast<const uint4*>(tok_emb + tok * w + c * 8);
  const float4 p0 = *reinterpret_cast<const float4*>(pos_emb + (size_t)t * w + c * 8);
  const float4 p1 = *reinterpret_cast<const float4*>(pos_emb + (size_t)t * w + c * 8 + 4);
  const __nv_bfloat162* e2 = reinterpret_cast<const __nv_bfloat162*>(&e);
  const float2 a = __bfloat1622float2(e2[0]), b = __bfloat1622float2(e2[1]), cc = __bfloat1622float2(e2[2]),
               d = __bfloat1622float2(e2[3]);
  uint4 o;
  __nv_bfloat162 t0 = __floats2bfloat162_rn(a.x + p0.x, a.y + p0.y);
  __nv_bfloat162 t1 = __floats2bfloat162_rn(b.x + p0.z, b.y + p0.w);
  __nv_bfloat162 t2 = __floats2bfloat162_rn(cc.x + p1.x, cc.y + p1.y);
  __nv_bfloat162 t3 = __floats2bfloat162_rn(d.x + p1.z, d.y + p1.w);
  o.x = *reinterpret_cast<uint32_t*>(&t0);
  o.y = *reinterpret_cast<uint32_t*>(&t1);
  o.z = *reinterpret_cast<uint32_t*>(&t2);
  o.w = *reinterpret_cast<uint32_t*>(&t3);
  *reinterpret_cast<uint4*>(x + r * w + c * 8) = o;
}
int text_embed(const int64_t* tokens, const __nv_bfloat16* tok_emb, const float* pos_emb, __nv_bfloat16* x, int B, int T,
               int w, int vocab, cudaStream_t st) {
  const int64_t rows = (int64_t)B * T;
  const int64_t n = rows * (w / 8);
  text_embed_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(tokens, tok_emb, pos_emb, x, T, w, vocab, rows);
  B200_LAUNCH_OK();
  return B200_OK;
}

__global__ void token_argmax_kernel(const int64_t* __restrict__ tokens, int* __restrict__ out, int B, int T) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int64_t* row = tokens + (size_t)b * T;
  int64_t best = row[0];
  int bi = 0;
  for (int t = 1; t < T; t++)
    if (row[t] > best) { best = row[t]; bi = t; }
  out[b] = bi;
}
int token_argmax(const int64_t* tokens, int* pool_idx, int B, int T, cudaStream_t st) {
  token_argmax_kernel<<<(B + 127) / 128, 128, 0, st>>>(tokens, pool_idx, B, T);
  B200_LAUNCH_OK();
  return B200_OK;
}

// ---- LayerNorm: one warp per row, the row lives in registers between the two passes -------------
constexpr int LN_MAXC = 8;  // 16-byte chunks per lane: w <= 2048
template <int CPL>          // chunks per lane actually present: ceil(w / 256)
__global__ void __launch_bounds__(256)
layernorm_kernel(const __nv_bfloat16* __restrict__ in, int64_t in_ld, __nv_bfloat16* __restrict__ out, int64_t out_ld,
                 const float* __restrict__ gamma, const float* __restrict__ beta, int64_t rows, int w, float eps) {
  // persistent warps: row = gwarp, gwarp + total, ...; the next row's 16-byte chunks are loaded
  // before the current row is reduced and stored, so a warp always has a row in flight.
  const int lane = threadIdx.x & 31;
  const int64_t gw = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t total = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int chunks = w >> 3;
  // affine parameters of this lane's columns stay in registers across rows
  float gg[CPL][8], bb[CPL][8];
#pragma unroll
  for (int c = 0; c < CPL; c++) {
    const int ci = c * 32 + lane;
    if (ci < chunks) {
      const float4 g0 = *reinterpret_cast<const float4*>(gamma + ci * 8);
      const float4 g1 = *reinterpret_cast<const float4*>(gamma + ci * 8 + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(beta + ci * 8);
      const float4 b1 = *reinterpret_cast<const float4*>(beta + ci * 8 + 4);
      gg[c][0] = g0.x; gg[c][1] = g0.y; gg[c][2] = g0.z; gg[c][3] = g0.w;
      gg[c][4] = g1.x; gg[c][5] = g1.y; gg[c][6] = g1.z; gg[c][7] = g1.w;
      bb[c][0] = b0.x; bb[c][1] = b0.y; bb[c][2] = b0.z; bb[c][3] = b0.w;
      bb[c][4] = b1.x; bb[c][5] = b1.y; bb[c][6] = b1.z; bb[c][7] = b1.w;
    }
  }
  uint4 nxt[CPL];
  if (gw < rows) {
#pragma unroll
    for (int c = 0; c < CPL; c++) {
      const int ci = c * 32 + lane;
      nxt[c] = ci < chunks ? *reinterpret_cast<const uint4*>(in + gw * in_ld + ci * 8) : make_uint4(0u, 0u, 0u, 0u);
    }
  }
  for (int64_t row = gw; row < rows; row += total) {
    uint4 cur[CPL];
#pragma unroll
    for (int c = 0; c < CPL; c++) cur[c] = nxt[c];
    if (row + total < rows) {
#pragma unroll
      for (int c = 0; c < CPL; c++) {
        const int ci = c * 32 + lane;
        nxt[c] = ci < chunks ? *reinterpret_cast<const uint4*>(in + (row + total) * in_ld + ci * 8) : make_uint4(0u, 0u, 0u, 0u);
      }
    }
    float v[CPL][8];
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < CPL; c++) {
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&cur[c]);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const float2 f = __bfloat1622float2(h[j]);
        v[c][2 * j] = f.x;
        v[c][2 * j + 1] = f.y;
        sum += f.x + f.y;   // chunks past the row are zeros
      }
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)w;
    float ss = 0.f;
#pragma unroll
    for (int c = 0; c < CPL; c++) {
      if (c * 32 + lane < chunks) {
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float dlt = v[c][j] - mean;
          ss += dlt * dlt;
        }
      }
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rstd = rsqrtf(ss / (float)w + eps);
    __nv_bfloat16* dst = out + row * out_ld;
#pragma unroll
    for (int c = 0; c < CPL; c++) {
      const int ci = c * 32 + lane;
      if (ci < chunks) {
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const float a = (v[c][2 * j] - mean) * rstd * gg[c][2 * j] + bb[c][2 * j];
          const float b = (v[c][2 * j + 1] - mean) * rstd * gg[c][2 * j + 1] + bb[c][2 * j + 1];
          __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
          o[j] = *reinterpret_cast<uint32_t*>(&t);
        }
        *reinterpret_cast<uint4*>(dst + ci * 8) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}
int layernorm_rows(const __nv_bfloat16* in, int64_t in_ld, __nv_bfloat16* out, int64_t out_ld, const float* gamma,
                   const float* beta, int64_t rows, int w, cudaStream_t st) {
  return layernorm_rows_eps(in, in_ld, out, out_ld, gamma, beta, rows, w, 1e-5f, st);
}
int layernorm_rows_eps(const __nv_bfloat16* in, int64_t in_ld, __nv_bfloat16* out, int64_t out_ld, const float* gamma,
                       const float* beta, int64_t rows, int w, float eps, cudaStream_t st) {
  B200_CHECK(w % 8 == 0 && w <= LN_MAXC * 256, B200_ERR_UNSUPPORTED, "layernorm: width %d (need %%8, <= 2048)", w);
  if (rows == 0) return B200_OK;
  // persistent: enough blocks to fill the chip, each warp strides over rows
  const unsigned grid = (unsigned)std::min<int64_t>((rows + 7) / 8, (int64_t)132 * 6);
  switch ((w / 8 + 31) / 32) {
    case 1: layernorm_kernel<1><<<grid, 256, 0, st>>>(in, in_ld, out, out_ld, gamma, beta, rows, w, eps); break;
    case 2: layernorm_kernel<2><<<grid, 256, 0, st>>>(in, in_ld, out, out_ld, gamma, beta, rows, w, eps); break;
    case 3: layernorm_kernel<3><<<grid, 256, 0, st>>>(in, in_ld, out, out_ld, gamma, beta, rows, w, eps); break;
    case 4: layernorm_kernel<4><<<grid, 256, 0, st>>>(in, in_ld, out, out_ld, gamma, beta, rows, w, eps); break;
    case 5: layernorm_kernel<5><<<grid, 256, 0, st>>>(in, in_ld, out, out_ld, gamma, beta, rows, w, eps); break;
    case 6: layernorm_kernel<6><<<grid, 256, 0, st>>>(in, in_ld, out, out_ld, gamma, beta, rows, w, eps); break;
    case 7: layernorm_kernel<7><<<grid, 256, 0, st>>>(in, in_ld, out, out_ld, gamma, beta, rows, w, eps); break;
    default: layernorm_kernel<8><<<grid, 256, 0, st>>>(in, in_ld, out, out_ld, gamma, beta, rows, w, eps); break;
  }
  B200_LAUNCH_OK();
  return B200_OK;
}

// ---- K8/K10/K11: pooled LN + projection + L2 normalise + cast --------------------------------------
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  const int nw = blockDim.x >> 5;
  for (int i = 0; i < nw; i++) t += red[i];
  return t;
}

// A block owns 64 output columns of one sample, so that batch 1 (clip_back.py:226-246's shape) still spreads the
// projection over D / 64 SMs instead of a w-long dependent loop per thread on one: the pooled row is normalised
// redundantly per block (w values), the projection is split over 64 columns x 4 quarters of the reduction dimension,
// raw features go to `feat` and a second tiny kernel normalises.
__global__ void __launch_bounds__(256)
pool_proj_split_kernel(const __nv_bfloat16* __restrict__ x, int T, int w, const int* __restrict__ pool_idx,
                       const float* __restrict__ gamma, const float* __restrict__ beta,
                       const __nv_bfloat16* __restrict__ proj, int D, const float* __restrict__ bias,
                       float* __restrict__ feat) {
  extern __shared__ float sm[];
  float* s_row = sm;                // [w]
  float* s_part = sm + w;           // [4][64]
  __shared__ float red[8];
  const int b = blockIdx.y, j0 = blockIdx.x * 64;
  const int t = pool_idx ? pool_idx[b] : 0;
  const __nv_bfloat16* src = x + ((size_t)b * T + t) * w;
  float part = 0.f;
  for (int j = threadIdx.x; j < w; j += blockDim.x) {
    const float f = __bfloat162float(src[j]);
    s_row[j] = f;
    part += f;
  }
  if (gamma != nullptr) {   // null: the ResNet attention pool's c_proj, no LayerNorm
    const float mean = block_sum(part, red) / (float)w;
    part = 0.f;
    for (int j = threadIdx.x; j < w; j += blockDim.x) {
      const float dlt = s_row[j] - mean;
      part += dlt * dlt;
    }
    const float rstd = rsqrtf(block_sum(part, red) / (float)w + 1e-5f);
    for (int j = threadIdx.x; j < w; j += blockDim.x) s_row[j] = (s_row[j] - mean) * rstd * gamma[j] + beta[j];
  }
  __syncthreads();
  const int jj = threadIdx.x & 63, quarter = threadIdx.x >> 6;
  const int j = j0 + jj;
  const int per = (w + 3) / 4, i0 = quarter * per, i1 = min(w, i0 + per);
  float acc0 = 0.f, acc1 = 0.f;   // two interleaved chains halve the latency; the order is fixed, so deterministic
  if (j < D) {
    int i = i0;
    for (; i + 1 < i1; i += 2) {
      acc0 = fmaf(s_row[i], __bfloat162float(proj[(size_t)i * D + j]), acc0);
      acc1 = fmaf(s_row[i + 1], __bfloat162float(proj[(size_t)(i + 1) * D + j]), acc1);
    }
    if (i < i1) acc0 = fmaf(s_row[i], __bfloat162float(proj[(size_t)i * D + j]), acc0);
  }
  s_part[quarter * 64 + jj] = acc0 + acc1;
  __syncthreads();
  if (quarter == 0 && j < D) {
    const float f = (s_part[jj] + s_part[64 + jj]) + (s_part[128 + jj] + s_part[192 + jj]);
    feat[(size_t)b * D + j] = bias != nullptr ? f + bias[j] : f;
  }
}

// SigLIP's text tail, pool_proj_split_kernel's arithmetic on the last row of each sample (the tower attends
// bidirectionally over every position, pads included, and pools position T - 1), with LayerNorm at `eps` and a bias.
__global__ void __launch_bounds__(256)
pool_last_proj_split_kernel(const __nv_bfloat16* __restrict__ x, int T, int w, const float* __restrict__ gamma,
                            const float* __restrict__ beta, float eps, const __nv_bfloat16* __restrict__ proj, int D,
                            const float* __restrict__ bias, float* __restrict__ feat) {
  extern __shared__ float sm[];
  float* s_row = sm;                // [w]
  float* s_part = sm + w;           // [4][64]
  __shared__ float red[8];
  const int b = blockIdx.y, j0 = blockIdx.x * 64;
  const __nv_bfloat16* src = x + ((size_t)b * T + T - 1) * w;
  float part = 0.f;
  for (int j = threadIdx.x; j < w; j += blockDim.x) {
    const float f = __bfloat162float(src[j]);
    s_row[j] = f;
    part += f;
  }
  const float mean = block_sum(part, red) / (float)w;
  part = 0.f;
  for (int j = threadIdx.x; j < w; j += blockDim.x) {
    const float dlt = s_row[j] - mean;
    part += dlt * dlt;
  }
  const float rstd = rsqrtf(block_sum(part, red) / (float)w + eps);
  for (int j = threadIdx.x; j < w; j += blockDim.x) s_row[j] = (s_row[j] - mean) * rstd * gamma[j] + beta[j];
  __syncthreads();
  const int jj = threadIdx.x & 63, quarter = threadIdx.x >> 6;
  const int j = j0 + jj;
  const int per = (w + 3) / 4, i0 = quarter * per, i1 = min(w, i0 + per);
  float acc0 = 0.f, acc1 = 0.f;
  if (j < D) {
    int i = i0;
    for (; i + 1 < i1; i += 2) {
      acc0 = fmaf(s_row[i], __bfloat162float(proj[(size_t)i * D + j]), acc0);
      acc1 = fmaf(s_row[i + 1], __bfloat162float(proj[(size_t)(i + 1) * D + j]), acc1);
    }
    if (i < i1) acc0 = fmaf(s_row[i], __bfloat162float(proj[(size_t)i * D + j]), acc0);
  }
  s_part[quarter * 64 + jj] = acc0 + acc1;
  __syncthreads();
  if (quarter == 0 && j < D)
    feat[(size_t)b * D + j] = ((s_part[jj] + s_part[64 + jj]) + (s_part[128 + jj] + s_part[192 + jj])) + bias[j];
}

__global__ void __launch_bounds__(256)
feat_norm_cast_kernel(const float* __restrict__ feat, int D, void* __restrict__ out, int out_f16, int normalize) {
  __shared__ float red[8];
  const int b = blockIdx.x;
  float part = 0.f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const float v = feat[(size_t)b * D + j];
    part += v * v;
  }
  const float ss = block_sum(part, red);
  // reference: `features /= features.norm(dim=-1, keepdim=True)` — no epsilon (mapper.py:58,66)
  const float inv = normalize ? 1.0f / sqrtf(ss) : 1.0f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const float v = feat[(size_t)b * D + j] * inv;
    if (out_f16) reinterpret_cast<__half*>(out)[(size_t)b * D + j] = __float2half_rn(v);
    else reinterpret_cast<float*>(out)[(size_t)b * D + j] = v;
  }
}

int pool_ln_proj_norm(const __nv_bfloat16* x, int T, int w, const int* pool_idx, const float* gamma, const float* beta,
                      const __nv_bfloat16* proj, int D, float* feat, void* out, int out_f16, int normalize, int B,
                      cudaStream_t st) {
  if (B == 0) return B200_OK;
  const size_t smem = (size_t)(w + 256) * sizeof(float);
  B200_CHECK(smem <= 48 * 1024, B200_ERR_UNSUPPORTED, "pool_proj: width %d too large", w);
  pool_proj_split_kernel<<<dim3((D + 63) / 64, B), 256, smem, st>>>(x, T, w, pool_idx, gamma, beta, proj, D, nullptr,
                                                                     feat);
  B200_LAUNCH_OK();
  feat_norm_cast_kernel<<<B, 256, 0, st>>>(feat, D, out, out_f16, normalize);
  B200_LAUNCH_OK();
  return B200_OK;
}

int pool_last_ln_proj_bias_norm(const __nv_bfloat16* x, int T, int w, const float* gamma, const float* beta, float eps,
                                const __nv_bfloat16* proj, const float* bias, int D, float* feat, void* out, int out_f16,
                                int normalize, int B, cudaStream_t st) {
  if (B == 0) return B200_OK;
  const size_t smem = (size_t)(w + 256) * sizeof(float);
  B200_CHECK(smem <= 48 * 1024, B200_ERR_UNSUPPORTED, "pool_proj: width %d too large", w);
  pool_last_proj_split_kernel<<<dim3((D + 63) / 64, B), 256, smem, st>>>(x, T, w, gamma, beta, eps, proj, D, bias,
                                                                          feat);
  B200_LAUNCH_OK();
  feat_norm_cast_kernel<<<B, 256, 0, st>>>(feat, D, out, out_f16, normalize);
  B200_LAUNCH_OK();
  return B200_OK;
}

// feat[b] = x[b] (bf16 -> fp32), then normalised and cast as feat_norm_cast_kernel does.
__global__ void __launch_bounds__(256)
rows_feat_norm_cast_kernel(const __nv_bfloat16* __restrict__ x, int D, float* __restrict__ feat,
                           void* __restrict__ out, int out_f16, int normalize) {
  __shared__ float red[8];
  const int b = blockIdx.x;
  float part = 0.f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const float v = __bfloat162float(x[(size_t)b * D + j]);
    feat[(size_t)b * D + j] = v;
    part += v * v;
  }
  const float ss = block_sum(part, red);
  const float inv = normalize ? 1.0f / sqrtf(ss) : 1.0f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const float v = __bfloat162float(x[(size_t)b * D + j]) * inv;
    if (out_f16) reinterpret_cast<__half*>(out)[(size_t)b * D + j] = __float2half_rn(v);
    else reinterpret_cast<float*>(out)[(size_t)b * D + j] = v;
  }
}

int rows_feat_norm_cast(const __nv_bfloat16* x, int D, float* feat, void* out, int out_f16, int normalize, int B,
                        cudaStream_t st) {
  if (B == 0) return B200_OK;
  rows_feat_norm_cast_kernel<<<B, 256, 0, st>>>(x, D, feat, out, out_f16, normalize);
  B200_LAUNCH_OK();
  return B200_OK;
}

int pool_proj_bias_norm(const __nv_bfloat16* x, int T, int w, const __nv_bfloat16* proj, const float* bias, int D,
                        float* feat, void* out, int out_f16, int normalize, int B, cudaStream_t st) {
  if (B == 0) return B200_OK;
  const size_t smem = (size_t)(w + 256) * sizeof(float);
  B200_CHECK(smem <= 48 * 1024, B200_ERR_UNSUPPORTED, "pool_proj: width %d too large", w);
  pool_proj_split_kernel<<<dim3((D + 63) / 64, B), 256, smem, st>>>(x, T, w, nullptr, nullptr, nullptr, proj, D, bias,
                                                                     feat);
  B200_LAUNCH_OK();
  feat_norm_cast_kernel<<<B, 256, 0, st>>>(feat, D, out, out_f16, normalize);
  B200_LAUNCH_OK();
  return B200_OK;
}

// ---- BERT-family encoders (text_encoder.cu) --------------------------------------------------------------
// Embedding + LayerNorm: one block per row, 8 columns per thread in registers between the two passes.
__global__ void __launch_bounds__(256)
encoder_embed_kernel(const int64_t* __restrict__ ids, const __nv_bfloat16* __restrict__ word,
                     const float* __restrict__ tt0, const float* __restrict__ pos, int pos_off,
                     const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                     __nv_bfloat16* __restrict__ x, int T, int w, int vocab) {
  __shared__ float red[8];
  const int64_t r = blockIdx.x;
  const int t = (int)(r % T);
  const int c = threadIdx.x;          // 8-column chunk
  const bool live = c * 8 < w;
  int64_t tok = ids[r];
  if (tok < 0) tok = 0;
  if (tok >= vocab) tok = vocab - 1;
  float v[8];
  float part = 0.f;
  if (live) {
    const uint4 e = *reinterpret_cast<const uint4*>(word + tok * w + c * 8);
    const __nv_bfloat162* e2 = reinterpret_cast<const __nv_bfloat162*>(&e);
    const float* pr = pos + (size_t)(pos_off + t) * w + c * 8;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float2 f = __bfloat1622float2(e2[j]);
      float a = f.x, b = f.y;
      if (tt0 != nullptr) { a = a + tt0[c * 8 + 2 * j]; b = b + tt0[c * 8 + 2 * j + 1]; }
      v[2 * j] = a + pr[2 * j];
      v[2 * j + 1] = b + pr[2 * j + 1];
    }
#pragma unroll
    for (int j = 0; j < 8; j++) part += v[j];
  }
  const float mean = block_sum(part, red) / (float)w;
  part = 0.f;
  if (live) {
#pragma unroll
    for (int j = 0; j < 8; j++) part += (v[j] - mean) * (v[j] - mean);
  }
  const float rstd = rsqrtf(block_sum(part, red) / (float)w + eps);
  if (live) {
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int k = c * 8 + 2 * j;
      __nv_bfloat162 h = __floats2bfloat162_rn((v[2 * j] - mean) * rstd * gamma[k] + beta[k],
                                               (v[2 * j + 1] - mean) * rstd * gamma[k + 1] + beta[k + 1]);
      o[j] = *reinterpret_cast<uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(x + r * w + c * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}
int encoder_embed(const int64_t* ids, const __nv_bfloat16* word, const float* tt0, const float* pos, int pos_off,
                  const float* gamma, const float* beta, float eps, __nv_bfloat16* x, int B, int T, int w, int vocab,
                  cudaStream_t st) {
  B200_CHECK(w % 8 == 0 && w <= 2048, B200_ERR_UNSUPPORTED, "encoder_embed: width %d (need %%8, <= 2048)", w);
  if (B == 0) return B200_OK;
  const int threads = (w / 8 + 31) / 32 * 32;
  encoder_embed_kernel<<<(unsigned)((int64_t)B * T), threads, 0, st>>>(ids, word, tt0, pos, pos_off, gamma, beta, eps,
                                                                       x, T, w, vocab);
  B200_LAUNCH_OK();
  return B200_OK;
}

// The pieces of the masked-mean heads below.  s_row[j] = (sum over t < L, ascending, of x[b*T + t, j] in fp32) / L
// with L = len[b] clamped to 1..T: one thread per column.
__device__ __forceinline__ void masked_mean_row(const __nv_bfloat16* __restrict__ x, int T, int w,
                                                const int* __restrict__ len, int b, float* s_row) {
  const int L = min(max(len[b], 1), T);
  const __nv_bfloat16* src = x + (size_t)b * T * w;
  for (int j = threadIdx.x; j < w; j += blockDim.x) {
    float acc = 0.f;
    for (int t = 0; t < L; t++) acc += __bfloat162float(src[(size_t)t * w + j]);
    s_row[j] = acc / (float)L;
  }
}

// Column j0 + (threadIdx.x & 63) of s_row [K] @ WT [K, N] for a block of 256 threads: the reduction dimension is split
// over 4 quarters, each summed in two interleaved fma chains, and the quarters are added in a fixed order.  Every
// thread of the block must call it (it synchronises); the value is meaningful in threads 0..63 with column < N.
__device__ __forceinline__ float split_column_dot(const float* s_row, int K, const float* __restrict__ WT, int N,
                                                  int j0, float* s_part) {
  const int jj = threadIdx.x & 63, quarter = threadIdx.x >> 6;
  const int j = j0 + jj;
  const int per = (K + 3) / 4, i0 = quarter * per, i1 = min(K, i0 + per);
  float acc0 = 0.f, acc1 = 0.f;
  if (j < N) {
    int i = i0;
    for (; i + 1 < i1; i += 2) {
      acc0 = fmaf(s_row[i], WT[(size_t)i * N + j], acc0);
      acc1 = fmaf(s_row[i + 1], WT[(size_t)(i + 1) * N + j], acc1);
    }
    if (i < i1) acc0 = fmaf(s_row[i], WT[(size_t)i * N + j], acc0);
  }
  s_part[quarter * 64 + jj] = acc0 + acc1;
  __syncthreads();
  return (s_part[jj] + s_part[64 + jj]) + (s_part[128 + jj] + s_part[192 + jj]);
}

// Masked mean + projection, split like pool_proj_split_kernel: a block owns 64 output columns of one sample, forms
// the mean row itself (one thread per column, tokens in ascending order) and splits the projection over 4 quarters
// of the reduction dimension.
__global__ void __launch_bounds__(256)
masked_mean_proj_kernel(const __nv_bfloat16* __restrict__ x, int T, int w, const int* __restrict__ len,
                        const float* __restrict__ projT, const float* __restrict__ bias, int D,
                        float* __restrict__ feat) {
  extern __shared__ float sm[];
  float* s_row = sm;                // [w]
  float* s_part = sm + w;           // [4][64]
  const int b = blockIdx.y, j0 = blockIdx.x * 64;
  masked_mean_row(x, T, w, len, b, s_row);
  __syncthreads();
  const float f = split_column_dot(s_row, w, projT, D, j0, s_part);
  const int j = j0 + threadIdx.x;
  if (threadIdx.x < 64 && j < D) feat[(size_t)b * D + j] = bias != nullptr ? f + bias[j] : f;
}

// open_clip's MLP text head (proj "mlp": Linear(w, h, bias=False), GELU, Linear(h, D, bias=False)) on the masked
// mean, in two launches so that each layer is spread over (columns / 64) x B blocks.  Layer 1: every block forms the
// mean row of its sample, then hid[b, j] = gelu_erf(mean . W1T[:, j]) for its 64 columns j.
__global__ void __launch_bounds__(256)
masked_mean_mlp1_kernel(const __nv_bfloat16* __restrict__ x, int T, int w, const int* __restrict__ len,
                        const float* __restrict__ w1T, int h, float* __restrict__ hid) {
  extern __shared__ float sm[];
  float* s_row = sm;                // [w]
  float* s_part = sm + w;           // [4][64]
  const int b = blockIdx.y, j0 = blockIdx.x * 64;
  masked_mean_row(x, T, w, len, b, s_row);
  __syncthreads();
  const float y = split_column_dot(s_row, w, w1T, h, j0, s_part);
  const int j = j0 + threadIdx.x;
  if (threadIdx.x < 64 && j < h) hid[(size_t)b * h + j] = 0.5f * y * (1.0f + erff(y * 0.70710678118654752f));
}

// Layer 2: feat[b, j] = hid[b, :] . W2T[:, j] for the block's 64 columns j.
__global__ void __launch_bounds__(256)
mlp2_kernel(const float* __restrict__ hid, int h, const float* __restrict__ w2T, int D, float* __restrict__ feat) {
  extern __shared__ float sm[];
  float* s_row = sm;                // [h]
  float* s_part = sm + h;           // [4][64]
  const int b = blockIdx.y, j0 = blockIdx.x * 64;
  for (int i = threadIdx.x; i < h; i += blockDim.x) s_row[i] = hid[(size_t)b * h + i];
  __syncthreads();
  const float f = split_column_dot(s_row, h, w2T, D, j0, s_part);
  const int j = j0 + threadIdx.x;
  if (threadIdx.x < 64 && j < D) feat[(size_t)b * D + j] = f;
}

// len[b] = the first t with ids[b, t] == pad_id, or T when the row has none (right-padded rows: the token count).
__global__ void token_lengths_kernel(const int64_t* __restrict__ ids, int B, int T, int64_t pad_id,
                                     int* __restrict__ len) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int64_t* row = ids + (size_t)b * T;
  int t = 0;
  while (t < T && row[t] != pad_id) t++;
  len[b] = t;
}

// clip_back.py normalized(): a / |a|, with |a| == 0 replaced by 1 (a zero row stays zero, never NaN).
__global__ void __launch_bounds__(256)
feat_normalized_cast_kernel(const float* __restrict__ feat, int D, void* __restrict__ out, int out_f16, int normalize) {
  __shared__ float red[8];
  const int b = blockIdx.x;
  float part = 0.f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const float v = feat[(size_t)b * D + j];
    part += v * v;
  }
  float nrm = sqrtf(block_sum(part, red));
  if (!normalize || nrm == 0.f) nrm = 1.f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const float v = feat[(size_t)b * D + j] / nrm;
    if (out_f16) reinterpret_cast<__half*>(out)[(size_t)b * D + j] = __float2half_rn(v);
    else reinterpret_cast<float*>(out)[(size_t)b * D + j] = v;
  }
}

int masked_mean_proj_norm(const __nv_bfloat16* x, int T, int w, const int* len, const float* projT, const float* bias,
                          int D, float* feat, void* out, int out_f16, int normalize, int B, cudaStream_t st) {
  if (B == 0) return B200_OK;
  const size_t smem = (size_t)(w + 256) * sizeof(float);
  B200_CHECK(smem <= 48 * 1024, B200_ERR_UNSUPPORTED, "masked_mean_proj: width %d too large", w);
  masked_mean_proj_kernel<<<dim3((D + 63) / 64, B), 256, smem, st>>>(x, T, w, len, projT, bias, D, feat);
  B200_LAUNCH_OK();
  feat_normalized_cast_kernel<<<B, 256, 0, st>>>(feat, D, out, out_f16, normalize);
  B200_LAUNCH_OK();
  return B200_OK;
}

int masked_mean_mlp_norm(const __nv_bfloat16* x, int T, int w, const int* len, const float* w1T, int h,
                         const float* w2T, int D, float* hid, float* feat, void* out, int out_f16, int normalize, int B,
                         cudaStream_t st) {
  if (B == 0) return B200_OK;
  const size_t smem = (size_t)(std::max(w, h) + 256) * sizeof(float);
  B200_CHECK(smem <= 48 * 1024, B200_ERR_UNSUPPORTED, "masked_mean_mlp: width %d / hidden %d too large", w, h);
  masked_mean_mlp1_kernel<<<dim3((h + 63) / 64, B), 256, (size_t)(w + 256) * sizeof(float), st>>>(x, T, w, len, w1T, h,
                                                                                                   hid);
  B200_LAUNCH_OK();
  mlp2_kernel<<<dim3((D + 63) / 64, B), 256, (size_t)(h + 256) * sizeof(float), st>>>(hid, h, w2T, D, feat);
  B200_LAUNCH_OK();
  feat_normalized_cast_kernel<<<B, 256, 0, st>>>(feat, D, out, out_f16, normalize);
  B200_LAUNCH_OK();
  return B200_OK;
}

// The ConvNeXt head's first MLP layer on fp32 rows: hid[b, j] = gelu_erf(rows[b, :] . w1T[:, j] + b1[j]).
__global__ void __launch_bounds__(256)
rows_mlp1_bias_kernel(const float* __restrict__ rows, int w, const float* __restrict__ w1T,
                      const float* __restrict__ b1, int h, float* __restrict__ hid) {
  extern __shared__ float sm[];
  float* s_row = sm;                // [w]
  float* s_part = sm + w;           // [4][64]
  const int b = blockIdx.y, j0 = blockIdx.x * 64;
  for (int i = threadIdx.x; i < w; i += blockDim.x) s_row[i] = rows[(size_t)b * w + i];
  __syncthreads();
  const float y = split_column_dot(s_row, w, w1T, h, j0, s_part);
  const int j = j0 + threadIdx.x;
  if (threadIdx.x < 64 && j < h) {
    const float v = y + b1[j];
    hid[(size_t)b * h + j] = 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
  }
}

int rows_head_norm(const float* rows, int w, const float* w1T, const float* b1, int h, const float* w2T, int D,
                   float* hid, float* feat, void* out, int out_f16, int normalize, int B, cudaStream_t st) {
  if (B == 0) return B200_OK;
  const int k2 = w1T != nullptr ? h : w;
  B200_CHECK((size_t)(std::max(w, k2) + 256) * sizeof(float) <= 48 * 1024, B200_ERR_UNSUPPORTED,
             "rows_head: width %d / hidden %d too large", w, h);
  if (w1T != nullptr) {
    rows_mlp1_bias_kernel<<<dim3((h + 63) / 64, B), 256, (size_t)(w + 256) * sizeof(float), st>>>(rows, w, w1T, b1, h,
                                                                                                   hid);
    B200_LAUNCH_OK();
  }
  mlp2_kernel<<<dim3((D + 63) / 64, B), 256, (size_t)(k2 + 256) * sizeof(float), st>>>(w1T != nullptr ? hid : rows, k2,
                                                                                       w2T, D, feat);
  B200_LAUNCH_OK();
  feat_norm_cast_kernel<<<B, 256, 0, st>>>(feat, D, out, out_f16, normalize);
  B200_LAUNCH_OK();
  return B200_OK;
}

int token_lengths(const int64_t* ids, int B, int T, int64_t pad_id, int* len, cudaStream_t st) {
  if (B == 0) return B200_OK;
  token_lengths_kernel<<<(B + 127) / 128, 128, 0, st>>>(ids, B, T, pad_id, len);
  B200_LAUNCH_OK();
  return B200_OK;
}

}  // namespace b200
