// Non-GEMM kernels of the embed path (declarations; embed_kernels.cu, attention.cu).
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace b200 {

// K1 (SURVEY.md §2.2): pixels fp32 NCHW [B,3,S,S] -> patch matrix bf16 [B*g*g, Kp], column index
// c*p*p + i*p + j (the conv weight's own flattening); columns >= 3*p*p are never written (zero).
int im2col_patches(const float* pixels, __nv_bfloat16* cols, int B, int S, int p, int Kp, cudaStream_t st);
// x[b*T + 0, :] = class_embedding + positional_embedding[0]  (K2)
int write_cls_rows(__nv_bfloat16* x, const float* cls_plus_pos0, int B, int T, int w, cudaStream_t st);
// K9: x[b*T + t, :] = token_embedding[tokens[b,t]] + positional_embedding[t]
int text_embed(const int64_t* tokens, const __nv_bfloat16* tok_emb, const float* pos_emb, __nv_bfloat16* x, int B, int T,
               int w, int vocab, cudaStream_t st);
// LayerNorm over the last dimension, eps 1e-5, fp32 statistics: out = (x - mean) * rstd * g + b.
// rows of `w` bf16 elements, in_ld/out_ld in elements; in == out allowed.
int layernorm_rows(const __nv_bfloat16* in, int64_t in_ld, __nv_bfloat16* out, int64_t out_ld, const float* gamma,
                   const float* beta, int64_t rows, int w, cudaStream_t st);
// (mean, M2) per 64-column slot of every row of x [rows, w] (w % 64 == 0): seeds GemmEpilogue::ln_stats.
int row_stats(const __nv_bfloat16* x, int64_t rows, int w, float2* stats, cudaStream_t st);
// K4: multi-head attention over the fused qkv buffer [B*T, 3w] -> out [B*T, w]; causal for text.  mma.sync kernel
// (attention.cu) for the head dimensions the wgmma kernel does not take (80, 96, 128).
int attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int T, int heads, int w, int causal, cudaStream_t st);
// K4 on wgmma (attention_wgmma.cu) for head dim 64, T <= 320: tmQKV is a map over the qkv buffer [rows, 3w] with
// boxes of 64 rows x 64 columns (128B swizzle), rows >= B*T of it are never used unmasked.
bool attention_wgmma_supported(int T, int heads, int w);
int attention_wgmma(const CUtensorMap& tmQKV, const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int T, int heads, int w,
                    int causal, cudaStream_t st);
// K8/K10/K11: pooled row (x[b*T + pool_index(b)]) -> LN -> @ proj [w, D] -> optional L2 normalise
// -> fp16 or fp32.  pool_idx == nullptr pools token 0 (vision); else row pool_idx[b] (text EOT).
int pool_ln_proj_norm(const __nv_bfloat16* x, int T, int w, const int* pool_idx, const float* gamma, const float* beta,
                      const __nv_bfloat16* proj, int D, void* out, int out_f16, int normalize, int B, cudaStream_t st,
                      float* feat_scratch = nullptr);   // fp32 [B, D]: when given, the projection is split over D / 64 blocks per sample
// argmax(tokens, dim=-1) (first maximum) -> pool_idx[b]
int token_argmax(const int64_t* tokens, int* pool_idx, int B, int T, cudaStream_t st);

}  // namespace b200
