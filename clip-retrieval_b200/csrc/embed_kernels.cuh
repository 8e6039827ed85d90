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
// The same LayerNorm with the epsilon as an argument (BERT-family encoders carry it in their config: 1e-5, 1e-12).
int layernorm_rows_eps(const __nv_bfloat16* in, int64_t in_ld, __nv_bfloat16* out, int64_t out_ld, const float* gamma,
                       const float* beta, int64_t rows, int w, float eps, cudaStream_t st);
// K4: multi-head attention over the fused qkv buffer [B*T, 3w] -> out [B*T, w]; causal for text.  mma.sync kernels
// (attention.cu) for the head dimensions the wgmma kernel does not take (80, 88, 96, 104, 128) and for head dim 64 past
// T = 320:
// whole K/V of a head in shared memory while it fits in 200 KB, K/V streamed through a ring of 64-key stages beyond.
// len (device int32 [B], values 1..T, or nullptr = T): sample b attends to its keys < len[b], and its rows >= len[b]
// of `out` are zeros — the key-padding mask of a bidirectional encoder (both kernels).
int attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int T, int heads, int w, int causal, cudaStream_t st,
              const int* len = nullptr);
// K4 on wgmma (attention_wgmma.cu) for head dim 64, T <= 320: tmQKV is a 3-D map over the qkv buffer seen as
// [samples >= B, T, 3w] (make_tmap_3d, row pitch 3w, plane pitch T * 3w) with boxes of 64 tokens x 64 columns (128B
// swizzle); a box is clipped at token T of its sample, so keys and values past the end read as zeros.
bool attention_wgmma_supported(int T, int heads, int w);
int attention_wgmma(const CUtensorMap& tmQKV, __nv_bfloat16* out, int B, int T, int heads, int w, int causal,
                    cudaStream_t st, const int* len = nullptr);
// K8/K10/K11: pooled row (x[b*T + pool_index(b)]) -> LN -> @ proj [w, D] into feat fp32 [B, D] (blocks of 64 output
// columns per sample) -> optional L2 normalise -> fp16 or fp32.  pool_idx == nullptr pools token 0 (vision); else row
// pool_idx[b] (text EOT).
int pool_ln_proj_norm(const __nv_bfloat16* x, int T, int w, const int* pool_idx, const float* gamma, const float* beta,
                      const __nv_bfloat16* proj, int D, float* feat, void* out, int out_f16, int normalize, int B,
                      cudaStream_t st);
// BERT-family embedding: x[b*T + t, :] = LN_eps((word[ids[b,t]] + tt0) + pos[pos_off + t]) in fp32, stored bf16
// (HF's order of additions; tt0 = token-type row 0, or nullptr when the model has no token types).  word bf16
// [vocab, w]; tt0, pos, gamma, beta fp32.  Ids outside [0, vocab) are clamped.
int encoder_embed(const int64_t* ids, const __nv_bfloat16* word, const float* tt0, const float* pos, int pos_off,
                  const float* gamma, const float* beta, float eps, __nv_bfloat16* x, int B, int T, int w, int vocab,
                  cudaStream_t st);
// Masked mean pool + projection + normalise: m = (sum over t < len[b], ascending, of x[b*T + t, :] in fp32) / len[b];
// f = m @ projT [w, D] fp32 (+ bias[D] fp32 | nullptr) into feat fp32 [B, D] (blocks of 64 output columns per
// sample); out = f / (normalize ? (|f| == 0 ? 1 : |f|) : 1) as fp16 or fp32 (clip_back.py normalized()).
int masked_mean_proj_norm(const __nv_bfloat16* x, int T, int w, const int* len, const float* projT, const float* bias,
                          int D, float* feat, void* out, int out_f16, int normalize, int B, cudaStream_t st);
// open_clip's MLP text head on the masked mean m of masked_mean_proj_norm: hid = gelu_erf(m @ w1T [w, h]) into hid
// fp32 [B, h], f = hid @ w2T [h, D] into feat fp32 [B, D], all in fp32 (each layer in blocks of 64 output columns
// per sample); out as masked_mean_proj_norm writes it.
int masked_mean_mlp_norm(const __nv_bfloat16* x, int T, int w, const int* len, const float* w1T, int h,
                         const float* w2T, int D, float* hid, float* feat, void* out, int out_f16, int normalize, int B,
                         cudaStream_t st);
// len[b] = index of the first pad_id in row b of ids [B, T], T when there is none (0 for a row of padding only).
int token_lengths(const int64_t* ids, int B, int T, int64_t pad_id, int* len, cudaStream_t st);
// argmax(tokens, dim=-1) (first maximum) -> pool_idx[b]
int token_argmax(const int64_t* tokens, int* pool_idx, int B, int T, cudaStream_t st);

}  // namespace b200
