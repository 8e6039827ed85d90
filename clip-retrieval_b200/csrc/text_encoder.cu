// BERT-family text encoder handle: the multilingual text towers behind `use_mclip` (M-CLIP XLM-RoBERTa-Large for the
// query service, clip_back.py:836-859; the SentenceTransformer DistilBERT of the mapper, mapper.py:44-47,62-63).
//
// Forward of a batch right-padded to T tokens with per-sample lengths len[b]:
//   x = LN_eps((word[id] + token_type[0]) + position[position_offset + t])
//   per layer (post-LN):  x = LN1(x + Wo · attn(Wqkv · x + b, keys < len[b]) + bo)
//                         x = LN2(x + W2 · gelu_erf(W1 · x + b1) + b2)
//   out = normalized(mean over t < len[b] of x, @ projection (+ bias))
//   or, with the MLP head of open_clip's HF text towers (b200_text_encoder_create_mlp):
//   out = normalized(W2 · gelu_erf(W1 · mean over t < len[b] of x)), no biases, all in fp32
// Weights bf16 [N, K] for the GEMMs (q, k, v concatenated into one [3w, w] in-projection at load time), LayerNorm
// affine, biases, position / token-type tables and the projection fp32.  Activations bf16 [rows, width] sized for
// max_batch x max_tokens rows, so the GEMM operand maps are built once; the 3-D map of the wgmma attention depends
// on T and is cached per T.
#include "common.cuh"
#include "embed_kernels.cuh"
#include "gemm.cuh"
#include "layers.cuh"
#include "weights.cuh"
#include <algorithm>
#include <map>
#include <mutex>
#include <string>
#include <vector>

namespace b200 {
namespace {

struct EncLayer {
  Linear qkv, out, fc1, fc2;
  float *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
};

enum { ENC_GEMM = 0, ENC_ATTN = 1, ENC_LN = 2, ENC_OTHER = 3, ENC_CLASSES = 4 };

}  // namespace
}  // namespace b200

struct b200_text_encoder {
  b200_text_encoder_config cfg;
  int device = 0, sms = 132;
  bool loaded = false;
  b200::DeviceAllocs allocs;
  // weights
  __nv_bfloat16* word = nullptr;   // [vocab, w]
  float* tt0 = nullptr;            // token type 0 [w] or null
  float* pos = nullptr;            // [positions, w]
  float *emb_g = nullptr, *emb_b = nullptr;
  std::vector<b200::EncLayer> L;
  float* projT = nullptr;          // [w, D] (linear head)
  float* proj_b = nullptr;         // [D] or null
  int hidden = 0;                  // > 0: the MLP head, w -> hidden -> D
  float *w1T = nullptr, *w2T = nullptr;   // [w, hidden], [hidden, D]
  float* hid = nullptr;            // [max_batch, hidden]
  // activations
  __nv_bfloat16 *x = nullptr, *qkv = nullptr, *a = nullptr, *f = nullptr;
  CUtensorMap tm_x, tm_a, tm_f;
  std::map<int, CUtensorMap> tm_qkv;   // per T: make_qkv_map over max_batch samples
  float* feat = nullptr;               // [max_batch, D]
  // staging of the host entry
  int64_t* s_ids = nullptr;
  int* s_len = nullptr;
  float* s_out = nullptr;
  std::mutex mu;                  // held by both encode entries while they enqueue
  b200::StreamFence act;          // orders calls on different streams: they share the activation buffers
  b200::SpanTimer timer;          // timing; timer.launches = kernels of the last encode call
};

namespace b200 {
namespace {

int enc_gemm(b200_text_encoder* m, const CUtensorMap& tmA, const Linear& l, int M, const GemmEpilogue& ep,
             cudaStream_t st) {
  TimedSpan sp(m->timer, ENC_GEMM, st, 1);
  return linear_gemm(l, tmA, M, ep, m->sms, st);
}

int enc_ln(b200_text_encoder* m, const float* g, const float* b, int64_t rows, cudaStream_t st) {
  TimedSpan sp(m->timer, ENC_LN, st, 1);
  const int w = m->cfg.width;
  return layernorm_rows_eps(m->x, w, m->x, w, g, b, rows, w, m->cfg.layer_norm_eps, st);
}

// One chunk of at most max_batch samples.
int enc_forward(b200_text_encoder* m, const int64_t* d_ids, const int* d_len, int B, int T, void* d_out, int out_f16,
                int normalize, cudaStream_t st) {
  const b200_text_encoder_config& c = m->cfg;
  const int w = c.width, M = B * T;
  const CUtensorMap* tmq = nullptr;
  if (attention_wgmma_supported(T, c.heads, w)) {
    auto it = m->tm_qkv.find(T);
    if (it == m->tm_qkv.end()) {
      CUtensorMap tm;
      B200_TRY(make_qkv_map(&tm, m->qkv, c.max_batch, T, w));
      it = m->tm_qkv.emplace(T, tm).first;
    }
    tmq = &it->second;
  }
  { TimedSpan sp(m->timer, ENC_OTHER, st, 1);
    B200_TRY(encoder_embed(d_ids, m->word, m->tt0, m->pos, c.position_offset, m->emb_g, m->emb_b, c.layer_norm_eps,
                           m->x, B, T, w, c.vocab_size, st)); }
  for (const EncLayer& L : m->L) {
    GemmEpilogue e1; e1.out = m->qkv; e1.out_ld = 3 * w;
    B200_TRY(enc_gemm(m, m->tm_x, L.qkv, M, e1, st));
    { TimedSpan sp(m->timer, ENC_ATTN, st, 1);
      B200_TRY(qkv_attention(tmq, m->qkv, m->a, B, T, c.heads, w, 0, st, d_len)); }
    GemmEpilogue e2; e2.out = m->x; e2.out_ld = w; e2.residual = m->x; e2.res_ld = w;
    B200_TRY(enc_gemm(m, m->tm_a, L.out, M, e2, st));
    B200_TRY(enc_ln(m, L.ln1_g, L.ln1_b, M, st));
    GemmEpilogue e3; e3.out = m->f; e3.out_ld = c.ffn; e3.act = ACT_GELU;
    B200_TRY(enc_gemm(m, m->tm_x, L.fc1, M, e3, st));
    GemmEpilogue e4; e4.out = m->x; e4.out_ld = w; e4.residual = m->x; e4.res_ld = w;
    B200_TRY(enc_gemm(m, m->tm_f, L.fc2, M, e4, st));
    B200_TRY(enc_ln(m, L.ln2_g, L.ln2_b, M, st));
  }
  if (m->hidden > 0) {
    TimedSpan sp(m->timer, ENC_OTHER, st, 3);
    return masked_mean_mlp_norm(m->x, T, w, d_len, m->w1T, m->hidden, m->w2T, c.out_dim, m->hid, m->feat, d_out, out_f16,
                                normalize, B, st);
  }
  TimedSpan sp(m->timer, ENC_OTHER, st, 2);
  return masked_mean_proj_norm(m->x, T, w, d_len, m->projT, m->proj_b, c.out_dim, m->feat, d_out, out_f16, normalize,
                               B, st);
}

int enc_encode(b200_text_encoder* m, const int64_t* d_ids, const int* d_len, int B, int T, void* d_out, int out_dtype,
               int normalize, cudaStream_t st) {
  B200_CHECK(m->loaded, B200_ERR_STATE, "text_encoder: weights not loaded");
  B200_CHECK(B >= 0 && (B == 0 || (d_ids && d_len && d_out)), B200_ERR_INVALID, "text_encoder: bad argument");
  B200_CHECK(T >= 1 && T <= m->cfg.max_tokens, B200_ERR_INVALID, "text_encoder: T = %d outside 1..%d (max_tokens)", T,
             m->cfg.max_tokens);
  B200_CHECK(out_dtype == B200_OUT_F16 || out_dtype == B200_OUT_F32, B200_ERR_INVALID, "text_encoder: out_dtype %d",
             out_dtype);
  m->timer.launches = 0;
  const int mb = m->cfg.max_batch;
  const size_t out_stride = (size_t)m->cfg.out_dim * (out_dtype == B200_OUT_F16 ? 2 : 4);
  for (int b0 = 0; b0 < B; b0 += mb) {
    const int nb = std::min(mb, B - b0);
    B200_TRY(enc_forward(m, d_ids + (size_t)b0 * T, d_len + b0, nb, T, (char*)d_out + b0 * out_stride,
                         out_dtype == B200_OUT_F16, normalize, st));
  }
  return B200_OK;
}

}  // namespace
}  // namespace b200

using namespace b200;

namespace b200 {
namespace {

// hidden == 0: the linear projection head; > 0: the MLP head (cfg->proj_bias must be 0).
int text_encoder_create(const b200_text_encoder_config* cfg, int hidden, int device, b200_text_encoder** out) {
  B200_CHECK(cfg && out, B200_ERR_INVALID, "text_encoder_create: null argument");
  const b200_text_encoder_config& c = *cfg;
  B200_CHECK(c.layers >= 1 && c.heads >= 1 && c.width == 64 * c.heads && c.width <= 2048 && c.ffn >= 64 &&
                 c.ffn % 64 == 0 && c.vocab_size >= 1 && c.type_vocab_size >= 0 && c.position_offset >= 0 &&
                 c.max_positions >= 1 && c.layer_norm_eps > 0.f && c.out_dim >= 1 && c.max_batch >= 1 &&
                 c.max_tokens >= 1 && c.position_offset + c.max_tokens <= c.max_positions && c.max_tokens <= 512,
             B200_ERR_INVALID,
             "text_encoder_create: bad config (head dim 64, width <= 2048, ffn %% 64 == 0, eps > 0, "
             "position_offset + max_tokens <= max_positions, max_tokens <= 512)");
  int ndev = 0;
  B200_CUDA(cudaGetDeviceCount(&ndev));
  B200_CHECK(device >= 0 && device < ndev, B200_ERR_INVALID, "text_encoder_create: device %d of %d", device, ndev);
  DeviceGuard g(device);
  b200_text_encoder* m = new (std::nothrow) b200_text_encoder();
  B200_CHECK(m != nullptr, B200_ERR_OOM, "text_encoder_create: host allocation failed");
  m->cfg = c;
  m->device = device;
  m->sms = sm_count(device);
  m->hidden = hidden;
  auto build = [&]() -> int {
    const int w = c.width;
    const size_t rows = (size_t)c.max_batch * c.max_tokens;
    DeviceAllocs& al = m->allocs;
    B200_TRY(al.alloc(&m->word, (size_t)c.vocab_size * w));
    if (c.type_vocab_size > 0) B200_TRY(al.alloc(&m->tt0, (size_t)w));
    B200_TRY(al.alloc(&m->pos, (size_t)c.max_positions * w));
    B200_TRY(al.alloc(&m->emb_g, (size_t)w));
    B200_TRY(al.alloc(&m->emb_b, (size_t)w));
    m->L.resize(c.layers);
    for (EncLayer& L : m->L) {
      B200_TRY(make_linear(al, &L.qkv, 3 * w, w, true));
      B200_TRY(make_linear(al, &L.out, w, w, true));
      B200_TRY(make_linear(al, &L.fc1, c.ffn, w, true));
      B200_TRY(make_linear(al, &L.fc2, w, c.ffn, true));
      B200_TRY(al.alloc(&L.ln1_g, (size_t)w)); B200_TRY(al.alloc(&L.ln1_b, (size_t)w));
      B200_TRY(al.alloc(&L.ln2_g, (size_t)w)); B200_TRY(al.alloc(&L.ln2_b, (size_t)w));
    }
    if (hidden > 0) {
      B200_TRY(al.alloc(&m->w1T, (size_t)w * hidden));
      B200_TRY(al.alloc(&m->w2T, (size_t)hidden * c.out_dim));
      B200_TRY(al.alloc(&m->hid, (size_t)c.max_batch * hidden));
    } else {
      B200_TRY(al.alloc(&m->projT, (size_t)w * c.out_dim));
      if (c.proj_bias) B200_TRY(al.alloc(&m->proj_b, (size_t)c.out_dim));
    }
    B200_TRY(al.alloc(&m->x, rows * w));
    B200_TRY(al.alloc(&m->qkv, rows * 3 * w));
    B200_TRY(al.alloc(&m->a, rows * w));
    B200_TRY(al.alloc(&m->f, rows * c.ffn));
    B200_TRY(make_tmap_2d(&m->tm_x, m->x, 1, rows, w, w, GEMM_BM, GEMM_BK));
    B200_TRY(make_tmap_2d(&m->tm_a, m->a, 1, rows, w, w, GEMM_BM, GEMM_BK));
    B200_TRY(make_tmap_2d(&m->tm_f, m->f, 1, rows, c.ffn, c.ffn, GEMM_BM, GEMM_BK));
    B200_TRY(al.alloc(&m->feat, (size_t)c.max_batch * c.out_dim));
    B200_TRY(al.alloc(&m->s_ids, rows));
    B200_TRY(al.alloc(&m->s_len, (size_t)c.max_batch));
    B200_TRY(al.alloc(&m->s_out, (size_t)c.max_batch * c.out_dim));
    return B200_OK;
  };
  const int rc = build();
  if (rc != B200_OK) {
    b200_text_encoder_destroy(m);
    return rc;
  }
  *out = m;
  return B200_OK;
}

}  // namespace

}  // namespace b200

extern "C" {

int b200_text_encoder_create(const b200_text_encoder_config* cfg, int device, b200_text_encoder** out) {
  return text_encoder_create(cfg, 0, device, out);
}

int b200_text_encoder_create_mlp(const b200_text_encoder_config* cfg, int hidden, int device, b200_text_encoder** out) {
  B200_CHECK(cfg && hidden >= 1 && hidden <= 12 * 1024 - 256 && cfg->proj_bias == 0, B200_ERR_INVALID,
             "text_encoder_create_mlp: hidden %d (1..%d) and proj_bias 0 required", hidden, 12 * 1024 - 256);
  return text_encoder_create(cfg, hidden, device, out);
}

int b200_text_encoder_destroy(b200_text_encoder* m) {
  if (!m) return B200_OK;
  DeviceGuard g(m->device);
  cudaDeviceSynchronize();
  m->allocs.free_all();
  delete m;
  return B200_OK;
}

int b200_text_encoder_load_weights(b200_text_encoder* m, const b200_tensor_view* tensors, int n) {
  B200_CHECK(m && tensors && n > 0, B200_ERR_INVALID, "text_encoder_load_weights: bad argument");
  DeviceGuard g(m->device);
  Loader ld;
  B200_TRY(ld.index(tensors, n));
  const b200_text_encoder_config& c = m->cfg;
  const size_t w = c.width, D = c.out_dim, ffn = c.ffn;
  B200_TRY(ld.put_bf16("embeddings.word_embeddings.weight", m->word, (size_t)c.vocab_size, w, w));
  B200_TRY(ld.put_f32("embeddings.position_embeddings.weight", m->pos, (size_t)c.max_positions * w));
  if (c.type_vocab_size > 0) {
    // token type 0 only: the first row of the table
    const b200_tensor_view* tt = ld.find("embeddings.token_type_embeddings.weight", (size_t)c.type_vocab_size * w);
    if (!tt) return B200_ERR_INVALID;
    std::vector<float> row(w);
    for (size_t j = 0; j < w; j++) row[j] = view_get(*tt, j);
    B200_CUDA(cudaMemcpy(m->tt0, row.data(), w * 4, cudaMemcpyHostToDevice));
  }
  B200_TRY(ld.put_f32("embeddings.LayerNorm.weight", m->emb_g, w));
  B200_TRY(ld.put_f32("embeddings.LayerNorm.bias", m->emb_b, w));
  for (int i = 0; i < c.layers; i++) {
    EncLayer& L = m->L[i];
    const std::string p = "encoder.layer." + std::to_string(i) + ".";
    const char* qkv[3] = {"query", "key", "value"};
    for (int k = 0; k < 3; k++) {
      B200_TRY(ld.put_bf16(p + "attention.self." + qkv[k] + ".weight", L.qkv.w + k * w * w, w, w, w));
      B200_TRY(ld.put_f32(p + "attention.self." + qkv[k] + ".bias", L.qkv.b + k * w, w));
    }
    B200_TRY(ld.put_bf16(p + "attention.output.dense.weight", L.out.w, w, w, w));
    B200_TRY(ld.put_f32(p + "attention.output.dense.bias", L.out.b, w));
    B200_TRY(ld.put_f32(p + "attention.output.LayerNorm.weight", L.ln1_g, w));
    B200_TRY(ld.put_f32(p + "attention.output.LayerNorm.bias", L.ln1_b, w));
    B200_TRY(ld.put_bf16(p + "intermediate.dense.weight", L.fc1.w, ffn, w, w));
    B200_TRY(ld.put_f32(p + "intermediate.dense.bias", L.fc1.b, ffn));
    B200_TRY(ld.put_bf16(p + "output.dense.weight", L.fc2.w, w, ffn, ffn));
    B200_TRY(ld.put_f32(p + "output.dense.bias", L.fc2.b, w));
    B200_TRY(ld.put_f32(p + "output.LayerNorm.weight", L.ln2_g, w));
    B200_TRY(ld.put_f32(p + "output.LayerNorm.bias", L.ln2_b, w));
  }
  // nn.Linear weight [N, K] -> fp32 [K, N]: a projection thread reads one output column, consecutive threads
  // consecutive columns
  auto put_transposed = [&](const char* name, float* dst, size_t N, size_t K) -> int {
    const b200_tensor_view* pw = ld.find(name, N * K);
    if (!pw) return B200_ERR_INVALID;
    std::vector<float> t(K * N);
    for (size_t d = 0; d < N; d++)
      for (size_t k = 0; k < K; k++) t[k * N + d] = view_get(*pw, d * K + k);
    B200_CUDA(cudaMemcpy(dst, t.data(), t.size() * 4, cudaMemcpyHostToDevice));
    return B200_OK;
  };
  if (m->hidden > 0) {
    B200_TRY(put_transposed("projection.0.weight", m->w1T, (size_t)m->hidden, w));
    B200_TRY(put_transposed("projection.2.weight", m->w2T, D, (size_t)m->hidden));
  } else {
    B200_TRY(put_transposed("projection.weight", m->projT, D, w));
  }
  if (c.proj_bias) B200_TRY(ld.put_f32("projection.bias", m->proj_b, D));
  B200_CUDA(cudaDeviceSynchronize());
  m->loaded = true;
  return B200_OK;
}

int b200_text_encoder_encode_device(b200_text_encoder* m, const int64_t* d_ids, const int32_t* d_len, int B, int T,
                                    void* d_out, int out_dtype, int normalize, void* stream) {
  B200_CHECK(m, B200_ERR_INVALID, "text_encoder_encode: null handle");
  std::lock_guard<std::mutex> lock(m->mu);
  DeviceGuard g(m->device);
  const cudaStream_t st = (cudaStream_t)stream;
  B200_TRY(m->act.acquire(st));
  const int rc = enc_encode(m, d_ids, d_len, B, T, d_out, out_dtype, normalize, st);
  B200_TRY(m->act.release(st));
  return rc;
}

int b200_text_encoder_encode(b200_text_encoder* m, const int64_t* h_ids, const int32_t* h_len, int B, int T,
                             void* h_out, int out_dtype, int normalize) {
  B200_CHECK(m && B >= 0 && (B == 0 || (h_ids && h_len && h_out)), B200_ERR_INVALID, "text_encoder_encode: bad argument");
  B200_CHECK(T >= 1 && T <= m->cfg.max_tokens, B200_ERR_INVALID, "text_encoder_encode: T = %d outside 1..%d", T,
             m->cfg.max_tokens);
  for (int b = 0; b < B; b++)
    B200_CHECK(h_len[b] >= 1 && h_len[b] <= T, B200_ERR_INVALID, "text_encoder_encode: len[%d] = %d outside 1..%d", b,
               h_len[b], T);
  std::lock_guard<std::mutex> lock(m->mu);
  DeviceGuard g(m->device);
  B200_TRY(m->act.acquire(nullptr));   // the legacy stream, which does not wait for work on non-blocking streams
  const int mb = m->cfg.max_batch;
  const size_t out_stride = (size_t)m->cfg.out_dim * (out_dtype == B200_OUT_F16 ? 2 : 4);
  int launches = 0;
  for (int b0 = 0; b0 < B; b0 += mb) {
    const int nb = std::min(mb, B - b0);
    B200_CUDA(cudaMemcpy(m->s_ids, h_ids + (size_t)b0 * T, (size_t)nb * T * 8, cudaMemcpyHostToDevice));
    B200_CUDA(cudaMemcpy(m->s_len, h_len + b0, (size_t)nb * 4, cudaMemcpyHostToDevice));
    B200_TRY(enc_encode(m, m->s_ids, m->s_len, nb, T, m->s_out, out_dtype, normalize, nullptr));
    launches += m->timer.launches;
    B200_CUDA(cudaMemcpy((char*)h_out + b0 * out_stride, m->s_out, nb * out_stride, cudaMemcpyDeviceToHost));
  }
  B200_TRY(m->act.release(nullptr));
  m->timer.launches = launches;
  return B200_OK;
}

int b200_text_encoder_set_profiling(b200_text_encoder* m, int on) {
  B200_CHECK(m, B200_ERR_INVALID, "text_encoder_set_profiling: null handle");
  m->timer.set_profiling(on != 0);
  return B200_OK;
}

int b200_text_encoder_last_timing(b200_text_encoder* m, float* ms_by_class, int* launches) {
  B200_CHECK(m && ms_by_class, B200_ERR_INVALID, "text_encoder_last_timing: null argument");
  DeviceGuard g(m->device);
  B200_TRY(m->timer.collect(ms_by_class, ENC_CLASSES));
  if (launches) *launches = m->timer.launches;
  return B200_OK;
}

int b200_layernorm_eps_bf16_device(const void* d_in, void* d_out, const float* d_gamma, const float* d_beta,
                                   int64_t rows, int w, float eps, int device, void* stream) {
  B200_CHECK(d_in && d_out && d_gamma && d_beta && rows >= 0 && eps > 0.f, B200_ERR_INVALID, "layernorm: bad argument");
  DeviceGuard g(device);
  return layernorm_rows_eps((const __nv_bfloat16*)d_in, w, (__nv_bfloat16*)d_out, w, d_gamma, d_beta, rows, w, eps,
                            (cudaStream_t)stream);
}

int b200_attention_len_bf16_device(const void* d_qkv, const int32_t* d_len, void* d_out, int B, int T, int heads, int w,
                                   int device, void* stream) {
  B200_CHECK(d_qkv && d_len && d_out && B >= 0 && T >= 1, B200_ERR_INVALID, "attention_len: bad argument");
  DeviceGuard g(device);
  return qkv_attention(nullptr, (const __nv_bfloat16*)d_qkv, (__nv_bfloat16*)d_out, B, T, heads, w, 0,
                       (cudaStream_t)stream, d_len);
}

int b200_text_lengths_device(const int64_t* d_ids, int B, int T, int64_t pad_id, int32_t* d_len, void* stream) {
  B200_CHECK(B >= 0 && T >= 1 && (B == 0 || (d_ids && d_len)), B200_ERR_INVALID, "text_lengths: bad argument");
  return token_lengths(d_ids, B, T, pad_id, d_len, (cudaStream_t)stream);
}

int b200_mean_mlp_head_device(const void* d_x, int B, int T, int w, const int32_t* d_len, const float* d_w1T,
                              int hidden, const float* d_w2T, int D, float* d_hid, float* d_feat, void* d_out,
                              int out_dtype, int normalize, int device, void* stream) {
  B200_CHECK(B >= 0 && T >= 1 && w >= 1 && hidden >= 1 && D >= 1 &&
                 (B == 0 || (d_x && d_len && d_w1T && d_w2T && d_hid && d_feat && d_out)) &&
                 (out_dtype == B200_OUT_F16 || out_dtype == B200_OUT_F32),
             B200_ERR_INVALID, "mean_mlp_head: bad argument");
  DeviceGuard g(device);
  return masked_mean_mlp_norm((const __nv_bfloat16*)d_x, T, w, d_len, d_w1T, hidden, d_w2T, D, d_hid, d_feat, d_out,
                              out_dtype == B200_OUT_F16, normalize, B, (cudaStream_t)stream);
}

int b200_mean_proj_head_device(const void* d_x, int B, int T, int w, const int32_t* d_len, const float* d_projT,
                               const float* d_bias, int D, float* d_feat, void* d_out, int out_dtype, int normalize,
                               int device, void* stream) {
  B200_CHECK(B >= 0 && T >= 1 && w >= 1 && D >= 1 && (B == 0 || (d_x && d_len && d_projT && d_feat && d_out)) &&
                 (out_dtype == B200_OUT_F16 || out_dtype == B200_OUT_F32),
             B200_ERR_INVALID, "mean_proj_head: bad argument");
  DeviceGuard g(device);
  return masked_mean_proj_norm((const __nv_bfloat16*)d_x, T, w, d_len, d_projT, d_bias, D, d_feat, d_out,
                               out_dtype == B200_OUT_F16, normalize, B, (cudaStream_t)stream);
}

int b200_encoder_embed_bf16_device(const int64_t* d_ids, const void* d_word, const float* d_tt0, const float* d_pos,
                                   int position_offset, const float* d_gamma, const float* d_beta, float eps,
                                   void* d_out, int B, int T, int w, int vocab, int device, void* stream) {
  B200_CHECK(d_ids && d_word && d_pos && d_gamma && d_beta && d_out && B >= 0 && T >= 1 && eps > 0.f, B200_ERR_INVALID,
             "encoder_embed: bad argument");
  DeviceGuard g(device);
  return encoder_embed(d_ids, (const __nv_bfloat16*)d_word, d_tt0, d_pos, position_offset, d_gamma, d_beta, eps,
                       (__nv_bfloat16*)d_out, B, T, w, vocab, (cudaStream_t)stream);
}

}  // extern "C"
