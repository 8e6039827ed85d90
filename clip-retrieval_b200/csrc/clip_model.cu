// Embed path handle: the object behind model.encode_image / model.encode_text (reference
// clip_retrieval/clip_inference/mapper.py:42-43,57-59,65-67 and clip_back.py:230-232,244-246),
// fused with the L2-normalise + cast that follows each call in the reference.
//
// Data layout in HBM: weights packed once as bf16 [N, K] row-major (the layout both open_clip's
// state_dict and the wgmma B operand use), LayerNorm affine / biases / positional tables fp32;
// activations bf16 [B*T, width] row-major, one buffer per role (x residual stream, h LN output,
// qkv, a attention output, f MLP hidden), sized for max_batch at create time so every TMA
// descriptor is built once.
#include "common.cuh"
#include "embed_kernels.cuh"
#include "gemm.cuh"
#include <map>
#include <mutex>
#include <string>
#include <vector>
#include <cstring>
#include <cmath>
#include <cstdlib>

namespace b200 {

struct Linear {
  __nv_bfloat16* w = nullptr;  // [N, K]
  float* b = nullptr;          // [N] or null (folded LayerNorm: d[n] = sum_k beta[k] W[n,k] + b[n])
  float* lnc = nullptr;        // folded LayerNorm: c[n] = sum_k W'[n,k], W' = bf16(W * gamma)  (gemm.cuh)
  int N = 0, K = 0;
  CUtensorMap tm128, tm64, tm32;   // weight boxes of BN rows x 64 columns for every tile width
};

struct Layer {
  float *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
  Linear qkv, out, fc, proj;
};

struct Tower {
  int width = 0, layers = 0, heads = 0, mlp = 0, T = 0;
  std::vector<Layer> L;
  // activations
  __nv_bfloat16 *x = nullptr, *h = nullptr, *qkv = nullptr, *a = nullptr, *f = nullptr;
  CUtensorMap tm_h, tm_a, tm_f, tm_x;
  CUtensorMap tm_qkv;          // qkv in boxes of 64 rows x 64 columns: Q / K tiles of the wgmma attention
  bool wgmma_attn = false;
  float2* stats = nullptr;     // folded LayerNorm: (mean, M2) per 64-column slot of every row of x
  float *lnf_g = nullptr, *lnf_b = nullptr;  // ln_post / ln_final
  __nv_bfloat16* proj = nullptr;             // [width, D]
};

constexpr int GRAPH_MAX_B = 8;   // forwards of at most this many samples are replayed from a captured graph

enum { CLS_GEMM = 0, CLS_ATTN = 1, CLS_LN = 2, CLS_OTHER = 3,
       CLS_G_QKV = 4, CLS_G_OUT = 5, CLS_G_FC = 6, CLS_G_PROJ = 7, CLS_COUNT = 8 };  // 4..7: per-kind share of CLS_GEMM

}  // namespace b200

struct b200_clip {
  b200_clip_config cfg;
  int device = 0, sms = 132;
  bool loaded = false;
  b200::Tower vis, txt;
  // vision front end
  int grid = 0, Kp = 0;
  b200::Linear conv;          // [w, Kp]
  __nv_bfloat16* cols = nullptr;  // [max_batch*g*g, Kp]
  CUtensorMap tm_cols;
  __nv_bfloat16* vpos = nullptr;  // positional_embedding bf16 [T, w] (residual operand of the patch GEMM)
  float* cls_pos0 = nullptr;      // class_embedding + positional_embedding[0]
  float *lnpre_g = nullptr, *lnpre_b = nullptr;
  // text front end
  __nv_bfloat16* tok_emb = nullptr;  // [vocab, w]
  float* tpos = nullptr;             // [ctx, w]
  int* pool_idx = nullptr;
  float* feat = nullptr;             // raw projected features fp32 [max_batch, D] (pool/projection split over D / 64 blocks)
  // staging for the host entry points
  void* stage_in = nullptr;
  void* stage_out = nullptr;
  cudaStream_t s_copy = nullptr, s_comp = nullptr;   // host entry: H2D of sub-batch i+1 overlaps compute of i
  cudaEvent_t ev_in[4] = {}, ev_done[4] = {};
  std::vector<void*> allocs;
  std::mutex mu;                  // held by every encode entry (host and device) while it enqueues
  cudaEvent_t act_ev = nullptr;   // end of the last forward; a forward on another stream waits on it
  cudaStream_t act_stream = nullptr;
  bool act_used = false;
  // timing
  bool profiling = false;
  // Serving shapes (batch <= GRAPH_MAX_B, clip_back.py:226-246 issues batch 1): the whole tower is captured once into a
  // CUDA graph per (modality, batch, output type) and replayed — ~75-150 kernel launches become one submission.
  // The graph works on fixed device buffers (g_in / g_out); a call copies its input in and its result out.
  struct TowerGraph { cudaGraphExec_t exec = nullptr; int seen = 0; int kernels = 0; };
  std::map<int, TowerGraph> graphs;   // key: image | B << 1 | f16 << 12 | normalize << 13
  void* g_in = nullptr;
  void* g_out = nullptr;
  bool use_graphs = true;      // B200_GRAPHS=0 disables (A/B, debugging)
  cudaStream_t cap_stream = nullptr;
  bool fuse_ln = false;        // LayerNorm folded into the qkv / fc GEMMs (B200_FUSE_LN=1)
  struct Span { int cls; cudaEvent_t a, b; };
  std::vector<Span> spans;
  int span_used = 0;
  int last_launches = 0;
};

namespace b200 {

template <typename T>
static int dev_alloc(b200_clip* m, T** p, size_t count) {
  void* q = nullptr;
  B200_CUDA(cudaMalloc(&q, count * sizeof(T)));
  m->allocs.push_back(q);
  *p = (T*)q;
  return B200_OK;
}

static int make_linear(b200_clip* m, Linear* l, int N, int K, bool bias) {
  l->N = N;
  l->K = K;
  B200_TRY(dev_alloc(m, &l->w, (size_t)N * K));
  B200_CUDA(cudaMemset(l->w, 0, (size_t)N * K * 2));
  if (bias) {
    B200_TRY(dev_alloc(m, &l->b, (size_t)N));
    B200_CUDA(cudaMemset(l->b, 0, (size_t)N * 4));
  }
  B200_TRY(make_tmap_2d(&l->tm128, l->w, 1, N, K, K, 128, GEMM_BK));
  B200_TRY(make_tmap_2d(&l->tm64, l->w, 1, N, K, K, 64, GEMM_BK));
  B200_TRY(make_tmap_2d(&l->tm32, l->w, 1, N, K, K, 32, GEMM_BK));
  return B200_OK;
}

static int make_tower(b200_clip* m, Tower* t, const b200_tower_config& c, int T, int D) {
  t->width = c.width; t->layers = c.layers; t->heads = c.heads; t->mlp = c.mlp; t->T = T;
  const int w = c.width;
  const size_t rows = (size_t)m->cfg.max_batch * T;
  B200_CHECK(w % 8 == 0 && c.mlp % 8 == 0 && w % c.heads == 0, B200_ERR_INVALID, "tower: width/mlp must be multiples of 8");
  t->L.resize(c.layers);
  for (auto& L : t->L) {
    B200_TRY(dev_alloc(m, &L.ln1_g, (size_t)w)); B200_TRY(dev_alloc(m, &L.ln1_b, (size_t)w));
    B200_TRY(dev_alloc(m, &L.ln2_g, (size_t)w)); B200_TRY(dev_alloc(m, &L.ln2_b, (size_t)w));
    B200_TRY(make_linear(m, &L.qkv, 3 * w, w, true));
    B200_TRY(make_linear(m, &L.out, w, w, true));
    B200_TRY(make_linear(m, &L.fc, c.mlp, w, true));
    B200_TRY(make_linear(m, &L.proj, w, c.mlp, true));
  }
  B200_TRY(dev_alloc(m, &t->lnf_g, (size_t)w)); B200_TRY(dev_alloc(m, &t->lnf_b, (size_t)w));
  B200_TRY(dev_alloc(m, &t->proj, (size_t)w * D));
  B200_TRY(dev_alloc(m, &t->x, rows * w));
  B200_TRY(dev_alloc(m, &t->h, rows * w));
  B200_TRY(dev_alloc(m, &t->qkv, rows * 3 * w));
  B200_TRY(dev_alloc(m, &t->a, rows * w));
  B200_TRY(dev_alloc(m, &t->f, rows * c.mlp));
  B200_TRY(make_tmap_2d(&t->tm_h, t->h, 1, rows, w, w, GEMM_BM, GEMM_BK));
  B200_TRY(make_tmap_2d(&t->tm_a, t->a, 1, rows, w, w, GEMM_BM, GEMM_BK));
  B200_TRY(make_tmap_2d(&t->tm_f, t->f, 1, rows, c.mlp, c.mlp, GEMM_BM, GEMM_BK));
  B200_TRY(make_tmap_2d(&t->tm_x, t->x, 1, rows, w, w, GEMM_BM, GEMM_BK));
  t->wgmma_attn = attention_wgmma_supported(T, c.heads, w);
  if (t->wgmma_attn) B200_TRY(make_tmap_2d(&t->tm_qkv, t->qkv, 1, rows, 3 * (size_t)w, 3 * (size_t)w, 64, 64));
  if (m->fuse_ln && w % 64 == 0 && w <= 64 * LN_MAX_SLOTS) {
    B200_TRY(dev_alloc(m, &t->stats, rows * (size_t)(w / 64)));
    for (auto& L : t->L) {
      B200_TRY(dev_alloc(m, &L.qkv.lnc, (size_t)3 * w));
      B200_TRY(dev_alloc(m, &L.fc.lnc, (size_t)c.mlp));
    }
  }
  return B200_OK;
}

// ---- timing spans ------------------------------------------------------------------------------
struct SpanGuard {
  b200_clip* m; cudaStream_t st; int idx = -1;
  SpanGuard(b200_clip* m_, int cls, cudaStream_t s) : m(m_), st(s) {
    if (!m->profiling) return;
    if (m->span_used == (int)m->spans.size()) {
      b200_clip::Span sp;
      sp.cls = cls;
      if (cudaEventCreate(&sp.a) != cudaSuccess || cudaEventCreate(&sp.b) != cudaSuccess) return;
      m->spans.push_back(sp);
    }
    idx = m->span_used++;
    m->spans[idx].cls = cls;
    cudaEventRecord(m->spans[idx].a, st);
  }
  ~SpanGuard() {
    if (idx >= 0) cudaEventRecord(m->spans[idx].b, st);
  }
};

static int run_linear(b200_clip* m, const CUtensorMap& tmA, const Linear& l, int M, GemmEpilogue ep, cudaStream_t st,
                      int kind = CLS_GEMM) {
  SpanGuard sg(m, kind, st);
  int bn = gemm_pick_bn(M, l.N, m->sms);
  // row statistics are written per 64-column slot by ONE thread: the narrow tiles split a slot over two warps
  if (ep.stats_out != nullptr && bn < 128) bn = 128;
  ep.bias = l.b;
  m->last_launches++;
  const CUtensorMap& tmB = bn == 64 ? l.tm64 : (bn == 32 ? l.tm32 : l.tm128);
  return gemm_bf16_launch(tmA, tmB, bn, M, l.N, l.K, ep, st);
}

static int run_blocks(b200_clip* m, Tower& t, int B, int causal, cudaStream_t st) {
  const int w = t.width;
  const int M = B * t.T;
  const int act = m->cfg.quick_gelu ? ACT_QUICK_GELU : ACT_GELU;
  const bool fused = t.stats != nullptr;   // LayerNorm folded into the qkv / fc GEMMs (weights carry gamma)
  if (fused) {
    // records of the stream as it enters the first block (after ln_pre / the embedding lookup); every later
    // version of x comes out of a residual GEMM whose epilogue writes them
    SpanGuard sg(m, CLS_LN, st); m->last_launches++;
    B200_TRY(row_stats(t.x, M, w, t.stats, st));
  }
  for (auto& L : t.L) {
    if (!fused) { SpanGuard sg(m, CLS_LN, st); m->last_launches++;
      B200_TRY(layernorm_rows(t.x, w, t.h, w, L.ln1_g, L.ln1_b, M, w, st)); }
    GemmEpilogue e1; e1.out = t.qkv; e1.out_ld = 3 * w;
    if (fused) { e1.ln_stats = t.stats; e1.ln_c = L.qkv.lnc; e1.ln_w = w; }
    B200_TRY(run_linear(m, fused ? t.tm_x : t.tm_h, L.qkv, M, e1, st, CLS_G_QKV));
    { SpanGuard sg(m, CLS_ATTN, st); m->last_launches++;
      if (t.wgmma_attn) B200_TRY(attention_wgmma(t.tm_qkv, t.qkv, t.a, B, t.T, t.heads, w, causal, st));
      else B200_TRY(attention(t.qkv, t.a, B, t.T, t.heads, w, causal, st)); }
    GemmEpilogue e2; e2.out = t.x; e2.out_ld = w; e2.residual = t.x; e2.res_ld = w;
    if (fused) e2.stats_out = t.stats;
    B200_TRY(run_linear(m, t.tm_a, L.out, M, e2, st, CLS_G_OUT));
    if (!fused) { SpanGuard sg(m, CLS_LN, st); m->last_launches++;
      B200_TRY(layernorm_rows(t.x, w, t.h, w, L.ln2_g, L.ln2_b, M, w, st)); }
    GemmEpilogue e3; e3.out = t.f; e3.out_ld = t.mlp; e3.act = act;
    if (fused) { e3.ln_stats = t.stats; e3.ln_c = L.fc.lnc; e3.ln_w = w; }
    B200_TRY(run_linear(m, fused ? t.tm_x : t.tm_h, L.fc, M, e3, st, CLS_G_FC));
    GemmEpilogue e4; e4.out = t.x; e4.out_ld = w; e4.residual = t.x; e4.res_ld = w;
    if (fused) e4.stats_out = t.stats;
    B200_TRY(run_linear(m, t.tm_f, L.proj, M, e4, st, CLS_G_PROJ));
  }
  return B200_OK;
}

static int encode_image_chunk(b200_clip* m, const float* d_px, int B, void* d_out, int out_f16, int normalize,
                              cudaStream_t st) {
  Tower& t = m->vis;
  const int g = m->grid, w = t.width, T = t.T;
  { SpanGuard sg(m, CLS_OTHER, st); m->last_launches += 2;
    B200_TRY(im2col_patches(d_px, m->cols, B, m->cfg.image_size, m->cfg.patch, m->Kp, st));
    B200_TRY(write_cls_rows(t.x, m->cls_pos0, B, T, w, st)); }
  // patch embedding: x[b*T + 1 + p, :] = cols[b*g*g + p, :] · conv^T + positional_embedding[1 + p]
  GemmEpilogue ep; ep.out = t.x; ep.out_ld = w; ep.out_group = g * g;
  ep.residual = m->vpos; ep.res_ld = w; ep.res_row_mod = g * g; ep.res_row_off = 1;
  B200_TRY(run_linear(m, m->tm_cols, m->conv, B * g * g, ep, st, CLS_GEMM));
  { SpanGuard sg(m, CLS_LN, st); m->last_launches++;
    B200_TRY(layernorm_rows(t.x, w, t.x, w, m->lnpre_g, m->lnpre_b, (int64_t)B * T, w, st)); }
  B200_TRY(run_blocks(m, t, B, 0, st));
  { SpanGuard sg(m, CLS_OTHER, st); m->last_launches++;
    B200_TRY(pool_ln_proj_norm(t.x, T, w, nullptr, t.lnf_g, t.lnf_b, t.proj, m->cfg.embed_dim, d_out, out_f16, normalize, B, st, m->feat)); }
  return B200_OK;
}

static int encode_text_chunk(b200_clip* m, const int64_t* d_tok, int B, void* d_out, int out_f16, int normalize,
                             cudaStream_t st) {
  Tower& t = m->txt;
  const int w = t.width, T = t.T;
  { SpanGuard sg(m, CLS_OTHER, st); m->last_launches += 2;
    B200_TRY(text_embed(d_tok, m->tok_emb, m->tpos, t.x, B, T, w, m->cfg.vocab_size, st));
    B200_TRY(token_argmax(d_tok, m->pool_idx, B, T, st)); }
  B200_TRY(run_blocks(m, t, B, 1, st));
  { SpanGuard sg(m, CLS_OTHER, st); m->last_launches++;
    B200_TRY(pool_ln_proj_norm(t.x, T, w, m->pool_idx, t.lnf_g, t.lnf_b, t.proj, m->cfg.embed_dim, d_out, out_f16, normalize, B, st, m->feat)); }
  return B200_OK;
}

// ---- weight upload -------------------------------------------------------------------------------
static inline float view_get(const b200_tensor_view& v, size_t i) {
  if (v.dtype == 0) return ((const float*)v.data)[i];
  return __half2float(((const __half*)v.data)[i]);
}
static inline uint16_t f32_to_bf16_rn(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);  // NaN
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
static size_t view_count(const b200_tensor_view& v) {
  size_t n = 1;
  for (int i = 0; i < v.ndim; i++) n *= (size_t)v.shape[i];
  return n;
}

struct Loader {
  std::map<std::string, const b200_tensor_view*> by_name;
  std::vector<uint16_t> tmp16;
  std::vector<float> tmp32;
  const b200_tensor_view* find(const std::string& name, size_t count) {
    auto it = by_name.find(name);
    if (it == by_name.end()) { set_error("load_weights: tensor '%s' is missing", name.c_str()); return nullptr; }
    if (view_count(*it->second) != count) {
      set_error("load_weights: tensor '%s' has %zu elements, expected %zu", name.c_str(), view_count(*it->second), count);
      return nullptr;
    }
    return it->second;
  }
  // dst bf16 [rows, dst_ld] <- src [rows, cols] (zero padded columns keep their zeros)
  int put_bf16(const std::string& name, __nv_bfloat16* dst, size_t rows, size_t cols, size_t dst_ld) {
    const b200_tensor_view* v = find(name, rows * cols);
    if (!v) return B200_ERR_INVALID;
    tmp16.assign(rows * dst_ld, 0);
    for (size_t r = 0; r < rows; r++)
      for (size_t c = 0; c < cols; c++) tmp16[r * dst_ld + c] = f32_to_bf16_rn(view_get(*v, r * cols + c));
    B200_CUDA(cudaMemcpy(dst, tmp16.data(), tmp16.size() * 2, cudaMemcpyHostToDevice));
    return B200_OK;
  }
  int put_f32(const std::string& name, float* dst, size_t count) {
    const b200_tensor_view* v = find(name, count);
    if (!v) return B200_ERR_INVALID;
    tmp32.resize(count);
    for (size_t i = 0; i < count; i++) tmp32[i] = view_get(*v, i);
    B200_CUDA(cudaMemcpy(dst, tmp32.data(), count * 4, cudaMemcpyHostToDevice));
    return B200_OK;
  }
};

// Folded LayerNorm (gemm.cuh): W' = bf16(W * gamma) replaces W; c[n] = sum_k W'[n,k] (of the ROUNDED weights — what
// the tensor core multiplies); d[n] = sum_k beta[k] W[n,k] + b[n] replaces the bias.
static int put_folded(Loader& ld, const std::string& wname, const std::string& bname, const std::string& gname,
                      const std::string& betaname, Linear& l) {
  const size_t N = l.N, K = l.K;
  const b200_tensor_view* W = ld.find(wname, N * K);
  const b200_tensor_view* bv = ld.find(bname, N);
  const b200_tensor_view* g = ld.find(gname, K);
  const b200_tensor_view* be = ld.find(betaname, K);
  if (!W || !bv || !g || !be) return B200_ERR_INVALID;
  std::vector<uint16_t> w16(N * K);
  std::vector<float> c(N), d(N);
  for (size_t n = 0; n < N; n++) {
    double cs = 0.0, ds = 0.0;
    for (size_t k = 0; k < K; k++) {
      const float wv = view_get(*W, n * K + k);
      const uint16_t h = f32_to_bf16_rn(wv * view_get(*g, k));
      w16[n * K + k] = h;
      uint32_t u = (uint32_t)h << 16;
      float hf;
      memcpy(&hf, &u, 4);
      cs += (double)hf;
      ds += (double)view_get(*be, k) * (double)wv;
    }
    c[n] = (float)cs;
    d[n] = (float)(ds + (double)view_get(*bv, n));
  }
  B200_CUDA(cudaMemcpy(l.w, w16.data(), w16.size() * 2, cudaMemcpyHostToDevice));
  B200_CUDA(cudaMemcpy(l.lnc, c.data(), N * 4, cudaMemcpyHostToDevice));
  B200_CUDA(cudaMemcpy(l.b, d.data(), N * 4, cudaMemcpyHostToDevice));
  return B200_OK;
}

static int load_tower(Loader& ld, Tower& t, const std::string& prefix) {
  const size_t w = t.width, mlp = t.mlp;
  const bool fused = t.stats != nullptr;
  for (int i = 0; i < t.layers; i++) {
    Layer& L = t.L[i];
    const std::string p = prefix + "transformer.resblocks." + std::to_string(i) + ".";
    B200_TRY(ld.put_f32(p + "ln_1.weight", L.ln1_g, w));
    B200_TRY(ld.put_f32(p + "ln_1.bias", L.ln1_b, w));
    if (fused) {
      B200_TRY(put_folded(ld, p + "attn.in_proj_weight", p + "attn.in_proj_bias", p + "ln_1.weight", p + "ln_1.bias", L.qkv));
      B200_TRY(put_folded(ld, p + "mlp.c_fc.weight", p + "mlp.c_fc.bias", p + "ln_2.weight", p + "ln_2.bias", L.fc));
      B200_TRY(ld.put_bf16(p + "attn.out_proj.weight", L.out.w, w, w, w));
      B200_TRY(ld.put_f32(p + "attn.out_proj.bias", L.out.b, w));
      B200_TRY(ld.put_f32(p + "ln_2.weight", L.ln2_g, w));
      B200_TRY(ld.put_f32(p + "ln_2.bias", L.ln2_b, w));
      B200_TRY(ld.put_bf16(p + "mlp.c_proj.weight", L.proj.w, w, mlp, mlp));
      B200_TRY(ld.put_f32(p + "mlp.c_proj.bias", L.proj.b, w));
      continue;
    }
    B200_TRY(ld.put_bf16(p + "attn.in_proj_weight", L.qkv.w, 3 * w, w, w));
    B200_TRY(ld.put_f32(p + "attn.in_proj_bias", L.qkv.b, 3 * w));
    B200_TRY(ld.put_bf16(p + "attn.out_proj.weight", L.out.w, w, w, w));
    B200_TRY(ld.put_f32(p + "attn.out_proj.bias", L.out.b, w));
    B200_TRY(ld.put_f32(p + "ln_2.weight", L.ln2_g, w));
    B200_TRY(ld.put_f32(p + "ln_2.bias", L.ln2_b, w));
    B200_TRY(ld.put_bf16(p + "mlp.c_fc.weight", L.fc.w, mlp, w, w));
    B200_TRY(ld.put_f32(p + "mlp.c_fc.bias", L.fc.b, mlp));
    B200_TRY(ld.put_bf16(p + "mlp.c_proj.weight", L.proj.w, w, mlp, mlp));
    B200_TRY(ld.put_f32(p + "mlp.c_proj.bias", L.proj.b, w));
  }
  return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_clip_create(const b200_clip_config* cfg, int device, b200_clip** out) {
  B200_CHECK(cfg && out, B200_ERR_INVALID, "clip_create: null argument");
  B200_CHECK(cfg->max_batch >= 1 && cfg->embed_dim >= 8 && cfg->patch >= 1 && cfg->image_size >= cfg->patch &&
                 cfg->context_length >= 1 && cfg->vocab_size >= 2,
             B200_ERR_INVALID, "clip_create: bad config");
  int ndev = 0;
  B200_CUDA(cudaGetDeviceCount(&ndev));
  B200_CHECK(device >= 0 && device < ndev, B200_ERR_INVALID, "clip_create: device %d of %d", device, ndev);
  DeviceGuard g(device);
  b200_clip* m = new (std::nothrow) b200_clip();
  B200_CHECK(m != nullptr, B200_ERR_OOM, "clip_create: host allocation failed");
  m->cfg = *cfg;
  m->device = device;
  m->sms = sm_count(device);
  // LayerNorm folded into the qkv / fc GEMMs stays opt-in: it adds per-row statistics work to the GEMM epilogue, and at
  // serving batch sizes the row statistics need >= 128-column tiles, which undoes the narrow-tile weight streaming.
  if (const char* g = getenv("B200_FUSE_LN")) m->fuse_ln = atoi(g) != 0;
  if (const char* g = getenv("B200_GRAPHS")) m->use_graphs = atoi(g) != 0;
  m->grid = cfg->image_size / cfg->patch;
  const int k_raw = 3 * cfg->patch * cfg->patch;
  m->Kp = (k_raw + 63) / 64 * 64;
  const int T = m->grid * m->grid + 1;
  int rc = B200_OK;
  auto build = [&]() -> int {
    B200_TRY(make_tower(m, &m->vis, cfg->vision, T, cfg->embed_dim));
    B200_TRY(make_tower(m, &m->txt, cfg->text, cfg->context_length, cfg->embed_dim));
    B200_TRY(make_linear(m, &m->conv, cfg->vision.width, m->Kp, false));
    const size_t prow = (size_t)cfg->max_batch * m->grid * m->grid;
    B200_TRY(dev_alloc(m, &m->cols, prow * m->Kp));
    B200_CUDA(cudaMemset(m->cols, 0, prow * m->Kp * 2));
    B200_TRY(make_tmap_2d(&m->tm_cols, m->cols, 1, prow, m->Kp, m->Kp, GEMM_BM, GEMM_BK));
    B200_TRY(dev_alloc(m, &m->vpos, (size_t)T * cfg->vision.width));
    B200_TRY(dev_alloc(m, &m->cls_pos0, (size_t)cfg->vision.width));
    B200_TRY(dev_alloc(m, &m->lnpre_g, (size_t)cfg->vision.width));
    B200_TRY(dev_alloc(m, &m->lnpre_b, (size_t)cfg->vision.width));
    B200_TRY(dev_alloc(m, &m->tok_emb, (size_t)cfg->vocab_size * cfg->text.width));
    B200_TRY(dev_alloc(m, &m->tpos, (size_t)cfg->context_length * cfg->text.width));
    B200_TRY(dev_alloc(m, &m->pool_idx, (size_t)cfg->max_batch));
    B200_TRY(dev_alloc(m, &m->feat, (size_t)cfg->max_batch * cfg->embed_dim));
    const size_t in_bytes = std::max((size_t)cfg->max_batch * 3 * cfg->image_size * cfg->image_size * 4,
                                     (size_t)cfg->max_batch * cfg->context_length * 8);
    B200_CUDA(cudaMalloc(&m->stage_in, in_bytes));
    m->allocs.push_back(m->stage_in);
    B200_CUDA(cudaMalloc(&m->stage_out, (size_t)cfg->max_batch * cfg->embed_dim * 4));
    m->allocs.push_back(m->stage_out);
    const int gb = std::min(GRAPH_MAX_B, cfg->max_batch);
    B200_CUDA(cudaMalloc(&m->g_in, std::max((size_t)gb * 3 * cfg->image_size * cfg->image_size * 4, (size_t)gb * cfg->context_length * 8)));
    m->allocs.push_back(m->g_in);
    B200_CUDA(cudaMalloc(&m->g_out, (size_t)gb * cfg->embed_dim * 4));
    m->allocs.push_back(m->g_out);
    return B200_OK;
  };
  rc = build();
  if (rc != B200_OK) {
    b200_clip_destroy(m);
    return rc;
  }
  *out = m;
  return B200_OK;
}

int b200_clip_destroy(b200_clip* m) {
  if (!m) return B200_OK;
  DeviceGuard g(m->device);
  cudaDeviceSynchronize();
  for (void* p : m->allocs) cudaFree(p);
  for (auto& s : m->spans) { cudaEventDestroy(s.a); cudaEventDestroy(s.b); }
  if (m->act_ev) cudaEventDestroy(m->act_ev);
  for (auto& kv : m->graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
  if (m->cap_stream) cudaStreamDestroy(m->cap_stream);
  if (m->s_copy) {
    cudaStreamDestroy(m->s_copy); cudaStreamDestroy(m->s_comp);
    for (int i = 0; i < 4; i++) { cudaEventDestroy(m->ev_in[i]); cudaEventDestroy(m->ev_done[i]); }
  }
  delete m;
  return B200_OK;
}

int b200_clip_load_weights(b200_clip* m, const b200_tensor_view* tensors, int n) {
  B200_CHECK(m && tensors && n > 0, B200_ERR_INVALID, "load_weights: bad argument");
  DeviceGuard g(m->device);
  Loader ld;
  for (int i = 0; i < n; i++) {
    B200_CHECK(tensors[i].name && tensors[i].data && (tensors[i].dtype == 0 || tensors[i].dtype == 1) &&
                   tensors[i].ndim >= 0 && tensors[i].ndim <= 4,
               B200_ERR_INVALID, "load_weights: malformed tensor view %d", i);
    ld.by_name[tensors[i].name] = &tensors[i];
  }
  const b200_clip_config& c = m->cfg;
  const size_t vw = c.vision.width, tw = c.text.width, D = c.embed_dim;
  const size_t T = (size_t)m->grid * m->grid + 1, kraw = (size_t)3 * c.patch * c.patch;
  B200_TRY(ld.put_bf16("visual.conv1.weight", m->conv.w, vw, kraw, m->Kp));
  B200_TRY(ld.put_bf16("visual.positional_embedding", m->vpos, T, vw, vw));
  {
    const b200_tensor_view* cls = ld.find("visual.class_embedding", vw);
    const b200_tensor_view* pos = ld.find("visual.positional_embedding", T * vw);
    if (!cls || !pos) return B200_ERR_INVALID;
    std::vector<float> v(vw);
    for (size_t j = 0; j < vw; j++) v[j] = view_get(*cls, j) + view_get(*pos, j);
    B200_CUDA(cudaMemcpy(m->cls_pos0, v.data(), vw * 4, cudaMemcpyHostToDevice));
  }
  B200_TRY(ld.put_f32("visual.ln_pre.weight", m->lnpre_g, vw));
  B200_TRY(ld.put_f32("visual.ln_pre.bias", m->lnpre_b, vw));
  B200_TRY(load_tower(ld, m->vis, "visual."));
  B200_TRY(ld.put_f32("visual.ln_post.weight", m->vis.lnf_g, vw));
  B200_TRY(ld.put_f32("visual.ln_post.bias", m->vis.lnf_b, vw));
  B200_TRY(ld.put_bf16("visual.proj", m->vis.proj, vw, D, D));
  B200_TRY(ld.put_bf16("token_embedding.weight", m->tok_emb, (size_t)c.vocab_size, tw, tw));
  B200_TRY(ld.put_f32("positional_embedding", m->tpos, (size_t)c.context_length * tw));
  B200_TRY(load_tower(ld, m->txt, ""));
  B200_TRY(ld.put_f32("ln_final.weight", m->txt.lnf_g, tw));
  B200_TRY(ld.put_f32("ln_final.bias", m->txt.lnf_b, tw));
  B200_TRY(ld.put_bf16("text_projection", m->txt.proj, tw, D, D));
  B200_CUDA(cudaDeviceSynchronize());
  m->loaded = true;
  return B200_OK;
}

static int encode_device(b200_clip* m, const void* d_in, int B, void* d_out, int out_dtype, int normalize, bool image,
                         cudaStream_t st) {
  B200_CHECK(m && (B == 0 || (d_in && d_out)) && B >= 0, B200_ERR_INVALID, "encode: bad argument");
  B200_CHECK(m->loaded, B200_ERR_STATE, "encode: weights not loaded");
  B200_CHECK(out_dtype == B200_OUT_F16 || out_dtype == B200_OUT_F32, B200_ERR_INVALID, "encode: out_dtype %d", out_dtype);
  DeviceGuard g(m->device);
  m->last_launches = 0;
  const int mb = m->cfg.max_batch;
  const size_t in_stride = image ? (size_t)3 * m->cfg.image_size * m->cfg.image_size * 4 : (size_t)m->cfg.context_length * 8;
  const size_t out_stride = (size_t)m->cfg.embed_dim * (out_dtype == B200_OUT_F16 ? 2 : 4);
  if (B >= 1 && B <= GRAPH_MAX_B && B <= mb && m->use_graphs && !m->profiling) {
    // serving shape: replay the captured tower.  First call of a shape runs eagerly (sets kernel attributes,
    // touches every buffer), the second captures, later ones replay.
    const int key = (image ? 1 : 0) | (B << 1) | ((out_dtype == B200_OUT_F16 ? 1 : 0) << 12) | ((normalize ? 1 : 0) << 13);
    b200_clip::TowerGraph& tg = m->graphs[key];
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    B200_CUDA(cudaStreamIsCapturing(st, &cs));
    if (cs == cudaStreamCaptureStatusNone && tg.seen >= 1) {
      if (tg.exec == nullptr) {
        cudaGraph_t graph = nullptr;
        // captured on a private stream (the caller's may be the legacy default stream, which cannot capture)
        if (!m->cap_stream) B200_CUDA(cudaStreamCreateWithFlags(&m->cap_stream, cudaStreamNonBlocking));
        cudaStream_t cst = m->cap_stream;
        B200_CUDA(cudaStreamBeginCapture(cst, cudaStreamCaptureModeThreadLocal));
        int rc = image ? encode_image_chunk(m, (const float*)m->g_in, B, m->g_out, out_dtype == B200_OUT_F16, normalize, cst)
                       : encode_text_chunk(m, (const int64_t*)m->g_in, B, m->g_out, out_dtype == B200_OUT_F16, normalize, cst);
        const cudaError_t ce = cudaStreamEndCapture(cst, &graph);
        if (rc != B200_OK || ce != cudaSuccess || graph == nullptr) {
          if (graph) cudaGraphDestroy(graph);
          cudaGetLastError();
          m->use_graphs = false;   // fall back to eager launches for the life of the handle
          B200_CHECK(rc == B200_OK, rc, "encode: kernel launch failed during graph capture");
        } else {
          const cudaError_t ie = cudaGraphInstantiate(&tg.exec, graph, 0);
          cudaGraphDestroy(graph);
          tg.kernels = m->last_launches;   // kernels inside the graph (they were counted once, at capture)
          if (ie != cudaSuccess) { cudaGetLastError(); tg.exec = nullptr; m->use_graphs = false; }
        }
      }
      if (tg.exec != nullptr) {
        B200_CUDA(cudaMemcpyAsync(m->g_in, d_in, (size_t)B * in_stride, cudaMemcpyDeviceToDevice, st));
        B200_CUDA(cudaGraphLaunch(tg.exec, st));
        B200_CUDA(cudaMemcpyAsync(d_out, m->g_out, (size_t)B * out_stride, cudaMemcpyDeviceToDevice, st));
        count_launch(tg.kernels);
        m->last_launches = tg.kernels;
        return B200_OK;
      }
    }
    tg.seen++;
  }
  for (int b0 = 0; b0 < B; b0 += mb) {
    const int nb = std::min(mb, B - b0);
    const char* in = (const char*)d_in + (size_t)b0 * in_stride;
    char* o = (char*)d_out + (size_t)b0 * out_stride;
    if (image) B200_TRY(encode_image_chunk(m, (const float*)in, nb, o, out_dtype == B200_OUT_F16, normalize, st));
    else B200_TRY(encode_text_chunk(m, (const int64_t*)in, nb, o, out_dtype == B200_OUT_F16, normalize, st));
  }
  return B200_OK;
}

// The activation buffers of a handle are shared by every forward on it: calls hold m->mu while they enqueue,
// and a call on a different stream than the previous one first waits (event) for the previous forward's kernels.
static int act_acquire(b200_clip* m, cudaStream_t st) {
  if (!m->act_ev) B200_CUDA(cudaEventCreateWithFlags(&m->act_ev, cudaEventDisableTiming));
  if (m->act_used && m->act_stream != st) B200_CUDA(cudaStreamWaitEvent(st, m->act_ev, 0));
  return B200_OK;
}
static int act_release(b200_clip* m, cudaStream_t st) {
  B200_CUDA(cudaEventRecord(m->act_ev, st));
  m->act_stream = st;
  m->act_used = true;
  return B200_OK;
}
static int encode_device_locked(b200_clip* m, const void* d_in, int B, void* d_out, int out_dtype, int normalize,
                                bool image, cudaStream_t st) {
  B200_CHECK(m, B200_ERR_INVALID, "encode: null handle");
  std::lock_guard<std::mutex> lock(m->mu);
  DeviceGuard g(m->device);
  B200_TRY(act_acquire(m, st));
  const int rc = encode_device(m, d_in, B, d_out, out_dtype, normalize, image, st);
  B200_TRY(act_release(m, st));
  return rc;
}

int b200_clip_encode_image_device(b200_clip* m, const float* d_pixels, int B, void* d_out, int out_dtype, int normalize,
                                  void* stream) {
  return encode_device_locked(m, d_pixels, B, d_out, out_dtype, normalize, true, (cudaStream_t)stream);
}
int b200_clip_encode_text_device(b200_clip* m, const int64_t* d_tokens, int B, void* d_out, int out_dtype, int normalize,
                                 void* stream) {
  return encode_device_locked(m, d_tokens, B, d_out, out_dtype, normalize, false, (cudaStream_t)stream);
}

// Host-buffer entry (the mapper call).  Images are pipelined in sub-batches: the H2D copy of
// sub-batch i+1 (copy stream) overlaps the forward of sub-batch i (compute stream); the staging
// buffer is a ring of max_batch / sub-batch slots guarded by events.
static int encode_host(b200_clip* m, const void* h_in, int B, void* h_out, int out_dtype, int normalize, bool image) {
  B200_CHECK(m && (B == 0 || (h_in && h_out)) && B >= 0, B200_ERR_INVALID, "encode: bad argument");
  B200_CHECK(m->loaded, B200_ERR_STATE, "encode: weights not loaded");
  std::lock_guard<std::mutex> lock(m->mu);
  DeviceGuard g(m->device);
  if (!m->s_copy) {
    B200_CUDA(cudaStreamCreateWithFlags(&m->s_copy, cudaStreamNonBlocking));
    B200_CUDA(cudaStreamCreateWithFlags(&m->s_comp, cudaStreamNonBlocking));
    for (int i = 0; i < 4; i++) {
      B200_CUDA(cudaEventCreateWithFlags(&m->ev_in[i], cudaEventDisableTiming));
      B200_CUDA(cudaEventCreateWithFlags(&m->ev_done[i], cudaEventDisableTiming));
    }
  }
  B200_TRY(act_acquire(m, m->s_comp));
  const int mb = m->cfg.max_batch;
  const size_t in_stride = image ? (size_t)3 * m->cfg.image_size * m->cfg.image_size * 4 : (size_t)m->cfg.context_length * 8;
  const size_t out_stride = (size_t)m->cfg.embed_dim * (out_dtype == B200_OUT_F16 ? 2 : 4);
  const int slots = (image && mb >= 256) ? 4 : 1;
  const int SB = mb / slots;
  int launches = 0;
  long gi = 0;  // sub-batches issued so far (slot = gi % slots)
  for (int b0 = 0; b0 < B; b0 += mb) {
    const int nb = std::min(mb, B - b0);
    if (b0 > 0) B200_CUDA(cudaStreamSynchronize(m->s_comp));  // stage_out is reused per chunk
    for (int s0 = 0; s0 < nb; s0 += SB, gi++) {
      const int ns = std::min(SB, nb - s0);
      const int slot = (int)(gi % slots);
      char* stage = (char*)m->stage_in + (size_t)slot * SB * in_stride;
      if (gi >= slots) B200_CUDA(cudaStreamWaitEvent(m->s_copy, m->ev_done[slot], 0));
      B200_CUDA(cudaMemcpyAsync(stage, (const char*)h_in + (size_t)(b0 + s0) * in_stride, ns * in_stride,
                                cudaMemcpyHostToDevice, m->s_copy));
      B200_CUDA(cudaEventRecord(m->ev_in[slot], m->s_copy));
      B200_CUDA(cudaStreamWaitEvent(m->s_comp, m->ev_in[slot], 0));
      B200_TRY(encode_device(m, stage, ns, (char*)m->stage_out + (size_t)s0 * out_stride, out_dtype, normalize, image,
                             m->s_comp));
      B200_CUDA(cudaEventRecord(m->ev_done[slot], m->s_comp));
      launches += m->last_launches;
    }
    B200_CUDA(cudaMemcpyAsync((char*)h_out + (size_t)b0 * out_stride, m->stage_out, nb * out_stride, cudaMemcpyDeviceToHost,
                              m->s_comp));
  }
  B200_CUDA(cudaStreamSynchronize(m->s_comp));
  B200_TRY(act_release(m, m->s_comp));
  m->last_launches = launches;
  return B200_OK;
}

int b200_clip_encode_image(b200_clip* m, const float* h_pixels, int B, void* h_out, int out_dtype, int normalize) {
  return encode_host(m, h_pixels, B, h_out, out_dtype, normalize, true);
}
int b200_clip_encode_text(b200_clip* m, const int64_t* h_tokens, int B, void* h_out, int out_dtype, int normalize) {
  return encode_host(m, h_tokens, B, h_out, out_dtype, normalize, false);
}

int b200_layernorm_bf16_device(const void* d_in, void* d_out, const float* d_gamma, const float* d_beta, int64_t rows,
                               int w, int device, void* stream) {
  B200_CHECK(d_in && d_out && d_gamma && d_beta && rows >= 0, B200_ERR_INVALID, "layernorm: bad argument");
  DeviceGuard g(device);
  return layernorm_rows((const __nv_bfloat16*)d_in, w, (__nv_bfloat16*)d_out, w, d_gamma, d_beta, rows, w,
                        (cudaStream_t)stream);
}
int b200_attention_bf16_device(const void* d_qkv, void* d_out, int B, int T, int heads, int w, int causal, int device,
                               void* stream) {
  B200_CHECK(d_qkv && d_out && B >= 0 && T >= 1, B200_ERR_INVALID, "attention: bad argument");
  DeviceGuard g(device);
  if (B > 0 && attention_wgmma_supported(T, heads, w)) {
    CUtensorMap tm;
    B200_TRY(make_tmap_2d(&tm, d_qkv, 1, (uint64_t)B * T, 3 * (uint64_t)w, 3 * (uint64_t)w, 64, 64));
    return attention_wgmma(tm, (const __nv_bfloat16*)d_qkv, (__nv_bfloat16*)d_out, B, T, heads, w, causal, (cudaStream_t)stream);
  }
  return attention((const __nv_bfloat16*)d_qkv, (__nv_bfloat16*)d_out, B, T, heads, w, causal, (cudaStream_t)stream);
}

int b200_clip_set_profiling(b200_clip* m, int on) {
  B200_CHECK(m, B200_ERR_INVALID, "set_profiling: null handle");
  m->profiling = on != 0;
  m->span_used = 0;
  return B200_OK;
}

int b200_clip_last_timing(b200_clip* m, float* ms_by_class, int* launches) {
  B200_CHECK(m && ms_by_class, B200_ERR_INVALID, "last_timing: null argument");
  DeviceGuard g(m->device);
  for (int i = 0; i < CLS_COUNT; i++) ms_by_class[i] = 0.f;
  for (int i = 0; i < m->span_used; i++) {
    const auto& s = m->spans[i];
    B200_CUDA(cudaEventSynchronize(s.b));
    float t = 0.f;
    B200_CUDA(cudaEventElapsedTime(&t, s.a, s.b));
    if (s.cls >= 0 && s.cls < CLS_COUNT) ms_by_class[s.cls] += t;
    if (s.cls >= CLS_G_QKV && s.cls <= CLS_G_PROJ) ms_by_class[CLS_GEMM] += t;
  }
  if (launches) *launches = m->span_used;
  m->span_used = 0;
  return B200_OK;
}

}  // extern "C"
