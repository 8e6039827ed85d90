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
#include "convnext.cuh"
#include "embed_kernels.cuh"
#include "gemm.cuh"
#include "layers.cuh"
#include "resnet.cuh"
#include "weights.cuh"
#include <map>
#include <mutex>
#include <string>
#include <vector>
#include <cstring>
#include <cmath>
#include <cstdlib>

namespace b200 {

struct Layer {
  float *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
  Linear qkv, out, fc, proj;
};

// How a tower turns its last residual stream into features.
enum Pool {
  POOL_FIRST = 0,    // LN(row 0) @ proj (CLIP image tower: the class token)
  POOL_EOT = 1,      // LN(row argmax(tokens)) @ proj (CLIP text tower)
  POOL_LAST = 2,     // LN(row T - 1) @ proj + proj_b (SigLIP text tower)
  POOL_LATENT = 3,   // LN over every row, then the latent-query attention-pool head (SigLIP image tower)
};

struct Tower {
  int width = 0, layers = 0, heads = 0, mlp = 0, T = 0;
  float ln_eps = 1e-5f;        // every LayerNorm of the tower, its final one included
  int causal = 0;
  int pool = POOL_FIRST;
  std::vector<Layer> L;
  // activations
  __nv_bfloat16 *x = nullptr, *h = nullptr, *qkv = nullptr, *a = nullptr, *f = nullptr;
  CUtensorMap tm_h, tm_a, tm_f;
  CUtensorMap tm_qkv;          // make_qkv_map over max_batch samples, built when the wgmma attention takes the tower
  float *lnf_g = nullptr, *lnf_b = nullptr;  // ln_post / ln_final
  __nv_bfloat16* proj = nullptr;             // [width, D]
  float* proj_b = nullptr;                   // [D] (POOL_LAST) or null
};

// SigLIP's image head (timm AttentionPoolLatent): out = y + fc2(gelu(fc1(LN(y)))) with y = proj(attn(q, kv(LN(x)))),
// where q = q_proj(latent) is input-independent and computed once at load time.
struct LatentHead {
  Linear kv, proj, fc1, fc2;   // [2w, w], [w, w], [mlp, w], [w, mlp], all with biases
  float* q = nullptr;          // [w] fp32
  float *ln_g = nullptr, *ln_b = nullptr;
};

constexpr int GRAPH_MAX_B = 8;   // forwards of at most this many samples are replayed from a captured graph

enum { CLS_GEMM = 0, CLS_ATTN = 1, CLS_LN = 2, CLS_OTHER = 3,
       CLS_G_QKV = 4, CLS_G_OUT = 5, CLS_G_FC = 6, CLS_G_PROJ = 7, CLS_COUNT = 8 };  // 4..7: per-kind share of CLS_GEMM

}  // namespace b200

struct b200_clip {
  b200_clip_config cfg;
  int device = 0, sms = 132;
  bool loaded = false;
  bool has_text = true;       // false: an image-only handle (all-zero text tower config), no text weights or buffers
  b200::Tower vis, txt;
  b200::ResNetTower* rn = nullptr;   // the ResNet image tower (b200_clip_create_resnet) in place of vis and its front
  b200::ConvNeXtTower* cnx = nullptr;   // the ConvNeXt image tower (b200_clip_create_convnext), likewise
  bool siglip = false;               // b200_clip_create_siglip: timm/open_clip SigLIP towers
  b200::LatentHead head;             // SigLIP's image head
  // vision front end
  int grid = 0, Kp = 0;
  b200::Linear conv;          // [w, Kp]
  __nv_bfloat16* cols = nullptr;  // [max_batch*g*g, Kp]
  CUtensorMap tm_cols;
  __nv_bfloat16* vpos = nullptr;  // positional_embedding bf16 [T, w] (residual operand of the patch GEMM)
  float* cls_pos0 = nullptr;      // class_embedding + positional_embedding[0] (not SigLIP)
  float *lnpre_g = nullptr, *lnpre_b = nullptr;
  // text front end
  __nv_bfloat16* tok_emb = nullptr;  // [vocab, w]
  float* tpos = nullptr;             // [ctx, w]
  int* pool_idx = nullptr;
  float* feat = nullptr;             // raw projected features fp32 [max_batch, D] (pool/projection split over D / 64 blocks)
  // staging for the host entry points
  char* stage_in = nullptr;
  char* stage_out = nullptr;
  cudaStream_t s_copy = nullptr, s_comp = nullptr;   // host entry: H2D of sub-batch i+1 overlaps compute of i
  cudaEvent_t ev_in[4] = {}, ev_done[4] = {};
  b200::DeviceAllocs allocs;
  std::mutex mu;                  // held by every encode entry (host and device) while it enqueues
  b200::StreamFence act;          // orders forwards on different streams: they share the activation buffers
  b200::SpanTimer timer;          // timing; timer.launches = kernels of the last encode call
  // Serving shapes (batch <= GRAPH_MAX_B, clip_back.py:226-246 issues batch 1): the whole tower is captured once into a
  // CUDA graph per (modality, batch, output type) and replayed — ~75-150 kernel launches become one submission.
  // The graph works on fixed device buffers (g_in / g_out); a call copies its input in and its result out.
  struct TowerGraph { cudaGraphExec_t exec = nullptr; int seen = 0; int kernels = 0; };
  std::map<int, TowerGraph> graphs;   // key: image | B << 1 | f16 << 12 | normalize << 13
  char* g_in = nullptr;
  char* g_out = nullptr;
  bool use_graphs = true;      // B200_GRAPHS=0 disables (A/B, debugging)
  cudaStream_t cap_stream = nullptr;
};

namespace b200 {

static int make_tower(b200_clip* m, Tower* t, const b200_tower_config& c, int T, int D) {
  t->width = c.width; t->layers = c.layers; t->heads = c.heads; t->mlp = c.mlp; t->T = T;
  const int w = c.width;
  const size_t rows = (size_t)m->cfg.max_batch * T;
  B200_CHECK(w % 8 == 0 && c.mlp % 8 == 0 && w % c.heads == 0, B200_ERR_INVALID, "tower: width/mlp must be multiples of 8");
  DeviceAllocs& al = m->allocs;
  t->L.resize(c.layers);
  for (auto& L : t->L) {
    B200_TRY(al.alloc(&L.ln1_g, (size_t)w)); B200_TRY(al.alloc(&L.ln1_b, (size_t)w));
    B200_TRY(al.alloc(&L.ln2_g, (size_t)w)); B200_TRY(al.alloc(&L.ln2_b, (size_t)w));
    B200_TRY(make_linear(al, &L.qkv, 3 * w, w, true));
    B200_TRY(make_linear(al, &L.out, w, w, true));
    B200_TRY(make_linear(al, &L.fc, c.mlp, w, true));
    B200_TRY(make_linear(al, &L.proj, w, c.mlp, true));
  }
  B200_TRY(al.alloc(&t->lnf_g, (size_t)w)); B200_TRY(al.alloc(&t->lnf_b, (size_t)w));
  B200_TRY(al.alloc(&t->proj, (size_t)w * D));
  B200_TRY(al.alloc(&t->x, rows * w));
  B200_TRY(al.alloc(&t->h, rows * w));
  B200_TRY(al.alloc(&t->qkv, rows * 3 * w));
  B200_TRY(al.alloc(&t->a, rows * w));
  B200_TRY(al.alloc(&t->f, rows * c.mlp));
  B200_TRY(make_tmap_2d(&t->tm_h, t->h, 1, rows, w, w, GEMM_BM, GEMM_BK));
  B200_TRY(make_tmap_2d(&t->tm_a, t->a, 1, rows, w, w, GEMM_BM, GEMM_BK));
  B200_TRY(make_tmap_2d(&t->tm_f, t->f, 1, rows, c.mlp, c.mlp, GEMM_BM, GEMM_BK));
  if (attention_wgmma_supported(T, c.heads, w)) B200_TRY(make_qkv_map(&t->tm_qkv, t->qkv, m->cfg.max_batch, T, w));
  return B200_OK;
}

static int run_linear(b200_clip* m, const CUtensorMap& tmA, const Linear& l, int M, const GemmEpilogue& ep,
                      cudaStream_t st, int kind = CLS_GEMM) {
  TimedSpan sp(m->timer, kind, st, 1);
  return linear_gemm(l, tmA, M, ep, m->sms, st);
}

static int run_blocks(b200_clip* m, Tower& t, int B, cudaStream_t st) {
  const int w = t.width;
  const int M = B * t.T;
  const int act = m->cfg.quick_gelu ? ACT_QUICK_GELU : ACT_GELU;
  for (auto& L : t.L) {
    { TimedSpan sp(m->timer, CLS_LN, st, 1);
      B200_TRY(layernorm_rows_eps(t.x, w, t.h, w, L.ln1_g, L.ln1_b, M, w, t.ln_eps, st)); }
    GemmEpilogue e1; e1.out = t.qkv; e1.out_ld = 3 * w;
    B200_TRY(run_linear(m, t.tm_h, L.qkv, M, e1, st, CLS_G_QKV));
    { TimedSpan sp(m->timer, CLS_ATTN, st, 1);
      B200_TRY(qkv_attention(&t.tm_qkv, t.qkv, t.a, B, t.T, t.heads, w, t.causal, st)); }
    GemmEpilogue e2; e2.out = t.x; e2.out_ld = w; e2.residual = t.x; e2.res_ld = w;
    B200_TRY(run_linear(m, t.tm_a, L.out, M, e2, st, CLS_G_OUT));
    { TimedSpan sp(m->timer, CLS_LN, st, 1);
      B200_TRY(layernorm_rows_eps(t.x, w, t.h, w, L.ln2_g, L.ln2_b, M, w, t.ln_eps, st)); }
    GemmEpilogue e3; e3.out = t.f; e3.out_ld = t.mlp; e3.act = act;
    B200_TRY(run_linear(m, t.tm_h, L.fc, M, e3, st, CLS_G_FC));
    GemmEpilogue e4; e4.out = t.x; e4.out_ld = w; e4.residual = t.x; e4.res_ld = w;
    B200_TRY(run_linear(m, t.tm_f, L.proj, M, e4, st, CLS_G_PROJ));
  }
  return B200_OK;
}

// SigLIP image tower: patch GEMM with its bias and the positional rows as the residual (no class row, no ln_pre),
// the blocks, LN of every row, then the latent attention-pool head on M = B rows.
static int encode_image_chunk_siglip(b200_clip* m, const float* d_px, int B, void* d_out, int out_f16, int normalize,
                                     cudaStream_t st) {
  Tower& t = m->vis;
  LatentHead& hd = m->head;
  const int g = m->grid, w = t.width, T = t.T;
  { TimedSpan sp(m->timer, CLS_OTHER, st, 1);
    B200_TRY(im2col_patches(d_px, m->cols, B, m->cfg.image_size, m->cfg.patch, m->Kp, st)); }
  GemmEpilogue ep; ep.out = t.x; ep.out_ld = w;
  ep.residual = m->vpos; ep.res_ld = w; ep.res_row_mod = g * g; ep.res_row_off = 0;
  B200_TRY(run_linear(m, m->tm_cols, m->conv, B * T, ep, st, CLS_GEMM));
  B200_TRY(run_blocks(m, t, B, st));
  { TimedSpan sp(m->timer, CLS_LN, st, 1);
    B200_TRY(layernorm_rows_eps(t.x, w, t.h, w, t.lnf_g, t.lnf_b, (int64_t)B * T, w, t.ln_eps, st)); }
  GemmEpilogue e1; e1.out = t.qkv; e1.out_ld = 2 * w;
  B200_TRY(run_linear(m, t.tm_h, hd.kv, B * T, e1, st, CLS_GEMM));
  { TimedSpan sp(m->timer, CLS_ATTN, st, 1);
    B200_TRY(latent_pool_attention(t.qkv, hd.q, t.a, B, T, t.heads, w, st)); }
  GemmEpilogue e2; e2.out = t.x; e2.out_ld = w;
  B200_TRY(run_linear(m, t.tm_a, hd.proj, B, e2, st, CLS_GEMM));
  { TimedSpan sp(m->timer, CLS_LN, st, 1);
    B200_TRY(layernorm_rows_eps(t.x, w, t.h, w, hd.ln_g, hd.ln_b, B, w, t.ln_eps, st)); }
  GemmEpilogue e3; e3.out = t.f; e3.out_ld = t.mlp; e3.act = ACT_GELU;
  B200_TRY(run_linear(m, t.tm_h, hd.fc1, B, e3, st, CLS_GEMM));
  GemmEpilogue e4; e4.out = t.x; e4.out_ld = w; e4.residual = t.x; e4.res_ld = w;
  B200_TRY(run_linear(m, t.tm_f, hd.fc2, B, e4, st, CLS_GEMM));
  { TimedSpan sp(m->timer, CLS_OTHER, st, 1);
    B200_TRY(rows_feat_norm_cast(t.x, w, m->feat, d_out, out_f16, normalize, B, st)); }
  return B200_OK;
}

static int encode_image_chunk(b200_clip* m, const float* d_px, int B, void* d_out, int out_f16, int normalize,
                              cudaStream_t st) {
  if (m->rn)
    return resnet_encode(*m->rn, m->timer, CLS_GEMM, CLS_ATTN, CLS_OTHER, m->sms, d_px, B, m->feat, d_out, out_f16,
                         normalize, st);
  if (m->cnx)
    return convnext_encode(*m->cnx, m->timer, CLS_GEMM, CLS_OTHER, m->sms, d_px, B, m->feat, d_out, out_f16, normalize,
                           st);
  if (m->siglip) return encode_image_chunk_siglip(m, d_px, B, d_out, out_f16, normalize, st);
  Tower& t = m->vis;
  const int g = m->grid, w = t.width, T = t.T;
  { TimedSpan sp(m->timer, CLS_OTHER, st, 2);
    B200_TRY(im2col_patches(d_px, m->cols, B, m->cfg.image_size, m->cfg.patch, m->Kp, st));
    B200_TRY(write_cls_rows(t.x, m->cls_pos0, B, T, w, st)); }
  // patch embedding: x[b*T + 1 + p, :] = cols[b*g*g + p, :] · conv^T + positional_embedding[1 + p]
  GemmEpilogue ep; ep.out = t.x; ep.out_ld = w; ep.out_group = g * g;
  ep.residual = m->vpos; ep.res_ld = w; ep.res_row_mod = g * g; ep.res_row_off = 1;
  B200_TRY(run_linear(m, m->tm_cols, m->conv, B * g * g, ep, st, CLS_GEMM));
  { TimedSpan sp(m->timer, CLS_LN, st, 1);
    B200_TRY(layernorm_rows(t.x, w, t.x, w, m->lnpre_g, m->lnpre_b, (int64_t)B * T, w, st)); }
  B200_TRY(run_blocks(m, t, B, st));
  { TimedSpan sp(m->timer, CLS_OTHER, st, 1);
    B200_TRY(pool_ln_proj_norm(t.x, T, w, nullptr, t.lnf_g, t.lnf_b, t.proj, m->cfg.embed_dim, m->feat, d_out, out_f16, normalize, B, st)); }
  return B200_OK;
}

static int encode_text_chunk(b200_clip* m, const int64_t* d_tok, int B, void* d_out, int out_f16, int normalize,
                             cudaStream_t st) {
  Tower& t = m->txt;
  const int w = t.width, T = t.T;
  if (t.pool == POOL_LAST) {
    { TimedSpan sp(m->timer, CLS_OTHER, st, 1);
      B200_TRY(text_embed(d_tok, m->tok_emb, m->tpos, t.x, B, T, w, m->cfg.vocab_size, st)); }
    B200_TRY(run_blocks(m, t, B, st));
    TimedSpan sp(m->timer, CLS_OTHER, st, 2);
    return pool_last_ln_proj_bias_norm(t.x, T, w, t.lnf_g, t.lnf_b, t.ln_eps, t.proj, t.proj_b, m->cfg.embed_dim,
                                       m->feat, d_out, out_f16, normalize, B, st);
  }
  { TimedSpan sp(m->timer, CLS_OTHER, st, 2);
    B200_TRY(text_embed(d_tok, m->tok_emb, m->tpos, t.x, B, T, w, m->cfg.vocab_size, st));
    B200_TRY(token_argmax(d_tok, m->pool_idx, B, T, st)); }
  B200_TRY(run_blocks(m, t, B, st));
  { TimedSpan sp(m->timer, CLS_OTHER, st, 1);
    B200_TRY(pool_ln_proj_norm(t.x, T, w, m->pool_idx, t.lnf_g, t.lnf_b, t.proj, m->cfg.embed_dim, m->feat, d_out, out_f16, normalize, B, st)); }
  return B200_OK;
}

static int load_tower(Loader& ld, Tower& t, const std::string& prefix) {
  const size_t w = t.width, mlp = t.mlp;
  for (int i = 0; i < t.layers; i++) {
    Layer& L = t.L[i];
    const std::string p = prefix + "transformer.resblocks." + std::to_string(i) + ".";
    B200_TRY(ld.put_f32(p + "ln_1.weight", L.ln1_g, w));
    B200_TRY(ld.put_f32(p + "ln_1.bias", L.ln1_b, w));
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

// What both image towers share: the text tower and its front, the projected features, and the staging buffers of the
// host and graph entries.
static int make_text_and_staging(b200_clip* m) {
  const b200_clip_config* cfg = &m->cfg;
  DeviceAllocs& al = m->allocs;
  if (m->has_text) {
    B200_TRY(make_tower(m, &m->txt, cfg->text, cfg->context_length, cfg->embed_dim));
    m->txt.causal = 1;
    m->txt.pool = POOL_EOT;
    B200_TRY(al.alloc(&m->tok_emb, (size_t)cfg->vocab_size * cfg->text.width));
    B200_TRY(al.alloc(&m->tpos, (size_t)cfg->context_length * cfg->text.width));
    B200_TRY(al.alloc(&m->pool_idx, (size_t)cfg->max_batch));
  }
  const size_t tok_bytes = m->has_text ? (size_t)cfg->context_length * 8 : 0;
  B200_TRY(al.alloc(&m->feat, (size_t)cfg->max_batch * cfg->embed_dim));
  const size_t in_bytes = std::max((size_t)cfg->max_batch * 3 * cfg->image_size * cfg->image_size * 4,
                                   (size_t)cfg->max_batch * tok_bytes);
  B200_TRY(al.alloc(&m->stage_in, in_bytes));
  B200_TRY(al.alloc(&m->stage_out, (size_t)cfg->max_batch * cfg->embed_dim * 4));
  const int gb = std::min(GRAPH_MAX_B, cfg->max_batch);
  B200_TRY(al.alloc(&m->g_in, std::max((size_t)gb * 3 * cfg->image_size * cfg->image_size * 4, (size_t)gb * tok_bytes)));
  B200_TRY(al.alloc(&m->g_out, (size_t)gb * cfg->embed_dim * 4));
  return B200_OK;
}

// The ViT image tower's visual.* tensors.
static int load_vit(b200_clip* m, Loader& ld) {
  const b200_clip_config& c = m->cfg;
  const size_t vw = c.vision.width, D = c.embed_dim;
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
  return B200_OK;
}

// SigLIP's tensors in open_clip's layout: the timm trunk under visual.trunk.*, the text tower under text.*.
static int load_siglip(b200_clip* m, Loader& ld) {
  const b200_clip_config& c = m->cfg;
  const size_t w = c.vision.width, mlp = c.vision.mlp, T = m->vis.T, kraw = (size_t)3 * c.patch * c.patch;
  const std::string v = "visual.trunk.";
  B200_TRY(ld.put_bf16(v + "patch_embed.proj.weight", m->conv.w, w, kraw, m->Kp));
  B200_TRY(ld.put_f32(v + "patch_embed.proj.bias", m->conv.b, w));
  B200_TRY(ld.put_bf16(v + "pos_embed", m->vpos, T, w, w));
  for (int i = 0; i < m->vis.layers; i++) {
    Layer& L = m->vis.L[i];
    const std::string p = v + "blocks." + std::to_string(i) + ".";
    B200_TRY(ld.put_f32(p + "norm1.weight", L.ln1_g, w));
    B200_TRY(ld.put_f32(p + "norm1.bias", L.ln1_b, w));
    B200_TRY(ld.put_bf16(p + "attn.qkv.weight", L.qkv.w, 3 * w, w, w));
    B200_TRY(ld.put_f32(p + "attn.qkv.bias", L.qkv.b, 3 * w));
    B200_TRY(ld.put_bf16(p + "attn.proj.weight", L.out.w, w, w, w));
    B200_TRY(ld.put_f32(p + "attn.proj.bias", L.out.b, w));
    B200_TRY(ld.put_f32(p + "norm2.weight", L.ln2_g, w));
    B200_TRY(ld.put_f32(p + "norm2.bias", L.ln2_b, w));
    B200_TRY(ld.put_bf16(p + "mlp.fc1.weight", L.fc.w, mlp, w, w));
    B200_TRY(ld.put_f32(p + "mlp.fc1.bias", L.fc.b, mlp));
    B200_TRY(ld.put_bf16(p + "mlp.fc2.weight", L.proj.w, w, mlp, mlp));
    B200_TRY(ld.put_f32(p + "mlp.fc2.bias", L.proj.b, w));
  }
  B200_TRY(ld.put_f32(v + "norm.weight", m->vis.lnf_g, w));
  B200_TRY(ld.put_f32(v + "norm.bias", m->vis.lnf_b, w));
  const std::string a = v + "attn_pool.";
  LatentHead& hd = m->head;
  {
    // q = q_proj(latent) in fp64 from the checkpoint's values, stored fp32
    const b200_tensor_view* lat = ld.find(a + "latent", w);
    const b200_tensor_view* qw = ld.find(a + "q.weight", w * w);
    const b200_tensor_view* qb = ld.find(a + "q.bias", w);
    if (!lat || !qw || !qb) return B200_ERR_INVALID;
    std::vector<float> q(w);
    for (size_t i = 0; i < w; i++) {
      double acc = view_get(*qb, i);
      for (size_t j = 0; j < w; j++) acc += (double)view_get(*qw, i * w + j) * (double)view_get(*lat, j);
      q[i] = (float)acc;
    }
    B200_CUDA(cudaMemcpy(hd.q, q.data(), w * 4, cudaMemcpyHostToDevice));
  }
  B200_TRY(ld.put_bf16(a + "kv.weight", hd.kv.w, 2 * w, w, w));
  B200_TRY(ld.put_f32(a + "kv.bias", hd.kv.b, 2 * w));
  B200_TRY(ld.put_bf16(a + "proj.weight", hd.proj.w, w, w, w));
  B200_TRY(ld.put_f32(a + "proj.bias", hd.proj.b, w));
  B200_TRY(ld.put_f32(a + "norm.weight", hd.ln_g, w));
  B200_TRY(ld.put_f32(a + "norm.bias", hd.ln_b, w));
  B200_TRY(ld.put_bf16(a + "mlp.fc1.weight", hd.fc1.w, mlp, w, w));
  B200_TRY(ld.put_f32(a + "mlp.fc1.bias", hd.fc1.b, mlp));
  B200_TRY(ld.put_bf16(a + "mlp.fc2.weight", hd.fc2.w, w, mlp, mlp));
  B200_TRY(ld.put_f32(a + "mlp.fc2.bias", hd.fc2.b, w));
  if (m->has_text) {
    const size_t tw = c.text.width, D = c.embed_dim;
    B200_TRY(ld.put_bf16("text.token_embedding.weight", m->tok_emb, (size_t)c.vocab_size, tw, tw));
    B200_TRY(ld.put_f32("text.positional_embedding", m->tpos, (size_t)c.context_length * tw));
    B200_TRY(load_tower(ld, m->txt, "text."));
    B200_TRY(ld.put_f32("text.ln_final.weight", m->txt.lnf_g, tw));
    B200_TRY(ld.put_f32("text.ln_final.bias", m->txt.lnf_b, tw));
    B200_TRY(ld.put_bf16_t("text.text_projection.weight", m->txt.proj, D, tw));
    B200_TRY(ld.put_f32("text.text_projection.bias", m->txt.proj_b, D));
  }
  return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_clip_create(const b200_clip_config* cfg, int device, b200_clip** out) {
  B200_CHECK(cfg && out, B200_ERR_INVALID, "clip_create: null argument");
  const bool has_text = cfg->text.width != 0 || cfg->text.layers != 0 || cfg->text.heads != 0 || cfg->text.mlp != 0;
  B200_CHECK(cfg->max_batch >= 1 && cfg->embed_dim >= 8 && cfg->patch >= 1 && cfg->image_size >= cfg->patch &&
                 (!has_text || (cfg->context_length >= 1 && cfg->vocab_size >= 2)),
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
  m->has_text = has_text;
  if (const char* g = getenv("B200_GRAPHS")) m->use_graphs = atoi(g) != 0;
  m->grid = cfg->image_size / cfg->patch;
  const int k_raw = 3 * cfg->patch * cfg->patch;
  m->Kp = (k_raw + 63) / 64 * 64;
  const int T = m->grid * m->grid + 1;
  int rc = B200_OK;
  auto build = [&]() -> int {
    B200_TRY(make_tower(m, &m->vis, cfg->vision, T, cfg->embed_dim));
    DeviceAllocs& al = m->allocs;
    B200_TRY(make_linear(al, &m->conv, cfg->vision.width, m->Kp, false));
    const size_t prow = (size_t)cfg->max_batch * m->grid * m->grid;
    B200_TRY(al.alloc(&m->cols, prow * m->Kp));
    B200_CUDA(cudaMemset(m->cols, 0, prow * m->Kp * 2));
    B200_TRY(make_tmap_2d(&m->tm_cols, m->cols, 1, prow, m->Kp, m->Kp, GEMM_BM, GEMM_BK));
    B200_TRY(al.alloc(&m->vpos, (size_t)T * cfg->vision.width));
    B200_TRY(al.alloc(&m->cls_pos0, (size_t)cfg->vision.width));
    B200_TRY(al.alloc(&m->lnpre_g, (size_t)cfg->vision.width));
    B200_TRY(al.alloc(&m->lnpre_b, (size_t)cfg->vision.width));
    return make_text_and_staging(m);
  };
  rc = build();
  if (rc != B200_OK) {
    b200_clip_destroy(m);
    return rc;
  }
  *out = m;
  return B200_OK;
}

// The ResNet image tower (resnet.cuh) with the same text tower, staging, graphs and entries as b200_clip_create.
int b200_clip_create_resnet(const b200_clip_config* cfg, const b200_resnet_config* rc, int device, b200_clip** out) {
  B200_CHECK(cfg && rc && out, B200_ERR_INVALID, "clip_create_resnet: null argument");
  const bool has_text = cfg->text.width != 0 || cfg->text.layers != 0 || cfg->text.heads != 0 || cfg->text.mlp != 0;
  const bool no_vit = cfg->patch == 0 && cfg->vision.width == 0 && cfg->vision.layers == 0 && cfg->vision.heads == 0 &&
                      cfg->vision.mlp == 0;
  B200_CHECK(no_vit && cfg->max_batch >= 1 && cfg->embed_dim >= 8 && cfg->image_size >= 32 && cfg->image_size % 32 == 0 &&
                 (!has_text || (cfg->context_length >= 1 && cfg->vocab_size >= 2)),
             B200_ERR_INVALID, "clip_create_resnet: bad config (vision and patch must be zero, image_size a multiple of 32)");
  int ndev = 0;
  B200_CUDA(cudaGetDeviceCount(&ndev));
  B200_CHECK(device >= 0 && device < ndev, B200_ERR_INVALID, "clip_create_resnet: device %d of %d", device, ndev);
  DeviceGuard g(device);
  b200_clip* m = new (std::nothrow) b200_clip();
  B200_CHECK(m != nullptr, B200_ERR_OOM, "clip_create_resnet: host allocation failed");
  m->cfg = *cfg;
  m->device = device;
  m->sms = sm_count(device);
  m->has_text = has_text;
  if (const char* e = getenv("B200_GRAPHS")) m->use_graphs = atoi(e) != 0;
  m->rn = new (std::nothrow) ResNetTower();
  int rc_ = m->rn == nullptr ? B200_ERR_OOM : B200_OK;
  if (rc_ == B200_OK) rc_ = resnet_create(m->allocs, m->rn, *rc, cfg->image_size, cfg->embed_dim, cfg->max_batch);
  if (rc_ == B200_OK) rc_ = make_text_and_staging(m);
  if (rc_ != B200_OK) {
    b200_clip_destroy(m);
    return rc_;
  }
  *out = m;
  return B200_OK;
}

// The ConvNeXt image tower (convnext.cuh) with the same text tower, staging, graphs and entries as b200_clip_create.
int b200_clip_create_convnext(const b200_clip_config* cfg, const b200_convnext_config* nc, int device, b200_clip** out) {
  B200_CHECK(cfg && nc && out, B200_ERR_INVALID, "clip_create_convnext: null argument");
  const bool has_text = cfg->text.width != 0 || cfg->text.layers != 0 || cfg->text.heads != 0 || cfg->text.mlp != 0;
  const bool no_vit = cfg->patch == 0 && cfg->vision.width == 0 && cfg->vision.layers == 0 && cfg->vision.heads == 0 &&
                      cfg->vision.mlp == 0;
  B200_CHECK(no_vit && cfg->max_batch >= 1 && cfg->embed_dim >= 8 && cfg->image_size >= 32 && cfg->image_size % 32 == 0 &&
                 (!has_text || (cfg->context_length >= 1 && cfg->vocab_size >= 2)),
             B200_ERR_INVALID, "clip_create_convnext: bad config (vision and patch must be zero, image_size a multiple of "
             "32)");
  int ndev = 0;
  B200_CUDA(cudaGetDeviceCount(&ndev));
  B200_CHECK(device >= 0 && device < ndev, B200_ERR_INVALID, "clip_create_convnext: device %d of %d", device, ndev);
  DeviceGuard g(device);
  b200_clip* m = new (std::nothrow) b200_clip();
  B200_CHECK(m != nullptr, B200_ERR_OOM, "clip_create_convnext: host allocation failed");
  m->cfg = *cfg;
  m->device = device;
  m->sms = sm_count(device);
  m->has_text = has_text;
  if (const char* e = getenv("B200_GRAPHS")) m->use_graphs = atoi(e) != 0;
  m->cnx = new (std::nothrow) ConvNeXtTower();
  int rc = m->cnx == nullptr ? B200_ERR_OOM : B200_OK;
  if (rc == B200_OK) rc = convnext_create(m->allocs, m->cnx, *nc, cfg->image_size, cfg->embed_dim, cfg->max_batch);
  if (rc == B200_OK) rc = make_text_and_staging(m);
  if (rc != B200_OK) {
    b200_clip_destroy(m);
    return rc;
  }
  *out = m;
  return B200_OK;
}

// SigLIP (open_clip's timm-trunk configs): the ViT handle with no class row and no ln_pre, a patch bias, the latent
// attention-pool head, a bidirectional text tower pooled at its last position with a biased projection, and LayerNorm
// eps 1e-6 everywhere.
int b200_clip_create_siglip(const b200_clip_config* cfg, int device, b200_clip** out) {
  B200_CHECK(cfg && out, B200_ERR_INVALID, "clip_create_siglip: null argument");
  const bool has_text = cfg->text.width != 0 || cfg->text.layers != 0 || cfg->text.heads != 0 || cfg->text.mlp != 0;
  B200_CHECK(cfg->max_batch >= 1 && cfg->patch >= 1 && cfg->image_size >= cfg->patch && cfg->vision.heads >= 1 &&
                 cfg->embed_dim == cfg->vision.width && cfg->quick_gelu == 0 &&
                 (!has_text || (cfg->context_length >= 1 && cfg->vocab_size >= 2)),
             B200_ERR_INVALID, "clip_create_siglip: bad config (embed_dim must equal the vision width, quick_gelu 0)");
  int ndev = 0;
  B200_CUDA(cudaGetDeviceCount(&ndev));
  B200_CHECK(device >= 0 && device < ndev, B200_ERR_INVALID, "clip_create_siglip: device %d of %d", device, ndev);
  DeviceGuard g(device);
  b200_clip* m = new (std::nothrow) b200_clip();
  B200_CHECK(m != nullptr, B200_ERR_OOM, "clip_create_siglip: host allocation failed");
  m->cfg = *cfg;
  m->device = device;
  m->sms = sm_count(device);
  m->has_text = has_text;
  m->siglip = true;
  if (const char* e = getenv("B200_GRAPHS")) m->use_graphs = atoi(e) != 0;
  m->grid = cfg->image_size / cfg->patch;
  m->Kp = (3 * cfg->patch * cfg->patch + 63) / 64 * 64;
  const int T = m->grid * m->grid;
  auto build = [&]() -> int {
    const int w = cfg->vision.width;
    B200_TRY(make_tower(m, &m->vis, cfg->vision, T, cfg->embed_dim));
    m->vis.ln_eps = 1e-6f;
    m->vis.pool = POOL_LATENT;
    DeviceAllocs& al = m->allocs;
    B200_TRY(make_linear(al, &m->conv, w, m->Kp, true));
    const size_t prow = (size_t)cfg->max_batch * T;
    B200_TRY(al.alloc(&m->cols, prow * m->Kp));
    B200_CUDA(cudaMemset(m->cols, 0, prow * m->Kp * 2));
    B200_TRY(make_tmap_2d(&m->tm_cols, m->cols, 1, prow, m->Kp, m->Kp, GEMM_BM, GEMM_BK));
    B200_TRY(al.alloc(&m->vpos, (size_t)T * w));
    LatentHead& hd = m->head;
    B200_TRY(make_linear(al, &hd.kv, 2 * w, w, true));
    B200_TRY(make_linear(al, &hd.proj, w, w, true));
    B200_TRY(make_linear(al, &hd.fc1, cfg->vision.mlp, w, true));
    B200_TRY(make_linear(al, &hd.fc2, w, cfg->vision.mlp, true));
    B200_TRY(al.alloc(&hd.q, (size_t)w));
    B200_TRY(al.alloc(&hd.ln_g, (size_t)w));
    B200_TRY(al.alloc(&hd.ln_b, (size_t)w));
    B200_TRY(make_text_and_staging(m));
    if (has_text) {
      m->txt.ln_eps = 1e-6f;
      m->txt.causal = 0;
      m->txt.pool = POOL_LAST;
      B200_TRY(al.alloc(&m->txt.proj_b, (size_t)cfg->embed_dim));
    }
    return B200_OK;
  };
  const int rc = build();
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
  m->allocs.free_all();
  delete m->rn;
  delete m->cnx;
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
  B200_TRY(ld.index(tensors, n));
  const b200_clip_config& c = m->cfg;
  const size_t tw = c.text.width, D = c.embed_dim;
  if (m->siglip) {
    B200_TRY(load_siglip(m, ld));
    B200_CUDA(cudaDeviceSynchronize());
    m->loaded = true;
    return B200_OK;
  }
  if (m->rn) B200_TRY(resnet_load(ld, *m->rn));
  else if (m->cnx) B200_TRY(convnext_load(ld, *m->cnx));
  else B200_TRY(load_vit(m, ld));
  if (m->has_text) {
    B200_TRY(ld.put_bf16("token_embedding.weight", m->tok_emb, (size_t)c.vocab_size, tw, tw));
    B200_TRY(ld.put_f32("positional_embedding", m->tpos, (size_t)c.context_length * tw));
    B200_TRY(load_tower(ld, m->txt, ""));
    B200_TRY(ld.put_f32("ln_final.weight", m->txt.lnf_g, tw));
    B200_TRY(ld.put_f32("ln_final.bias", m->txt.lnf_b, tw));
    B200_TRY(ld.put_bf16("text_projection", m->txt.proj, tw, D, D));
  }
  B200_CUDA(cudaDeviceSynchronize());
  m->loaded = true;
  return B200_OK;
}

static int encode_device(b200_clip* m, const void* d_in, int B, void* d_out, int out_dtype, int normalize, bool image,
                         cudaStream_t st) {
  B200_CHECK(m && (B == 0 || (d_in && d_out)) && B >= 0, B200_ERR_INVALID, "encode: bad argument");
  B200_CHECK(m->loaded, B200_ERR_STATE, "encode: weights not loaded");
  B200_CHECK(image || m->has_text, B200_ERR_UNSUPPORTED, "encode_text: this handle has no text tower");
  B200_CHECK(out_dtype == B200_OUT_F16 || out_dtype == B200_OUT_F32, B200_ERR_INVALID, "encode: out_dtype %d", out_dtype);
  DeviceGuard g(m->device);
  m->timer.launches = 0;
  const int mb = m->cfg.max_batch;
  const size_t in_stride = image ? (size_t)3 * m->cfg.image_size * m->cfg.image_size * 4 : (size_t)m->cfg.context_length * 8;
  const size_t out_stride = (size_t)m->cfg.embed_dim * (out_dtype == B200_OUT_F16 ? 2 : 4);
  if (B >= 1 && B <= GRAPH_MAX_B && B <= mb && m->use_graphs && !m->timer.profiling) {
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
          tg.kernels = m->timer.launches;   // kernels inside the graph (they were counted once, at capture)
          if (ie != cudaSuccess) { cudaGetLastError(); tg.exec = nullptr; m->use_graphs = false; }
        }
      }
      if (tg.exec != nullptr) {
        B200_CUDA(cudaMemcpyAsync(m->g_in, d_in, (size_t)B * in_stride, cudaMemcpyDeviceToDevice, st));
        B200_CUDA(cudaGraphLaunch(tg.exec, st));
        B200_CUDA(cudaMemcpyAsync(d_out, m->g_out, (size_t)B * out_stride, cudaMemcpyDeviceToDevice, st));
        count_launch(tg.kernels);
        m->timer.launches = tg.kernels;
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

static int encode_device_locked(b200_clip* m, const void* d_in, int B, void* d_out, int out_dtype, int normalize,
                                bool image, cudaStream_t st) {
  B200_CHECK(m, B200_ERR_INVALID, "encode: null handle");
  std::lock_guard<std::mutex> lock(m->mu);
  DeviceGuard g(m->device);
  B200_TRY(m->act.acquire(st));
  const int rc = encode_device(m, d_in, B, d_out, out_dtype, normalize, image, st);
  B200_TRY(m->act.release(st));
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
  B200_CHECK(image || m->has_text, B200_ERR_UNSUPPORTED, "encode_text: this handle has no text tower");
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
  B200_TRY(m->act.acquire(m->s_comp));
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
      char* stage = m->stage_in + (size_t)slot * SB * in_stride;
      if (gi >= slots) B200_CUDA(cudaStreamWaitEvent(m->s_copy, m->ev_done[slot], 0));
      B200_CUDA(cudaMemcpyAsync(stage, (const char*)h_in + (size_t)(b0 + s0) * in_stride, ns * in_stride,
                                cudaMemcpyHostToDevice, m->s_copy));
      B200_CUDA(cudaEventRecord(m->ev_in[slot], m->s_copy));
      B200_CUDA(cudaStreamWaitEvent(m->s_comp, m->ev_in[slot], 0));
      B200_TRY(encode_device(m, stage, ns, m->stage_out + (size_t)s0 * out_stride, out_dtype, normalize, image,
                             m->s_comp));
      B200_CUDA(cudaEventRecord(m->ev_done[slot], m->s_comp));
      launches += m->timer.launches;
    }
    B200_CUDA(cudaMemcpyAsync((char*)h_out + (size_t)b0 * out_stride, m->stage_out, nb * out_stride, cudaMemcpyDeviceToHost,
                              m->s_comp));
  }
  B200_CUDA(cudaStreamSynchronize(m->s_comp));
  B200_TRY(m->act.release(m->s_comp));
  m->timer.launches = launches;
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
  return qkv_attention(nullptr, (const __nv_bfloat16*)d_qkv, (__nv_bfloat16*)d_out, B, T, heads, w, causal,
                       (cudaStream_t)stream);
}
int b200_vision_front_bf16_device(const float* d_pixels, int B, int S, int p, int Kp, void* d_cols, const float* d_cls,
                                  int T, int w, void* d_x, int device, void* stream) {
  B200_CHECK(B >= 0 && p >= 1 && S >= p && Kp >= 3 * p * p && (B == 0 || (d_pixels && d_cols)) &&
                 (d_x == nullptr || (d_cls && T >= 1 && w >= 1)),
             B200_ERR_INVALID, "vision_front: bad argument");
  if (B == 0) return B200_OK;
  DeviceGuard g(device);
  B200_TRY(im2col_patches(d_pixels, (__nv_bfloat16*)d_cols, B, S, p, Kp, (cudaStream_t)stream));
  if (d_x) B200_TRY(write_cls_rows((__nv_bfloat16*)d_x, d_cls, B, T, w, (cudaStream_t)stream));
  return B200_OK;
}
int b200_text_embed_bf16_device(const int64_t* d_tokens, const void* d_tok_emb, const float* d_pos, void* d_x, int B,
                                int T, int w, int vocab, int device, void* stream) {
  B200_CHECK(B >= 0 && T >= 1 && w >= 8 && w % 8 == 0 && vocab >= 1 && (B == 0 || (d_tokens && d_tok_emb && d_pos && d_x)),
             B200_ERR_INVALID, "text_embed: bad argument");
  if (B == 0) return B200_OK;
  DeviceGuard g(device);
  return text_embed(d_tokens, (const __nv_bfloat16*)d_tok_emb, d_pos, (__nv_bfloat16*)d_x, B, T, w, vocab,
                    (cudaStream_t)stream);
}
int b200_token_argmax_device(const int64_t* d_tokens, int B, int T, int32_t* d_idx, int device, void* stream) {
  B200_CHECK(B >= 0 && T >= 1 && (B == 0 || (d_tokens && d_idx)), B200_ERR_INVALID, "token_argmax: bad argument");
  if (B == 0) return B200_OK;
  DeviceGuard g(device);
  return token_argmax(d_tokens, d_idx, B, T, (cudaStream_t)stream);
}
int b200_pool_ln_proj_device(const void* d_x, int B, int T, int w, const int32_t* d_pool_idx, const float* d_gamma,
                             const float* d_beta, const void* d_proj, int D, float* d_feat, void* d_out, int out_dtype,
                             int normalize, int device, void* stream) {
  B200_CHECK(B >= 0 && T >= 1 && w >= 1 && D >= 1 && (B == 0 || (d_x && d_gamma && d_beta && d_proj && d_feat && d_out)) &&
                 (out_dtype == B200_OUT_F16 || out_dtype == B200_OUT_F32),
             B200_ERR_INVALID, "pool_ln_proj: bad argument");
  DeviceGuard g(device);
  return pool_ln_proj_norm((const __nv_bfloat16*)d_x, T, w, d_pool_idx, d_gamma, d_beta, (const __nv_bfloat16*)d_proj,
                           D, d_feat, d_out, out_dtype == B200_OUT_F16, normalize, B, (cudaStream_t)stream);
}

int b200_latent_pool_attention_device(const void* d_kv, int B, int T, int heads, int w, const float* d_q, void* d_out,
                                      int device, void* stream) {
  B200_CHECK(B >= 0 && T >= 1 && (B == 0 || (d_kv && d_q && d_out)), B200_ERR_INVALID, "latent_pool: bad argument");
  DeviceGuard g(device);
  return latent_pool_attention((const __nv_bfloat16*)d_kv, d_q, (__nv_bfloat16*)d_out, B, T, heads, w,
                               (cudaStream_t)stream);
}
int b200_pool_last_ln_proj_bias_device(const void* d_x, int B, int T, int w, const float* d_gamma, const float* d_beta,
                                       float eps, const void* d_proj, const float* d_bias, int D, float* d_feat,
                                       void* d_out, int out_dtype, int normalize, int device, void* stream) {
  B200_CHECK(B >= 0 && T >= 1 && w >= 1 && D >= 1 && eps > 0.f &&
                 (B == 0 || (d_x && d_gamma && d_beta && d_proj && d_bias && d_feat && d_out)) &&
                 (out_dtype == B200_OUT_F16 || out_dtype == B200_OUT_F32),
             B200_ERR_INVALID, "pool_last_ln_proj_bias: bad argument");
  DeviceGuard g(device);
  return pool_last_ln_proj_bias_norm((const __nv_bfloat16*)d_x, T, w, d_gamma, d_beta, eps,
                                     (const __nv_bfloat16*)d_proj, d_bias, D, d_feat, d_out,
                                     out_dtype == B200_OUT_F16, normalize, B, (cudaStream_t)stream);
}

int b200_dwconv7_ln_bf16_device(const void* d_x, int B, int H, int W, int C, const float* d_w49, const float* d_bias,
                                const float* d_gamma, const float* d_beta, float eps, void* d_out, int device,
                                void* stream) {
  B200_CHECK(B >= 0 && (B == 0 || (d_x && d_w49 && d_bias && d_out)) && (d_gamma == nullptr || (d_beta && eps > 0.f)),
             B200_ERR_INVALID, "dwconv7_ln: bad argument");
  DeviceGuard g(device);
  return dwconv7_ln((const __nv_bfloat16*)d_x, d_w49, d_bias, d_gamma, d_beta, eps, (__nv_bfloat16*)d_out, B, H, W, C,
                    (cudaStream_t)stream);
}
int b200_ln_s2d_bf16_device(const void* d_x, int B, int H, int W, int C, const float* d_gamma, const float* d_beta,
                            float eps, void* d_out, int device, void* stream) {
  B200_CHECK(B >= 0 && eps > 0.f && (B == 0 || (d_x && d_gamma && d_beta && d_out)), B200_ERR_INVALID,
             "ln_s2d: bad argument");
  DeviceGuard g(device);
  return ln_s2d((const __nv_bfloat16*)d_x, d_gamma, d_beta, eps, (__nv_bfloat16*)d_out, B, H, W, C,
                (cudaStream_t)stream);
}
int b200_convnext_head_device(const void* d_x, int B, int HW, int C, const float* d_gamma, const float* d_beta, float eps,
                              const float* d_w1T, const float* d_b1, int h, const float* d_w2T, int D, float* d_pooled,
                              float* d_hid, float* d_feat, void* d_out, int out_dtype, int normalize, int device,
                              void* stream) {
  B200_CHECK(B >= 0 && HW >= 1 && C >= 1 && D >= 1 && eps > 0.f && (d_w1T == nullptr || (d_b1 && d_hid && h >= 1)) &&
                 (B == 0 || (d_x && d_gamma && d_beta && d_w2T && d_pooled && d_feat && d_out)) &&
                 (out_dtype == B200_OUT_F16 || out_dtype == B200_OUT_F32),
             B200_ERR_INVALID, "convnext_head: bad argument");
  DeviceGuard g(device);
  const cudaStream_t st = (cudaStream_t)stream;
  B200_TRY(mean_ln_rows((const __nv_bfloat16*)d_x, B, HW, C, d_gamma, d_beta, eps, d_pooled, st));
  return rows_head_norm(d_pooled, C, d_w1T, d_b1, h, d_w2T, D, d_hid, d_feat, d_out, out_dtype == B200_OUT_F16,
                        normalize, B, st);
}

int b200_clip_set_profiling(b200_clip* m, int on) {
  B200_CHECK(m, B200_ERR_INVALID, "set_profiling: null handle");
  m->timer.set_profiling(on != 0);
  return B200_OK;
}

int b200_clip_last_timing(b200_clip* m, float* ms_by_class, int* launches) {
  B200_CHECK(m && ms_by_class, B200_ERR_INVALID, "last_timing: null argument");
  DeviceGuard g(m->device);
  const int spans = m->timer.used;
  B200_TRY(m->timer.collect(ms_by_class, CLS_COUNT));
  for (int c = CLS_G_QKV; c <= CLS_G_PROJ; c++) ms_by_class[CLS_GEMM] += ms_by_class[c];
  if (launches) *launches = spans;
  return B200_OK;
}

}  // extern "C"
