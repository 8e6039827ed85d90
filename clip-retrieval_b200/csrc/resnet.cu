// The ResNet image tower (resnet.cuh): buffers, the BatchNorm-folding loader and the forward.
#include "resnet.cuh"
#include <algorithm>
#include <cmath>
#include <string>

namespace b200 {

static int conv_cb(int cin) { return (cin + GEMM_BK - 1) / GEMM_BK; }

int resnet_create(DeviceAllocs& al, ResNetTower* r, const b200_resnet_config& rc, int S, int D, int mb) {
  B200_CHECK(S >= 32 && S % 32 == 0 && rc.width >= 16 && rc.width % 16 == 0 && rc.heads >= 1 &&
                 (32 * rc.width) % rc.heads == 0 && D >= 8,
             B200_ERR_INVALID, "resnet: image_size a multiple of 32, width a multiple of 16 (S=%d width=%d heads=%d)", S,
             rc.width, rc.heads);
  for (int i = 0; i < 4; i++) B200_CHECK(rc.layers[i] >= 1, B200_ERR_INVALID, "resnet: layers[%d]=%d", i, rc.layers[i]);
  const int w = rc.width;
  for (int i = 0; i < 4; i++) r->layers[i] = rc.layers[i];
  r->w = w; r->heads = rc.heads; r->S = S; r->C = 32 * w; r->D = D; r->mb = mb;
  const int Hf = S / 32;
  r->T = Hf * Hf + 1;
  const size_t B = (size_t)mb;
  const size_t g = S / 2;
  // buffer sizes, walking the tower
  size_t n_buf = std::max(B * g * g * w, B * (g / 2) * (g / 2) * w), n_t1 = B * g * g * (w / 2), n_t3 = 1, n_xp = 1,
         n_idn = 1;
  {
    int H = S / 4, cin = w;
    for (int s = 0; s < 4; s++) {
      const int planes = w << s;
      for (int j = 0; j < rc.layers[s]; j++) {
        const int stride = (j == 0 && s > 0) ? 2 : 1, Ho = H / stride;
        n_t1 = std::max(n_t1, B * H * H * planes);
        n_buf = std::max(n_buf, B * Ho * Ho * 4 * planes);
        if (stride > 1) {
          n_t3 = std::max(n_t3, B * Ho * Ho * planes);
          n_xp = std::max(n_xp, B * Ho * Ho * cin);
        }
        if (stride > 1 || cin != 4 * planes) n_idn = std::max(n_idn, B * Ho * Ho * 4 * planes);
        cin = 4 * planes;
        H = Ho;
      }
    }
  }
  B200_TRY(al.alloc(&r->cols, B * g * g * GEMM_BK));
  B200_CUDA(cudaMemset(r->cols, 0, B * g * g * GEMM_BK * 2));   // columns 27..63 stay zero
  for (int i = 0; i < 2; i++) B200_TRY(al.alloc(&r->buf[i], n_buf));
  B200_TRY(al.alloc(&r->t1, n_t1));
  B200_TRY(al.alloc(&r->t2, n_t1));
  B200_TRY(al.alloc(&r->t3, n_t3));
  B200_TRY(al.alloc(&r->xp, n_xp));
  B200_TRY(al.alloc(&r->idn, n_idn));
  // stem: gather -> stem1 (t1) -> stem2 (t2) -> stem3 (buf[1]) -> pool (buf[0])
  B200_TRY(make_linear(al, &r->stem1, w / 2, GEMM_BK, true));
  B200_TRY(make_linear(al, &r->stem2, w / 2, 9 * conv_cb(w / 2) * GEMM_BK, true));
  B200_TRY(make_linear(al, &r->stem3, w, 9 * conv_cb(w / 2) * GEMM_BK, true));
  B200_TRY(make_tmap_2d(&r->tm_cols, r->cols, 1, B * g * g, GEMM_BK, GEMM_BK, GEMM_BM, GEMM_BK));
  B200_TRY(make_tmap_im2col_3x3(&r->tm_s1, r->t1, mb, (int)g, (int)g, w / 2));
  B200_TRY(make_tmap_im2col_3x3(&r->tm_s2, r->t2, mb, (int)g, (int)g, w / 2));
  int H = S / 4, cin = w, idx = 0;
  for (int s = 0; s < 4; s++) {
    const int planes = w << s;
    for (int j = 0; j < rc.layers[s]; j++, idx++) {
      RnBlock b;
      b.cin = cin; b.planes = planes; b.H = H;
      b.stride = (j == 0 && s > 0) ? 2 : 1;
      b.has_ds = b.stride > 1 || cin != 4 * planes;
      const int Ho = H / b.stride;
      b.x = r->buf[idx % 2];
      b.y = r->buf[(idx + 1) % 2];
      B200_TRY(make_linear(al, &b.c1, planes, cin, true));
      B200_TRY(make_linear(al, &b.c2, planes, 9 * conv_cb(planes) * GEMM_BK, true));
      B200_TRY(make_linear(al, &b.c3, 4 * planes, planes, true));
      if (b.has_ds) B200_TRY(make_linear(al, &b.ds, 4 * planes, cin, true));
      B200_TRY(make_tmap_2d(&b.tm_x, b.x, 1, B * H * H, cin, cin, GEMM_BM, GEMM_BK));
      B200_TRY(make_tmap_im2col_3x3(&b.tm_t1, r->t1, mb, H, H, planes));
      B200_TRY(make_tmap_2d(&b.tm_a3, b.stride > 1 ? r->t3 : r->t2, 1, B * Ho * Ho, planes, planes, GEMM_BM, GEMM_BK));
      if (b.stride > 1) B200_TRY(make_tmap_2d(&b.tm_xp, r->xp, 1, B * Ho * Ho, cin, cin, GEMM_BM, GEMM_BK));
      r->blocks.push_back(b);
      cin = 4 * planes;
      H = Ho;
    }
  }
  // attention pool
  const int C = r->C, T = r->T;
  B200_TRY(al.alloc(&r->tok, B * T * C));
  B200_TRY(al.alloc(&r->qkv, B * T * 3 * C));
  B200_TRY(al.alloc(&r->att, B * T * C));
  B200_TRY(make_tmap_2d(&r->tm_tok, r->tok, 1, B * T, C, C, GEMM_BM, GEMM_BK));
  r->qkv_map = attention_wgmma_supported(T, rc.heads, C);
  if (r->qkv_map) B200_TRY(make_qkv_map(&r->tm_qkv, r->qkv, mb, T, C));
  B200_TRY(make_linear(al, &r->in_proj, 3 * C, C, true));
  B200_TRY(al.alloc(&r->cproj, (size_t)C * D));
  B200_TRY(al.alloc(&r->cproj_b, (size_t)D));
  B200_TRY(al.alloc(&r->pos, (size_t)T * C));
  return B200_OK;
}

// ---- loader ----------------------------------------------------------------------------------------------------

// scale = gamma / sqrt(var + 1e-5), shift = beta - mean * scale, in fp64 (eval-mode BatchNorm2d)
static int bn_fold(Loader& ld, const std::string& bn, size_t n, std::vector<double>& scale, std::vector<double>& shift) {
  const b200_tensor_view* g = ld.find(bn + ".weight", n);
  const b200_tensor_view* b = ld.find(bn + ".bias", n);
  const b200_tensor_view* m = ld.find(bn + ".running_mean", n);
  const b200_tensor_view* v = ld.find(bn + ".running_var", n);
  if (!g || !b || !m || !v) return B200_ERR_INVALID;
  scale.resize(n);
  shift.resize(n);
  for (size_t i = 0; i < n; i++) {
    scale[i] = (double)view_get(*g, i) / std::sqrt((double)view_get(*v, i) + 1e-5);
    shift[i] = (double)view_get(*b, i) - (double)view_get(*m, i) * scale[i];
  }
  return B200_OK;
}

// conv weight [cout, cin, k, k] with its BatchNorm folded -> l.w bf16 [cout, l.K] and l.b fp32 [cout].
// taps: the 3x3 implicit-GEMM packing, column (3 r + s) * C64 + c; otherwise the plain flattening c * k * k + r * k + s
// (1x1 convolutions, and the stem's gathered stride-2 convolution), columns past cin * k * k zero.
static int put_conv_bn(Loader& ld, const std::string& conv, const std::string& bn, Linear& l, int cout, int cin, int k,
                       bool taps) {
  const size_t kk = (size_t)k * k;
  const b200_tensor_view* wv = ld.find(conv + ".weight", (size_t)cout * cin * kk);
  if (!wv) return B200_ERR_INVALID;
  std::vector<double> scale, shift;
  B200_TRY(bn_fold(ld, bn, cout, scale, shift));
  const size_t K = l.K, c64 = (size_t)conv_cb(cin) * GEMM_BK;
  std::vector<uint16_t> w16((size_t)cout * K, 0);
  for (int o = 0; o < cout; o++)
    for (int c = 0; c < cin; c++)
      for (size_t t = 0; t < kk; t++) {
        const size_t col = taps ? t * c64 + c : c * kk + t;
        const double v = (double)view_get(*wv, ((size_t)o * cin + c) * kk + t) * scale[o];
        w16[(size_t)o * K + col] = f32_to_bf16_rn((float)v);
      }
  std::vector<float> b32(cout);
  for (int o = 0; o < cout; o++) b32[o] = (float)shift[o];
  B200_CUDA(cudaMemcpy(l.w, w16.data(), w16.size() * 2, cudaMemcpyHostToDevice));
  B200_CUDA(cudaMemcpy(l.b, b32.data(), b32.size() * 4, cudaMemcpyHostToDevice));
  return B200_OK;
}

int resnet_load(Loader& ld, ResNetTower& r) {
  const int w = r.w, C = r.C, D = r.D;
  B200_TRY(put_conv_bn(ld, "visual.conv1", "visual.bn1", r.stem1, w / 2, 3, 3, false));
  B200_TRY(put_conv_bn(ld, "visual.conv2", "visual.bn2", r.stem2, w / 2, w / 2, 3, true));
  B200_TRY(put_conv_bn(ld, "visual.conv3", "visual.bn3", r.stem3, w, w / 2, 3, true));
  size_t idx = 0;
  for (int s = 0; s < 4; s++)
    for (int j = 0; j < r.layers[s]; j++, idx++) {
      RnBlock& b = r.blocks[idx];
      const std::string p = "visual.layer" + std::to_string(s + 1) + "." + std::to_string(j) + ".";
      B200_TRY(put_conv_bn(ld, p + "conv1", p + "bn1", b.c1, b.planes, b.cin, 1, false));
      B200_TRY(put_conv_bn(ld, p + "conv2", p + "bn2", b.c2, b.planes, b.planes, 3, true));
      B200_TRY(put_conv_bn(ld, p + "conv3", p + "bn3", b.c3, 4 * b.planes, b.planes, 1, false));
      if (b.has_ds) B200_TRY(put_conv_bn(ld, p + "downsample.0", p + "downsample.1", b.ds, 4 * b.planes, b.cin, 1, false));
    }
  const std::string a = "visual.attnpool.";
  B200_TRY(ld.put_f32(a + "positional_embedding", r.pos, (size_t)r.T * C));
  const char* qkv[3] = {"q_proj", "k_proj", "v_proj"};
  for (int i = 0; i < 3; i++) {
    B200_TRY(ld.put_bf16(a + qkv[i] + ".weight", r.in_proj.w + (size_t)i * C * C, C, C, C));
    B200_TRY(ld.put_f32(a + qkv[i] + ".bias", r.in_proj.b + (size_t)i * C, C));
  }
  {
    const b200_tensor_view* v = ld.find(a + "c_proj.weight", (size_t)D * C);   // [D, C] -> [C, D]
    if (!v) return B200_ERR_INVALID;
    std::vector<uint16_t> t((size_t)C * D);
    for (int d = 0; d < D; d++)
      for (int c = 0; c < C; c++) t[(size_t)c * D + d] = f32_to_bf16_rn(view_get(*v, (size_t)d * C + c));
    B200_CUDA(cudaMemcpy(r.cproj, t.data(), t.size() * 2, cudaMemcpyHostToDevice));
  }
  B200_TRY(ld.put_f32(a + "c_proj.bias", r.cproj_b, (size_t)D));
  return B200_OK;
}

// ---- forward -------------------------------------------------------------------------------------------------------

static int conv3(const Linear& l, const CUtensorMap& tm_im2col, int B, int H, int cin, const GemmEpilogue& ep, int sms,
                 cudaStream_t st) {
  const int M = B * H * H;
  const int bn = conv_pick_bn(M, l.N, sms);
  GemmEpilogue e = ep;
  e.bias = l.b;
  ConvGeom cg;
  cg.H = H; cg.W = H; cg.cb = conv_cb(cin);
  const CUtensorMap& tmB = bn == 64 ? l.tm64 : (bn == 32 ? l.tm32 : l.tm128);
  return conv3x3_launch(tm_im2col, tmB, bn, M, l.N, cg, e, st);
}

static GemmEpilogue epi(__nv_bfloat16* out, int ld, int act, const __nv_bfloat16* res = nullptr) {
  GemmEpilogue e;
  e.out = out; e.out_ld = ld; e.act = act;
  e.residual = res; e.res_ld = ld;
  return e;
}

int resnet_encode(ResNetTower& r, SpanTimer& timer, int cls_gemm, int cls_attn, int cls_other, int sms, const float* px,
                  int B, float* feat, void* out, int out_f16, int normalize, cudaStream_t st) {
  const int w = r.w, g = r.S / 2;
  { TimedSpan sp(timer, cls_other, st, 1);
    B200_TRY(stem_gather(px, r.cols, B, r.S, GEMM_BK, st)); }
  { TimedSpan sp(timer, cls_gemm, st, 3);
    B200_TRY(linear_gemm(r.stem1, r.tm_cols, B * g * g, epi(r.t1, w / 2, ACT_RELU), sms, st));
    B200_TRY(conv3(r.stem2, r.tm_s1, B, g, w / 2, epi(r.t2, w / 2, ACT_RELU), sms, st));
    B200_TRY(conv3(r.stem3, r.tm_s2, B, g, w / 2, epi(r.buf[1], w, ACT_RELU), sms, st)); }
  { TimedSpan sp(timer, cls_other, st, 1);
    B200_TRY(avgpool_nhwc(r.buf[1], r.buf[0], B, g, g, w, 2, st)); }
  for (const RnBlock& b : r.blocks) {
    const int H = b.H, Ho = H / b.stride, p = b.planes;
    { TimedSpan sp(timer, cls_gemm, st, 2);
      B200_TRY(linear_gemm(b.c1, b.tm_x, B * H * H, epi(r.t1, p, ACT_RELU), sms, st));
      B200_TRY(conv3(b.c2, b.tm_t1, B, H, p, epi(r.t2, p, ACT_RELU), sms, st)); }
    if (b.stride > 1) {
      TimedSpan sp(timer, cls_other, st, 2);
      B200_TRY(avgpool_nhwc(r.t2, r.t3, B, H, H, p, b.stride, st));
      B200_TRY(avgpool_nhwc(b.x, r.xp, B, H, H, b.cin, b.stride, st));
    }
    { TimedSpan sp(timer, cls_gemm, st, b.has_ds ? 2 : 1);
      if (b.has_ds)
        B200_TRY(linear_gemm(b.ds, b.stride > 1 ? b.tm_xp : b.tm_x, B * Ho * Ho, epi(r.idn, 4 * p, ACT_NONE), sms, st));
      B200_TRY(linear_gemm(b.c3, b.tm_a3, B * Ho * Ho, epi(b.y, 4 * p, ACT_RELU, b.has_ds ? r.idn : b.x), sms, st)); }
  }
  // attention pool: tokens -> q, k, v of every token -> attention -> c_proj of token 0 -> normalise
  const int C = r.C, T = r.T;
  const __nv_bfloat16* fmap = r.blocks.back().y;
  { TimedSpan sp(timer, cls_other, st, 1);
    B200_TRY(attnpool_tokens(fmap, B, T - 1, C, r.pos, r.tok, st)); }
  { TimedSpan sp(timer, cls_gemm, st, 1);
    B200_TRY(linear_gemm(r.in_proj, r.tm_tok, B * T, epi(r.qkv, 3 * C, ACT_NONE), sms, st)); }
  { TimedSpan sp(timer, cls_attn, st, 1);
    B200_TRY(qkv_attention(r.qkv_map ? &r.tm_qkv : nullptr, r.qkv, r.att, B, T, r.heads, C, 0, st)); }
  { TimedSpan sp(timer, cls_other, st, 2);
    B200_TRY(pool_proj_bias_norm(r.att, T, C, r.cproj, r.cproj_b, r.D, feat, out, out_f16, normalize, B, st)); }
  return B200_OK;
}

}  // namespace b200
