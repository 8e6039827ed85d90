// The ConvNeXt image tower (convnext.cuh): buffers, the loader that packs open_clip's timm-trunk tensors, and the forward.
#include "convnext.cuh"
#include <algorithm>
#include <string>

namespace b200 {

int convnext_create(DeviceAllocs& al, ConvNeXtTower* t, const b200_convnext_config& cc, int S, int D, int mb) {
  B200_CHECK(S >= 32 && S % 32 == 0 && D >= 8 && D % 8 == 0 && cc.eps > 0.f, B200_ERR_INVALID,
             "convnext: image_size a multiple of 32, embed_dim a multiple of 8, eps > 0 (S=%d D=%d)", S, D);
  for (int s = 0; s < 4; s++)
    B200_CHECK(cc.depths[s] >= 1 && cc.dims[s] >= 64 && cc.dims[s] % 64 == 0 && cc.dims[s] <= 3072 &&
                   (s == 3 || cc.dims[s] <= 1536) && (s > 0 || cc.dims[0] <= 2048),
               B200_ERR_INVALID, "convnext: stage %d depth %d width %d (widths multiples of 64, <= 1536 before the last "
               "stage, <= 3072)", s, cc.depths[s], cc.dims[s]);
  t->S = S; t->D = D; t->mb = mb; t->eps = cc.eps; t->head_mlp = cc.head_mlp ? 1 : 0;
  const size_t B = (size_t)mb;
  const int g = S / 4;
  // buffer sizes, walking the stages: x and h hold one activation map (stage 0's B g^2 C0 is the largest, each stage
  // halving it, and ln_s2d's output is the size of its input), f the 4C hidden
  size_t n_x = 0, n_f = 0;
  for (int s = 0; s < 4; s++) {
    const size_t H = (size_t)(g >> s);
    n_x = std::max(n_x, B * H * H * cc.dims[s]);
    if (s > 0) n_x = std::max(n_x, B * H * H * 4 * cc.dims[s - 1]);
    n_f = std::max(n_f, B * H * H * 4 * cc.dims[s]);
  }
  const size_t prow = B * g * g;
  B200_TRY(al.alloc(&t->cols, prow * GEMM_BK));
  B200_CUDA(cudaMemset(t->cols, 0, prow * GEMM_BK * 2));   // im2col_patches never writes columns 48..63
  B200_TRY(al.alloc(&t->x, n_x));
  B200_TRY(al.alloc(&t->h, n_x));
  B200_TRY(al.alloc(&t->f, n_f));
  B200_TRY(make_tmap_2d(&t->tm_cols, t->cols, 1, prow, GEMM_BK, GEMM_BK, GEMM_BM, GEMM_BK));
  const int C0 = cc.dims[0];
  B200_TRY(make_linear(al, &t->stem, C0, GEMM_BK, true));
  B200_TRY(al.alloc(&t->stem_g, (size_t)C0));
  B200_TRY(al.alloc(&t->stem_b, (size_t)C0));
  for (int s = 0; s < 4; s++) {
    CnxStage& sg = t->st[s];
    sg.C = cc.dims[s]; sg.H = g >> s; sg.depth = cc.depths[s];
    const int C = sg.C;
    const size_t rows = B * sg.H * sg.H;
    if (s > 0) {
      const int Cp = cc.dims[s - 1];
      B200_TRY(al.alloc(&sg.ds_g, (size_t)Cp));
      B200_TRY(al.alloc(&sg.ds_b, (size_t)Cp));
      B200_TRY(make_linear(al, &sg.ds, C, 4 * Cp, true));
      B200_TRY(make_tmap_2d(&sg.tm_ds, t->h, 1, rows, 4 * Cp, 4 * Cp, GEMM_BM, GEMM_BK));
    }
    B200_TRY(make_tmap_2d(&sg.tm_h, t->h, 1, rows, C, C, GEMM_BM, GEMM_BK));
    B200_TRY(make_tmap_2d(&sg.tm_f, t->f, 1, rows, 4 * C, 4 * C, GEMM_BM, GEMM_BK));
    sg.blocks.resize(sg.depth);
    for (CnxBlock& b : sg.blocks) {
      B200_TRY(al.alloc(&b.dw, (size_t)49 * C));
      B200_TRY(al.alloc(&b.dw_b, (size_t)C));
      B200_TRY(al.alloc(&b.ln_g, (size_t)C));
      B200_TRY(al.alloc(&b.ln_b, (size_t)C));
      B200_TRY(make_linear(al, &b.fc1, 4 * C, C, true));
      B200_TRY(make_linear(al, &b.fc2, C, 4 * C, true));
    }
  }
  const int C3 = cc.dims[3];
  B200_TRY(al.alloc(&t->head_g, (size_t)C3));
  B200_TRY(al.alloc(&t->head_b, (size_t)C3));
  if (t->head_mlp) {
    B200_TRY(al.alloc(&t->w1T, (size_t)C3 * 2 * D));
    B200_TRY(al.alloc(&t->b1, (size_t)2 * D));
    B200_TRY(al.alloc(&t->w2T, (size_t)2 * D * D));
    B200_TRY(al.alloc(&t->hid, B * 2 * D));
  } else {
    B200_TRY(al.alloc(&t->w2T, (size_t)C3 * D));
  }
  B200_TRY(al.alloc(&t->pooled, B * C3));
  return B200_OK;
}

// ---- loader ----------------------------------------------------------------------------------------------------

// A [n_out, n_in] nn.Linear weight transposed into fp32 [n_in, n_out] (the head's fp32 projection layout).
static int put_f32_t(Loader& ld, const std::string& name, float* dst, size_t n_out, size_t n_in) {
  const b200_tensor_view* v = ld.find(name, n_out * n_in);
  if (!v) return B200_ERR_INVALID;
  std::vector<float> t(n_out * n_in);
  for (size_t o = 0; o < n_out; o++)
    for (size_t i = 0; i < n_in; i++) t[i * n_out + o] = view_get(*v, o * n_in + i);
  B200_CUDA(cudaMemcpy(dst, t.data(), t.size() * 4, cudaMemcpyHostToDevice));
  return B200_OK;
}

// conv_dw.weight [C, 1, 7, 7] -> fp32 [49, C], row 7 r + s.
static int put_dw(Loader& ld, const std::string& name, float* dst, size_t C) {
  const b200_tensor_view* v = ld.find(name, C * 49);
  if (!v) return B200_ERR_INVALID;
  std::vector<float> t(C * 49);
  for (size_t c = 0; c < C; c++)
    for (size_t k = 0; k < 49; k++) t[k * C + c] = view_get(*v, c * 49 + k);
  B200_CUDA(cudaMemcpy(dst, t.data(), t.size() * 4, cudaMemcpyHostToDevice));
  return B200_OK;
}

// downsample.1.weight [Cout, Cin, 2, 2] -> bf16 [Cout, 4 Cin], column (2 i + j) Cin + c: ln_s2d's column order.
static int put_s2d(Loader& ld, const std::string& name, Linear& l, size_t cout, size_t cin) {
  const b200_tensor_view* v = ld.find(name, cout * cin * 4);
  if (!v) return B200_ERR_INVALID;
  std::vector<uint16_t> t(cout * 4 * cin);
  for (size_t o = 0; o < cout; o++)
    for (size_t c = 0; c < cin; c++)
      for (size_t k = 0; k < 4; k++) t[o * 4 * cin + k * cin + c] = f32_to_bf16_rn(view_get(*v, (o * cin + c) * 4 + k));
  B200_CUDA(cudaMemcpy(l.w, t.data(), t.size() * 2, cudaMemcpyHostToDevice));
  return B200_OK;
}

// mlp.fc2 with the layer scale folded, in fp64 before the bf16 round: W2' = diag(gamma) W2, b2' = gamma * b2.
static int put_fc2_gamma(Loader& ld, const std::string& p, Linear& l, size_t C) {
  const b200_tensor_view* w = ld.find(p + "mlp.fc2.weight", C * 4 * C);
  const b200_tensor_view* b = ld.find(p + "mlp.fc2.bias", C);
  const b200_tensor_view* g = ld.find(p + "gamma", C);
  if (!w || !b || !g) return B200_ERR_INVALID;
  std::vector<uint16_t> t(C * 4 * C);
  std::vector<float> bb(C);
  for (size_t o = 0; o < C; o++) {
    const double go = view_get(*g, o);
    for (size_t i = 0; i < 4 * C; i++) t[o * 4 * C + i] = f32_to_bf16_rn((float)(go * (double)view_get(*w, o * 4 * C + i)));
    bb[o] = (float)(go * (double)view_get(*b, o));
  }
  B200_CUDA(cudaMemcpy(l.w, t.data(), t.size() * 2, cudaMemcpyHostToDevice));
  B200_CUDA(cudaMemcpy(l.b, bb.data(), C * 4, cudaMemcpyHostToDevice));
  return B200_OK;
}

int convnext_load(Loader& ld, ConvNeXtTower& t) {
  const std::string v = "visual.trunk.";
  const size_t C0 = t.st[0].C, D = t.D;
  B200_TRY(ld.put_bf16(v + "stem.0.weight", t.stem.w, C0, 48, GEMM_BK));
  B200_TRY(ld.put_f32(v + "stem.0.bias", t.stem.b, C0));
  B200_TRY(ld.put_f32(v + "stem.1.weight", t.stem_g, C0));
  B200_TRY(ld.put_f32(v + "stem.1.bias", t.stem_b, C0));
  for (int s = 0; s < 4; s++) {
    CnxStage& sg = t.st[s];
    const size_t C = sg.C;
    const std::string sp = v + "stages." + std::to_string(s) + ".";
    if (s > 0) {
      const size_t Cp = t.st[s - 1].C;
      B200_TRY(ld.put_f32(sp + "downsample.0.weight", sg.ds_g, Cp));
      B200_TRY(ld.put_f32(sp + "downsample.0.bias", sg.ds_b, Cp));
      B200_TRY(put_s2d(ld, sp + "downsample.1.weight", sg.ds, C, Cp));
      B200_TRY(ld.put_f32(sp + "downsample.1.bias", sg.ds.b, C));
    }
    for (int j = 0; j < sg.depth; j++) {
      CnxBlock& b = sg.blocks[j];
      const std::string p = sp + "blocks." + std::to_string(j) + ".";
      B200_TRY(put_dw(ld, p + "conv_dw.weight", b.dw, C));
      B200_TRY(ld.put_f32(p + "conv_dw.bias", b.dw_b, C));
      B200_TRY(ld.put_f32(p + "norm.weight", b.ln_g, C));
      B200_TRY(ld.put_f32(p + "norm.bias", b.ln_b, C));
      B200_TRY(ld.put_bf16(p + "mlp.fc1.weight", b.fc1.w, 4 * C, C, C));
      B200_TRY(ld.put_f32(p + "mlp.fc1.bias", b.fc1.b, 4 * C));
      B200_TRY(put_fc2_gamma(ld, p, b.fc2, C));
    }
  }
  const size_t C3 = t.st[3].C;
  B200_TRY(ld.put_f32(v + "head.norm.weight", t.head_g, C3));
  B200_TRY(ld.put_f32(v + "head.norm.bias", t.head_b, C3));
  if (t.head_mlp) {
    B200_TRY(put_f32_t(ld, "visual.head.mlp.fc1.weight", t.w1T, 2 * D, C3));
    B200_TRY(ld.put_f32("visual.head.mlp.fc1.bias", t.b1, 2 * D));
    B200_TRY(put_f32_t(ld, "visual.head.mlp.fc2.weight", t.w2T, D, 2 * D));
  } else {
    B200_TRY(put_f32_t(ld, "visual.head.proj.weight", t.w2T, D, C3));
  }
  return B200_OK;
}

// ---- forward -------------------------------------------------------------------------------------------------------

static GemmEpilogue cnx_epi(__nv_bfloat16* out, int ld, int act, const __nv_bfloat16* res = nullptr) {
  GemmEpilogue e;
  e.out = out; e.out_ld = ld; e.act = act;
  e.residual = res; e.res_ld = ld;
  return e;
}

int convnext_encode(ConvNeXtTower& t, SpanTimer& timer, int cls_gemm, int cls_other, int sms, const float* px, int B,
                    float* feat, void* out, int out_f16, int normalize, cudaStream_t st) {
  const int g = t.S / 4, C0 = t.st[0].C;
  { TimedSpan sp(timer, cls_other, st, 1);
    B200_TRY(im2col_patches(px, t.cols, B, t.S, 4, GEMM_BK, st)); }
  { TimedSpan sp(timer, cls_gemm, st, 1);
    B200_TRY(linear_gemm(t.stem, t.tm_cols, B * g * g, cnx_epi(t.x, C0, ACT_NONE), sms, st)); }
  { TimedSpan sp(timer, cls_other, st, 1);
    B200_TRY(layernorm_rows_eps(t.x, C0, t.x, C0, t.stem_g, t.stem_b, (int64_t)B * g * g, C0, t.eps, st)); }
  for (int s = 0; s < 4; s++) {
    CnxStage& sg = t.st[s];
    const int C = sg.C, H = sg.H, M = B * H * H;
    if (s > 0) {
      const int Cp = t.st[s - 1].C;
      { TimedSpan sp(timer, cls_other, st, 1);
        B200_TRY(ln_s2d(t.x, sg.ds_g, sg.ds_b, t.eps, t.h, B, 2 * H, 2 * H, Cp, st)); }
      TimedSpan sp(timer, cls_gemm, st, 1);
      B200_TRY(linear_gemm(sg.ds, sg.tm_ds, M, cnx_epi(t.x, C, ACT_NONE), sms, st));
    }
    for (const CnxBlock& b : sg.blocks) {
      { TimedSpan sp(timer, cls_other, st, 1);
        B200_TRY(dwconv7_ln(t.x, b.dw, b.dw_b, b.ln_g, b.ln_b, t.eps, t.h, B, H, H, C, st)); }
      TimedSpan sp(timer, cls_gemm, st, 2);
      B200_TRY(linear_gemm(b.fc1, sg.tm_h, M, cnx_epi(t.f, 4 * C, ACT_GELU), sms, st));
      B200_TRY(linear_gemm(b.fc2, sg.tm_f, M, cnx_epi(t.x, C, ACT_NONE, t.x), sms, st));
    }
  }
  const CnxStage& last = t.st[3];
  TimedSpan sp(timer, cls_other, st, t.head_mlp ? 4 : 3);
  B200_TRY(mean_ln_rows(t.x, B, last.H * last.H, last.C, t.head_g, t.head_b, t.eps, t.pooled, st));
  return rows_head_norm(t.pooled, last.C, t.head_mlp ? t.w1T : nullptr, t.b1, 2 * t.D, t.w2T, t.D, t.hid, feat, out,
                        out_f16, normalize, B, st);
}

}  // namespace b200
