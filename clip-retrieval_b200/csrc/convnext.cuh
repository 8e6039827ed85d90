// The ConvNeXt image tower of open_clip's convnext_* CLIPs (timm's ConvNeXt trunk + open_clip's linear or MLP head),
// inside the b200_clip handle (clip_model.cu) beside the shared text tower.  convnext.cu; the kernels are in dwconv.cu.
//
// Activations are NHWC bf16 [B * H * W, C] rows.  Stem: the 4x4 stride-4 patch GEMM (im2col_patches) with its bias,
// then LayerNorm.  A block: dwconv7_ln (depthwise 7x7 + bias + LayerNorm, fused) -> fc1 GEMM with erf GELU -> fc2 GEMM
// whose residual epilogue adds the block input in place; the layer scale gamma is folded into fc2's rows and bias at load
// time (fp64).  A downsample: ln_s2d (LayerNorm + 2x2 space-to-depth) -> one GEMM with bias.  Head: fp32 spatial mean +
// LayerNorm, then the projection (or MLP) in fp32.  Every buffer and tensor map is built once for max_batch.
#pragma once
#include "layers.cuh"
#include "weights.cuh"
#include <vector>

namespace b200 {

struct CnxBlock {
  float *dw = nullptr, *dw_b = nullptr;    // depthwise weight fp32 [49, C] (tap-major), bias [C]
  float *ln_g = nullptr, *ln_b = nullptr;  // the block's LayerNorm
  Linear fc1, fc2;                         // [4C, C] + bias, [C, 4C] + bias with gamma folded in
};

struct CnxStage {
  int C = 0, H = 0, depth = 0;             // width, spatial size (square) and blocks
  float *ds_g = nullptr, *ds_b = nullptr;  // the downsample's LayerNorm over the previous stage's width (s > 0)
  Linear ds;                               // [C, 4 C_prev] + bias, columns (2 i + j) C_prev + c (s > 0)
  CUtensorMap tm_ds;                       // A of ds: ln_s2d's output [mb * H^2, 4 C_prev] (s > 0)
  CUtensorMap tm_h, tm_f;                  // A of fc1 [mb * H^2, C] and of fc2 [mb * H^2, 4C]
  std::vector<CnxBlock> blocks;
};

struct ConvNeXtTower {
  int S = 0, D = 0, mb = 0, head_mlp = 0;
  float eps = 1e-6f;
  CnxStage st[4];
  Linear stem;                             // [C0, 64] + bias (columns 48..63 zero)
  float *stem_g = nullptr, *stem_b = nullptr;
  float *head_g = nullptr, *head_b = nullptr;
  float *w1T = nullptr, *b1 = nullptr;     // MLP head: fc1 transposed [C3, 2D] + bias (null for the linear head)
  float* w2T = nullptr;                    // [C3, D] (linear) or [2D, D] (MLP)
  __nv_bfloat16 *cols = nullptr, *x = nullptr, *h = nullptr, *f = nullptr;
  float *pooled = nullptr, *hid = nullptr;
  CUtensorMap tm_cols;
};

// Allocates every weight and buffer of the tower for max_batch samples of image_size px (a multiple of 32).
int convnext_create(DeviceAllocs& al, ConvNeXtTower* t, const b200_convnext_config& cc, int image_size, int D,
                    int max_batch);
// visual.trunk.* and visual.head.* tensors of open_clip's state_dict; a missing or mis-shaped one is B200_ERR_INVALID
// naming it.
int convnext_load(Loader& ld, ConvNeXtTower& t);
// Pixels fp32 NCHW [B, 3, S, S] (B <= mb) -> feat fp32 [B, D] and out (normalised, fp16 / fp32).  Time classes: the
// GEMMs `gemm`, the rest (im2col, LayerNorms, dwconv7_ln, ln_s2d, head) `other`.
int convnext_encode(ConvNeXtTower& t, SpanTimer& timer, int cls_gemm, int cls_other, int sms, const float* px, int B,
                    float* feat, void* out, int out_f16, int normalize, cudaStream_t st);

}  // namespace b200
