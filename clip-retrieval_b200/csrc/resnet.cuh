// The ResNet image tower of OpenAI's RN50 / RN101 / RN50x4 / RN50x16 / RN50x64 CLIPs (ModifiedResNet), inside the
// b200_clip handle (clip_model.cu) beside the shared text tower.  resnet.cu; the kernels are in conv.cu.
//
// Activations are NHWC bf16 [B * H * W, C] rows throughout: a 1x1 convolution is the GEMM of those rows, a 3x3 one the
// implicit GEMM of conv.cu, every BatchNorm is folded into its convolution at load time (fp64, eps 1e-5), and ReLU
// (after the residual add) runs in the GEMM epilogue.  Every buffer and tensor map is built once for max_batch.
#pragma once
#include "layers.cuh"
#include "weights.cuh"
#include <vector>

namespace b200 {

// One Bottleneck block: conv1 1x1 -> relu -> conv2 3x3 -> relu -> [AvgPool(stride)] -> conv3 1x1, + identity, relu.
// The identity is the input, or downsample = [AvgPool(stride)] -> 1x1 conv (-> BN, folded) when stride > 1 or
// cin != 4 planes.
struct RnBlock {
  int cin = 0, planes = 0, stride = 1, H = 0;   // H: the input's spatial size (square)
  bool has_ds = false;
  Linear c1, c2, c3, ds;                        // c2: [planes, 9 * cb * 64], tap-major (conv.cu)
  __nv_bfloat16 *x = nullptr, *y = nullptr;     // block input and output (the tower's two ping-pong buffers)
  CUtensorMap tm_x;    // A of c1 (and of ds at stride 1): x [mb * H^2, cin]
  CUtensorMap tm_t1;   // im2col over c1's output [mb, H, H, planes]
  CUtensorMap tm_a3;   // A of c3: c2's output, pooled at stride 2 [mb * Ho^2, planes]
  CUtensorMap tm_xp;   // A of ds at stride 2: the pooled input [mb * Ho^2, cin]
};

struct ResNetTower {
  int layers[4] = {0, 0, 0, 0};
  int w = 0, heads = 0, S = 0, C = 0, T = 0, D = 0, mb = 0;   // C = 32 w: the attention pool's width
  Linear stem1, stem2, stem3;   // stem1 on the gathered patch matrix [.., 64]; stem2 / stem3 implicit 3x3
  std::vector<RnBlock> blocks;
  __nv_bfloat16 *cols = nullptr, *buf[2] = {nullptr, nullptr}, *t1 = nullptr, *t2 = nullptr, *t3 = nullptr,
                *xp = nullptr, *idn = nullptr, *tok = nullptr, *qkv = nullptr, *att = nullptr;
  CUtensorMap tm_cols, tm_s1, tm_s2, tm_tok, tm_qkv;
  bool qkv_map = false;         // tm_qkv built (the wgmma attention takes the shape)
  Linear in_proj;               // cat(q, k, v) [3C, C] + bias
  __nv_bfloat16* cproj = nullptr;   // c_proj transposed [C, D]
  float* cproj_b = nullptr;
  float* pos = nullptr;             // attention-pool positional embedding [T, C]
};

// Allocates every weight and buffer of the tower for max_batch samples of image_size px (a multiple of 32).
int resnet_create(DeviceAllocs& al, ResNetTower* r, const b200_resnet_config& rc, int image_size, int D, int max_batch);
// visual.* tensors of the OpenAI / open_clip state_dict; each BatchNorm's weight, bias and running statistics are
// folded into its convolution here.  num_batches_tracked is never looked up.
int resnet_load(Loader& ld, ResNetTower& r);
// Pixels fp32 NCHW [B, 3, S, S] (B <= mb) -> feat fp32 [B, D] and out (normalised, fp16 / fp32).  Time classes: the
// convolutions and GEMMs `gemm`, the attention `attention`, the rest `other`.
int resnet_encode(ResNetTower& r, SpanTimer& timer, int cls_gemm, int cls_attn, int cls_other, int sms, const float* px,
                  int B, float* feat, void* out, int out_f16, int normalize, cudaStream_t st);

}  // namespace b200
