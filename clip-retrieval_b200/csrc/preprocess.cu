// GPU image transform in front of the embed path (SURVEY §8(f) row 1).
//
// Replaces the CPU transform the reference runs per image in its DataLoader workers
// (`preprocess(PIL.Image)`, reference clip_retrieval/clip_inference/reader.py:98-106,158-165):
//   Resize(n_px, BICUBIC) -> CenterCrop(n_px) -> ToTensor -> Normalize(mean, std)
// bit for bit: Pillow's 8-bit resampler (double-precision Keys bicubic weights normalised and
// rounded to 22-bit fixed point, horizontal pass then vertical pass with a uint8 intermediate)
// followed by torchvision's float32 `/255`, `-mean`, `/std`.
//
// Three kernels per batch:
//   resize_coeff_kernel   one thread per (image, axis, output index inside the crop window):
//                         window bounds + fixed-point weights, IEEE double with explicit
//                         round-to-nearest intrinsics in Pillow's operation order (no FMA).
//   resize_h_kernel       horizontal pass over the input rows the vertical pass will touch, only
//                         for the n_px output columns that survive the crop -> uint8 [rows,n_px,3].
//   resize_v_norm_kernel  vertical pass + normalise -> float32 NCHW, coalesced along x.
// Work is O(rows · n_px · 3 · taps) integer MACs per image and the traffic is one read of the
// source pixels plus one write of the output: neither is near any roofline of the device; the
// point of the kernel is to take the resize off the host cores and to put the batch in HBM.
#include <vector>
#include <mutex>
#include <new>
#include <math.h>
#include <stdlib.h>
#include "common.cuh"

using namespace b200;

namespace {

constexpr int PRECISION_BITS = 32 - 8 - 2;   // Pillow Resample.c
constexpr int KSIZE_MAX = 1024;              // taps per output sample (scale up to ~255x)

struct ImgDesc {
  long long pix_off;    // byte offset of the image's first pixel in the packed buffer
  long long tmp_off;    // byte offset of its intermediate rows
  long long coef_off;   // int offset of its coefficient block: [axis][n_px][2 + ksize_axis]
  int h, w;             // source size
  int new_h, new_w;     // size after Resize
  int top, left;        // crop origin inside the resized image
  int ksize_h, ksize_v; // taps per sample of each pass (1 when the pass is the identity)
  int y0, rows;         // source rows [y0, y0+rows) the vertical pass reads
};

struct Axis {           // per-axis resampling parameters, computed identically on host and device
  double scale, filterscale, support;
  int ksize;
};

__host__ __device__ inline Axis axis_params(int in_size, int out_size) {
  Axis a;
  a.scale = (double)in_size / (double)out_size;
  a.filterscale = a.scale < 1.0 ? 1.0 : a.scale;
  a.support = 2.0 * a.filterscale;            // bicubic support 2.0
  a.ksize = (int)ceil(a.support) * 2 + 1;
  return a;
}

// Pillow `bicubic_filter`, a = -0.5, same association order, every op rounded separately.
__device__ __forceinline__ double bicubic_w(double x) {
  if (x < 0.0) x = -x;
  if (x < 1.0) {
    double t = __dmul_rn(1.5, x);
    t = __dsub_rn(t, 2.5);
    t = __dmul_rn(t, x);
    t = __dmul_rn(t, x);
    return __dadd_rn(t, 1.0);
  }
  if (x < 2.0) {
    double t = __dsub_rn(x, 5.0);
    t = __dmul_rn(t, x);
    t = __dadd_rn(t, 8.0);
    t = __dmul_rn(t, x);
    t = __dsub_rn(t, 4.0);
    return __dmul_rn(t, -0.5);
  }
  return 0.0;
}

// blockIdx.x = image, blockIdx.y = axis (0 horizontal, 1 vertical); thread = crop-window index.
__global__ void resize_coeff_kernel(const ImgDesc* __restrict__ descs, int* __restrict__ coefs, int n_px) {
  const ImgDesc d = descs[blockIdx.x];
  const int axis = blockIdx.y;
  const int in_size = axis ? d.h : d.w;
  const int out_size = axis ? d.new_h : d.new_w;
  const int first = axis ? d.top : d.left;
  const int ks = axis ? d.ksize_v : d.ksize_h;
  int* base = coefs + d.coef_off + (axis ? (long long)n_px * (2 + d.ksize_h) : 0);
  for (int j = threadIdx.x; j < n_px; j += blockDim.x) {
    int* row = base + (long long)j * (2 + ks);
    const int xx = first + j;
    if (in_size == out_size) {            // Pillow skips the pass: identity tap
      row[0] = xx; row[1] = 1; row[2] = 1 << PRECISION_BITS;
      continue;
    }
    const Axis a = axis_params(in_size, out_size);
    const double ss = __ddiv_rn(1.0, a.filterscale);
    const double center = __dmul_rn(__dadd_rn((double)xx, 0.5), a.scale);
    int xmin = __double2int_rz(__dadd_rn(__dsub_rn(center, a.support), 0.5));
    if (xmin < 0) xmin = 0;
    int xmax = __double2int_rz(__dadd_rn(__dadd_rn(center, a.support), 0.5));
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    if (xmax > ks) xmax = ks;   // the window never exceeds ks = 2*ceil(support)+1; bounds the store loop for the compiler
    double ww = 0.0;
    for (int x = 0; x < xmax; x++) {
      const double arg = __dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss);
      ww = __dadd_rn(ww, bicubic_w(arg));
    }
    for (int x = 0; x < xmax; x++) {
      const double arg = __dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss);
      double w = bicubic_w(arg);
      if (ww != 0.0) w = __ddiv_rn(w, ww);
      const double f = __dmul_rn(w, (double)(1 << PRECISION_BITS));
      row[2 + x] = w < 0.0 ? __double2int_rz(__dadd_rn(-0.5, f)) : __double2int_rz(__dadd_rn(0.5, f));
    }
    row[0] = xmin; row[1] = xmax;
  }
}

__device__ __forceinline__ int clip8(int acc) {
  acc >>= PRECISION_BITS;
  return acc < 0 ? 0 : (acc > 255 ? 255 : acc);
}

// grid (row blocks, images); block (256): thread = output column, ROWS_PER_BLOCK rows per block.
constexpr int H_ROWS_PER_BLOCK = 8;
__global__ void __launch_bounds__(256) resize_h_kernel(const uint8_t* __restrict__ pixels,
                                                       const ImgDesc* __restrict__ descs,
                                                       const int* __restrict__ coefs,
                                                       uint8_t* __restrict__ tmp, int n_px) {
  const ImgDesc d = descs[blockIdx.y];
  const int r0 = blockIdx.x * H_ROWS_PER_BLOCK;
  if (r0 >= d.rows) return;
  const int r1 = min(d.rows, r0 + H_ROWS_PER_BLOCK);
  const uint8_t* img = pixels + d.pix_off;
  uint8_t* out = tmp + d.tmp_off;
  for (int j = threadIdx.x; j < n_px; j += blockDim.x) {
    const int* row = coefs + d.coef_off + (long long)j * (2 + d.ksize_h);
    const int xmin = row[0], cnt = row[1];
    for (int r = r0; r < r1; r++) {
      const uint8_t* src = img + ((long long)(d.y0 + r) * d.w + xmin) * 3;
      int s0 = 1 << (PRECISION_BITS - 1), s1 = s0, s2 = s0;
      for (int x = 0; x < cnt; x++) {
        const int k = __ldg(row + 2 + x);
        s0 += (int)src[3 * x + 0] * k;
        s1 += (int)src[3 * x + 1] * k;
        s2 += (int)src[3 * x + 2] * k;
      }
      uint8_t* o = out + ((long long)r * n_px + j) * 3;
      o[0] = (uint8_t)clip8(s0); o[1] = (uint8_t)clip8(s1); o[2] = (uint8_t)clip8(s2);
    }
  }
}

// grid (n_px rows, images); thread = output column.
__global__ void __launch_bounds__(256) resize_v_norm_kernel(const ImgDesc* __restrict__ descs,
                                                            const int* __restrict__ coefs,
                                                            const uint8_t* __restrict__ tmp,
                                                            float* __restrict__ out, int n_px,
                                                            float m0, float m1, float m2,
                                                            float sd0, float sd1, float sd2) {
  const ImgDesc d = descs[blockIdx.y];
  const int i = blockIdx.x;
  const int* row = coefs + d.coef_off + (long long)n_px * (2 + d.ksize_h) + (long long)i * (2 + d.ksize_v);
  const int ymin = row[0] - d.y0, cnt = row[1];
  const uint8_t* src = tmp + d.tmp_off;
  float* o = out + (long long)blockIdx.y * 3 * n_px * n_px + (long long)i * n_px;
  for (int j = threadIdx.x; j < n_px; j += blockDim.x) {
    int s0 = 1 << (PRECISION_BITS - 1), s1 = s0, s2 = s0;
    for (int y = 0; y < cnt; y++) {
      const int k = __ldg(row + 2 + y);
      const uint8_t* p = src + ((long long)(ymin + y) * n_px + j) * 3;
      s0 += (int)p[0] * k;
      s1 += (int)p[1] * k;
      s2 += (int)p[2] * k;
    }
    // torchvision to_tensor + normalize: float32 divide, subtract, divide — no contraction.
    const float v0 = __fdiv_rn((float)clip8(s0), 255.0f);
    const float v1 = __fdiv_rn((float)clip8(s1), 255.0f);
    const float v2 = __fdiv_rn((float)clip8(s2), 255.0f);
    o[j] = __fdiv_rn(__fsub_rn(v0, m0), sd0);
    o[(long long)n_px * n_px + j] = __fdiv_rn(__fsub_rn(v1, m1), sd1);
    o[2ll * n_px * n_px + j] = __fdiv_rn(__fsub_rn(v2, m2), sd2);
  }
}

}  // namespace

struct b200_preproc {
  int device = 0, n_px = 224;
  int resize_mode = B200_RESIZE_SHORTEST;
  float mean[3], stdv[3];
  std::mutex mu;                       // one batch at a time per handle (workspaces are shared)
  void* ws[4] = {nullptr, nullptr, nullptr, nullptr};   // descs, coefs, tmp, staged pixels
  size_t ws_bytes[4] = {0, 0, 0, 0};
  std::vector<ImgDesc> host_descs;
};

static int ws_reserve(b200_preproc* p, int slot, size_t bytes) {
  if (bytes <= p->ws_bytes[slot]) return B200_OK;
  if (p->ws[slot]) { B200_CUDA(cudaDeviceSynchronize()); B200_CUDA(cudaFree(p->ws[slot])); }
  p->ws[slot] = nullptr; p->ws_bytes[slot] = 0;
  const size_t want = bytes + bytes / 4;
  B200_CUDA(cudaMalloc(&p->ws[slot], want));
  p->ws_bytes[slot] = want;
  return B200_OK;
}

// torchvision `_compute_resized_output_size` (int size) and `center_crop` (Python round: half to even).
static void resized_shape(int h, int w, int n_px, int* new_h, int* new_w) {
  const int shrt = w <= h ? w : h, lng = w <= h ? h : w;
  const int new_long = (int)((double)((long long)n_px * lng) / (double)shrt);
  if (w <= h) { *new_w = n_px; *new_h = new_long; }
  else { *new_h = n_px; *new_w = new_long; }
}
static int crop_origin(int new_size, int n_px) { return (int)nearbyint((double)(new_size - n_px) / 2.0); }

extern "C" {

int b200_preproc_create(int n_px, const float* mean3, const float* std3, int device, b200_preproc** out) {
  return b200_preproc_create_mode(n_px, mean3, std3, B200_RESIZE_SHORTEST, device, out);
}

int b200_preproc_create_mode(int n_px, const float* mean3, const float* std3, int resize_mode, int device,
                             b200_preproc** out) {
  B200_CHECK(out && mean3 && std3, B200_ERR_INVALID, "preproc_create: null argument");
  B200_CHECK(resize_mode == B200_RESIZE_SHORTEST || resize_mode == B200_RESIZE_SQUASH, B200_ERR_INVALID,
             "preproc_create: resize mode %d (0 shortest side + centre crop, 1 squash)", resize_mode);
  B200_CHECK(n_px >= 1 && n_px <= 4096, B200_ERR_INVALID, "preproc_create: n_px %d out of range", n_px);
  int ndev = 0;
  B200_CUDA(cudaGetDeviceCount(&ndev));
  B200_CHECK(device >= 0 && device < ndev, B200_ERR_INVALID, "preproc_create: device %d of %d", device, ndev);
  b200_preproc* p = new (std::nothrow) b200_preproc();
  B200_CHECK(p != nullptr, B200_ERR_OOM, "preproc_create: host allocation failed");
  p->device = device; p->n_px = n_px; p->resize_mode = resize_mode;
  for (int c = 0; c < 3; c++) { p->mean[c] = mean3[c]; p->stdv[c] = std3[c]; }
  *out = p;
  return B200_OK;
}

int b200_preproc_destroy(b200_preproc* p) {
  if (!p) return B200_OK;
  DeviceGuard g(p->device);
  cudaDeviceSynchronize();
  for (void* w : p->ws) if (w) cudaFree(w);
  delete p;
  return B200_OK;
}

int b200_preproc_run(b200_preproc* p, const uint8_t* pixels, int pixels_on_device, const int64_t* h_offsets,
                     const int32_t* h_heights, const int32_t* h_widths, int n, float* d_out, void* stream) {
  B200_CHECK(p && h_offsets && h_heights && h_widths && (pixels || n == 0) && (d_out || n == 0), B200_ERR_INVALID,
             "preproc_run: null argument");
  B200_CHECK(n >= 0 && n <= 65535, B200_ERR_INVALID, "preproc_run: n=%d (0..65535 images per call)", n);
  if (n == 0) return B200_OK;
  std::lock_guard<std::mutex> lock(p->mu);
  DeviceGuard g(p->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int n_px = p->n_px;
  p->host_descs.resize(n);
  long long tmp_total = 0, coef_total = 0, pix_end = 0;
  int max_rows = 0;
  for (int i = 0; i < n; i++) {
    ImgDesc& d = p->host_descs[i];
    d.h = h_heights[i]; d.w = h_widths[i]; d.pix_off = h_offsets[i];
    B200_CHECK(d.h >= 1 && d.w >= 1 && d.h <= 65536 && d.w <= 65536 && d.pix_off >= 0, B200_ERR_INVALID,
               "preproc_run: image %d has size %dx%d offset %lld", i, d.h, d.w, (long long)d.pix_off);
    if (p->resize_mode == B200_RESIZE_SQUASH) {   // Resize((n_px, n_px)): both sides to n_px, nothing cropped
      d.new_h = d.new_w = n_px;
      d.top = d.left = 0;
    } else {
      resized_shape(d.h, d.w, n_px, &d.new_h, &d.new_w);
      d.top = crop_origin(d.new_h, n_px); d.left = crop_origin(d.new_w, n_px);
    }
    const Axis ah = axis_params(d.w, d.new_w), av = axis_params(d.h, d.new_h);
    d.ksize_h = d.w == d.new_w ? 1 : ah.ksize;
    d.ksize_v = d.h == d.new_h ? 1 : av.ksize;
    B200_CHECK(d.ksize_h <= KSIZE_MAX && d.ksize_v <= KSIZE_MAX, B200_ERR_UNSUPPORTED,
               "preproc_run: image %d (%dx%d) needs %d taps per sample (max %d)", i, d.h, d.w,
               d.ksize_h > d.ksize_v ? d.ksize_h : d.ksize_v, KSIZE_MAX);
    if (d.h == d.new_h) { d.y0 = d.top; d.rows = n_px; }
    else {   // rows [ymin(first crop row), ymax(last crop row)) — same doubles as the device computes
      const double c0 = ((double)d.top + 0.5) * av.scale, c1 = ((double)(d.top + n_px - 1) + 0.5) * av.scale;
      int y0 = (int)(c0 - av.support + 0.5); if (y0 < 0) y0 = 0;
      int y1 = (int)(c1 + av.support + 0.5); if (y1 > d.h) y1 = d.h;
      y0 = y0 > 0 ? y0 - 1 : 0; y1 = y1 < d.h ? y1 + 1 : d.h;   // one row of slack either side
      d.y0 = y0; d.rows = y1 - y0;
    }
    d.tmp_off = tmp_total; tmp_total += (long long)d.rows * n_px * 3;
    d.coef_off = coef_total; coef_total += (long long)n_px * (4 + d.ksize_h + d.ksize_v);
    if (d.rows > max_rows) max_rows = d.rows;
    const long long e = d.pix_off + (long long)d.h * d.w * 3;
    if (e > pix_end) pix_end = e;
  }
  B200_CHECK(tmp_total <= (16ll << 30), B200_ERR_UNSUPPORTED,
             "preproc_run: batch needs %.1f GB of intermediate rows; split the batch", tmp_total / 1e9);
  B200_TRY(ws_reserve(p, 0, sizeof(ImgDesc) * (size_t)n));
  B200_TRY(ws_reserve(p, 1, sizeof(int) * (size_t)coef_total));
  B200_TRY(ws_reserve(p, 2, (size_t)tmp_total));
  const uint8_t* d_pix = pixels;
  if (!pixels_on_device) {
    B200_TRY(ws_reserve(p, 3, (size_t)pix_end));
    B200_CUDA(cudaMemcpyAsync(p->ws[3], pixels, (size_t)pix_end, cudaMemcpyHostToDevice, st));
    d_pix = (const uint8_t*)p->ws[3];
  }
  B200_CUDA(cudaMemcpyAsync(p->ws[0], p->host_descs.data(), sizeof(ImgDesc) * (size_t)n, cudaMemcpyHostToDevice, st));
  const ImgDesc* dd = (const ImgDesc*)p->ws[0];
  int* dc = (int*)p->ws[1];
  uint8_t* dt = (uint8_t*)p->ws[2];
  if (getenv("B200_PREPROC_DEBUG")) {
    const ImgDesc& d = p->host_descs[0];
    fprintf(stderr, "preproc: n=%d descs=%p coefs=%p (%zu B) tmp=%p (%zu B) pix=%p coef_total=%lld tmp_total=%lld\n"
            "  img0 %dx%d -> %dx%d crop (%d,%d) ks %d/%d rows [%d,+%d) offs pix %lld tmp %lld coef %lld sizeof(desc)=%zu\n",
            n, (void*)dd, (void*)dc, p->ws_bytes[1], (void*)dt, p->ws_bytes[2], (const void*)d_pix, coef_total, tmp_total,
            d.h, d.w, d.new_h, d.new_w, d.top, d.left, d.ksize_h, d.ksize_v, d.y0, d.rows, d.pix_off, d.tmp_off, d.coef_off,
            sizeof(ImgDesc));
  }
  resize_coeff_kernel<<<dim3(n, 2), 256, 0, st>>>(dd, dc, n_px);
  B200_LAUNCH_OK();
  resize_h_kernel<<<dim3((max_rows + H_ROWS_PER_BLOCK - 1) / H_ROWS_PER_BLOCK, n), 256, 0, st>>>(d_pix, dd, dc, dt, n_px);
  B200_LAUNCH_OK();
  resize_v_norm_kernel<<<dim3(n_px, n), 256, 0, st>>>(dd, dc, dt, d_out, n_px, p->mean[0], p->mean[1], p->mean[2],
                                                       p->stdv[0], p->stdv[1], p->stdv[2]);
  B200_LAUNCH_OK();
  // host_descs / pageable source pixels are read by the async copies above
  B200_CUDA(cudaStreamSynchronize(st));
  return B200_OK;
}

}  // extern "C"
