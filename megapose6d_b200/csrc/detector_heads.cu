// The RoI heads of torchvision's Mask R-CNN (torchvision.models.detection.roi_heads.RoIHeads, eval mode) on the engine:
// the box branch (MultiScaleRoIAlign 7x7, TwoMLPHead, FastRCNNPredictor) and the mask branch (MultiScaleRoIAlign 14x14,
// MaskRCNNHeads, MaskRCNNPredictor).  Every matrix product is the wgmma convolution of conv_wgmma.cu (act16 operands,
// fp32 accumulation, bias and ReLU in the epilogue, one rounding per layer):
//   fc6                 the 7x7 convolution of the [P, 7, 7, 256] pooled map (1x1 output), 256 * 49 -> hidden
//   fc7                 1x1 on the [P, 1, 1, hidden] map
//   predictor           cls_score | bbox_pred merged into one 1x1, zero rows up to a multiple of 64
//   mask_head           four 3x3 convolutions, 256 channels, ReLU
//   conv5_mask          the 2x2/s2 ConvTranspose2d as a 1x1 convolution 256 -> 4 x 256, channel (dy * 2 + dx) * 256 + c;
//                       the taps of a stride-2 2x2 deconvolution do not overlap, so the output pixel (2y + dy, 2x + dx)
//                       is exactly channel group (dy, dx) of input pixel (y, x)
//   mask_fcn_logits     1x1 over the [N, S, 4S, 256] view of that output (the four sub-pixels of (y, x) side by side),
//                       classes zero-padded to a multiple of 64
// Three kernels move data around them:
//   roi_pool_kernel         level mapping and roi_align of every RoI on its level -> act16 NHWC (fp32 for tests)
//   roi_box_output_kernel   merged predictor rows -> fp32 class_logits [P, C] and box_regression [P, 4C]
//   roi_mask_output_kernel  logits of the four sub-pixels -> fp32 [N, C, 2S, 2S] (depth-to-space)
#include <cmath>
#include "mpx_common.cuh"

namespace mpx {

// The FPN levels the pool reads ('0'..'3', strides 4..32), feature channels.
constexpr int kRoiLevels = 4;
constexpr int kRoiChannels = 256;

struct RoiPoolParams {
  const float* feat[kRoiLevels];  // [n_images, 256, h_l, w_l] fp32
  int h[kRoiLevels], w[kRoiLevels];
  float scale[kRoiLevels];        // spatial_scale of each level (MultiScaleRoIAlign's inferred 2^-k)
  int start[kMaskMaxImages + 1];  // first RoI of each image; start[n_images] = n_rois
  int n_images, n_rois, out, sampling;
  int k_min;                      // LevelMapper.k_min: -log2(scale[0])
  float inv_s0, lvl0, eps;        // fp32(1 / fp32(canonical_scale)), canonical_level, fp32(1e-6)
};

// LevelMapper: floor(lvl0 + log2(sqrt(box_area) / s0) + eps) clamped to [k_min, k_min + 3], minus k_min.  torchvision
// runs each operation as an ATen kernel of its own, so each is rounded here on its own (no FMA contraction); the
// division by the Python int s0 is ATen's multiplication by the fp32 reciprocal of a CPU scalar divisor.  A box of
// negative area (x1 < x0 or y1 < y0, not both) has a NaN level, which torch.clamp keeps and the int64 conversion turns
// into 0: level -k_min, outside 0..3 for the FPN's k_min = 2, so torchvision pools no level for it and leaves zeros.
__device__ __forceinline__ int roi_level(const float* b, const RoiPoolParams& p) {
  const float area = __fmul_rn(__fsub_rn(b[2], b[0]), __fsub_rn(b[3], b[1]));
  const float s = __fsqrt_rn(area);
  float lv = log2f(__fmul_rn(s, p.inv_s0));
  lv = floorf(__fadd_rn(__fadd_rn(lv, p.lvl0), p.eps));
  if (isnan(lv)) return -p.k_min;
  lv = fminf(fmaxf(lv, static_cast<float>(p.k_min)), static_cast<float>(p.k_min + kRoiLevels - 1));
  return static_cast<int>(lv) - p.k_min;
}

// torchvision's bilinear_interpolate (ops/cuda/roi_align_kernel.cu) for 8 channels of one sample, with each rounding of
// its compiled form written out: `w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4` is fma(w4, v4, fma(w3, v3, fma(w2, v2, w1 * v1)))
// there.  Left to the compiler the chain may instead fuse w1 * v1 and round w2 * v2 on its own, which moves the pooled
// value by an ulp.
__device__ __forceinline__ void roi_bilinear8(const float* __restrict__ f, size_t plane, int height, int width, float y,
                                              float x, float acc[8]) {
  if (y < -1.0f || y > static_cast<float>(height) || x < -1.0f || x > static_cast<float>(width)) {
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] += 0.f;
    return;
  }
  if (y <= 0) y = 0;
  if (x <= 0) x = 0;
  int y_low = static_cast<int>(y), x_low = static_cast<int>(x), y_high, x_high;
  if (y_low >= height - 1) {
    y_high = y_low = height - 1;
    y = static_cast<float>(y_low);
  } else {
    y_high = y_low + 1;
  }
  if (x_low >= width - 1) {
    x_high = x_low = width - 1;
    x = static_cast<float>(x_low);
  } else {
    x_high = x_low + 1;
  }
  const float ly = __fsub_rn(y, static_cast<float>(y_low)), lx = __fsub_rn(x, static_cast<float>(x_low));
  const float hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
  const float w1 = __fmul_rn(hy, hx), w2 = __fmul_rn(hy, lx), w3 = __fmul_rn(ly, hx), w4 = __fmul_rn(ly, lx);
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const float* fc = f + c * plane;
    const float v1 = __ldg(fc + y_low * width + x_low), v2 = __ldg(fc + y_low * width + x_high);
    const float v3 = __ldg(fc + y_high * width + x_low), v4 = __ldg(fc + y_high * width + x_high);
    const float val = __fmaf_rn(w4, v4, __fmaf_rn(w3, v3, __fmaf_rn(w2, v2, __fmul_rn(w1, v1))));
    acc[c] = __fadd_rn(acc[c], val);
  }
}

// One thread per (RoI, 8-channel group, output bin), bins fastest: neighbouring threads sample neighbouring positions
// of the same feature planes.  Writes [n_rois, out, out, 256] NHWC, act16 (F32 = false) or fp32 (F32 = true), and the
// level index of each RoI when `levels` is not NULL.
template <bool F32>
__global__ void __launch_bounds__(256)
roi_pool_kernel(const __grid_constant__ RoiPoolParams p, const float* __restrict__ boxes, void* __restrict__ out,
                int* __restrict__ levels) {
  pdl_trigger();
  pdl_wait();
  const int bins = p.out * p.out;
  const long long total = static_cast<long long>(p.n_rois) * (kRoiChannels / 8) * bins;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int bin = static_cast<int>(i % bins);
    const long long t = i / bins;
    const int cg = static_cast<int>(t % (kRoiChannels / 8));
    const int r = static_cast<int>(t / (kRoiChannels / 8));
    int img = 0;
    while (img + 1 < p.n_images && r >= p.start[img + 1]) ++img;
    const float* b = boxes + 4 * static_cast<size_t>(r);
    const int l = roi_level(b, p);
    if (levels != nullptr && cg == 0 && bin == 0) levels[r] = l;
    const size_t o = (static_cast<size_t>(r) * bins + bin) * kRoiChannels + 8 * cg;
    if (l < 0 || l >= kRoiLevels) {
      if (F32) {
        float4* d = reinterpret_cast<float4*>(static_cast<float*>(out) + o);
        d[0] = d[1] = make_float4(0.f, 0.f, 0.f, 0.f);
      } else {
        *reinterpret_cast<uint4*>(static_cast<act_t*>(out) + o) = make_uint4(0u, 0u, 0u, 0u);
      }
      continue;
    }
    const int height = p.h[l], width = p.w[l];
    const size_t plane = static_cast<size_t>(height) * width;
    const float* f = p.feat[l] + (static_cast<size_t>(img) * kRoiChannels + 8 * cg) * plane;
    // roi_align_forward_kernel_impl, aligned = false.  There each corner is `box * spatial_scale - offset`, whose
    // subtraction keeps the product from contracting into the width's subtraction; here explicit roundings do that.
    const float spatial_scale = p.scale[l];
    const float roi_start_w = __fmul_rn(b[0], spatial_scale), roi_start_h = __fmul_rn(b[1], spatial_scale);
    const float roi_end_w = __fmul_rn(b[2], spatial_scale), roi_end_h = __fmul_rn(b[3], spatial_scale);
    const float roi_width = fmaxf(__fsub_rn(roi_end_w, roi_start_w), 1.f);
    const float roi_height = fmaxf(__fsub_rn(roi_end_h, roi_start_h), 1.f);
    const float bin_size_h = __fdiv_rn(roi_height, static_cast<float>(p.out));
    const float bin_size_w = __fdiv_rn(roi_width, static_cast<float>(p.out));
    const int ph = bin / p.out, pw = bin % p.out;
    const int grid_h = p.sampling, grid_w = p.sampling;
    const float count = static_cast<float>(grid_h * grid_w);
    float acc[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = 0.f;
    // roi_start + p * bin_size + (i + .5f) * bin_size / grid: the first sum is one FMA in torchvision's kernel
    for (int iy = 0; iy < grid_h; iy++) {
      const float y = __fadd_rn(__fmaf_rn(static_cast<float>(ph), bin_size_h, roi_start_h),
                                __fdiv_rn(__fmul_rn(iy + .5f, bin_size_h), static_cast<float>(grid_h)));
      for (int ix = 0; ix < grid_w; ix++) {
        const float x = __fadd_rn(__fmaf_rn(static_cast<float>(pw), bin_size_w, roi_start_w),
                                  __fdiv_rn(__fmul_rn(ix + .5f, bin_size_w), static_cast<float>(grid_w)));
        roi_bilinear8(f, plane, height, width, y, x, acc);
      }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = __fdiv_rn(acc[c], count);
    if (F32) {
      float4* d = reinterpret_cast<float4*>(static_cast<float*>(out) + o);
      d[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
      d[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    } else {
      *reinterpret_cast<uint4*>(static_cast<act_t*>(out) + o) =
          make_uint4(pack_act2(acc[0], acc[1]), pack_act2(acc[2], acc[3]), pack_act2(acc[4], acc[5]),
                     pack_act2(acc[6], acc[7]));
    }
  }
}

// [n_rois, rows] act16 -> class_logits [n_rois, C] (rows 0..C-1) and box_regression [n_rois, 4C] (rows C..5C-1), fp32
__global__ void __launch_bounds__(256)
roi_box_output_kernel(const act_t* __restrict__ src, int rows, int n_rois, int n_classes, float* __restrict__ logits,
                      float* __restrict__ deltas) {
  pdl_trigger();
  pdl_wait();
  const int cols = 5 * n_classes;
  const long long total = static_cast<long long>(n_rois) * cols;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / cols;
    const int k = static_cast<int>(i % cols);
    const float v = static_cast<float>(src[r * rows + k]);
    if (k < n_classes) logits[r * n_classes + k] = v;
    else deltas[r * 4 * n_classes + (k - n_classes)] = v;
  }
}

// [n, s, s, 4, rows] act16 (sub-pixel (dy, dx) = index dy * 2 + dx) -> [n, C, 2s, 2s] fp32
__global__ void __launch_bounds__(256)
roi_mask_output_kernel(const act_t* __restrict__ src, int rows, int n, int s, int n_classes, float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const int m = 2 * s;
  const long long total = static_cast<long long>(n) * n_classes * m * m;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int X = static_cast<int>(i % m);
    long long t = i / m;
    const int Y = static_cast<int>(t % m);
    t /= m;
    const int c = static_cast<int>(t % n_classes);
    const long long b = t / n_classes;
    const long long q = ((b * s + (Y >> 1)) * s + (X >> 1)) * 4 + (Y & 1) * 2 + (X & 1);
    out[i] = static_cast<float>(src[q * rows + c]);
  }
}

static unsigned roi_grid(long long items) {
  long long blocks = (items + 255) / 256;
  const long long cap = static_cast<long long>(sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  return static_cast<unsigned>(blocks > 0 ? blocks : 1);
}

static size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

struct RoiHeads {
  const void* w[kRoiHeadConvs];
  const float* b[kRoiHeadConvs];
  int n_classes, hidden, box_rows, mask_rows;
};

int roi_heads_create(const void* const* w, const float* const* b, int n_classes, int hidden, RoiHeads** out) {
  RoiHeads* h = new RoiHeads();
  for (int i = 0; i < kRoiHeadConvs; ++i) {
    h->w[i] = w[i];
    h->b[i] = b[i];
  }
  h->n_classes = n_classes;
  h->hidden = hidden;
  h->box_rows = roi_box_rows(n_classes);
  h->mask_rows = roi_mask_rows(n_classes);
  *out = h;
  return MPX_OK;
}

void roi_heads_destroy(RoiHeads* h) { delete h; }

// Box branch: pooled [P, 7, 7, 256] | fc6 out [P, hidden] | fc7 out [P, hidden] | predictor out [P, box_rows].
// Mask branch: pooled [N, s, s, 256] | two 3x3 ping-pong buffers of the same size | deconvolution [N, s, s, 1024] |
// logits [N, s, s, 4, mask_rows].  One workspace serves both; the branches run one after the other.
static size_t box_bytes(const RoiHeads* h, int n_rois, size_t off[4]) {
  const size_t p = static_cast<size_t>(n_rois);
  const size_t bytes[4] = {p * kRoiBoxPool * kRoiBoxPool * kRoiChannels * 2, p * h->hidden * 2, p * h->hidden * 2,
                           p * h->box_rows * 2};
  size_t total = 0;
  for (int i = 0; i < 4; ++i) {
    off[i] = total;
    total += align256(bytes[i]);
  }
  return total;
}

static size_t mask_bytes(const RoiHeads* h, int n_rois, int s, size_t off[5]) {
  const size_t px = static_cast<size_t>(n_rois) * s * s;
  const size_t bytes[5] = {px * kRoiChannels * 2, px * kRoiChannels * 2, px * kRoiChannels * 2, px * 4 * kRoiChannels * 2,
                           px * 4 * h->mask_rows * 2};
  size_t total = 0;
  for (int i = 0; i < 5; ++i) {
    off[i] = total;
    total += align256(bytes[i]);
  }
  return total;
}

size_t roi_heads_workspace_bytes(const RoiHeads* h, int n_box_rois, int n_mask_rois, int mask_pool) {
  size_t ob[4], om[5];
  const size_t a = box_bytes(h, n_box_rois, ob), b = mask_bytes(h, n_mask_rois, mask_pool, om);
  return a > b ? a : b;
}

static RoiPoolParams pool_params(const float* const* features, int n_images, int h, int w, const float* scales,
                                 int canonical_scale, int canonical_level, int sampling, const int* counts, int out) {
  RoiPoolParams p{};
  for (int l = 0; l < kRoiLevels; ++l) {
    p.feat[l] = features[l];
    p.h[l] = h >> (l + 2);
    p.w[l] = w >> (l + 2);
    p.scale[l] = scales[l];
  }
  p.n_images = n_images;
  int start = 0;
  for (int i = 0; i < n_images; ++i) {
    p.start[i] = start;
    start += counts[i];
  }
  p.start[n_images] = start;
  p.n_rois = start;
  p.out = out;
  p.sampling = sampling;
  p.k_min = static_cast<int>(std::lround(-std::log2(static_cast<double>(scales[0]))));
  p.inv_s0 = 1.0f / static_cast<float>(canonical_scale);
  p.lvl0 = static_cast<float>(canonical_level);
  p.eps = static_cast<float>(1e-6);
  return p;
}

int roi_pool(const float* const* features, int n_images, int h, int w, const float* scales, int canonical_scale,
             int canonical_level, int sampling, const float* boxes, const int* counts, int out_size, void* out, bool f32,
             int* levels, cudaStream_t stream) {
  const RoiPoolParams p =
      pool_params(features, n_images, h, w, scales, canonical_scale, canonical_level, sampling, counts, out_size);
  if (p.n_rois == 0) return MPX_OK;
  const long long items = static_cast<long long>(p.n_rois) * (kRoiChannels / 8) * out_size * out_size;
  if (f32)
    MPX_CHECK_CUDA(launch_pdl(roi_pool_kernel<true>, dim3(roi_grid(items)), dim3(256), 0, stream, 1, p, boxes, out, levels));
  else
    MPX_CHECK_CUDA(launch_pdl(roi_pool_kernel<false>, dim3(roi_grid(items)), dim3(256), 0, stream, 1, p, boxes, out, levels));
  ++g_launches;
  return MPX_OK;
}

static int heads_splitk() { return (conv_get_mode() & MPX_CONV_NET_SPLITK) != 0 ? -1 : 0; }

int roi_box_forward(const RoiHeads* hd, const float* const* features, int n_images, int h, int w, const float* scales,
                    int canonical_scale, int canonical_level, int sampling, const float* boxes, const int* counts,
                    float* class_logits, float* box_regression, void* workspace, cudaStream_t stream) {
  int n_rois = 0;
  for (int i = 0; i < n_images; ++i) n_rois += counts[i];
  if (n_rois == 0) return MPX_OK;
  size_t off[4];
  box_bytes(hd, n_rois, off);
  uint8_t* base = static_cast<uint8_t*>(workspace);
  int rc = roi_pool(features, n_images, h, w, scales, canonical_scale, canonical_level, sampling, boxes, counts,
                    kRoiBoxPool, base + off[0], false, nullptr, stream);
  if (rc != MPX_OK) return rc;
  const int sk = heads_splitk();
  const ConvDesc fc6{n_rois, kRoiBoxPool, kRoiBoxPool, kRoiChannels, hd->hidden, kRoiBoxPool, kRoiBoxPool, 1, 0, 0, 0, 0, 1, 0};
  rc = conv_forward(fc6, base + off[0], hd->w[0], hd->b[0], nullptr, base + off[1], 0, 0, stream, sk, 2048);
  if (rc != MPX_OK) return rc;
  const ConvDesc fc7{n_rois, 1, 1, hd->hidden, hd->hidden, 1, 1, 1, 0, 0, 0, 0, 1, 0};
  rc = conv_forward(fc7, base + off[1], hd->w[1], hd->b[1], nullptr, base + off[2], 0, 0, stream, sk, 2048);
  if (rc != MPX_OK) return rc;
  const ConvDesc pred{n_rois, 1, 1, hd->hidden, hd->box_rows, 1, 1, 1, 0, 0, 0, 0, 0, 0};
  rc = conv_forward(pred, base + off[2], hd->w[2], hd->b[2], nullptr, base + off[3], 0, 0, stream, sk, 2048);
  if (rc != MPX_OK) return rc;
  const long long items = static_cast<long long>(n_rois) * 5 * hd->n_classes;
  MPX_CHECK_CUDA(launch_pdl(roi_box_output_kernel, dim3(roi_grid(items)), dim3(256), 0, stream, 1,
                            reinterpret_cast<const act_t*>(base + off[3]), hd->box_rows, n_rois, hd->n_classes,
                            class_logits, box_regression));
  ++g_launches;
  return MPX_OK;
}

int roi_mask_forward(const RoiHeads* hd, const float* const* features, int n_images, int h, int w, const float* scales,
                     int canonical_scale, int canonical_level, int sampling, int s, const float* boxes,
                     const int* counts, float* mask_logits, void* workspace, cudaStream_t stream) {
  int n = 0;
  for (int i = 0; i < n_images; ++i) n += counts[i];
  if (n == 0) return MPX_OK;
  size_t off[5];
  mask_bytes(hd, n, s, off);
  uint8_t* base = static_cast<uint8_t*>(workspace);
  int rc = roi_pool(features, n_images, h, w, scales, canonical_scale, canonical_level, sampling, boxes, counts, s,
                    base + off[0], false, nullptr, stream);
  if (rc != MPX_OK) return rc;
  const int sk = heads_splitk();
  void* x = base + off[0];
  for (int k = 0; k < 4; ++k) {
    void* y = base + off[1 + (k & 1)];
    const ConvDesc d{n, s, s, kRoiChannels, kRoiChannels, 3, 3, 1, 1, 1, 1, 1, 1, 0};
    rc = conv_forward(d, x, hd->w[3 + k], hd->b[3 + k], nullptr, y, 0, 0, stream, sk, 2048);
    if (rc != MPX_OK) return rc;
    x = y;
  }
  const ConvDesc up{n, s, s, kRoiChannels, 4 * kRoiChannels, 1, 1, 1, 0, 0, 0, 0, 1, 0};
  rc = conv_forward(up, x, hd->w[7], hd->b[7], nullptr, base + off[3], 0, 0, stream, sk, 2048);
  if (rc != MPX_OK) return rc;
  const ConvDesc logits{n, s, 4 * s, kRoiChannels, hd->mask_rows, 1, 1, 1, 0, 0, 0, 0, 0, 0};
  rc = conv_forward(logits, base + off[3], hd->w[8], hd->b[8], nullptr, base + off[4], 0, 0, stream, sk, 2048);
  if (rc != MPX_OK) return rc;
  const long long items = static_cast<long long>(n) * hd->n_classes * 4 * s * s;
  MPX_CHECK_CUDA(launch_pdl(roi_mask_output_kernel, dim3(roi_grid(items)), dim3(256), 0, stream, 1,
                            reinterpret_cast<const act_t*>(base + off[4]), hd->mask_rows, n, s, hd->n_classes,
                            mask_logits));
  ++g_launches;
  return MPX_OK;
}

}  // namespace mpx
