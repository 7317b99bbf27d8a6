// BOP 2019 pose-error kernels (include/mpx.h: mpx_bop_vsd, mpx_bop_point_errors).
//
// VSD: one pass over the test depth and the two rendered depths of each (estimate, ground truth) pair.  The arithmetic is
// the BOP toolkit's, in its order and without FMA contraction (every float64 step is an explicit _rn intrinsic): test depth
// in mm = fp32(raw) * fp32(depth_scale); rendered depth in mm = fp32(metres * 1000); distance image
// sqrt((X d)^2 + (Y d)^2 + d^2) with X = (x - cx) / fx in float64; visibility masks from the fp32 difference of the two
// distance images against delta ("bop19" mode: pixels without test depth count as visible).  Each CTA counts its pixels in
// registers, reduces the counts with warp shuffles and adds them to the pair's int64 counters with one atomic per counter,
// so the counts do not depend on the launch shape.  A second kernel turns the counts into (count + comp) / union.
//
// Point errors: one CTA per pair.  MSSD / MSPD take the max over the model points of each (pair, symmetry) and the min over
// the symmetries (first minimum wins, as Python's min); ADD is the mean point distance; ADI the mean nearest-neighbour
// distance, by brute force over shared-memory tiles of the estimate's points, all in float64.
//
// CUS counts the two silhouettes of the VSD layout's renders as the VSD count kernel counts; PROJ / RE / TE
// (mpx_bop_pose_errors) take one CTA per pair, PROJ with ADD's block sum.
#include "mpx_common.cuh"
#include "../../include/mpx.h"

namespace mpx {

constexpr int kVsdThreads = 256;
constexpr int kVsdPixelsPerThread = 16;
constexpr int kPointThreads = 256;
constexpr int kSymChunk = 4;  // symmetries per pass over the points (running maxima held in registers)

struct VsdTaus {
  double tau[MPX_BOP_MAX_TAUS];
};

__device__ __forceinline__ double dist_from_depth(double X, double Y, double d) {
  const double a = __dmul_rn(X, d);
  const double b = __dmul_rn(Y, d);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), __dmul_rn(d, d)));
}

// misc.depth_im_to_dist_im (calc_gt_masks.py): X d = ((x - cx) d) (1 / fx) in float64, then the same norm
__device__ __forceinline__ double dist_from_depth_px(double xc, double yc, double rfx, double rfy, double d) {
  const double a = __dmul_rn(__dmul_rn(xc, d), rfx);
  const double b = __dmul_rn(__dmul_rn(yc, d), rfy);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), __dmul_rn(d, d)));
}

// visibility.estimate_visib_mask_gt, "bop19" mode: fp32(dist_model) - fp32(dist_test) <= delta, or no test depth, and a
// model surface
__device__ __forceinline__ bool visib_bop19(double dist_model, float dist_test_f32, bool test_missing, float delta) {
  return (__fsub_rn(__double2float_rn(dist_model), dist_test_f32) <= delta || test_missing) && dist_model > 0.0;
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ bool vsd_pair_valid(int p, const int* est_idx, const int* gt_idx, const int* img_idx, int n_est,
                                               int n_gt, int n_img) {
  const int e = est_idx[p], g = gt_idx[p], i = img_idx[p];
  return e >= 0 && e < n_est && g >= 0 && g < n_gt && i >= 0 && i < n_img;
}

// counts[p] = {union, intersection, count(tau_0), ..., count(tau_{n_taus-1})}, zeroed before the launch
__global__ void __launch_bounds__(kVsdThreads) bop_vsd_count_kernel(
    int pair0, int w, int hw, const uint16_t* __restrict__ test, int n_img, const float* __restrict__ depth_scale,
    const double* __restrict__ K, const float* __restrict__ dest, int n_est, const float* __restrict__ dgt, int n_gt,
    const int* __restrict__ est_idx, const int* __restrict__ gt_idx, const int* __restrict__ img_idx,
    const double* __restrict__ diameter, VsdTaus taus, int n_taus, float delta, unsigned long long* __restrict__ counts) {
  const int p = pair0 + blockIdx.y;
  if (!vsd_pair_valid(p, est_idx, gt_idx, img_idx, n_est, n_gt, n_img)) return;
  const int img = img_idx[p];
  const uint16_t* t_im = test + static_cast<size_t>(img) * hw;
  const float* e_im = dest + static_cast<size_t>(est_idx[p]) * hw;
  const float* g_im = dgt + static_cast<size_t>(gt_idx[p]) * hw;
  const double* k = K + 9 * img;
  const double fx = k[0], cx = k[2], fy = k[4], cy = k[5];
  const float scale = depth_scale[img];
  const double diam = diameter[p];

  unsigned n_union = 0, n_inter = 0;
  unsigned n_tau[MPX_BOP_MAX_TAUS];
#pragma unroll
  for (int j = 0; j < MPX_BOP_MAX_TAUS; ++j) n_tau[j] = 0;

  for (int px = blockIdx.x * blockDim.x + threadIdx.x; px < hw; px += gridDim.x * blockDim.x) {
    const float de = __fmul_rn(e_im[px], 1000.f);
    const float dg = __fmul_rn(g_im[px], 1000.f);
    if (!(de > 0.f) && !(dg > 0.f)) continue;  // neither mask can hold here
    const float dt = __fmul_rn(static_cast<float>(t_im[px]), scale);
    const int y = px / w, x = px - y * w;
    const double X = __ddiv_rn(__dadd_rn(static_cast<double>(x), -cx), fx);
    const double Y = __ddiv_rn(__dadd_rn(static_cast<double>(y), -cy), fy);
    const double dist_t = dist_from_depth(X, Y, static_cast<double>(dt));
    const double dist_e = dist_from_depth(X, Y, static_cast<double>(de));
    const double dist_g = dist_from_depth(X, Y, static_cast<double>(dg));
    const float ft = __double2float_rn(dist_t);
    const bool test_missing = dist_t == 0.0;
    const bool vg = visib_bop19(dist_g, ft, test_missing, delta);
    const bool ve = visib_bop19(dist_e, ft, test_missing, delta) || (vg && dist_e > 0.0);
    n_union += (vg || ve);
    if (vg && ve) {
      ++n_inter;
      const double dd = __ddiv_rn(fabs(__dadd_rn(dist_g, -dist_e)), diam);
#pragma unroll
      for (int j = 0; j < MPX_BOP_MAX_TAUS; ++j)
        if (j < n_taus) n_tau[j] += (dd >= taus.tau[j]);
    }
  }

  __shared__ unsigned long long part[kVsdThreads / 32][2 + MPX_BOP_MAX_TAUS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long v = warp_sum_u64(n_union);
  if (lane == 0) part[warp][0] = v;
  v = warp_sum_u64(n_inter);
  if (lane == 0) part[warp][1] = v;
#pragma unroll
  for (int j = 0; j < MPX_BOP_MAX_TAUS; ++j) {
    if (j < n_taus) {
      v = warp_sum_u64(n_tau[j]);
      if (lane == 0) part[warp][2 + j] = v;
    }
  }
  __syncthreads();
  if (threadIdx.x < 2 + n_taus) {
    unsigned long long s = 0;
    for (int i = 0; i < kVsdThreads / 32; ++i) s += part[i][threadIdx.x];
    if (s) atomicAdd(counts + static_cast<size_t>(p) * (2 + n_taus) + threadIdx.x, s);
  }
}

__global__ void bop_vsd_finish_kernel(int n_pairs, int n_taus, const int* __restrict__ est_idx,
                                      const int* __restrict__ gt_idx, const int* __restrict__ img_idx, int n_est, int n_gt,
                                      int n_img, const unsigned long long* __restrict__ counts, double* __restrict__ err) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pairs) return;
  const unsigned long long* c = counts + static_cast<size_t>(p) * (2 + n_taus);
  const bool ok = vsd_pair_valid(p, est_idx, gt_idx, img_idx, n_est, n_gt, n_img);
  const unsigned long long uni = c[0], comp = c[0] - c[1];
  for (int j = 0; j < n_taus; ++j) {
    double e;
    if (!ok) e = __longlong_as_double(0x7ff8000000000000ll);
    else if (uni == 0) e = 1.0;
    else e = __ddiv_rn(static_cast<double>(c[2 + j] + comp), static_cast<double>(uni));
    err[static_cast<size_t>(p) * n_taus + j] = e;
  }
}

int bop_vsd(int n_pairs, int h, int w, const uint16_t* test, int n_img, const float* depth_scale, const double* K,
            const float* dest, int n_est, const float* dgt, int n_gt, const int* est_idx, const int* gt_idx,
            const int* img_idx, const double* diameter, const double* h_taus, int n_taus, float delta,
            int64_t* counts, double* err, cudaStream_t stream) {
  if (n_pairs == 0) return MPX_OK;
  VsdTaus taus;
  for (int j = 0; j < MPX_BOP_MAX_TAUS; ++j) taus.tau[j] = j < n_taus ? h_taus[j] : 0.0;
  const int hw = h * w;
  MPX_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * static_cast<size_t>(n_pairs) * (2 + n_taus), stream));
  const int bx = (hw + kVsdThreads * kVsdPixelsPerThread - 1) / (kVsdThreads * kVsdPixelsPerThread);
  auto* cnt = reinterpret_cast<unsigned long long*>(counts);
  for (int p0 = 0; p0 < n_pairs; p0 += 65535) {  // gridDim.y limit
    const int np = n_pairs - p0 < 65535 ? n_pairs - p0 : 65535;
    bop_vsd_count_kernel<<<dim3(bx, np), kVsdThreads, 0, stream>>>(p0, w, hw, test, n_img, depth_scale, K, dest, n_est,
                                                                   dgt, n_gt, est_idx, gt_idx, img_idx, diameter, taus,
                                                                   n_taus, delta, cnt);
    MPX_CHECK_CUDA(cudaGetLastError());
    ++g_launches;
  }
  bop_vsd_finish_kernel<<<(n_pairs + 127) / 128, 128, 0, stream>>>(n_pairs, n_taus, est_idx, gt_idx, img_idx, n_est, n_gt,
                                                                   n_img, cnt, err);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// CUS: complement over union of the two silhouettes (pose_error.cus), on the VSD kernel's render-sharing layout
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool cus_pair_valid(int p, const int* est_idx, const int* gt_idx, int n_est, int n_gt) {
  const int e = est_idx[p], g = gt_idx[p];
  return e >= 0 && e < n_est && g >= 0 && g < n_gt;
}

// counts[p] = {intersection, union}, zeroed before the launch
__global__ void __launch_bounds__(kVsdThreads) bop_cus_count_kernel(
    int pair0, int hw, const float* __restrict__ dest, int n_est, const float* __restrict__ dgt, int n_gt,
    const int* __restrict__ est_idx, const int* __restrict__ gt_idx, unsigned long long* __restrict__ counts) {
  const int p = pair0 + blockIdx.y;
  if (!cus_pair_valid(p, est_idx, gt_idx, n_est, n_gt)) return;
  const float* e_im = dest + static_cast<size_t>(est_idx[p]) * hw;
  const float* g_im = dgt + static_cast<size_t>(gt_idx[p]) * hw;
  unsigned n_inter = 0, n_union = 0;
  for (int px = blockIdx.x * blockDim.x + threadIdx.x; px < hw; px += gridDim.x * blockDim.x) {
    // fp32(metres * 1000) > 0 exactly when metres > 0: the mask of the toolkit's depth in mm
    const bool me = e_im[px] > 0.f, mg = g_im[px] > 0.f;
    n_inter += me && mg;
    n_union += me || mg;
  }
  __shared__ unsigned long long part[kVsdThreads / 32][2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long v = warp_sum_u64(n_inter);
  if (lane == 0) part[warp][0] = v;
  v = warp_sum_u64(n_union);
  if (lane == 0) part[warp][1] = v;
  __syncthreads();
  if (threadIdx.x < 2) {
    unsigned long long s = 0;
    for (int i = 0; i < kVsdThreads / 32; ++i) s += part[i][threadIdx.x];
    if (s) atomicAdd(counts + 2 * static_cast<size_t>(p) + threadIdx.x, s);
  }
}

// 1.0 - inter / float(union) in float64, as the toolkit writes it; 1.0 for an empty union, NaN for out-of-range indices
__global__ void bop_cus_finish_kernel(int n_pairs, const int* __restrict__ est_idx, const int* __restrict__ gt_idx,
                                      int n_est, int n_gt, const unsigned long long* __restrict__ counts,
                                      double* __restrict__ err) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pairs) return;
  const unsigned long long inter = counts[2 * static_cast<size_t>(p)], uni = counts[2 * static_cast<size_t>(p) + 1];
  double e;
  if (!cus_pair_valid(p, est_idx, gt_idx, n_est, n_gt)) e = __longlong_as_double(0x7ff8000000000000ll);
  else if (uni == 0) e = 1.0;
  else e = __dadd_rn(1.0, -__ddiv_rn(static_cast<double>(inter), static_cast<double>(uni)));
  err[p] = e;
}

int bop_cus(int n_pairs, int h, int w, const float* dest, int n_est, const float* dgt, int n_gt, const int* est_idx,
            const int* gt_idx, int64_t* counts, double* err, cudaStream_t stream) {
  if (n_pairs == 0) return MPX_OK;
  const int hw = h * w;
  MPX_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * 2 * static_cast<size_t>(n_pairs), stream));
  const int bx = (hw + kVsdThreads * kVsdPixelsPerThread - 1) / (kVsdThreads * kVsdPixelsPerThread);
  auto* cnt = reinterpret_cast<unsigned long long*>(counts);
  for (int p0 = 0; p0 < n_pairs; p0 += 65535) {  // gridDim.y limit
    const int np = n_pairs - p0 < 65535 ? n_pairs - p0 : 65535;
    bop_cus_count_kernel<<<dim3(bx, np), kVsdThreads, 0, stream>>>(p0, hw, dest, n_est, dgt, n_gt, est_idx, gt_idx, cnt);
    MPX_CHECK_CUDA(cudaGetLastError());
    ++g_launches;
  }
  bop_cus_finish_kernel<<<(n_pairs + 127) / 128, 128, 0, stream>>>(n_pairs, est_idx, gt_idx, n_est, n_gt, cnt, err);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// ground-truth annotation (scripts/calc_gt_info.py, calc_gt_masks.py)
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kGtThreads = 256;
constexpr int kGtPixelsPerThread = 16;
constexpr int kGtBoxWords = 8;  // {obj, visib} x {-xmin, -ymin, xmax, ymax} while counting: every slot is a running max
constexpr int kGtBoxInit = static_cast<int>(0x80808080u);  // cudaMemset byte 0x80: below any coordinate

__device__ __forceinline__ bool gt_img_valid(const int* img_idx, int g, int n_img) {
  const int i = img_idx[g];
  return i >= 0 && i < n_img;
}

// counts[g] = {px_count_all, px_count_valid, px_count_visib}, zeroed before the launch; box[g] as kGtBoxWords above.
// One CTA row per gt (grid-stride over gts in y), grid-stride over the 3h x 3w canvas in x.
__global__ void __launch_bounds__(kGtThreads) bop_gt_info_count_kernel(
    int n_gt, int h, int w, const uint16_t* __restrict__ test, int n_img, const float* __restrict__ depth_scale,
    const double* __restrict__ K, const float* __restrict__ large, const int* __restrict__ img_idx, float delta,
    unsigned long long* __restrict__ counts, int* __restrict__ box, uint8_t* __restrict__ mask,
    uint8_t* __restrict__ mask_visib) {
  const int W = 3 * w, HW = 9 * h * w, hw = h * w;
  __shared__ unsigned long long part_n[kGtThreads / 32][3];
  __shared__ int part_b[kGtThreads / 32][kGtBoxWords];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int g = blockIdx.y; g < n_gt; g += gridDim.y) {
    const bool ok = gt_img_valid(img_idx, g, n_img);
    const int img = ok ? img_idx[g] : 0;
    const uint16_t* t_im = test + static_cast<size_t>(img) * hw;
    const float* l_im = large + static_cast<size_t>(g) * HW;
    const double* k = K + 9 * img;
    const double fx = k[0], cx = k[2], fy = k[4], cy = k[5];
    const double rfx = __ddiv_rn(1.0, fx), rfy = __ddiv_rn(1.0, fy);
    const float scale = depth_scale[img];
    unsigned n_all = 0, n_valid = 0, n_visib = 0;
    int b[kGtBoxWords];
#pragma unroll
    for (int j = 0; j < kGtBoxWords; ++j) b[j] = kGtBoxInit;

    // the running index is 64-bit: its last step may pass INT_MAX for canvases near the 2^31-pixel limit
    for (long long p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += static_cast<long long>(gridDim.x) * blockDim.x) {
      const int px = static_cast<int>(p);
      const int Y = px / W, X = px - Y * W;
      const int x = X - w, y = Y - h;  // image coordinates (the canvas' principal point is shifted by (w, h))
      const bool in_image = x >= 0 && x < w && y >= 0 && y < h;
      const float dl = ok ? l_im[px] : 0.f;
      bool m = false, mv = false;
      if (dl > 0.f) {
        ++n_all;
        b[0] = max(b[0], -x);
        b[1] = max(b[1], -y);
        b[2] = max(b[2], x);
        b[3] = max(b[3], y);
        if (in_image) {
          const float dg = __fmul_rn(dl, 1000.f);
          const float dt = __fmul_rn(static_cast<float>(t_im[y * w + x]), scale);
          const double xc = __dadd_rn(static_cast<double>(x), -cx), yc = __dadd_rn(static_cast<double>(y), -cy);
          // scene_gt_info: misc.depth_im_to_dist_im_fast, as the VSD kernel
          const double Xf = __ddiv_rn(xc, fx), Yf = __ddiv_rn(yc, fy);
          const double dist_t = dist_from_depth(Xf, Yf, static_cast<double>(dt));
          const double dist_g = dist_from_depth(Xf, Yf, static_cast<double>(dg));
          n_valid += dist_g > 0.0 && dist_t > 0.0;
          if (visib_bop19(dist_g, __double2float_rn(dist_t), dist_t == 0.0, delta)) {
            ++n_visib;
            b[4] = max(b[4], -x);
            b[5] = max(b[5], -y);
            b[6] = max(b[6], x);
            b[7] = max(b[7], y);
          }
          // mask / mask_visib: misc.depth_im_to_dist_im, whose rounding differs
          const double dist_ts = dist_from_depth_px(xc, yc, rfx, rfy, static_cast<double>(dt));
          const double dist_gs = dist_from_depth_px(xc, yc, rfx, rfy, static_cast<double>(dg));
          m = dist_gs > 0.0;
          mv = visib_bop19(dist_gs, __double2float_rn(dist_ts), dist_ts == 0.0, delta);
        }
      }
      if (in_image) {
        const size_t o = static_cast<size_t>(g) * hw + y * w + x;
        if (mask) mask[o] = m;
        if (mask_visib) mask_visib[o] = mv;
      }
    }

    unsigned long long v0 = warp_sum_u64(n_all), v1 = warp_sum_u64(n_valid), v2 = warp_sum_u64(n_visib);
#pragma unroll
    for (int j = 0; j < kGtBoxWords; ++j) b[j] = __reduce_max_sync(0xffffffffu, b[j]);
    if (lane == 0) {
      part_n[warp][0] = v0;
      part_n[warp][1] = v1;
      part_n[warp][2] = v2;
#pragma unroll
      for (int j = 0; j < kGtBoxWords; ++j) part_b[warp][j] = b[j];
    }
    __syncthreads();
    if (threadIdx.x < 3) {
      unsigned long long s = 0;
      for (int i = 0; i < kGtThreads / 32; ++i) s += part_n[i][threadIdx.x];
      if (s) atomicAdd(counts + 3 * static_cast<size_t>(g) + threadIdx.x, s);
    } else if (threadIdx.x >= 32 && threadIdx.x < 32 + kGtBoxWords) {
      const int j = threadIdx.x - 32;
      int s = kGtBoxInit;
      for (int i = 0; i < kGtThreads / 32; ++i) s = max(s, part_b[i][j]);
      if (s != kGtBoxInit) atomicMax(box + kGtBoxWords * static_cast<size_t>(g) + j, s);
    }
    __syncthreads();  // part_* are rewritten by the next gt
  }
}

// box[g]: running maxima -> {bbox_obj, bbox_visib} as misc.calc_2d_bbox (x, y, x_max - x_min, y_max - y_min), both
// [-1, -1, -1, -1] unless px_count_visib > 0; a gt with an out-of-range image index gets counts and boxes of -1
__global__ void bop_gt_info_finish_kernel(int n_gt, int n_img, const int* __restrict__ img_idx,
                                          unsigned long long* __restrict__ counts, int* __restrict__ box) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_gt) return;
  int* bx = box + kGtBoxWords * static_cast<size_t>(g);
  unsigned long long* c = counts + 3 * static_cast<size_t>(g);
  const bool ok = gt_img_valid(img_idx, g, n_img);
  if (!ok) c[0] = c[1] = c[2] = ~0ull;
  if (!ok || c[2] == 0) {
    for (int j = 0; j < kGtBoxWords; ++j) bx[j] = -1;
    return;
  }
  for (int k = 0; k < 2; ++k) {
    int* q = bx + 4 * k;
    const int x0 = -q[0], y0 = -q[1], x1 = q[2], y1 = q[3];
    q[0] = x0;
    q[1] = y0;
    q[2] = x1 - x0;
    q[3] = y1 - y0;
  }
}

int bop_gt_info(int n_gt, int h, int w, const uint16_t* test, int n_img, const float* depth_scale, const double* K,
                const float* large, const int* img_idx, float delta, int64_t* counts, int* bbox, uint8_t* mask,
                uint8_t* mask_visib, cudaStream_t stream) {
  if (n_gt == 0) return MPX_OK;
  MPX_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * 3 * static_cast<size_t>(n_gt), stream));
  MPX_CHECK_CUDA(cudaMemsetAsync(bbox, 0x80, sizeof(int) * kGtBoxWords * static_cast<size_t>(n_gt), stream));
  const long long HW = 9ll * h * w;
  const int bx = static_cast<int>((HW + kGtThreads * kGtPixelsPerThread - 1) / (kGtThreads * kGtPixelsPerThread));
  const int by = n_gt < 65535 ? n_gt : 65535;  // gridDim.y limit: the kernel strides over the rest
  auto* cnt = reinterpret_cast<unsigned long long*>(counts);
  bop_gt_info_count_kernel<<<dim3(bx, by), kGtThreads, 0, stream>>>(n_gt, h, w, test, n_img, depth_scale, K, large,
                                                                    img_idx, delta, cnt, bbox, mask, mask_visib);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  bop_gt_info_finish_kernel<<<(n_gt + 127) / 128, 128, 0, stream>>>(n_gt, n_img, img_idx, cnt, bbox);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// point errors
// ---------------------------------------------------------------------------------------------------------------------
struct Rt {
  double R[9], t[3];
};

__device__ __forceinline__ void apply(const Rt& T, double x, double y, double z, double& ox, double& oy, double& oz) {
  ox = T.R[0] * x + T.R[1] * y + T.R[2] * z + T.t[0];
  oy = T.R[3] * x + T.R[4] * y + T.R[5] * z + T.t[1];
  oz = T.R[6] * x + T.R[7] * y + T.R[8] * z + T.t[2];
}

// image coordinates of a point under pose T and intrinsics K (misc.project_pts: P = K [R|t], divide by the third row)
__device__ __forceinline__ void project(const double* P, double x, double y, double z, double& u, double& v) {
  const double a = P[0] * x + P[1] * y + P[2] * z + P[3];
  const double b = P[4] * x + P[5] * y + P[6] * z + P[7];
  const double c = P[8] * x + P[9] * y + P[10] * z + P[11];
  u = a / c;
  v = b / c;
}

__device__ void make_P(const double* K, const Rt& T, double* P) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) P[4 * i + j] = K[3 * i] * T.R[j] + K[3 * i + 1] * T.R[3 + j] + K[3 * i + 2] * T.R[6 + j];
    P[4 * i + 3] = K[3 * i] * T.t[0] + K[3 * i + 1] * T.t[1] + K[3 * i + 2] * T.t[2];
  }
}

__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// block-wide reduction (max or sum) in a fixed order; every thread gets the result
template <bool kMax>
__device__ double block_reduce(double v, double* red) {
  v = kMax ? warp_max_d(v) : warp_sum_d(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double r = red[0];
  for (int i = 1; i < kPointThreads / 32; ++i) r = kMax ? fmax(r, red[i]) : r + red[i];
  return r;
}

template <int kind>
__global__ void __launch_bounds__(kPointThreads) bop_point_kernel(
    int n_models, const double* __restrict__ pts, const int64_t* __restrict__ pt_off, long long n_pts_total,
    const double* __restrict__ syms, const int64_t* __restrict__ sym_off, long long n_syms_total,
    const int* __restrict__ model_idx, const double* __restrict__ pose_est, const double* __restrict__ pose_gt,
    const double* __restrict__ K, double* __restrict__ err, int* __restrict__ sym_argmin) {
  const int p = blockIdx.x;
  __shared__ Rt est, gt, gsym[kSymChunk];
  __shared__ double P_est[12], P_gsym[kSymChunk][12];
  __shared__ double red[kPointThreads / 32];
  __shared__ double tile[kPointThreads][3];
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  const int m = model_idx[p];
  long long p0 = 0, p1 = 0, s0 = 0, s1 = 0;
  if (m >= 0 && m < n_models) {
    p0 = max(0ll, min(static_cast<long long>(pt_off[m]), n_pts_total));
    p1 = max(p0, min(static_cast<long long>(pt_off[m + 1]), n_pts_total));
    if (syms) {
      s0 = max(0ll, min(static_cast<long long>(sym_off[m]), n_syms_total));
      s1 = max(s0, min(static_cast<long long>(sym_off[m + 1]), n_syms_total));
    }
  }
  constexpr bool with_syms = kind == MPX_BOP_MSSD || kind == MPX_BOP_MSPD;
  if (p1 == p0 || (with_syms && s1 == s0)) {
    if (threadIdx.x == 0) {
      err[p] = nan;
      if (sym_argmin) sym_argmin[p] = -1;
    }
    return;
  }
  const double* pe = pose_est + 12 * p;
  const double* pg = pose_gt + 12 * p;
  if (threadIdx.x < 12) (threadIdx.x < 9 ? est.R[threadIdx.x] : est.t[threadIdx.x - 9]) = pe[threadIdx.x];
  else if (threadIdx.x < 24) (threadIdx.x < 21 ? gt.R[threadIdx.x - 12] : gt.t[threadIdx.x - 21]) = pg[threadIdx.x - 12];
  __syncthreads();
  if (kind == MPX_BOP_MSPD && threadIdx.x == 0) make_P(K + 9 * p, est, P_est);
  __syncthreads();
  const long long n = p1 - p0;
  const double* P = pts + 3 * p0;

  if constexpr (with_syms) {
    double best = __longlong_as_double(0x7ff0000000000000ll);
    int best_s = -1;
    for (long long c0 = s0; c0 < s1; c0 += kSymChunk) {
      const int ns = static_cast<int>(min(static_cast<long long>(kSymChunk), s1 - c0));
      if (threadIdx.x < ns) {  // gt pose composed with symmetry: R_gt S_R, R_gt S_t + t_gt
        const double* S = syms + 12 * (c0 + threadIdx.x);
        Rt& G = gsym[threadIdx.x];
        for (int i = 0; i < 3; ++i) {
          for (int j = 0; j < 3; ++j) G.R[3 * i + j] = pg[3 * i] * S[j] + pg[3 * i + 1] * S[3 + j] + pg[3 * i + 2] * S[6 + j];
          G.t[i] = pg[3 * i] * S[9] + pg[3 * i + 1] * S[10] + pg[3 * i + 2] * S[11] + pg[9 + i];
        }
        if (kind == MPX_BOP_MSPD) make_P(K + 9 * p, G, P_gsym[threadIdx.x]);
      }
      __syncthreads();
      double mx[kSymChunk];
#pragma unroll
      for (int s = 0; s < kSymChunk; ++s) mx[s] = 0.0;
      for (long long i = threadIdx.x; i < n; i += kPointThreads) {
        const double x = P[3 * i], y = P[3 * i + 1], z = P[3 * i + 2];
        if constexpr (kind == MPX_BOP_MSSD) {
          double ex, ey, ez;
          apply(est, x, y, z, ex, ey, ez);
#pragma unroll
          for (int s = 0; s < kSymChunk; ++s) {
            if (s < ns) {
              double gx, gy, gz;
              apply(gsym[s], x, y, z, gx, gy, gz);
              const double dx = ex - gx, dy = ey - gy, dz = ez - gz;
              mx[s] = fmax(mx[s], sqrt(dx * dx + dy * dy + dz * dz));
            }
          }
        } else {
          double eu, ev;
          project(P_est, x, y, z, eu, ev);
#pragma unroll
          for (int s = 0; s < kSymChunk; ++s) {
            if (s < ns) {
              double gu, gv;
              project(P_gsym[s], x, y, z, gu, gv);
              const double du = eu - gu, dv = ev - gv;
              mx[s] = fmax(mx[s], sqrt(du * du + dv * dv));
            }
          }
        }
      }
#pragma unroll
      for (int s = 0; s < kSymChunk; ++s) {
        if (s < ns) {
          const double v = block_reduce<true>(mx[s], red);
          if (v < best) {
            best = v;
            best_s = static_cast<int>(c0 - s0) + s;
          }
        }
      }
      __syncthreads();  // gsym is rewritten by the next chunk
    }
    if (threadIdx.x == 0) {
      err[p] = best;
      if (sym_argmin) sym_argmin[p] = best_s;
    }
    return;
  }

  double sum = 0.0;
  if constexpr (kind == MPX_BOP_ADD) {
    for (long long i = threadIdx.x; i < n; i += kPointThreads) {
      const double x = P[3 * i], y = P[3 * i + 1], z = P[3 * i + 2];
      double ex, ey, ez, gx, gy, gz;
      apply(est, x, y, z, ex, ey, ez);
      apply(gt, x, y, z, gx, gy, gz);
      const double dx = ex - gx, dy = ey - gy, dz = ez - gz;
      sum += sqrt(dx * dx + dy * dy + dz * dz);
    }
  } else {  // ADI: for each point in the gt pose, the nearest point in the estimated pose
    for (long long b0 = 0; b0 < n; b0 += kPointThreads) {
      const long long i = b0 + threadIdx.x;
      double gx = 0, gy = 0, gz = 0;
      if (i < n) apply(gt, P[3 * i], P[3 * i + 1], P[3 * i + 2], gx, gy, gz);
      double best = __longlong_as_double(0x7ff0000000000000ll);
      for (long long t0 = 0; t0 < n; t0 += kPointThreads) {
        const long long j = t0 + threadIdx.x;
        __syncthreads();
        if (j < n) apply(est, P[3 * j], P[3 * j + 1], P[3 * j + 2], tile[threadIdx.x][0], tile[threadIdx.x][1],
                         tile[threadIdx.x][2]);
        __syncthreads();
        const int nt = static_cast<int>(min(static_cast<long long>(kPointThreads), n - t0));
        for (int k = 0; k < nt; ++k) {
          const double dx = gx - tile[k][0], dy = gy - tile[k][1], dz = gz - tile[k][2];
          best = fmin(best, dx * dx + dy * dy + dz * dz);
        }
      }
      if (i < n) sum += sqrt(best);
    }
  }
  const double total = block_reduce<false>(sum, red);
  if (threadIdx.x == 0) {
    err[p] = total / static_cast<double>(n);
    if (sym_argmin) sym_argmin[p] = 0;
  }
}

int bop_point_errors(int kind, int n_pairs, int n_models, const double* pts, const int64_t* pt_off, long long n_pts_total,
                     const double* syms, const int64_t* sym_off, long long n_syms_total, const int* model_idx,
                     const double* pose_est, const double* pose_gt, const double* K, double* err, int* sym_argmin,
                     cudaStream_t stream) {
  if (n_pairs == 0) return MPX_OK;
  auto kernel = kind == MPX_BOP_MSSD ? bop_point_kernel<MPX_BOP_MSSD>
                : kind == MPX_BOP_MSPD ? bop_point_kernel<MPX_BOP_MSPD>
                : kind == MPX_BOP_ADD  ? bop_point_kernel<MPX_BOP_ADD>
                                       : bop_point_kernel<MPX_BOP_ADI>;
  kernel<<<n_pairs, kPointThreads, 0, stream>>>(n_models, pts, pt_off, n_pts_total, syms, sym_off, n_syms_total, model_idx,
                                                pose_est, pose_gt, K, err, sym_argmin);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// PROJ, RE, TE (pose_error.proj, re, te)
// ---------------------------------------------------------------------------------------------------------------------
// pose_error.re: acos of 0.5 (trace(R_est inv(R_gt)) - 1), clipped to [-1, 1], in degrees.  The inverse is the true one
// (adjugate over determinant), not the transpose: rotations read from text are orthonormal only to their printed digits.
__device__ double rotation_error_deg(const double* e, const double* g) {
  const double c00 = __dadd_rn(__dmul_rn(g[4], g[8]), -__dmul_rn(g[5], g[7]));
  const double c01 = __dadd_rn(__dmul_rn(g[5], g[6]), -__dmul_rn(g[3], g[8]));
  const double c02 = __dadd_rn(__dmul_rn(g[3], g[7]), -__dmul_rn(g[4], g[6]));
  const double det = __dadd_rn(__dadd_rn(__dmul_rn(g[0], c00), __dmul_rn(g[1], c01)), __dmul_rn(g[2], c02));
  double inv[9];  // row-major inv(R_gt)
  inv[0] = __ddiv_rn(c00, det);
  inv[3] = __ddiv_rn(c01, det);
  inv[6] = __ddiv_rn(c02, det);
  inv[1] = __ddiv_rn(__dadd_rn(__dmul_rn(g[2], g[7]), -__dmul_rn(g[1], g[8])), det);
  inv[2] = __ddiv_rn(__dadd_rn(__dmul_rn(g[1], g[5]), -__dmul_rn(g[2], g[4])), det);
  inv[4] = __ddiv_rn(__dadd_rn(__dmul_rn(g[0], g[8]), -__dmul_rn(g[2], g[6])), det);
  inv[5] = __ddiv_rn(__dadd_rn(__dmul_rn(g[2], g[3]), -__dmul_rn(g[0], g[5])), det);
  inv[7] = __ddiv_rn(__dadd_rn(__dmul_rn(g[1], g[6]), -__dmul_rn(g[0], g[7])), det);
  inv[8] = __ddiv_rn(__dadd_rn(__dmul_rn(g[0], g[4]), -__dmul_rn(g[1], g[3])), det);
  double tr = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double d = __dadd_rn(__dadd_rn(__dmul_rn(e[3 * i], inv[i]), __dmul_rn(e[3 * i + 1], inv[3 + i])),
                               __dmul_rn(e[3 * i + 2], inv[6 + i]));
    tr = i ? __dadd_rn(tr, d) : d;
  }
  const double c = fmin(1.0, fmax(-1.0, __dmul_rn(0.5, __dadd_rn(tr, -1.0))));
  return __ddiv_rn(__dmul_rn(180.0, acos(c)), 3.141592653589793);
}

// pose_error.te: |t_gt - t_est| (mm)
__device__ double translation_error(const double* e, const double* g) {
  const double dx = __dadd_rn(g[9], -e[9]), dy = __dadd_rn(g[10], -e[10]), dz = __dadd_rn(g[11], -e[11]);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

// One CTA per pair.  Thread 0 writes RE / TE; with PROJ the CTA projects the model's points under both poses (P = K [R|t]
// formed first, as misc.project_pts) and sums the distances in ADD's fixed-order block reduction.
__global__ void __launch_bounds__(kPointThreads) bop_pose_kernel(
    int n_models, const double* __restrict__ pts, const int64_t* __restrict__ pt_off, long long n_pts_total,
    const int* __restrict__ model_idx, const double* __restrict__ pose_est, const double* __restrict__ pose_gt,
    const double* __restrict__ K, double* __restrict__ proj, double* __restrict__ re, double* __restrict__ te) {
  const int p = blockIdx.x;
  const double* pe = pose_est + 12 * p;
  const double* pg = pose_gt + 12 * p;
  if (threadIdx.x == 0) {
    if (re) re[p] = rotation_error_deg(pe, pg);
    if (te) te[p] = translation_error(pe, pg);
  }
  if (!proj) return;
  __shared__ Rt est, gt;
  __shared__ double P_est[12], P_gt[12];
  __shared__ double red[kPointThreads / 32];
  const int m = model_idx[p];
  long long p0 = 0, p1 = 0;
  if (m >= 0 && m < n_models) {
    p0 = max(0ll, min(static_cast<long long>(pt_off[m]), n_pts_total));
    p1 = max(p0, min(static_cast<long long>(pt_off[m + 1]), n_pts_total));
  }
  if (p1 == p0) {
    if (threadIdx.x == 0) proj[p] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  if (threadIdx.x < 12) (threadIdx.x < 9 ? est.R[threadIdx.x] : est.t[threadIdx.x - 9]) = pe[threadIdx.x];
  else if (threadIdx.x < 24) (threadIdx.x < 21 ? gt.R[threadIdx.x - 12] : gt.t[threadIdx.x - 21]) = pg[threadIdx.x - 12];
  __syncthreads();
  if (threadIdx.x == 0) make_P(K + 9 * p, est, P_est);
  else if (threadIdx.x == 32) make_P(K + 9 * p, gt, P_gt);
  __syncthreads();
  const long long n = p1 - p0;
  const double* P = pts + 3 * p0;
  double sum = 0.0;
  for (long long i = threadIdx.x; i < n; i += kPointThreads) {
    const double x = P[3 * i], y = P[3 * i + 1], z = P[3 * i + 2];
    double eu, ev, gu, gv;
    project(P_est, x, y, z, eu, ev);
    project(P_gt, x, y, z, gu, gv);
    const double du = eu - gu, dv = ev - gv;
    sum += sqrt(du * du + dv * dv);
  }
  const double total = block_reduce<false>(sum, red);
  if (threadIdx.x == 0) proj[p] = total / static_cast<double>(n);
}

int bop_pose_errors(int n_pairs, int n_models, const double* pts, const int64_t* pt_off, long long n_pts_total,
                    const int* model_idx, const double* pose_est, const double* pose_gt, const double* K, double* proj,
                    double* re, double* te, cudaStream_t stream) {
  if (n_pairs == 0 || (!proj && !re && !te)) return MPX_OK;
  // without PROJ one warp per pair is enough
  bop_pose_kernel<<<n_pairs, proj ? kPointThreads : 32, 0, stream>>>(n_models, pts, pt_off, n_pts_total, model_idx,
                                                                     pose_est, pose_gt, K, proj, re, te);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

}  // namespace mpx
