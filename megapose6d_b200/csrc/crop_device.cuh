// Device-side roi_align arithmetic shared by crop.cu (stand-alone crop kernel) and raster.cu (crop fused
// into the render resolve pass).  torchvision.ops.roi_align semantics as used by the reference
// (src/megapose/lib3d/cropping.py:113-144: sampling_ratio 4, aligned=False, spatial_scale 1).
#pragma once
#include "mpx_common.cuh"

namespace mpx {

struct RoiParams {
  float x1, y1, bin_w, bin_h;
};

__device__ __forceinline__ RoiParams make_roi(const float* __restrict__ box, int oh, int ow) {
  RoiParams r;
  const float x1 = box[0], y1 = box[1], x2 = box[2], y2 = box[3];
  const float roi_w = fmaxf(x2 - x1, 1.f), roi_h = fmaxf(y2 - y1, 1.f);
  r.x1 = x1;
  r.y1 = y1;
  r.bin_w = roi_w / static_cast<float>(ow);
  r.bin_h = roi_h / static_cast<float>(oh);
  return r;
}

// One axis of a bilinear sample, torchvision rules: coordinate -> (low, high, l, h) or invalid.
struct AxisTap {
  int lo, hi;
  float l, h;
  bool ok;
};
__device__ __forceinline__ AxisTap axis_tap(float v, int size) {
  AxisTap t;
  t.ok = !(v < -1.0f || v > static_cast<float>(size));
  if (v <= 0.f) v = 0.f;
  int lo = static_cast<int>(v);
  if (lo >= size - 1) {
    t.hi = lo = size - 1;
    v = static_cast<float>(lo);
  } else {
    t.hi = lo + 1;
  }
  t.lo = lo;
  t.l = v - lo;
  t.h = 1.f - t.l;
  return t;
}

// Average of the 4x4 bilinear samples of output pixel (ph, pw); acc.w carries depth, vacc the averaged
// depth-validity mask (only accumulated when WITH_DEPTH).  The per-axis work (bounds, floor, weights) is done
// once per sample row / column instead of once per sample, and the 2x2 texel block of the previous sample is kept
// in registers: with bins smaller than a pixel most of the 16 samples share it.  Every floating-point operation
// and its order are those of torchvision's kernel, except that a tap of zero weight (a sample on an integer row /
// column, or clamped to the last one) adds 0 instead of 0 * texel: a NaN or inf texel reached only through zero weights
// does not make the sum NaN.  The collapsed form skips such taps, and a crop must not depend on which form its size
// selects.  Finite texels give the same sums either way.
template <bool WITH_DEPTH>
__device__ __forceinline__ void roi_align_pixel(const float4* __restrict__ img, int h, int w, const RoiParams& r,
                                                int ph, int pw, float4& acc, float& vacc) {
  acc = make_float4(0.f, 0.f, 0.f, 0.f);
  vacc = 0.f;
  AxisTap tx[4];
#pragma unroll
  for (int ix = 0; ix < 4; ++ix) tx[ix] = axis_tap(r.x1 + pw * r.bin_w + (ix + 0.5f) * r.bin_w / 4.f, w);
  int cy0 = -1, cy1 = -1, cx0 = -1, cx1 = -1;
  float4 v1 = acc, v2 = acc, v3 = acc, v4 = acc;
#pragma unroll
  for (int iy = 0; iy < 4; ++iy) {
    const AxisTap ty = axis_tap(r.y1 + ph * r.bin_h + (iy + 0.5f) * r.bin_h / 4.f, h);
    if (!ty.ok) continue;
#pragma unroll
    for (int ix = 0; ix < 4; ++ix) {
      if (!tx[ix].ok) continue;
      if (ty.lo != cy0 || ty.hi != cy1 || tx[ix].lo != cx0 || tx[ix].hi != cx1) {
        v1 = __ldg(img + ty.lo * w + tx[ix].lo);
        v2 = __ldg(img + ty.lo * w + tx[ix].hi);
        v3 = __ldg(img + ty.hi * w + tx[ix].lo);
        v4 = __ldg(img + ty.hi * w + tx[ix].hi);
        cy0 = ty.lo; cy1 = ty.hi; cx0 = tx[ix].lo; cx1 = tx[ix].hi;
      }
      const float w1 = ty.h * tx[ix].h, w2 = ty.h * tx[ix].l, w3 = ty.l * tx[ix].h, w4 = ty.l * tx[ix].l;
      // the high taps weigh 0 exactly when l == 0 on their axis (h = 1 - l is never 0): their texels count as 0
      const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
      const bool x0 = tx[ix].l == 0.f, y0 = ty.l == 0.f;
      const float4 u2 = x0 ? z4 : v2, u3 = y0 ? z4 : v3, u4 = (x0 || y0) ? z4 : v4;
      acc.x += w1 * v1.x + w2 * u2.x + w3 * u3.x + w4 * u4.x;
      acc.y += w1 * v1.y + w2 * u2.y + w3 * u3.y + w4 * u4.y;
      acc.z += w1 * v1.z + w2 * u2.z + w3 * u3.z + w4 * u4.z;
      if (WITH_DEPTH) {
        acc.w += w1 * v1.w + w2 * u2.w + w3 * u3.w + w4 * u4.w;
        vacc += w1 * (v1.w > 0.f ? 1.f : 0.f) + w2 * (u2.w > 0.f ? 1.f : 0.f) + w3 * (u3.w > 0.f ? 1.f : 0.f) +
                w4 * (u4.w > 0.f ? 1.f : 0.f);
      }
    }
  }
  acc.x /= 16.f;
  acc.y /= 16.f;
  acc.z /= 16.f;
  if (WITH_DEPTH) {
    acc.w /= 16.f;
    vacc /= 16.f;
  }
}

// ---------------------------------------------------------------------------------------------
// Collapsed form.  The bilinear weight of a sample factors into a row weight and a column weight, so the average
// of the 4x4 samples of one output pixel is  sum_a sum_b Wy[a] * Wx[b] * img[y0 + a][x0 + b]  with
// Wy[a] = (1/4) * sum over the 4 sample rows of their weight on image row y0 + a (same for columns).  When the four
// sample coordinates of an output row / column touch at most four consecutive image rows / columns (bin < 2.67 px:
// every crop that is not a strong minification) the 64 taps of the plain form become <= 16, usually 4-9.
// Sample coordinates, floor / clamp decisions and the validity rule are those of torchvision (axis_tap); only the
// order of the fp32 additions differs (tests: 2e-5).  AxisW entries live in shared memory, one per output row and
// one per output column of a crop, built once per crop.
// ---------------------------------------------------------------------------------------------
struct AxisW {
  int base;    // first image row / column touched
  float w[4];  // collapsed weights on base .. base+3 (1/4 folded in); zero weight = not touched
};

// returns false when the four samples span more than four image rows / columns
__device__ __forceinline__ bool axis_collapse(float start, float bin, int p, int size, AxisW& e) {
  AxisTap t[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) t[k] = axis_tap(start + p * bin + (k + 0.5f) * bin / 4.f, size);
  e.base = t[0].lo;
  float w0 = 0.f, w1 = 0.f, w2 = 0.f, w3 = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (!t[k].ok) continue;
    const int a = t[k].lo - e.base, b = t[k].hi - e.base;
    w0 += (a == 0 ? t[k].h : 0.f) + (b == 0 ? t[k].l : 0.f);
    w1 += (a == 1 ? t[k].h : 0.f) + (b == 1 ? t[k].l : 0.f);
    w2 += (a == 2 ? t[k].h : 0.f) + (b == 2 ? t[k].l : 0.f);
    w3 += (a == 3 ? t[k].h : 0.f) + (b == 3 ? t[k].l : 0.f);
  }
  e.w[0] = 0.25f * w0;
  e.w[1] = 0.25f * w1;
  e.w[2] = 0.25f * w2;
  e.w[3] = 0.25f * w3;
  return t[3].hi - e.base <= 3;
}

// Fills ay[0..oh) and ax[0..ow) (shared memory) with all threads of the CTA; returns (to every thread, via
// __syncthreads_and) whether the collapsed form is valid for this crop.  Contains a barrier.
__device__ __forceinline__ bool build_axis_tables(const RoiParams& r, int oh, int ow, int h, int w, AxisW* ay,
                                                  AxisW* ax) {
  bool ok = true;
  for (int p = threadIdx.x; p < oh + ow; p += blockDim.x) {
    AxisW e;
    if (p < oh) {
      ok = axis_collapse(r.y1, r.bin_h, p, h, e) && ok;
      ay[p] = e;
    } else {
      ok = axis_collapse(r.x1, r.bin_w, p - oh, w, e) && ok;
      ax[p - oh] = e;
    }
  }
  return __syncthreads_and(ok ? 1 : 0) != 0;
}

template <bool WITH_DEPTH>
__device__ __forceinline__ void roi_align_pixel_collapsed(const float4* __restrict__ img, int w, const AxisW& ey,
                                                          const AxisW& ex, float4& acc, float& vacc) {
  acc = make_float4(0.f, 0.f, 0.f, 0.f);
  vacc = 0.f;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const float wy = ey.w[a];
    if (wy == 0.f) continue;
    const float4* row = img + static_cast<size_t>(ey.base + a) * w + ex.base;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const float wx = ex.w[b];
      if (wx == 0.f) continue;
      const float4 v = __ldg(row + b);
      const float wgt = wy * wx;
      acc.x += wgt * v.x;
      acc.y += wgt * v.y;
      acc.z += wgt * v.z;
      if (WITH_DEPTH) {
        acc.w += wgt * v.w;
        vacc += v.w > 0.f ? wgt : 0.f;
      }
    }
  }
}

constexpr int kAxisTableMax = 1024;  // oh + ow entries of shared memory (20 KB) per CTA

}  // namespace mpx
