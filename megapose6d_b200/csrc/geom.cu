// Hypothesis geometry: the dozens of tiny ATen kernels the reference launches per batch for pose
// initialisation, projection, crop boxes, crop intrinsics, multi-view cameras and pose update are
// each one fused kernel here (one CTA or one thread per hypothesis).
//
// reference: src/megapose/lib3d/cosypose_ops.py:33-58,169-218; lib3d/camera_geometry.py:40-115;
//            lib3d/cropping.py:30-110; lib3d/transform_ops.py:106-119; lib3d/rotations.py:25-40;
//            lib3d/multiview.py:31-92,165-246; models/pose_rigid.py:180-303,305-312;
//            inference/pose_estimator.py:643-667.
#include <climits>

#include "mpx_common.cuh"

namespace mpx {

// ---------------------------------------------------------------------------------------------
// block-wide min/max helpers (blockDim.x multiple of 32, <= 1024)
// ---------------------------------------------------------------------------------------------
// fminf/fmaxf drop NaN; torch's min/max reductions and torch.max(a, b) return it.  The reductions below keep the fast
// fminf/fmaxf and carry an "any NaN" bit per coordinate instead (bit 0: coordinate 0, bit 1: coordinate 1); a flagged
// coordinate's min and max are NaN, as torch computes them.
__device__ __forceinline__ unsigned nan_bits(float c0, float c1) {
  return (c0 != c0 ? 1u : 0u) | (c1 != c1 ? 2u : 0u);
}
// torch.max(a, b) (elementwise): NaN if either operand is NaN, fmaxf otherwise
__device__ __forceinline__ float max_nan(float a, float b) { return a != a ? a : (b != b ? b : fmaxf(a, b)); }

__device__ __forceinline__ void block_minmax4(float& mn0, float& mx0, float& mn1, float& mx1, unsigned nan, float* sm) {
  __shared__ unsigned s_nan;
  if (threadIdx.x == 0) s_nan = 0u;
  mn0 = warp_min(mn0); mx0 = warp_max(mx0); mn1 = warp_min(mn1); mx1 = warp_max(mx1);
  nan = __reduce_or_sync(0xffffffffu, nan);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();  // s_nan cleared before any warp adds to it
  if (lane == 0) {
    sm[warp * 4 + 0] = mn0; sm[warp * 4 + 1] = mx0; sm[warp * 4 + 2] = mn1; sm[warp * 4 + 3] = mx1;
    if (nan) atomicOr(&s_nan, nan);
  }
  __syncthreads();
  if (warp == 0) {
    float a = lane < nw ? sm[lane * 4 + 0] : INFINITY;
    float b = lane < nw ? sm[lane * 4 + 1] : -INFINITY;
    float c = lane < nw ? sm[lane * 4 + 2] : INFINITY;
    float d = lane < nw ? sm[lane * 4 + 3] : -INFINITY;
    a = warp_min(a); b = warp_max(b); c = warp_min(c); d = warp_max(d);
    if (lane == 0) {
      const unsigned f = s_nan;
      if (f & 1u) a = b = NAN;
      if (f & 2u) c = d = NAN;
      sm[0] = a; sm[1] = b; sm[2] = c; sm[3] = d;
    }
  }
  __syncthreads();
  mn0 = sm[0]; mx0 = sm[1]; mn1 = sm[2]; mx1 = sm[3];
}

// ---------------------------------------------------------------------------------------------
// TCO_init_from_boxes_autodepth_with_R  (cosypose_ops.py:169-218)
// ---------------------------------------------------------------------------------------------
__global__ void pose_init_kernel(const float* __restrict__ points, int n_pts, const int* __restrict__ label_idx,
                                 const float* __restrict__ bboxes, const float* __restrict__ K,
                                 const float* __restrict__ R, float* __restrict__ TCO) {
  __shared__ float sm[128];
  const int n = blockIdx.x;
  const float* Kn = K + 9 * n;
  const float* Rn = R + 9 * n;
  const float* bb = bboxes + 4 * n;
  const float fx = Kn[0], fy = Kn[4], cx = Kn[2], cy = Kn[5];
  const float bcx = (bb[0] + bb[2]) / 2.f, bcy = (bb[1] + bb[3]) / 2.f;
  const float z_guess = 1.0f;
  const float tx = ((bcx - cx) * z_guess) / fx, ty = ((bcy - cy) * z_guess) / fy;
  const float* pts = points + static_cast<size_t>(label_idx[n]) * n_pts * 3;
  float mnx = INFINITY, mxx = -INFINITY, mny = INFINITY, mxy = -INFINITY;
  unsigned nan = 0u;
  for (int i = threadIdx.x; i < n_pts; i += blockDim.x) {
    const float px = __ldg(pts + 3 * i), py = __ldg(pts + 3 * i + 1), pz = __ldg(pts + 3 * i + 2);
    const float x = Rn[0] * px + Rn[1] * py + Rn[2] * pz + tx;
    const float y = Rn[3] * px + Rn[4] * py + Rn[5] * pz + ty;
    mnx = fminf(mnx, x); mxx = fmaxf(mxx, x);
    mny = fminf(mny, y); mxy = fmaxf(mxy, y);
    nan |= nan_bits(x, y);
  }
  block_minmax4(mnx, mxx, mny, mxy, nan, sm);
  if (threadIdx.x == 0) {
    const float deltax = mxx - mnx, deltay = mxy - mny;
    const float bb_dx = (bb[2] - bb[0]) + 1.f, bb_dy = (bb[3] - bb[1]) + 1.f;
    const float z_from_dx = fx * deltax / bb_dx;
    const float z_from_dy = fy * deltay / bb_dy;
    const float z = (z_from_dy + z_from_dx) / 2.f;
    float* T = TCO + 16 * n;
    T[0] = Rn[0]; T[1] = Rn[1]; T[2] = Rn[2];   T[3] = ((bcx - cx) * z) / fx;
    T[4] = Rn[3]; T[5] = Rn[4]; T[6] = Rn[5];   T[7] = ((bcy - cy) * z) / fy;
    T[8] = Rn[6]; T[9] = Rn[7]; T[10] = Rn[8];  T[11] = z;
    T[12] = 0.f;  T[13] = 0.f;  T[14] = 0.f;    T[15] = 1.f;
  }
}

int pose_init_autodepth(const float* points, int n_pts, const int* label_idx, const float* bboxes,
                        const float* K, const float* R, int n, float* TCO, cudaStream_t stream) {
  if (n == 0) return MPX_OK;
  MPX_REQUIRE(n_pts > 0, "pose_init: empty point set");
  pose_init_kernel<<<n, 256, 0, stream>>>(points, n_pts, label_idx, bboxes, K, R, TCO);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------
// ortho6d -> rotation (rotations.py:25-40); columns are (x, y, z)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void ortho6d(const float* xr, const float* yr, float* Rm /*row-major 3x3*/) {
  const float nx = sqrtf(xr[0] * xr[0] + xr[1] * xr[1] + xr[2] * xr[2]);
  const float x0 = xr[0] / nx, x1 = xr[1] / nx, x2 = xr[2] / nx;
  float z0 = x1 * yr[2] - x2 * yr[1];
  float z1 = x2 * yr[0] - x0 * yr[2];
  float z2 = x0 * yr[1] - x1 * yr[0];
  const float nz = sqrtf(z0 * z0 + z1 * z1 + z2 * z2);
  z0 /= nz; z1 /= nz; z2 /= nz;
  const float y0 = z1 * x2 - z2 * x1;
  const float y1 = z2 * x0 - z0 * x2;
  const float y2 = z0 * x1 - z1 * x0;
  Rm[0] = x0; Rm[1] = y0; Rm[2] = z0;
  Rm[3] = x1; Rm[4] = y1; Rm[5] = z1;
  Rm[6] = x2; Rm[7] = y2; Rm[8] = z2;
}

__global__ void normalize_T_kernel(const float* __restrict__ Tin, int n, float* __restrict__ Tout) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* T = Tin + 16 * i;
  const float c0[3] = {T[0], T[4], T[8]};
  const float c1[3] = {T[1], T[5], T[9]};
  const float t[3] = {T[3], T[7], T[11]};
  float Rm[9];
  ortho6d(c0, c1, Rm);
  float* o = Tout + 16 * i;
  o[0] = Rm[0]; o[1] = Rm[1]; o[2] = Rm[2];  o[3] = t[0];
  o[4] = Rm[3]; o[5] = Rm[4]; o[6] = Rm[5];  o[7] = t[1];
  o[8] = Rm[6]; o[9] = Rm[7]; o[10] = Rm[8]; o[11] = t[2];
  o[12] = 0.f;  o[13] = 0.f;  o[14] = 0.f;   o[15] = 1.f;
}

int normalize_T(const float* Tin, int n, float* Tout, cudaStream_t stream) {
  if (n == 0) return MPX_OK;
  normalize_T_kernel<<<(n + 127) / 128, 128, 0, stream>>>(Tin, n, Tout);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------
// crop geometry: project_points_robust + boxes_from_uv + deepim_boxes + get_K_crop_resize
// one CTA (128 threads) per hypothesis
// ---------------------------------------------------------------------------------------------
__global__ void crop_geometry_kernel(const float* __restrict__ points, int n_pts, const int* __restrict__ label_idx,
                                     const float* __restrict__ TCO, const float* __restrict__ K,
                                     const float* __restrict__ tCR, float lamb, int im_h, int im_w, int out_h,
                                     int out_w, float* __restrict__ boxes_rend, float* __restrict__ boxes_crop,
                                     float* __restrict__ K_crop) {
  __shared__ float sm[64];
  __shared__ float P[12];
  const int n = blockIdx.x;
  const float* Kn = K + 9 * n;
  const float* T = TCO + 16 * n;
  if (threadIdx.x < 12) {
    // P = K @ TCO[:3]  (3x4)
    const int r = threadIdx.x / 4, c = threadIdx.x % 4;
    P[threadIdx.x] = Kn[r * 3 + 0] * T[c] + Kn[r * 3 + 1] * T[4 + c] + Kn[r * 3 + 2] * T[8 + c];
  }
  __syncthreads();
  const float* pts = points + static_cast<size_t>(label_idx[n]) * n_pts * 3;
  float mnu = INFINITY, mxu = -INFINITY, mnv = INFINITY, mxv = -INFINITY;
  unsigned nan = 0u;
  for (int i = threadIdx.x; i < n_pts; i += blockDim.x) {
    const float px = __ldg(pts + 3 * i), py = __ldg(pts + 3 * i + 1), pz = __ldg(pts + 3 * i + 2);
    const float su = P[0] * px + P[1] * py + P[2] * pz + P[3];
    const float sv = P[4] * px + P[5] * py + P[6] * pz + P[7];
    float sz = P[8] * px + P[9] * py + P[10] * pz + P[11];
    sz = max_nan(0.1f, sz);
    const float u = su / sz, v = sv / sz;
    mnu = fminf(mnu, u); mxu = fmaxf(mxu, u);
    mnv = fminf(mnv, v); mxv = fmaxf(mxv, v);
    nan |= nan_bits(u, v);
  }
  block_minmax4(mnu, mxu, mnv, mxv, nan, sm);
  if (threadIdx.x == 0) {
    const float x1 = mnu, y1 = mnv, x2 = mxu, y2 = mxv;
    float* br = boxes_rend + 4 * n;
    br[0] = x1; br[1] = y1; br[2] = x2; br[3] = y2;
    // reference point projection: K @ tCR, z clamped.  The reference projects the origin through K @ [R | tCR], so a
    // non-finite entry of row r of K @ R reaches row r of its result as inf * 0 = NaN (or NaN * 0)
    const float* tr = tCR + 3 * n;
    float cu = Kn[0] * tr[0] + Kn[1] * tr[1] + Kn[2] * tr[2];
    float cv = Kn[3] * tr[0] + Kn[4] * tr[1] + Kn[5] * tr[2];
    float cz = Kn[6] * tr[0] + Kn[7] * tr[1] + Kn[8] * tr[2];
    if (!(isfinite(P[0]) && isfinite(P[1]) && isfinite(P[2]))) cu = NAN;
    if (!(isfinite(P[4]) && isfinite(P[5]) && isfinite(P[6]))) cv = NAN;
    if (!(isfinite(P[8]) && isfinite(P[9]) && isfinite(P[10]))) cz = NAN;
    cz = max_nan(0.1f, cz);
    const float xc = cu / cz, yc = cv / cz;
    // deepim_boxes with obs_boxes == rend_boxes (pose_rigid.py:218-229); torch.max propagates NaN
    const float wmax = static_cast<float>(max(im_h, im_w)), hmin = static_cast<float>(min(im_h, im_w));
    const float r = static_cast<float>(static_cast<double>(wmax) / static_cast<double>(hmin));
    const float xdist = max_nan(fabsf(x1 - xc), fabsf(x2 - xc));
    const float ydist = max_nan(fabsf(y1 - yc), fabsf(y2 - yc));
    const float width = max_nan(xdist, ydist * r) * 2.f * lamb;
    const float height = max_nan(xdist / r, ydist) * 2.f * lamb;
    const float bx1 = xc - width / 2.f, by1 = yc - height / 2.f;
    const float bx2 = xc + width / 2.f, by2 = yc + height / 2.f;
    float* bc = boxes_crop + 4 * n;
    bc[0] = bx1; bc[1] = by1; bc[2] = bx2; bc[3] = by2;
    // get_K_crop_resize (camera_geometry.py:67-115)
    const float final_w = static_cast<float>(max(out_h, out_w));
    const float final_h = static_cast<float>(min(out_h, out_w));
    const float crop_w = bx2 - bx1, crop_h = by2 - by1;
    const float crop_cj = (bx1 + bx2) / 2.f, crop_ci = (by1 + by2) / 2.f;
    const float cx = Kn[2] + (crop_w - 1.f) / 2.f - crop_cj;
    const float cy = Kn[5] + (crop_h - 1.f) / 2.f - crop_ci;
    const float center_x = (crop_w - 1.f) / 2.f, center_y = (crop_h - 1.f) / 2.f;
    const float dcx = cx - center_x, dcy = cy - center_y;
    const float sx = final_w / crop_w, sy = final_h / crop_h;
    float* Ko = K_crop + 9 * n;
    for (int i = 0; i < 9; ++i) Ko[i] = Kn[i];
    Ko[0] = sx * Kn[0];
    Ko[4] = sy * Kn[4];
    Ko[2] = (final_w - 1.f) / 2.f + sx * dcx;
    Ko[5] = (final_h - 1.f) / 2.f + sy * dcy;
  }
}

int crop_geometry(const float* points, int n_pts, const int* label_idx, const float* TCO, const float* K,
                  const float* tCR, int n, float lamb, int im_h, int im_w, int out_h, int out_w,
                  float* boxes_rend, float* boxes_crop, float* K_crop, cudaStream_t stream) {
  if (n == 0) return MPX_OK;
  MPX_REQUIRE(n_pts > 0, "crop_geometry: empty point set");
  crop_geometry_kernel<<<n, 128, 0, stream>>>(points, n_pts, label_idx, TCO, K, tCR, lamb, im_h, im_w, out_h,
                                              out_w, boxes_rend, boxes_crop, K_crop);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------
// multi-view cameras (multiview.py:31-92, 165-246), closed form in float64
// ---------------------------------------------------------------------------------------------
struct M4 { double m[16]; };

__device__ __forceinline__ void mat_mul4(const double* a, const double* b, double* o) {
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) {
      double s = 0.0;
      for (int k = 0; k < 4; ++k) s += a[r * 4 + k] * b[k * 4 + c];
      o[r * 4 + c] = s;
    }
}
__device__ __forceinline__ void rigid_inverse(const double* T, double* o) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) o[r * 4 + c] = T[c * 4 + r];
  for (int r = 0; r < 3; ++r)
    o[r * 4 + 3] = -(o[r * 4 + 0] * T[3] + o[r * 4 + 1] * T[7] + o[r * 4 + 2] * T[11]);
  o[12] = 0; o[13] = 0; o[14] = 0; o[15] = 1;
}
// Panda3D look-at in its Z-up right-handed frame: +Y forward, X = Y x up, Z = X x Y.
__device__ __forceinline__ void look_at(const double* fwd, const double* up, double* R /*3x3 row-major, cols x y z*/) {
  double y[3] = {fwd[0], fwd[1], fwd[2]};
  double ny = sqrt(y[0] * y[0] + y[1] * y[1] + y[2] * y[2]);
  for (int i = 0; i < 3; ++i) y[i] /= ny;
  double x[3] = {y[1] * up[2] - y[2] * up[1], y[2] * up[0] - y[0] * up[2], y[0] * up[1] - y[1] * up[0]};
  double nx = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
  for (int i = 0; i < 3; ++i) x[i] /= nx;
  const double z[3] = {x[1] * y[2] - x[2] * y[1], x[2] * y[0] - x[0] * y[2], x[0] * y[1] - x[1] * y[0]};
  for (int i = 0; i < 3; ++i) { R[i * 3 + 0] = x[i]; R[i * 3 + 1] = y[i]; R[i * 3 + 2] = z[i]; }
}

struct ViewOffsets { float v[96]; };

__global__ void multiview_kernel(const float* __restrict__ TCO, const float* __restrict__ tCR, int n,
                                 const ViewOffsets offs, int n_extra, float* __restrict__ TCV_O) {
  const float* offsets = offs.v;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int V = 1 + n_extra;
  double T[16], tcr[3];
  bool finite = true;
  for (int k = 0; k < 16; ++k) { T[k] = static_cast<double>(TCO[16 * i + k]); finite = finite && isfinite(T[k]); }
  for (int k = 0; k < 3; ++k) tcr[k] = static_cast<double>(tCR[3 * i + k]);
  float* out = TCV_O + static_cast<size_t>(i) * V * 16;
  for (int k = 0; k < 16; ++k) out[k] = TCO[16 * i + k];  // view 0 = inv(I) @ TCO
  double TOC[16];
  rigid_inverse(T, TOC);
  for (int k = 0; k < 16; ++k) finite = finite && isfinite(TOC[k]);
  if (!finite) {
    for (int k = 0; k < 16; ++k) TOC[k] = (k % 5 == 0) ? 1.0 : 0.0;
    tcr[0] = tcr[1] = tcr[2] = 0.0;
  }
  const double CCGL[16] = {1, 0, 0, 0, 0, 0, -1, 0, 0, 1, 0, 0, 0, 0, 0, 1};
  const double CCGL_inv[16] = {1, 0, 0, 0, 0, 0, 1, 0, 0, -1, 0, 0, 0, 0, 0, 1};
  double Wc0[16], Wc0_inv[16];
  mat_mul4(TOC, CCGL, Wc0);
  rigid_inverse(Wc0, Wc0_inv);
  const double c0[3] = {Wc0[3], Wc0[7], Wc0[11]};
  const double ref[3] = {TOC[0] * tcr[0] + TOC[1] * tcr[1] + TOC[2] * tcr[2] + TOC[3],
                         TOC[4] * tcr[0] + TOC[5] * tcr[1] + TOC[6] * tcr[2] + TOC[7],
                         TOC[8] * tcr[0] + TOC[9] * tcr[1] + TOC[10] * tcr[2] + TOC[11]};
  const double radius = sqrt(tcr[0] * tcr[0] + tcr[1] * tcr[1] + tcr[2] * tcr[2]);
  const double up[3] = {Wc0[2], Wc0[6], Wc0[10]};
  double fwd[3] = {ref[0] - c0[0], ref[1] - c0[1], ref[2] - c0[2]};
  double RP[9];
  look_at(fwd, up, RP);
  for (int v = 0; v < n_extra; ++v) {
    const double o[3] = {offsets[3 * v] * radius, offsets[3 * v + 1] * radius, offsets[3 * v + 2] * radius};
    double p[3];
    for (int r = 0; r < 3; ++r) p[r] = c0[r] + RP[r * 3] * o[0] + RP[r * 3 + 1] * o[1] + RP[r * 3 + 2] * o[2];
    double f2[3] = {ref[0] - p[0], ref[1] - p[1], ref[2] - p[2]};
    double Rn[9];
    look_at(f2, up, Rn);
    double Wn[16] = {Rn[0], Rn[1], Rn[2], p[0], Rn[3], Rn[4], Rn[5], p[1], Rn[6], Rn[7], Rn[8], p[2], 0, 0, 0, 1};
    double c0n[16], tmp[16], C0CV[16], CVC0[16], res[16];
    mat_mul4(Wc0_inv, Wn, c0n);
    mat_mul4(CCGL, c0n, tmp);
    mat_mul4(tmp, CCGL_inv, C0CV);
    rigid_inverse(C0CV, CVC0);
    mat_mul4(CVC0, T, res);
    float* ov = out + 16 * (v + 1);
    for (int k = 0; k < 16; ++k) ov[k] = static_cast<float>(res[k]);
  }
}

int multiview_cameras(const float* TCO, const float* tCR, int n, const float* h_offsets, int n_extra,
                      float* TCV_O, cudaStream_t stream) {
  if (n == 0) return MPX_OK;
  MPX_REQUIRE(n_extra >= 0 && n_extra <= 32, "multiview: n_extra=%d unsupported", n_extra);
  ViewOffsets offs;
  memset(&offs, 0, sizeof(offs));
  for (int i = 0; i < 3 * n_extra; ++i) offs.v[i] = h_offsets[i];
  multiview_kernel<<<(n + 63) / 64, 64, 0, stream>>>(TCO, tCR, n, offs, n_extra, TCV_O);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------
// pose update (pose_rigid.py:305-312, cosypose_ops.py:33-58)
// ---------------------------------------------------------------------------------------------
__global__ void pose_update_kernel(const float* __restrict__ TCO, const float* __restrict__ K_crop,
                                   const float* __restrict__ pose9, const float* __restrict__ tCR, int n,
                                   float* __restrict__ TCO_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* T = TCO + 16 * i;
  const float* Kc = K_crop + 9 * i;
  const float* o9 = pose9 + 9 * i;
  const float* tr = tCR + 3 * i;
  float dR[9];
  ortho6d(o9, o9 + 3, dR);
  const float vx = o9[6], vy = o9[7], vz = o9[8];
  const float zsrc = tr[2];
  const float ztgt = vz * zsrc;
  const float fx = Kc[0], fy = Kc[4];
  const float tox = (vx / fx + tr[0] / zsrc) * ztgt;
  const float toy = (vy / fy + tr[1] / zsrc) * ztgt;
  const float d0 = T[3] - tr[0], d1 = T[7] - tr[1], d2 = T[11] - tr[2];
  float* o = TCO_out + 16 * i;
  float Rn[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      Rn[r * 3 + c] = dR[r * 3 + 0] * T[0 * 4 + c] + dR[r * 3 + 1] * T[1 * 4 + c] + dR[r * 3 + 2] * T[2 * 4 + c];
  const float t0 = dR[0] * d0 + dR[1] * d1 + dR[2] * d2 + tox;
  const float t1 = dR[3] * d0 + dR[4] * d1 + dR[5] * d2 + toy;
  const float t2 = dR[6] * d0 + dR[7] * d1 + dR[8] * d2 + ztgt;
  o[0] = Rn[0]; o[1] = Rn[1]; o[2] = Rn[2];  o[3] = t0;
  o[4] = Rn[3]; o[5] = Rn[4]; o[6] = Rn[5];  o[7] = t1;
  o[8] = Rn[6]; o[9] = Rn[7]; o[10] = Rn[8]; o[11] = t2;
  o[12] = T[12]; o[13] = T[13]; o[14] = T[14]; o[15] = T[15];
}

int pose_update(const float* TCO, const float* K_crop, const float* pose9, const float* tCR, int n,
                float* TCO_out, cudaStream_t stream) {
  if (n == 0) return MPX_OK;
  pose_update_kernel<<<(n + 127) / 128, 128, 0, stream>>>(TCO, K_crop, pose9, tCR, n, TCO_out);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------
// top-K per detection (pose_estimator.py:643-667 for the coarse stage); one CTA per group
// ---------------------------------------------------------------------------------------------
// Logits are compared as order-preserving integer keys: a float's bits with the magnitude bits flipped when negative, -0
// taken as +0 (a tie, as in every sort).  NaN gets a key below -inf's, so it sorts after every number (pandas
// sort_values(ascending=False), numpy argsort of -x), and an entry already selected gets the lowest key of all.
constexpr int kTopkNanKey = INT_MIN + 1;
constexpr int kTopkTakenKey = INT_MIN;
__device__ __forceinline__ int topk_key(float v) {
  if (v != v) return kTopkNanKey;
  const int b = __float_as_int(v == 0.f ? 0.f : v);
  return b >= 0 ? b : b ^ 0x7fffffff;
}

__global__ void topk_kernel(const float* __restrict__ logits, int m, int k, int* __restrict__ idx) {
  extern __shared__ int keys[];  // [m]
  __shared__ int s_best[32];
  __shared__ int s_idx[32];
  const int g = blockIdx.x;
  for (int i = threadIdx.x; i < m; i += blockDim.x) keys[i] = topk_key(logits[static_cast<size_t>(g) * m + i]);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  // every untaken entry has a key above kTopkTakenKey, and k <= m leaves one untaken: each round selects a real entry,
  // the highest key with ties to the lowest index
  for (int sel = 0; sel < k; ++sel) {
    int best = kTopkTakenKey;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
      const int v = keys[i];
      if (v > best || (v == best && i < bi)) { best = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const int ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) { s_best[warp] = best; s_idx[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
      best = lane < nw ? s_best[lane] : kTopkTakenKey;
      bi = lane < nw ? s_idx[lane] : 0x7fffffff;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const int ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
      }
      if (lane == 0) {
        idx[static_cast<size_t>(g) * k + sel] = bi;
        keys[bi] = kTopkTakenKey;
      }
    }
    __syncthreads();
  }
}

int topk_per_group(const float* logits, int n_groups, int m, int k, int* idx, cudaStream_t stream) {
  if (n_groups == 0 || k == 0) return MPX_OK;
  MPX_REQUIRE(k <= m, "topk: k=%d > m=%d", k, m);
  MPX_REQUIRE(m <= 12000, "topk: m=%d too large", m);
  topk_kernel<<<n_groups, 256, m * sizeof(float), stream>>>(logits, m, k, idx);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

}  // namespace mpx
