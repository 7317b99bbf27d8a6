// Batched software rasteriser for sm_90a: one persistent CTA per view.
//
// Replaces the Panda3D/OpenGL path of the reference renderer
// (reference: src/megapose/panda3d_renderer/panda3d_batch_renderer.py:217-282 render,
//  :89-150 worker_loop; panda3d_scene_renderer.py:298-358 render_scene (pass 1 albedo under
//  ambient light, pass 2 eye-normal texture); types.py:58-101 camera model, near/far 0.1/10;
//  utils.py:44-68 depth linearisation and the 32^3 normal texture).
//
// Contract (restated in oracle/raster_ref.c, which this kernel must match bit for bit):
//   * pinhole projection u = fx*X/Z + cx, v = fy*Y/Z + cy; pixel (i, j) is sampled at
//     (u, v) = (j + 0.5, i + 0.5) (SURVEY A.2);
//   * vertices snapped to 1/256 pixel; coverage by exact 64-bit integer edge functions, edges
//     inclusive, two-sided; the fragment with the largest interpolated 1/z wins, ties go to the lower
//     triangle index;
//   * fragments with 1/z outside [1/10, 1/0.1] are rejected: 1/z is linear in screen space, so this per-sample test clips
//     every triangle exactly at the lens' near and far planes (types.py:63-64); only triangles with a vertex within 2^-10 m
//     of the eye plane or behind it (no projection) are dropped;
//   * barycentrics l_k = w_k * (1/area) from the integer edge values, 1/z interpolated linearly in
//     screen space, attributes perspective-correctly (b_k = l_k/z_k * z);
//   * rgb = interpolated vertex albedo (ambient light 1.0); normals = frac-wrapped eye normal
//     through the 32-level texture; depth = z = 1/(1/z) in metres, 0 for background or d > 0.999;
//   * every float operation is a single correctly-rounded IEEE operation in a fixed order
//     (reciprocals are 1/x, quantisation levels come from a k/255 table) so that the CPU restatement
//     reproduces it exactly.
//
// Per view: (A) clear a 64-bit visibility buffer (global scratch, L2 resident), (B) transform and
// snap the vertices once, (C) one thread per triangle walks its bounding box with incremental edge
// functions and atomicMin's (~1/z bits, triangle) keys -- large triangles are queued and rasterised by
// the whole CTA, (D) resolve: one thread per pixel re-derives the winning triangle's barycentrics,
// shades and writes the outputs.  In the fused single-view mode the resolve pass also computes the
// observation crop of its pixel (roi_align) and stores the complete channel vector of the network
// input with 16-byte stores.
#include <vector>
#include "crop_device.cuh"

namespace mpx {

constexpr float kProjMin = 0.0009765625f;  // 2^-10 m: nearer to the eye plane (or behind it) = not projectable; the near PLANE is the per-sample kIzMax test
constexpr float kIzMax = 10.0f;  // 1 / near
constexpr float kIzMin = 0.1f;   // 1 / far
constexpr int kSubBits = 8;
constexpr int kSub = 1 << kSubBits;  // 256 sub-pixel steps
constexpr int kHalf = kSub / 2;
constexpr float kClampUV = 1048576.0f;  // 2^20 pixels
constexpr int kRasterThreads = 512;
constexpr int kBigQueue = 2048;
constexpr long long kBigArea = 1024;  // pixels; larger bounding boxes go to the CTA-wide path
// tiled kernel
constexpr int kTileThreads = 512;
constexpr int kTileBatch = kTileThreads;  // triangles set up per batch, one per thread
constexpr int kTileMinRows = 16;          // fewer rows per strip than this: use the untiled kernel
constexpr int kTileMaxSpan = 6;           // strips a triangle of <= 65 rows can overlap when a strip has >= 16 rows
constexpr int kTileMaxStrips = 128;
constexpr int kRecFields = 16;
constexpr int kSmallExt = 16384;          // sub-pixel extent (64 px) up to which every edge value fits 32 bits

// k / 255 (uint8 read-back levels of the reference) and the 32 texel values uint8(k*255/32) / 255
struct QuantTables {
  float q8[256];
  float tex[32];
};
__constant__ QuantTables c_tables;
__constant__ int c_red_only = 1;
static bool g_tables_ready = false;
static bool g_scatter = true;  // small-batch scatter path (raster_set_scatter)
static bool g_tiled = true;    // tiled kernel for batches that fill the GPU (raster_set_tiled)
void raster_set_scatter(int on) { g_scatter = on != 0; }
void raster_set_tiled(int on) { g_tiled = on != 0; }
int raster_set_red_only(int on) {
  const int v = on != 0;
  MPX_CHECK_CUDA(cudaMemcpyToSymbol(c_red_only, &v, sizeof(v)));
  return MPX_OK;
}

__device__ __forceinline__ bool finite_f(float v) { return fabsf(v) <= 3.402823466e38f; }

// edge function of P against the directed edge a->b, exact in 64-bit
__device__ __forceinline__ long long edge_fn(int ax, int ay, int bx, int by, int px, int py) {
  return static_cast<long long>(bx - ax) * static_cast<long long>(py - ay) -
         static_cast<long long>(by - ay) * static_cast<long long>(px - ax);
}

// 32-level sawtooth of the reference's eye-normal texture with linear filtering and repeat wrap
__device__ __forceinline__ float normal_texture(float s) {
  const float u = __fmaf_rn(s, 32.0f, -0.5f);
  const float fl = floorf(u);
  const float f = __fsub_rn(u, fl);
  const int k0 = static_cast<int>(fl) & 31;
  const int k1 = (k0 + 1) & 31;
  const float t0 = c_tables.tex[k0];
  const float t1 = c_tables.tex[k1];
  return __fmaf_rn(f, __fsub_rn(t1, t0), t0);
}

__device__ __forceinline__ float quant8(float v, bool on) {
  v = fminf(fmaxf(v, 0.0f), 1.0f);
  if (!on) return v;
  return c_tables.q8[__float2int_rn(__fmul_rn(v, 255.0f))];
}

// Diffuse texture of a mesh (contract in oracle/raster_ref.c): uv wrapped to [0,1) (repeat), v up, bilinear over texel
// centres, texel = byte / 255 (the k/255 table), every step a single correctly rounded operation in a fixed order.
struct TexRef {
  const float* uv;           // this mesh's [nv,2]
  const unsigned char* tex;  // [th,tw,3], nullptr = untextured
  int th, tw, modulate;
};
__device__ __forceinline__ int wrap_idx(int i, int n) {
  const int r = i % n;
  return r < 0 ? r + n : r;
}
__device__ __forceinline__ void texture_sample(const TexRef& t, float u, float v, float (&out)[3]) {
  if (!(u == u)) u = 0.f;
  if (!(v == v)) v = 0.f;
  u = __fsub_rn(u, floorf(u));
  v = __fsub_rn(v, floorf(v));
  const float x = __fmaf_rn(u, static_cast<float>(t.tw), -0.5f);
  const float y = __fmaf_rn(__fsub_rn(1.0f, v), static_cast<float>(t.th), -0.5f);
  const float x0 = floorf(x), y0 = floorf(y);
  const float fx = __fsub_rn(x, x0), fy = __fsub_rn(y, y0);
  const int i0 = wrap_idx(static_cast<int>(x0), t.tw), i1 = wrap_idx(static_cast<int>(x0) + 1, t.tw);
  const int r0 = wrap_idx(static_cast<int>(y0), t.th), r1 = wrap_idx(static_cast<int>(y0) + 1, t.th);
  const unsigned char* p00 = t.tex + (static_cast<size_t>(r0) * t.tw + i0) * 3;
  const unsigned char* p10 = t.tex + (static_cast<size_t>(r0) * t.tw + i1) * 3;
  const unsigned char* p01 = t.tex + (static_cast<size_t>(r1) * t.tw + i0) * 3;
  const unsigned char* p11 = t.tex + (static_cast<size_t>(r1) * t.tw + i1) * 3;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float c00 = c_tables.q8[__ldg(p00 + k)], c10 = c_tables.q8[__ldg(p10 + k)];
    const float c01 = c_tables.q8[__ldg(p01 + k)], c11 = c_tables.q8[__ldg(p11 + k)];
    const float top = __fmaf_rn(fx, __fsub_rn(c10, c00), c00);
    const float bot = __fmaf_rn(fx, __fsub_rn(c11, c01), c01);
    out[k] = __fmaf_rn(fy, __fsub_rn(bot, top), top);
  }
}

struct TriSetup {
  int ax, ay, bx, by, cx, cy;
  float iza, izb, izc;
  float inv_area;
  bool flip;
  bool ok;
};

// camera transform, projection and 1/256-pixel snapping of one model vertex: {X, Y, 1/z bits, not projectable}
__device__ __forceinline__ int4 snap_vertex(const float* __restrict__ p, const float* sR, float fx, float cx, float fy,
                                            float cy) {
  const float px = __ldg(p), py = __ldg(p + 1), pz = __ldg(p + 2);
  const float xc = __fmaf_rn(sR[0], px, __fmaf_rn(sR[1], py, __fmaf_rn(sR[2], pz, sR[3])));
  const float yc = __fmaf_rn(sR[4], px, __fmaf_rn(sR[5], py, __fmaf_rn(sR[6], pz, sR[7])));
  const float zc = __fmaf_rn(sR[8], px, __fmaf_rn(sR[9], py, __fmaf_rn(sR[10], pz, sR[11])));
  int4 o;
  o.w = !(zc >= kProjMin);
  const float zs = o.w ? 1.0f : zc;
  const float iz = __frcp_rn(zs);
  float u = __fmaf_rn(fx, __fmul_rn(xc, iz), cx);
  float v = __fmaf_rn(fy, __fmul_rn(yc, iz), cy);
  u = fminf(fmaxf(u, -kClampUV), kClampUV);
  v = fminf(fmaxf(v, -kClampUV), kClampUV);
  if (!(u == u)) { u = 0.f; o.w = 1; }
  if (!(v == v)) { v = 0.f; o.w = 1; }
  o.x = __float2int_rn(__fmul_rn(u, static_cast<float>(kSub)));
  o.y = __float2int_rn(__fmul_rn(v, static_cast<float>(kSub)));
  o.z = __float_as_int(iz);
  return o;
}

// Where a triangle's snapped vertices come from: the per-CTA cache filled in phase (B) of raster_kernel, or (scatter
// path for a handful of views) recomputed from the model vertices -- same arithmetic, same result.
struct VtxSrc {
  const int4* cache;   // CACHED
  const float* verts;  // !CACHED: model vertices of this mesh
  const float* sR;     // pose rows (shared memory)
  float fx, cx, fy, cy;
};

template <bool CACHED>
__device__ __forceinline__ TriSetup load_tri(const VtxSrc& src, const int4* __restrict__ faces, int tri) {
  TriSetup t;
  const int4 f = __ldg(faces + tri);
  const int ia = f.x, ib = f.y, ic = f.z;
  int4 a, b, c;
  if (CACHED) {
    a = __ldcg(src.cache + ia); b = __ldcg(src.cache + ib); c = __ldcg(src.cache + ic);
  } else {
    a = snap_vertex(src.verts + 3 * ia, src.sR, src.fx, src.cx, src.fy, src.cy);
    b = snap_vertex(src.verts + 3 * ib, src.sR, src.fx, src.cx, src.fy, src.cy);
    c = snap_vertex(src.verts + 3 * ic, src.sR, src.fx, src.cx, src.fy, src.cy);
  }
  t.ax = a.x; t.ay = a.y; t.bx = b.x; t.by = b.y; t.cx = c.x; t.cy = c.y;
  t.iza = __int_as_float(a.z); t.izb = __int_as_float(b.z); t.izc = __int_as_float(c.z);
  long long area2 = edge_fn(t.ax, t.ay, t.bx, t.by, t.cx, t.cy);
  t.flip = area2 < 0;
  if (t.flip) area2 = -area2;
  t.ok = (area2 != 0) && !(a.w | b.w | c.w);
  t.inv_area = t.ok ? __frcp_rn(static_cast<float>(area2)) : 0.f;
  return t;
}

// interpolated 1/z of a covered sample from its (orientation-corrected) edge values
// W = long long, or int when the edge values are known to fit (same integers, same correctly rounded conversions: the
// 64-bit integer adds and int64 -> float conversions were a large part of the coverage loop's instructions)
template <typename W>
__device__ __forceinline__ float sample_iz(const TriSetup& t, W w0, W w1, W w2, float& l0, float& l1, float& l2) {
  l0 = __fmul_rn(static_cast<float>(w0), t.inv_area);
  l1 = __fmul_rn(static_cast<float>(w1), t.inv_area);
  l2 = __fmul_rn(static_cast<float>(w2), t.inv_area);
  return __fmaf_rn(l0, t.iza, __fmaf_rn(l1, t.izb, __fmul_rn(l2, t.izc)));
}

__device__ __forceinline__ void raster_bbox(const TriSetup& t, int h, int w, int& j0, int& j1, int& i0,
                                            int& i1) {
  const int minx = min(t.ax, min(t.bx, t.cx)), maxx = max(t.ax, max(t.bx, t.cx));
  const int miny = min(t.ay, min(t.by, t.cy)), maxy = max(t.ay, max(t.by, t.cy));
  // pixel j has its centre at j*256 + 128; kSub is a power of two: floor division = arithmetic shift
  j0 = max(0, (minx - kHalf + kSub - 1) >> kSubBits);  // ceil((minx-128)/256)
  j1 = min(w - 1, (maxx - kHalf) >> kSubBits);
  i0 = max(0, (miny - kHalf + kSub - 1) >> kSubBits);
  i1 = min(h - 1, (maxy - kHalf) >> kSubBits);
}

// key_id: the low 32 bits of the visibility key -- the triangle index within its mesh, or its scene index (scene renderer)
template <typename W>
__device__ __forceinline__ void emit_fragment(const TriSetup& t, W w0, W w1, W w2, int key_id,
                                              unsigned long long* __restrict__ cell) {
  if ((w0 | w1 | w2) < 0) return;
  float l0, l1, l2;
  const float iz = sample_iz(t, w0, w1, w2, l0, l1, l2);
  if (!(iz >= kIzMin && iz <= kIzMax)) return;
  const unsigned long long key =
      (static_cast<unsigned long long>(~__float_as_uint(iz)) << 32) | static_cast<unsigned>(key_id);
  // default: fire-and-forget reduction -- no dependent L2 read in the coverage loop (13.25 -> 13.06 ms per step, raster
  // microbench 8.17 -> 7.42 ms); mpx_raster_set_mode without bit 1 (2) restores read-then-atomic
  if (c_red_only) {
    atomicMin(cell, key);
  } else if (key < __ldcg(cell)) {
    atomicMin(cell, key);
  }
}

// (C) coverage of triangle `tri` of `faces` restricted to rows [row_lo, row_hi], its keys carrying `key_id`; bounding
// boxes above kBigArea pixels are queued (by key id) for the CTA-wide path
template <bool CACHED>
__device__ __forceinline__ void cover_triangle(const VtxSrc& src, const int4* __restrict__ faces, int tri, int key_id,
                                               int row_lo, int row_hi, int h, int w, unsigned long long* __restrict__ vis,
                                               int* s_big_count, int* s_big) {
  const TriSetup t = load_tri<CACHED>(src, faces, tri);
  if (!t.ok) return;
  int j0, j1, i0, i1;
  raster_bbox(t, h, w, j0, j1, i0, i1);
  i0 = max(i0, row_lo);
  i1 = min(i1, row_hi);
  if (j0 > j1 || i0 > i1) return;
  const long long area = static_cast<long long>(j1 - j0 + 1) * (i1 - i0 + 1);
  if (area > kBigArea) {
    const int slot = atomicAdd(s_big_count, 1);
    if (slot < kBigQueue) {
      s_big[slot] = key_id;
      return;
    }
  }
  // incremental edge functions (exact integers): d/dx = -(by-ay)*256, d/dy = (bx-ax)*256
  const int px0 = j0 * kSub + kHalf, py0 = i0 * kSub + kHalf;
  const long long sgn = t.flip ? -1 : 1;
  long long r0 = sgn * edge_fn(t.bx, t.by, t.cx, t.cy, px0, py0);
  long long r1 = sgn * edge_fn(t.cx, t.cy, t.ax, t.ay, px0, py0);
  long long r2 = sgn * edge_fn(t.ax, t.ay, t.bx, t.by, px0, py0);
  const long long dx0 = -sgn * static_cast<long long>(t.cy - t.by) * kSub, dy0 = sgn * static_cast<long long>(t.cx - t.bx) * kSub;
  const long long dx1 = -sgn * static_cast<long long>(t.ay - t.cy) * kSub, dy1 = sgn * static_cast<long long>(t.ax - t.cx) * kSub;
  const long long dx2 = -sgn * static_cast<long long>(t.by - t.ay) * kSub, dy2 = sgn * static_cast<long long>(t.bx - t.ax) * kSub;
  // Triangles spanning at most 64 pixels in x and y (practically all of them): every edge value at a pixel centre inside
  // the bounding box is below 2 * 2^14 * 2^14 = 2^29 in magnitude and every step below 2^22, so the walk runs in 32 bits
  const int ext_x = max(t.ax, max(t.bx, t.cx)) - min(t.ax, min(t.bx, t.cx));
  const int ext_y = max(t.ay, max(t.by, t.cy)) - min(t.ay, min(t.by, t.cy));
  if (ext_x <= 16384 && ext_y <= 16384) {
    int s0 = static_cast<int>(r0), s1 = static_cast<int>(r1), s2 = static_cast<int>(r2);
    const int ex0 = static_cast<int>(dx0), ex1 = static_cast<int>(dx1), ex2 = static_cast<int>(dx2);
    const int ey0 = static_cast<int>(dy0), ey1 = static_cast<int>(dy1), ey2 = static_cast<int>(dy2);
    for (int i = i0; i <= i1; ++i) {
      int w0 = s0, w1 = s1, w2 = s2;
      unsigned long long* row = vis + i * w;
      for (int j = j0; j <= j1; ++j) {
        emit_fragment<int>(t, w0, w1, w2, key_id, row + j);
        w0 += ex0; w1 += ex1; w2 += ex2;
      }
      s0 += ey0; s1 += ey1; s2 += ey2;
    }
    return;
  }
  for (int i = i0; i <= i1; ++i) {
    long long w0 = r0, w1 = r1, w2 = r2;
    for (int j = j0; j <= j1; ++j) {
      emit_fragment<long long>(t, w0, w1, w2, key_id, vis + i * w + j);
      w0 += dx0; w1 += dx1; w2 += dx2;
    }
    r0 += dy0; r1 += dy1; r2 += dy2;
  }
}

// A triangle named by its key id: where its vertices come from, its mesh's faces and its index among them
struct TriRef {
  VtxSrc src;
  const int4* faces;
  int tri;
};
// key id = triangle index of one mesh (the single-object kernels)
struct MeshTris {
  const VtxSrc& src;
  const int4* faces;
  __device__ __forceinline__ TriRef operator()(int key_id) const { return TriRef{src, faces, key_id}; }
};

// queued large triangles: the whole CTA shares each bounding box; `tri_of` maps a queued key id to its triangle
template <bool CACHED, typename TriOf>
__device__ __forceinline__ void cover_big_triangles(const TriOf& tri_of, int nbig, const int* s_big, int row_lo,
                                                    int row_hi, int h, int w, unsigned long long* __restrict__ vis) {
  for (int b = 0; b < nbig; ++b) {
    const int key_id = s_big[b];
    const TriRef r = tri_of(key_id);
    const TriSetup t = load_tri<CACHED>(r.src, r.faces, r.tri);
    int j0, j1, i0, i1;
    raster_bbox(t, h, w, j0, j1, i0, i1);
    i0 = max(i0, row_lo);
    i1 = min(i1, row_hi);
    const int bw = j1 - j0 + 1;
    const int cnt = bw * (i1 - i0 + 1);
    for (int k = threadIdx.x; k < cnt; k += blockDim.x) {
      const int i = i0 + k / bw, j = j0 + k % bw;
      const int px = j * kSub + kHalf, py = i * kSub + kHalf;
      long long w0 = edge_fn(t.bx, t.by, t.cx, t.cy, px, py);
      long long w1 = edge_fn(t.cx, t.cy, t.ax, t.ay, px, py);
      long long w2 = edge_fn(t.ax, t.ay, t.bx, t.by, px, py);
      if (t.flip) { w0 = -w0; w1 = -w1; w2 = -w2; }
      emit_fragment<long long>(t, w0, w1, w2, key_id, vis + i * w + j);
    }
  }
}

// pose / intrinsics of one view into shared memory (thread 0); returns nothing, *s_valid = 0 for non-finite input or an
// unknown label (such views render black)
__device__ __forceinline__ void load_view(const MeshDb& db, const int* __restrict__ label_idx, const float* __restrict__ TCO,
                                          const float* __restrict__ K, int view, float* sR, float* sK, int* s_valid) {
  bool ok = true;
  const float* T = TCO + 16 * view;
  const float* Kv = K + 9 * view;
  for (int i = 0; i < 16; ++i) ok = ok && finite_f(T[i]);
  for (int i = 0; i < 9; ++i) ok = ok && finite_f(Kv[i]);
  const int lab = label_idx[view];
  ok = ok && lab >= 0 && lab < db.n_meshes;
  *s_valid = ok ? 1 : 0;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) sR[r * 4 + c] = T[r * 4 + c];
  sK[0] = Kv[0]; sK[1] = Kv[2]; sK[2] = Kv[4]; sK[3] = Kv[5];
}

__device__ __forceinline__ TexRef mesh_texture(const MeshDb& db, int lab, long long v_off, bool valid) {
  TexRef t;
  t.uv = nullptr; t.tex = nullptr; t.th = t.tw = t.modulate = 0;
  if (valid && db.tex_info != nullptr) {
    const int4 info = db.tex_info[lab];
    if (info.x > 0 && info.y > 0) {
      t.uv = db.uv + 2 * v_off;
      t.tex = db.tex + db.tex_offsets[lab];
      t.th = info.x; t.tw = info.y; t.modulate = info.z;
    }
  }
  return t;
}

// (D) resolve + shade + write.  ResolveCtx holds what is constant over a view (output slots, fused-crop tables);
// resolve_pixel shades one pixel from its visibility key and writes every requested output.
struct ResolveCtx {
  int sample, vslot, npix;
  const float* verts;  // model vertices of this view's mesh, for the point-light shading (nullptr: ambient light)
  float light_dist;    // 10 x bounding radius
  bool fuse_crop, crop_collapsed;
  RoiParams roi;
  const float4* crop_img;
  const AxisW* s_axis;
};

// Called by every thread of the CTA (contains a barrier when the crop is fused).
__device__ __forceinline__ ResolveCtx make_resolve_ctx(const RasterOut& out, int view, int h, int w, AxisW* s_axis,
                                                        const float* verts = nullptr, float radius = 0.f) {
  ResolveCtx c;
  c.npix = h * w;
  c.verts = verts;
  c.light_dist = __fmul_rn(radius, 10.0f);
  c.sample = out.x ? view / out.views_per_sample : 0;
  c.vslot = out.x ? view % out.views_per_sample : 0;
  c.fuse_crop = out.x != nullptr && out.crop_images != nullptr;
  c.crop_img = nullptr;
  c.crop_collapsed = false;
  c.s_axis = s_axis;
  c.roi = RoiParams{0.f, 0.f, 0.f, 0.f};
  if (c.fuse_crop) {
    c.roi = make_roi(out.crop_boxes + 4 * c.sample, h, w);
    const int im = out.crop_im_idx ? out.crop_im_idx[c.sample] : c.sample;
    if (im >= 0 && im < out.crop_b) c.crop_img = out.crop_images + static_cast<size_t>(im) * out.crop_h * out.crop_w;
    // block-uniform: every thread sees the same sample / image
    if (c.crop_img != nullptr && h + w <= kAxisTableMax)
      c.crop_collapsed = build_axis_tables(c.roi, h, w, out.crop_h, out.crop_w, s_axis, s_axis + h);
  }
  return c;
}

template <bool CACHED, bool TEXTURED, bool COLOR_OVERRIDE = false>
__device__ __forceinline__ void resolve_pixel(const ResolveCtx& ctx, const VtxSrc& src, const int4* __restrict__ faces,
                                              const float4* __restrict__ vattr, const TexRef& texref,
                                              unsigned long long key, int view, int i, int j, int h, int w, bool q8,
                                              bool gl_axes, const RasterOut& out, const float* color = nullptr) {
  const int npix = ctx.npix;
  const int pix = i * w + j;
  const float* sR = src.sR;
  // d = a / z + b with a = 1 / (1/far - 1/near), b = -a / near (utils.py:44-55), as literals so
  // that host and device agree on the rounding
  const float dep_a = -0.10101010f;
  const float dep_b = 1.01010101f;
  const int sample = ctx.sample;
  float r = 0.f, g = 0.f, b = 0.f, n0 = 0.f, n1 = 0.f, n2 = 0.f, dep = 0.f;
  if (key != ~0ull) {
    const int tri = static_cast<int>(key & 0xffffffffu);
    const TriSetup t = load_tri<CACHED>(src, faces, tri);
    const int px = j * kSub + kHalf, py = i * kSub + kHalf;
    long long w0 = edge_fn(t.bx, t.by, t.cx, t.cy, px, py);
    long long w1 = edge_fn(t.cx, t.cy, t.ax, t.ay, px, py);
    long long w2 = edge_fn(t.ax, t.ay, t.bx, t.by, px, py);
    if (t.flip) { w0 = -w0; w1 = -w1; w2 = -w2; }
    float l0, l1, l2;
    const float iz = (((w0 | w1 | w2) >> 31) == 0)
                         ? sample_iz<int>(t, static_cast<int>(w0), static_cast<int>(w1), static_cast<int>(w2), l0, l1, l2)
                         : sample_iz<long long>(t, w0, w1, w2, l0, l1, l2);
    const float z = __frcp_rn(iz);
    const float b0 = __fmul_rn(__fmul_rn(l0, t.iza), z);
    const float b1 = __fmul_rn(__fmul_rn(l1, t.izb), z);
    const float b2 = __fmul_rn(__fmul_rn(l2, t.izc), z);
    const int4 f = __ldg(faces + tri);
    // packed per-vertex attributes {r, g, b, nx}, {ny, nz, u, v}
    const float4 a0 = __ldg(vattr + 2 * f.x), a1 = __ldg(vattr + 2 * f.x + 1);
    const float4 c0 = __ldg(vattr + 2 * f.y), c1 = __ldg(vattr + 2 * f.y + 1);
    const float4 e0 = __ldg(vattr + 2 * f.z), e1 = __ldg(vattr + 2 * f.z + 1);
#define MPX_INTERP(A, B, C) __fmaf_rn(b0, (A), __fmaf_rn(b1, (B), __fmul_rn(b2, (C))))
    float col[3], nrm[3];
    col[0] = MPX_INTERP(a0.x, c0.x, e0.x);
    col[1] = MPX_INTERP(a0.y, c0.y, e0.y);
    col[2] = MPX_INTERP(a0.z, c0.z, e0.z);
    nrm[0] = MPX_INTERP(a0.w, c0.w, e0.w);
    nrm[1] = MPX_INTERP(a1.x, c1.x, e1.x);
    nrm[2] = MPX_INTERP(a1.y, c1.y, e1.y);
    if (TEXTURED && texref.tex != nullptr) {
      const float tu = MPX_INTERP(a1.z, c1.z, e1.z);
      const float tv = MPX_INTERP(a1.w, c1.w, e1.w);
      float tc[3];
      texture_sample(texref, tu, tv, tc);
#pragma unroll
      for (int k = 0; k < 3; ++k) col[k] = texref.modulate ? __fmul_rn(tc[k], col[k]) : tc[k];
    }
    if (COLOR_OVERRIDE && color[0] >= 0.f) {  // scene renderer: the albedo replaced by the instance's colour
#pragma unroll
      for (int k = 0; k < 3; ++k) col[k] = color[k];
    }
    if (ctx.verts != nullptr) {
      // render_normals=False models: ambient 0.1 + six white point lights of 0.4 on the object's axes at 10 bounding radii
      // (make_scene_lights, panda3d_scene_renderer.py:104-136), Lambert term per fragment with the interpolated unit
      // normal and position in the object frame, no attenuation, no normal flip on back faces (contract: oracle/raster_ref.c)
      const float* pa = ctx.verts + 3 * f.x;
      const float* pb = ctx.verts + 3 * f.y;
      const float* pc = ctx.verts + 3 * f.z;
      const float p0 = MPX_INTERP(__ldg(pa), __ldg(pb), __ldg(pc));
      const float p1 = MPX_INTERP(__ldg(pa + 1), __ldg(pb + 1), __ldg(pc + 1));
      const float p2 = MPX_INTERP(__ldg(pa + 2), __ldg(pb + 2), __ldg(pc + 2));
      float u0 = nrm[0], u1 = nrm[1], u2 = nrm[2];
      const float ul = __fsqrt_rn(__fmaf_rn(u0, u0, __fmaf_rn(u1, u1, __fmul_rn(u2, u2))));
      if (ul > 0.f) {
        const float inv = __frcp_rn(ul);
        u0 = __fmul_rn(u0, inv); u1 = __fmul_rn(u1, inv); u2 = __fmul_rn(u2, inv);
      }
      float shade = 0.1f;
#pragma unroll
      for (int li = 0; li < 6; ++li) {
        const float sgn = (li & 1) ? -ctx.light_dist : ctx.light_dist;
        const float d0 = __fsub_rn(li < 2 ? sgn : 0.f, p0);
        const float d1 = __fsub_rn((li >> 1) == 1 ? sgn : 0.f, p1);
        const float d2 = __fsub_rn(li >= 4 ? sgn : 0.f, p2);
        const float dist = __fsqrt_rn(__fmaf_rn(d0, d0, __fmaf_rn(d1, d1, __fmul_rn(d2, d2))));
        if (dist > 0.f) {
          const float ndl = __fdiv_rn(__fmaf_rn(u0, d0, __fmaf_rn(u1, d1, __fmul_rn(u2, d2))), dist);
          shade = __fmaf_rn(0.4f, fmaxf(ndl, 0.f), shade);
        }
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) col[k] = __fmul_rn(col[k], shade);
    }
#undef MPX_INTERP
    r = quant8(col[0], q8);
    g = quant8(col[1], q8);
    b = quant8(col[2], q8);
    // eye-space normal (OpenCV camera axes), normalised
    float ex = __fmaf_rn(sR[0], nrm[0], __fmaf_rn(sR[1], nrm[1], __fmul_rn(sR[2], nrm[2])));
    float ey = __fmaf_rn(sR[4], nrm[0], __fmaf_rn(sR[5], nrm[1], __fmul_rn(sR[6], nrm[2])));
    float ez = __fmaf_rn(sR[8], nrm[0], __fmaf_rn(sR[9], nrm[1], __fmul_rn(sR[10], nrm[2])));
    const float nn = __fsqrt_rn(__fmaf_rn(ex, ex, __fmaf_rn(ey, ey, __fmul_rn(ez, ez))));
    if (nn > 0.f) {
      const float inv = __frcp_rn(nn);
      ex = __fmul_rn(ex, inv);
      ey = __fmul_rn(ey, inv);
      ez = __fmul_rn(ez, inv);
    }
    // Panda camera axes (x right, y forward, z up) or GL axes (x right, y up, z backward)
    const float px_ = ex;
    const float py_ = gl_axes ? -ey : ez;
    const float pz_ = gl_axes ? -ez : -ey;
    n0 = quant8(normal_texture(px_), q8);
    n1 = quant8(normal_texture(py_), q8);
    n2 = quant8(normal_texture(pz_), q8);
    const float d = __fmaf_rn(dep_a, iz, dep_b);
    dep = (d > 0.999f) ? 0.f : z;
  }
  if (out.rgb) {
    float* o = out.rgb + (static_cast<size_t>(view) * 3) * npix + pix;
    o[0] = r; o[npix] = g; o[2 * npix] = b;
  }
  if (out.normals) {
    float* o = out.normals + (static_cast<size_t>(view) * 3) * npix + pix;
    o[0] = n0; o[npix] = n1; o[2 * npix] = n2;
  }
  if (out.depth) out.depth[static_cast<size_t>(view) * npix + pix] = dep;
  if (out.x) {
    const int hs = h >> 1, ws = w >> 1;
    act_t* base = out.x + ((static_cast<size_t>(sample) * hs + (i >> 1)) * ws + (j >> 1)) * (4 * out.c_pad) +
                  ((i & 1) * 2 + (j & 1)) * out.c_pad;
    const bool has_n = out.ch_per_view >= 6, has_d = out.ch_per_view == 4 || out.ch_per_view == 7;
    float dn = dep;
    if (has_d && out.depth_norm_z) dn = depth_norm(dep, __ldg(out.depth_norm_z + sample), out.depth_norm_kind);
    if (ctx.fuse_crop) {
      // whole pixel vector: [crop rgb(d) | render rgb, normals(, depth) | zero pad], c_pad/8 16-byte stores
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      float vacc = 0.f;
      const AxisW* s_axis = ctx.s_axis;
      if (ctx.crop_collapsed) {
        if (out.crop_c == 4) roi_align_pixel_collapsed<true>(ctx.crop_img, out.crop_w, s_axis[i], s_axis[h + j], acc, vacc);
        else roi_align_pixel_collapsed<false>(ctx.crop_img, out.crop_w, s_axis[i], s_axis[h + j], acc, vacc);
      } else if (ctx.crop_img) {
        if (out.crop_c == 4) roi_align_pixel<true>(ctx.crop_img, out.crop_h, out.crop_w, ctx.roi, i, j, acc, vacc);
        else roi_align_pixel<false>(ctx.crop_img, out.crop_h, out.crop_w, ctx.roi, i, j, acc, vacc);
      }
      float ch[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) ch[k] = 0.f;
      int c = 0;
      ch[c++] = acc.x; ch[c++] = acc.y; ch[c++] = acc.z;
      if (out.crop_c == 4) {
        float d4 = (vacc < 0.99f) ? 0.f : acc.w;
        if (out.depth_norm_z) d4 = depth_norm(d4, __ldg(out.depth_norm_z + sample), out.depth_norm_kind);
        ch[c++] = d4;
      }
      ch[c++] = r; ch[c++] = g; ch[c++] = b;
      if (has_n) { ch[c++] = n0; ch[c++] = n1; ch[c++] = n2; }
      if (has_d) ch[c++] = dn;
      uint4* o4 = reinterpret_cast<uint4*>(base);
      uint4 v0, v1;
      v0.x = pack_act2(ch[0], ch[1]); v0.y = pack_act2(ch[2], ch[3]);
      v0.z = pack_act2(ch[4], ch[5]); v0.w = pack_act2(ch[6], ch[7]);
      v1.x = pack_act2(ch[8], ch[9]); v1.y = pack_act2(ch[10], ch[11]);
      v1.z = pack_act2(ch[12], ch[13]); v1.w = pack_act2(ch[14], ch[15]);
      o4[0] = v0;
      o4[1] = v1;
      for (int k = 2; k < out.c_pad / 8; ++k) o4[k] = make_uint4(0u, 0u, 0u, 0u);
    } else {
      act_t* o = base + out.ch_offset + ctx.vslot * out.ch_per_view;
      o[0] = to_act(r);
      o[1] = to_act(g);
      o[2] = to_act(b);
      if (has_n) {
        o[3] = to_act(n0);
        o[4] = to_act(n1);
        o[5] = to_act(n2);
      }
      if (has_d) o[has_n ? 6 : 3] = to_act(dn);
    }
  }
}

// rows [row_lo, row_hi] of one view from a global visibility buffer.  Called by every thread of the CTA.
template <bool CACHED, bool TEXTURED>
__device__ __forceinline__ void resolve_rows(const VtxSrc& src, const int4* __restrict__ faces,
                                             const float4* __restrict__ vattr, const TexRef& texref,
                                             const unsigned long long* __restrict__ vis, int view, int row_lo, int row_hi,
                                             int h, int w, bool q8, bool gl_axes, const RasterOut& out, AxisW* s_axis,
                                             const float* light_verts, float radius) {
  const ResolveCtx ctx = make_resolve_ctx(out, view, h, w, s_axis, light_verts, radius);
  for (int pix = row_lo * w + threadIdx.x; pix < (row_hi + 1) * w; pix += blockDim.x) {
    const int i = pix / w, j = pix - i * w;
    resolve_pixel<CACHED, TEXTURED>(ctx, src, faces, vattr, texref, __ldcg(vis + pix), view, i, j, h, w, q8, gl_axes, out);
  }
}

template <bool TEXTURED>  // instantiated for mesh stores with / without textures: the untextured kernel keeps its registers
__global__ void __launch_bounds__(kRasterThreads, 2)
raster_kernel(const MeshDb db, const int* __restrict__ label_idx, const float* __restrict__ TCO,
              const float* __restrict__ K, int n_views, int h, int w, unsigned flags, RasterOut out,
              unsigned long long* __restrict__ vis_all, int strips) {
  __shared__ float sR[12];
  __shared__ float sK[4];
  __shared__ int s_valid;
  __shared__ int s_big_count;
  __shared__ int s_big[kBigQueue];
  __shared__ AxisW s_axis[kAxisTableMax];  // fused crop: collapsed roi_align weights, rows then columns

  const int npix = h * w;
  unsigned long long* vis = vis_all + static_cast<size_t>(blockIdx.x) * npix;
  int4* vtx = db.vtx_cache + static_cast<size_t>(blockIdx.x) * db.nv_max;
  const bool q8 = (flags & 1u) != 0;
  const bool gl_axes = (flags & 2u) != 0;

  // work item = (view, horizontal strip of rows); strips > 1 only when there are fewer views than CTA slots
  const int rows_per_strip = (h + strips - 1) / strips;
  for (int item = blockIdx.x; item < n_views * strips; item += gridDim.x) {
    const int view = item / strips;
    const int row_lo = (item - view * strips) * rows_per_strip;
    const int row_hi = min(h, row_lo + rows_per_strip) - 1;  // inclusive
    __syncthreads();  // previous item fully resolved before scratch is reused
    if (threadIdx.x == 0) {
      load_view(db, label_idx, TCO, K, view, sR, sK, &s_valid);
      s_big_count = 0;
    }
    __syncthreads();
    const bool valid = s_valid != 0;
    const int lab = valid ? label_idx[view] : 0;
    const long long v_off = valid ? db.vert_offsets[lab] : 0;
    const int nv = valid ? static_cast<int>(db.vert_offsets[lab + 1] - v_off) : 0;
    const long long f_off = valid ? db.face_offsets[lab] : 0;
    const int nf = valid ? static_cast<int>(db.face_offsets[lab + 1] - f_off) : 0;
    const int4* faces = db.faces4 + f_off;

    // (A) clear visibility, (B) transform + snap vertices
    for (int i = row_lo * w + threadIdx.x; i < (row_hi + 1) * w; i += blockDim.x) vis[i] = ~0ull;
    const float fx = sK[0], cx = sK[1], fy = sK[2], cy = sK[3];
    for (int i = threadIdx.x; i < nv; i += blockDim.x)
      vtx[i] = snap_vertex(db.verts + 3 * (v_off + i), sR, fx, cx, fy, cy);
    __syncthreads();
    VtxSrc src;
    src.cache = vtx;
    src.verts = nullptr;
    src.sR = sR;
    src.fx = fx; src.cx = cx; src.fy = fy; src.cy = cy;

    // (C) triangles
    for (int tri = threadIdx.x; tri < nf; tri += blockDim.x)
      cover_triangle<true>(src, faces, tri, tri, row_lo, row_hi, h, w, vis, &s_big_count, s_big);
    __syncthreads();
    cover_big_triangles<true>(MeshTris{src, faces}, min(s_big_count, kBigQueue), s_big, row_lo, row_hi, h, w, vis);
    __syncthreads();

    resolve_rows<true, TEXTURED>(src, faces, db.vattr + 2 * v_off,
                                 TEXTURED ? mesh_texture(db, lab, v_off, valid) : TexRef{nullptr, nullptr, 0, 0, 0}, vis, view,
                                 row_lo, row_hi, h, w, q8, gl_axes, out, s_axis,
                                 (flags & 4u) != 0 && valid ? db.verts + 3 * v_off : nullptr, valid ? db.radius[lab] : 0.f);
  }
}

// ---------------------------------------------------------------------------------------------
// Scatter path for a handful of views (refiner iterations, final scoring): with one CTA per (view, strip) every CTA
// still transforms all vertices and sets up all triangles -- a ~180 us latency chain for 4 views.  Here the
// TRIANGLES of a view are spread over `parts` CTAs that share the view's visibility buffer through global atomics
// (each thread sets up about one triangle, recomputing its three vertices), and a second kernel resolves the
// pixels, again recomputing the winning triangle's vertices.  Same arithmetic per vertex / triangle / fragment and
// an order-independent atomicMin: results are identical to raster_kernel.
// ---------------------------------------------------------------------------------------------
constexpr int kCoverThreads = 256;
__global__ void __launch_bounds__(kCoverThreads)
raster_cover_kernel(const MeshDb db, const int* __restrict__ label_idx, const float* __restrict__ TCO,
                    const float* __restrict__ K, int n_views, int h, int w, unsigned long long* __restrict__ vis_all,
                    int parts) {
  __shared__ float sR[12];
  __shared__ float sK[4];
  __shared__ int s_valid;
  __shared__ int s_big_count;
  __shared__ int s_big[kBigQueue];
  const int view = blockIdx.x / parts, part = blockIdx.x - view * parts;
  if (threadIdx.x == 0) {
    load_view(db, label_idx, TCO, K, view, sR, sK, &s_valid);
    s_big_count = 0;
  }
  __syncthreads();
  if (s_valid == 0) return;
  const int lab = label_idx[view];
  const long long v_off = db.vert_offsets[lab];
  const long long f_off = db.face_offsets[lab];
  const int nf = static_cast<int>(db.face_offsets[lab + 1] - f_off);
  const int4* faces = db.faces4 + f_off;
  unsigned long long* vis = vis_all + static_cast<size_t>(view) * h * w;
  VtxSrc src;
  src.cache = nullptr;
  src.verts = db.verts + 3 * v_off;
  src.sR = sR;
  src.fx = sK[0]; src.cx = sK[1]; src.fy = sK[2]; src.cy = sK[3];
  for (int tri = part * kCoverThreads + threadIdx.x; tri < nf; tri += parts * kCoverThreads)
    cover_triangle<false>(src, faces, tri, tri, 0, h - 1, h, w, vis, &s_big_count, s_big);
  __syncthreads();
  cover_big_triangles<false>(MeshTris{src, faces}, min(s_big_count, kBigQueue), s_big, 0, h - 1, h, w, vis);
}

template <bool TEXTURED>
__global__ void __launch_bounds__(kRasterThreads, 2)
raster_resolve_kernel(const MeshDb db, const int* __restrict__ label_idx, const float* __restrict__ TCO,
                      const float* __restrict__ K, int n_views, int h, int w, unsigned flags, RasterOut out,
                      const unsigned long long* __restrict__ vis_all, int strips) {
  __shared__ float sR[12];
  __shared__ float sK[4];
  __shared__ int s_valid;
  __shared__ AxisW s_axis[kAxisTableMax];
  const int view = blockIdx.x / strips, strip = blockIdx.x - view * strips;
  const int rows_per_strip = (h + strips - 1) / strips;
  const int row_lo = strip * rows_per_strip;
  const int row_hi = min(h, row_lo + rows_per_strip) - 1;
  if (threadIdx.x == 0) load_view(db, label_idx, TCO, K, view, sR, sK, &s_valid);
  __syncthreads();
  const bool valid = s_valid != 0;
  const int lab = valid ? label_idx[view] : 0;
  const long long v_off = db.vert_offsets[lab];
  const long long f_off = db.face_offsets[lab];
  VtxSrc src;
  src.cache = nullptr;
  src.verts = db.verts + 3 * v_off;
  src.sR = sR;
  src.fx = sK[0]; src.cx = sK[1]; src.fy = sK[2]; src.cy = sK[3];
  // an invalid view has an untouched (all ~0) visibility buffer: every pixel resolves to background
  resolve_rows<false, TEXTURED>(src, db.faces4 + f_off, db.vattr + 2 * v_off,
                                TEXTURED ? mesh_texture(db, lab, v_off, valid) : TexRef{nullptr, nullptr, 0, 0, 0},
                                vis_all + static_cast<size_t>(view) * h * w, view, row_lo, row_hi, h, w, (flags & 1u) != 0,
                                (flags & 2u) != 0, out, s_axis, (flags & 4u) != 0 && valid ? db.verts + 3 * v_off : nullptr,
                                valid ? db.radius[lab] : 0.f);
}

// ---------------------------------------------------------------------------------------------
// Scene renderer: several posed instances per view with one shared visibility buffer
// (reference: panda3d_renderer/panda3d_scene_renderer.py:139-358 render_scene).  Modelled on the scatter path: a cover
// kernel spreads the view's SCENE triangles over `parts` CTAs, a resolve kernel shades the pixels.  Triangle t of instance
// k has scene index s = (face counts of the valid instances before k) + t, and the keys carry s: the largest 1/z wins,
// ties go to the lower instance, then to the lower triangle.  A one-instance scene therefore holds exactly the keys, and
// produces exactly the pixels, of mpx_raster_render.  Contract restated in tests/scene_ref.c.
// ---------------------------------------------------------------------------------------------
constexpr int kSceneMaxInst = 1024;

struct SceneIn {
  const int* inst_offsets;  // [n_views+1]
  const int* inst_label;    // [n_inst]
  const float* inst_TCO;    // [n_inst,16]
  const float* inst_color;  // [n_inst,3] or nullptr
  const float* K;           // [n_views,9]
  int n_inst;
};

// Shared-memory image of one view's instances (dynamic shared memory, n_cap = max instances per view):
//   R [n_cap,12] pose rows, pre [n_cap+1] exclusive prefix of the face counts, lab [n_cap] label (-1: contributes nothing),
//   col [n_cap,3] colour override (resolve only; first component < 0: none)
__host__ __device__ inline size_t scene_smem_bytes(int n_cap, bool colors) {
  return sizeof(float) * 12 * n_cap + sizeof(int) * (2 * n_cap + 1) + (colors ? sizeof(float) * 3 * n_cap : 0);
}

// exclusive prefix sum of s[0..n) in place, s[n] = total; called by every thread, blockDim a multiple of 32
__device__ __forceinline__ void block_exclusive_scan(int* s, int n, int* s_warp) {
  const int per = (n + blockDim.x - 1) / blockDim.x;
  const int lo = threadIdx.x * per, hi = min(n, lo + per);
  int sum = 0;
  for (int i = lo; i < hi; ++i) sum += s[i];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s_warp[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int x = lane < nw ? s_warp[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += t;
    }
    if (lane < nw) s_warp[lane] = x;
  }
  __syncthreads();
  int run = incl - sum + (wid > 0 ? s_warp[wid - 1] : 0);
  for (int i = lo; i < hi; ++i) {
    const int c = s[i];
    s[i] = run;
    run += c;
  }
  if (threadIdx.x == 0) s[n] = s_warp[nw - 1];
  __syncthreads();
}

// Stage view `view`'s instances; every thread calls it.  Returns the instance count: 0 for a view with non-finite K,
// no instances, or malformed offsets (clamped to [0, n_inst]; more than n_cap instances = malformed).
__device__ int stage_scene_view(const MeshDb& db, const SceneIn& in, int view, int n_cap, float* s_R, int* s_pre,
                                int* s_lab, float* s_col, float* sK, int* s_cnt, int* s_warp) {
  __shared__ int s_lo;
  if (threadIdx.x == 0) {
    const int lo = min(max(in.inst_offsets[view], 0), in.n_inst);
    const int hi = min(max(in.inst_offsets[view + 1], lo), in.n_inst);
    const float* Kv = in.K + 9 * view;
    bool ok = hi - lo <= n_cap;
    for (int i = 0; i < 9; ++i) ok = ok && finite_f(Kv[i]);
    s_lo = lo;
    *s_cnt = ok ? hi - lo : 0;
    sK[0] = Kv[0]; sK[1] = Kv[2]; sK[2] = Kv[4]; sK[3] = Kv[5];
  }
  __syncthreads();
  const int cnt = *s_cnt, lo = s_lo;
  for (int k = threadIdx.x; k < cnt; k += blockDim.x) {
    const int inst = lo + k;
    const float* T = in.inst_TCO + 16 * static_cast<size_t>(inst);
    bool ok = true;
    for (int i = 0; i < 16; ++i) ok = ok && finite_f(T[i]);
    const int lab = in.inst_label[inst];
    ok = ok && lab >= 0 && lab < db.n_meshes;
    for (int i = 0; i < 12; ++i) s_R[12 * k + i] = T[i];
    s_lab[k] = ok ? lab : -1;
    s_pre[k] = ok ? static_cast<int>(db.face_offsets[lab + 1] - db.face_offsets[lab]) : 0;
    if (s_col != nullptr) {
      const float* c = in.inst_color;
      const bool has = c != nullptr && c[3 * static_cast<size_t>(inst)] >= 0.f;
      for (int i = 0; i < 3; ++i) s_col[3 * k + i] = has ? c[3 * static_cast<size_t>(inst) + i] : -1.f;
    }
  }
  __syncthreads();
  block_exclusive_scan(s_pre, cnt, s_warp);
  return cnt;
}

// scene index -> instance and triangle (the instance by binary search over the prefix of the face counts)
struct SceneTris {
  const float* verts;
  const long long* vert_offsets;
  const int4* faces4;
  const long long* face_offsets;
  const float* s_R;
  const int* s_pre;
  const int* s_lab;
  int cnt;
  float fx, cx, fy, cy;
  __device__ __forceinline__ int instance(int s) const {  // largest k with pre[k] <= s; pre[k] <= s < pre[k+1]
    int lo = 0, hi = cnt - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_pre[mid] <= s) lo = mid;
      else hi = mid - 1;
    }
    return lo;
  }
  __device__ __forceinline__ TriRef at(int k, int s) const {
    const int lab = s_lab[k];
    TriRef r;
    r.src.cache = nullptr;
    r.src.verts = verts + 3 * vert_offsets[lab];
    r.src.sR = s_R + 12 * k;
    r.src.fx = fx; r.src.cx = cx; r.src.fy = fy; r.src.cy = cy;
    r.faces = faces4 + face_offsets[lab];
    r.tri = s - s_pre[k];
    return r;
  }
  __device__ __forceinline__ TriRef operator()(int s) const { return at(instance(s), s); }
};

__device__ __forceinline__ SceneTris make_scene_tris(const MeshDb& db, const float* s_R, const int* s_pre, const int* s_lab,
                                                     int cnt, const float* sK) {
  return SceneTris{db.verts, db.vert_offsets, db.faces4, db.face_offsets, s_R, s_pre, s_lab, cnt,
                   sK[0], sK[1], sK[2], sK[3]};
}

// grid = views of the chunk x parts; view = view0 + blockIdx.x / parts, its buffer vis_all[blockIdx.x / parts]
__global__ void __launch_bounds__(kCoverThreads)
scene_cover_kernel(const MeshDb db, const SceneIn in, int view0, int h, int w, unsigned long long* __restrict__ vis_all,
                   int parts, int n_cap) {
  extern __shared__ __align__(16) unsigned char s_dyn[];
  float* s_R = reinterpret_cast<float*>(s_dyn);
  int* s_pre = reinterpret_cast<int*>(s_R + 12 * n_cap);
  int* s_lab = s_pre + n_cap + 1;
  __shared__ float sK[4];
  __shared__ int s_cnt;
  __shared__ int s_warp[32];
  __shared__ int s_big_count;
  __shared__ int s_big[kBigQueue];
  const int lv = blockIdx.x / parts, part = blockIdx.x - lv * parts;
  if (threadIdx.x == 0) s_big_count = 0;
  const int cnt = stage_scene_view(db, in, view0 + lv, n_cap, s_R, s_pre, s_lab, nullptr, sK, &s_cnt, s_warp);
  if (cnt == 0) return;  // block-uniform
  const int total = s_pre[cnt];
  unsigned long long* vis = vis_all + static_cast<size_t>(lv) * h * w;
  const SceneTris tris = make_scene_tris(db, s_R, s_pre, s_lab, cnt, sK);
  for (int s = part * kCoverThreads + threadIdx.x; s < total; s += parts * kCoverThreads) {
    const TriRef r = tris(s);
    cover_triangle<false>(r.src, r.faces, r.tri, s, 0, h - 1, h, w, vis, &s_big_count, s_big);
  }
  __syncthreads();
  cover_big_triangles<false>(tris, min(s_big_count, kBigQueue), s_big, 0, h - 1, h, w, vis);
}

// grid = views of the chunk x row strips; `out` and inst_id point at the chunk's first view
template <bool TEXTURED>
__global__ void __launch_bounds__(kRasterThreads, 2)
scene_resolve_kernel(const MeshDb db, const SceneIn in, int view0, int h, int w, unsigned flags, RasterOut out,
                     int* __restrict__ inst_id, const unsigned long long* __restrict__ vis_all, int strips, int n_cap) {
  extern __shared__ __align__(16) unsigned char s_dyn[];
  float* s_R = reinterpret_cast<float*>(s_dyn);
  int* s_pre = reinterpret_cast<int*>(s_R + 12 * n_cap);
  int* s_lab = s_pre + n_cap + 1;
  float* s_col = reinterpret_cast<float*>(s_lab + n_cap);
  __shared__ float sK[4];
  __shared__ int s_cnt;
  __shared__ int s_warp[32];
  const int lv = blockIdx.x / strips, strip = blockIdx.x - lv * strips;
  const int rows_per_strip = (h + strips - 1) / strips;
  const int row_lo = strip * rows_per_strip;
  const int row_hi = min(h, row_lo + rows_per_strip) - 1;
  const int cnt = stage_scene_view(db, in, view0 + lv, n_cap, s_R, s_pre, s_lab, s_col, sK, &s_cnt, s_warp);
  const SceneTris tris = make_scene_tris(db, s_R, s_pre, s_lab, cnt, sK);
  const bool q8 = (flags & 1u) != 0, gl_axes = (flags & 2u) != 0;
  const ResolveCtx ctx = make_resolve_ctx(out, lv, h, w, nullptr);
  const unsigned long long* vis = vis_all + static_cast<size_t>(lv) * h * w;
  const int npix = h * w;
  const TexRef no_tex{nullptr, nullptr, 0, 0, 0};
  for (int pix = row_lo * w + threadIdx.x; pix < (row_hi + 1) * w; pix += blockDim.x) {
    const int i = pix / w, j = pix - i * w;
    const unsigned long long key = __ldcg(vis + pix);
    int k = -1;
    if (key == ~0ull) {  // background: no instance is looked up
      VtxSrc none;
      none.cache = nullptr; none.verts = nullptr; none.sR = s_R;
      none.fx = none.cx = none.fy = none.cy = 0.f;
      resolve_pixel<false, false>(ctx, none, db.faces4, db.vattr, no_tex, key, lv, i, j, h, w, q8, gl_axes, out);
    } else {
      const int s = static_cast<int>(key & 0xffffffffu);
      k = tris.instance(s);
      const TriRef r = tris.at(k, s);
      const int lab = s_lab[k];
      const long long v_off = db.vert_offsets[lab];
      // the key the single-object renderer holds for this pixel: same 1/z bits, instance-local triangle index
      const unsigned long long local = (key & 0xffffffff00000000ull) | static_cast<unsigned>(r.tri);
      resolve_pixel<false, TEXTURED, true>(ctx, r.src, r.faces, db.vattr + 2 * v_off,
                                           TEXTURED ? mesh_texture(db, lab, v_off, true) : no_tex, local, lv, i, j, h, w,
                                           q8, gl_axes, out, s_col + 3 * k);
    }
    if (inst_id != nullptr) inst_id[static_cast<size_t>(lv) * npix + pix] = k;
  }
}

// ---------------------------------------------------------------------------------------------
// Tiled kernel: per-view vertex transform -> triangles binned into screen strips -> z-test of one strip at a time in
// SHARED memory -> shade + coalesced stores.  No global visibility buffer (the untiled kernel keeps 2 x SMs of them, 182 MB at
// 240x320: more than the L2, so its clear / min-reduce / read-back traffic reached DRAM).
//
// One CTA (512 threads, two per SM) per (view, group of strips):
//   (B)  snap the vertices into the CTA's L2-resident cache;
//   (C0) one thread per triangle: bounding rows -> a range word per triangle; triangles are counted per strip, the counts
//        prefix-summed, and a second pass over the range words fills compact per-strip lists (global scratch, a few KB);
//        triangles wider or taller than 64 px (edge values beyond 32 bits) go to a list handled by the whole CTA;
//   per strip (rows_per_strip x w pixels, 64-bit keys in shared memory):
//   (C1) batches of 512 listed triangles, one per thread: edge functions at the corner of the strip-clipped bounding box,
//        per-pixel steps, 1/z, 1/area -> a record in shared memory; an exclusive scan of the boxes' pixel counts;
//   (C2) the batch's candidate fragments are dealt out EVENLY: thread t takes fragments [t*c, (t+1)*c) of the concatenated
//        boxes (binary search for its first triangle, then it walks boxes row by row).  One thread per triangle -- the
//        untiled kernel -- idles most of a warp while its largest box is walked (r01: 62% of the instructions, 64% lane
//        utilisation, warp time = the largest of 32 boxes);
//   (D)  resolve_pixel on the strip: keys from shared memory, triangle + packed attributes gathered with 16-byte loads.
// Same integers, same correctly rounded float operations, order-independent 64-bit minimum: bit-identical to
// raster_kernel and to oracle/raster_ref.c.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void smem_min64(unsigned long long* cell, unsigned long long key) {
  unsigned long long old = *reinterpret_cast<volatile unsigned long long*>(cell);
  while (key < old) {
    const unsigned long long prev = atomicCAS(cell, old, key);
    if (prev == old) break;
    old = prev;
  }
}

template <typename W>
__device__ __forceinline__ void emit_fragment_smem(W w0, W w1, W w2, float iza, float izb, float izc, float inv_area,
                                                   int tri, unsigned long long* cell) {
  if ((w0 | w1 | w2) < 0) return;
  const float l0 = __fmul_rn(static_cast<float>(w0), inv_area);
  const float l1 = __fmul_rn(static_cast<float>(w1), inv_area);
  const float l2 = __fmul_rn(static_cast<float>(w2), inv_area);
  const float iz = __fmaf_rn(l0, iza, __fmaf_rn(l1, izb, __fmul_rn(l2, izc)));
  if (!(iz >= kIzMin && iz <= kIzMax)) return;
  smem_min64(cell, (static_cast<unsigned long long>(~__float_as_uint(iz)) << 32) | static_cast<unsigned>(tri));
}

template <bool TEXTURED>
__global__ void __launch_bounds__(kTileThreads, 2)
raster_tiled_kernel(const MeshDb db, const int* __restrict__ label_idx, const float* __restrict__ TCO,
                    const float* __restrict__ K, int n_views, int h, int w, unsigned flags, RasterOut out, int R,
                    int n_strips, int groups) {
  extern __shared__ __align__(16) unsigned char s_dyn[];
  unsigned long long* s_vis = reinterpret_cast<unsigned long long*>(s_dyn);
  int* s_rec = reinterpret_cast<int*>(s_vis + static_cast<size_t>(R) * w);  // [kRecFields][kTileBatch]
  int* s_start = s_rec + kRecFields * kTileBatch;                            // [kTileBatch + 1]
  AxisW* s_axis = reinterpret_cast<AxisW*>(s_start + kTileBatch + 1);        // [h + w] when the crop is fused
  __shared__ float sR[12];
  __shared__ float sK[4];
  __shared__ int s_valid;
  __shared__ int s_nbig;
  __shared__ int s_counts[kTileMaxStrips + 1];
  __shared__ int s_cursor[kTileMaxStrips];
  __shared__ int s_wsum[kTileThreads / 32];

  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int4* vtx = db.vtx_cache + static_cast<size_t>(blockIdx.x) * db.nv_max;
  unsigned* scratch = db.tile_scratch + static_cast<size_t>(blockIdx.x) * db.tile_words;
  unsigned* g_range = scratch;                                   // [nf_max] row-range word per triangle
  unsigned* g_big = scratch + db.nf_max;                         // [nf_max] large triangles
  unsigned* g_list = scratch + 2 * static_cast<size_t>(db.nf_max);  // [kTileMaxSpan * nf_max] per-strip lists, back to back
  const bool q8 = (flags & 1u) != 0;
  const bool gl_axes = (flags & 2u) != 0;
  const int spg = (n_strips + groups - 1) / groups;

  for (int item = blockIdx.x; item < n_views * groups; item += gridDim.x) {
    const int view = item / groups, grp = item - view * groups;
    const int s_lo = grp * spg, s_hi = min(n_strips, s_lo + spg);
    const int grow_lo = s_lo * R, grow_hi = min(h, s_hi * R) - 1;
    __syncthreads();  // previous item fully resolved before shared / global scratch is reused
    if (tid == 0) {
      load_view(db, label_idx, TCO, K, view, sR, sK, &s_valid);
      s_nbig = 0;
    }
    for (int i = tid; i <= n_strips; i += kTileThreads) s_counts[i] = 0;
    __syncthreads();
    const bool valid = s_valid != 0;
    const int lab = valid ? label_idx[view] : 0;
    const long long v_off = valid ? db.vert_offsets[lab] : 0;
    const int nv = valid ? static_cast<int>(db.vert_offsets[lab + 1] - v_off) : 0;
    const long long f_off = valid ? db.face_offsets[lab] : 0;
    const int nf = valid ? static_cast<int>(db.face_offsets[lab + 1] - f_off) : 0;
    const int4* faces = db.faces4 + f_off;
    const float4* vattr = db.vattr + 2 * v_off;

    // (B) transform + snap vertices
    const float fx = sK[0], cx = sK[1], fy = sK[2], cy = sK[3];
    for (int i = tid; i < nv; i += kTileThreads) vtx[i] = snap_vertex(db.verts + 3 * (v_off + i), sR, fx, cx, fy, cy);
    __syncthreads();
    VtxSrc src;
    src.cache = vtx;
    src.verts = nullptr;
    src.sR = sR;
    src.fx = fx; src.cx = cx; src.fy = fy; src.cy = cy;

    // (C0) rows of every triangle, strip counts
    for (int tri = tid; tri < nf; tri += kTileThreads) {
      const TriSetup t = load_tri<true>(src, faces, tri);
      unsigned word = 0u;
      if (t.ok) {
        int j0, j1, i0, i1;
        raster_bbox(t, h, w, j0, j1, i0, i1);
        i0 = max(i0, grow_lo);
        i1 = min(i1, grow_hi);
        if (j0 <= j1 && i0 <= i1) {
          const int ext_x = max(t.ax, max(t.bx, t.cx)) - min(t.ax, min(t.bx, t.cx));
          const int ext_y = max(t.ay, max(t.by, t.cy)) - min(t.ay, min(t.by, t.cy));
          const bool big = ext_x > kSmallExt || ext_y > kSmallExt;
          word = 0x80000000u | (big ? 0x40000000u : 0u) | (static_cast<unsigned>(i1) << 12) | static_cast<unsigned>(i0);
          if (big) {
            g_big[atomicAdd(&s_nbig, 1)] = tri;
          } else {
            for (int s = i0 / R; s <= i1 / R; ++s) atomicAdd(&s_counts[s + 1], 1);
          }
        }
      }
      g_range[tri] = word;
    }
    __syncthreads();
    if (tid == 0)
      for (int s = 0; s < n_strips; ++s) s_counts[s + 1] += s_counts[s];  // s_counts[s] = first list entry of strip s
    __syncthreads();
    for (int i = tid; i < n_strips; i += kTileThreads) s_cursor[i] = s_counts[i];
    __syncthreads();
    for (int tri = tid; tri < nf; tri += kTileThreads) {
      const unsigned word = g_range[tri];
      if ((word & 0xC0000000u) == 0x80000000u) {
        const int i0 = static_cast<int>(word & 0xfffu), i1 = static_cast<int>((word >> 12) & 0xfffu);
        for (int s = i0 / R; s <= i1 / R; ++s) g_list[atomicAdd(&s_cursor[s], 1)] = static_cast<unsigned>(tri);
      }
    }
    const ResolveCtx ctx = make_resolve_ctx(out, view, h, w, s_axis, (flags & 4u) != 0 && valid ? db.verts + 3 * v_off : nullptr,
                                            valid ? db.radius[lab] : 0.f);
    const TexRef texref = TEXTURED ? mesh_texture(db, lab, v_off, valid) : TexRef{nullptr, nullptr, 0, 0, 0};
    __syncthreads();
    const int nbig = s_nbig;

    for (int s = s_lo; s < s_hi; ++s) {
      const int row_lo = s * R, row_hi = min(h, row_lo + R) - 1;
      const int strip_px = (row_hi - row_lo + 1) * w;
      for (int i = tid; i < strip_px; i += kTileThreads) s_vis[i] = ~0ull;
      const int seg0 = s_counts[s], seg1 = s_counts[s + 1];
      for (int b0 = seg0; b0 < seg1; b0 += kTileBatch) {
        const int n = min(kTileBatch, seg1 - b0);
        // (C1) one triangle per thread: record + number of candidate fragments
        int count = 0;
        if (tid < n) {
          const int tri = static_cast<int>(g_list[b0 + tid]);
          const TriSetup t = load_tri<true>(src, faces, tri);
          int j0, j1, i0, i1;
          raster_bbox(t, h, w, j0, j1, i0, i1);
          i0 = max(i0, row_lo);
          i1 = min(i1, row_hi);
          const int px0 = j0 * kSub + kHalf, py0 = i0 * kSub + kHalf;
          const long long sgn = t.flip ? -1 : 1;
          // exact integers; below 2^29 in magnitude for a triangle of at most 64 x 64 px (see cover_triangle)
          s_rec[0 * kTileBatch + tid] = static_cast<int>(sgn * edge_fn(t.bx, t.by, t.cx, t.cy, px0, py0));
          s_rec[1 * kTileBatch + tid] = static_cast<int>(sgn * edge_fn(t.cx, t.cy, t.ax, t.ay, px0, py0));
          s_rec[2 * kTileBatch + tid] = static_cast<int>(sgn * edge_fn(t.ax, t.ay, t.bx, t.by, px0, py0));
          const int isg = t.flip ? -1 : 1;
          s_rec[3 * kTileBatch + tid] = -isg * (t.cy - t.by) * kSub;
          s_rec[4 * kTileBatch + tid] = -isg * (t.ay - t.cy) * kSub;
          s_rec[5 * kTileBatch + tid] = -isg * (t.by - t.ay) * kSub;
          s_rec[6 * kTileBatch + tid] = isg * (t.cx - t.bx) * kSub;
          s_rec[7 * kTileBatch + tid] = isg * (t.ax - t.cx) * kSub;
          s_rec[8 * kTileBatch + tid] = isg * (t.bx - t.ax) * kSub;
          s_rec[9 * kTileBatch + tid] = __float_as_int(t.iza);
          s_rec[10 * kTileBatch + tid] = __float_as_int(t.izb);
          s_rec[11 * kTileBatch + tid] = __float_as_int(t.izc);
          s_rec[12 * kTileBatch + tid] = __float_as_int(t.inv_area);
          s_rec[13 * kTileBatch + tid] = (i0 - row_lo) * w + j0;  // strip-relative index of the box corner
          const int bw = j1 - j0 + 1;
          s_rec[14 * kTileBatch + tid] = bw;
          s_rec[15 * kTileBatch + tid] = tri;
          count = bw * (i1 - i0 + 1);
        }
        // exclusive scan of the counts over the CTA
        int incl = count;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int v = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += v;
        }
        if (lane == 31) s_wsum[wid] = incl;
        __syncthreads();
        if (wid == 0) {
          int v = lane < kTileThreads / 32 ? s_wsum[lane] : 0;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += u;
          }
          if (lane < kTileThreads / 32) s_wsum[lane] = v;  // inclusive over warps
        }
        __syncthreads();
        const int excl = incl - count + (wid > 0 ? s_wsum[wid - 1] : 0);
        s_start[tid] = excl;
        if (tid == kTileThreads - 1) s_start[kTileBatch] = excl + count;
        __syncthreads();
        // (C2) fragments dealt out evenly
        const int T = s_start[kTileBatch];
        const int c = (T + kTileThreads - 1) / kTileThreads;
        int f = tid * c;
        const int f1 = min(T, f + c);
        if (f < f1) {
          int lo = 0, hi = kTileBatch;  // s_start[lo] <= f < s_start[hi]
          while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (s_start[mid] <= f) lo = mid; else hi = mid;
          }
          int k = lo;
          while (f < f1) {
            const int st = s_start[k], en = s_start[k + 1];
            if (en <= f) { ++k; continue; }  // empty box
            const int r0 = s_rec[0 * kTileBatch + k], r1 = s_rec[1 * kTileBatch + k], r2 = s_rec[2 * kTileBatch + k];
            const int ex0 = s_rec[3 * kTileBatch + k], ex1 = s_rec[4 * kTileBatch + k], ex2 = s_rec[5 * kTileBatch + k];
            const int ey0 = s_rec[6 * kTileBatch + k], ey1 = s_rec[7 * kTileBatch + k], ey2 = s_rec[8 * kTileBatch + k];
            const float iza = __int_as_float(s_rec[9 * kTileBatch + k]), izb = __int_as_float(s_rec[10 * kTileBatch + k]);
            const float izc = __int_as_float(s_rec[11 * kTileBatch + k]), inv_area = __int_as_float(s_rec[12 * kTileBatch + k]);
            const int corner = s_rec[13 * kTileBatch + k], bw = s_rec[14 * kTileBatch + k], tri = s_rec[15 * kTileBatch + k];
            const int off = f - st;
            const int nfr = min(en, f1) - f;
            int di = off / bw, dj = off - di * bw;
            int w0 = r0 + dj * ex0 + di * ey0, w1 = r1 + dj * ex1 + di * ey1, w2 = r2 + dj * ex2 + di * ey2;
            int idx = corner + di * w + dj;
            for (int q = 0; q < nfr; ++q) {
              emit_fragment_smem<int>(w0, w1, w2, iza, izb, izc, inv_area, tri, s_vis + idx);
              ++dj; ++idx;
              w0 += ex0; w1 += ex1; w2 += ex2;
              if (dj == bw) {
                dj = 0; ++di;
                idx += w - bw;
                w0 = r0 + di * ey0; w1 = r1 + di * ey1; w2 = r2 + di * ey2;
              }
            }
            f += nfr;
            ++k;
          }
        }
        __syncthreads();  // the next batch overwrites the records
      }
      // large triangles (rare): the whole CTA shares each strip-clipped bounding box, 64-bit edge functions
      for (int b = 0; b < nbig; ++b) {
        const int tri = static_cast<int>(g_big[b]);
        const TriSetup t = load_tri<true>(src, faces, tri);
        int j0, j1, i0, i1;
        raster_bbox(t, h, w, j0, j1, i0, i1);
        i0 = max(i0, row_lo);
        i1 = min(i1, row_hi);
        if (i0 > i1) continue;
        const int bw = j1 - j0 + 1;
        const int cnt = bw * (i1 - i0 + 1);
        for (int k = tid; k < cnt; k += kTileThreads) {
          const int di = k / bw;
          const int i = i0 + di, j = j0 + (k - di * bw);
          const int px = j * kSub + kHalf, py = i * kSub + kHalf;
          long long w0 = edge_fn(t.bx, t.by, t.cx, t.cy, px, py);
          long long w1 = edge_fn(t.cx, t.cy, t.ax, t.ay, px, py);
          long long w2 = edge_fn(t.ax, t.ay, t.bx, t.by, px, py);
          if (t.flip) { w0 = -w0; w1 = -w1; w2 = -w2; }
          emit_fragment_smem<long long>(w0, w1, w2, t.iza, t.izb, t.izc, t.inv_area, tri, s_vis + (i - row_lo) * w + j);
        }
      }
      __syncthreads();
      // (D) resolve + shade + write the strip
      for (int p = tid; p < strip_px; p += kTileThreads) {
        const int di = p / w;
        resolve_pixel<true, TEXTURED>(ctx, src, faces, vattr, texref, s_vis[p], view, row_lo + di, p - di * w, h, w, q8,
                                      gl_axes, out);
      }
      __syncthreads();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------
static int upload_tables() {
  if (g_tables_ready) return MPX_OK;
  QuantTables t;
  for (int k = 0; k < 256; ++k) t.q8[k] = static_cast<float>(k) / 255.0f;
  for (int k = 0; k < 32; ++k) t.tex[k] = static_cast<float>((k * 255) >> 5) / 255.0f;
  MPX_CHECK_CUDA(cudaMemcpyToSymbol(c_tables, &t, sizeof(t)));
  g_tables_ready = true;
  return MPX_OK;
}

int meshdb_create(int n_meshes, const float* verts, const float* normals, const float* colors,
                  const int64_t* vert_offsets, const int32_t* faces, const int64_t* face_offsets,
                  MeshDb** out) {
  MPX_REQUIRE(n_meshes > 0, "meshdb: need at least one mesh");
  int rc = upload_tables();
  if (rc != MPX_OK) return rc;
  MeshDb* db = new MeshDb();
  memset(db, 0, sizeof(MeshDb));
  db->n_meshes = n_meshes;
  const long long nv = vert_offsets[n_meshes], nf = face_offsets[n_meshes];
  int nv_max = 0;
  for (int i = 0; i < n_meshes; ++i) {
    const long long c = vert_offsets[i + 1] - vert_offsets[i];
    if (c > nv_max) nv_max = static_cast<int>(c);
    const long long nfi = face_offsets[i + 1] - face_offsets[i];
    for (long long f = 3 * face_offsets[i]; f < 3 * (face_offsets[i] + nfi); ++f) {
      if (faces[f] < 0 || faces[f] >= c) {
        delete db;
        set_error("meshdb: mesh %d has a face index out of range", i);
        return MPX_ERR_INVALID;
      }
    }
  }
  db->nv_max = nv_max > 0 ? nv_max : 1;
  db->slots = 2 * sm_count();
  int nf_max = 1;
  for (int i = 0; i < n_meshes; ++i) {
    const long long c = face_offsets[i + 1] - face_offsets[i];
    if (c > nf_max) nf_max = static_cast<int>(c);
  }
  db->nf_max = nf_max;
  MPX_CHECK_CUDA(cudaMalloc(&db->verts, sizeof(float) * 3 * (nv > 0 ? nv : 1)));
  MPX_CHECK_CUDA(cudaMalloc(&db->normals, sizeof(float) * 3 * (nv > 0 ? nv : 1)));
  MPX_CHECK_CUDA(cudaMalloc(&db->colors, sizeof(float) * 3 * (nv > 0 ? nv : 1)));
  MPX_CHECK_CUDA(cudaMalloc(&db->faces, sizeof(int) * 3 * (nf > 0 ? nf : 1)));
  MPX_CHECK_CUDA(cudaMalloc(&db->vert_offsets, sizeof(long long) * (n_meshes + 1)));
  MPX_CHECK_CUDA(cudaMalloc(&db->face_offsets, sizeof(long long) * (n_meshes + 1)));
  MPX_CHECK_CUDA(cudaMalloc(&db->vtx_cache, sizeof(int4) * static_cast<size_t>(db->slots) * db->nv_max));
  MPX_CHECK_CUDA(cudaMemcpy(db->verts, verts, sizeof(float) * 3 * nv, cudaMemcpyHostToDevice));
  MPX_CHECK_CUDA(cudaMemcpy(db->normals, normals, sizeof(float) * 3 * nv, cudaMemcpyHostToDevice));
  MPX_CHECK_CUDA(cudaMemcpy(db->colors, colors, sizeof(float) * 3 * nv, cudaMemcpyHostToDevice));
  MPX_CHECK_CUDA(cudaMemcpy(db->faces, faces, sizeof(int) * 3 * nf, cudaMemcpyHostToDevice));
  MPX_CHECK_CUDA(cudaMemcpy(db->vert_offsets, vert_offsets, sizeof(long long) * (n_meshes + 1),
                            cudaMemcpyHostToDevice));
  MPX_CHECK_CUDA(cudaMemcpy(db->face_offsets, face_offsets, sizeof(long long) * (n_meshes + 1),
                            cudaMemcpyHostToDevice));
  {  // bounding radius about the object origin, in float with the oracle's operation order
    std::vector<float> rad(n_meshes, 0.f);
    for (int i = 0; i < n_meshes; ++i)
      for (long long v = vert_offsets[i]; v < vert_offsets[i + 1]; ++v) {
        const float x = verts[3 * v], y = verts[3 * v + 1], z = verts[3 * v + 2];
        const float r = sqrtf(fmaf(x, x, fmaf(y, y, z * z)));
        if (r > rad[i]) rad[i] = r;
      }
    MPX_CHECK_CUDA(cudaMalloc(&db->radius, sizeof(float) * n_meshes));
    MPX_CHECK_CUDA(cudaMemcpy(db->radius, rad.data(), sizeof(float) * n_meshes, cudaMemcpyHostToDevice));
  }
  // packed copies: 16-byte faces, two float4 of attributes per vertex (uv filled in by meshdb_set_textures)
  {
    std::vector<int4> f4(nf > 0 ? nf : 1);
    for (long long f = 0; f < nf; ++f) f4[f] = make_int4(faces[3 * f], faces[3 * f + 1], faces[3 * f + 2], 0);
    std::vector<float4> va(2 * (nv > 0 ? nv : 1));
    for (long long v = 0; v < nv; ++v) {
      va[2 * v] = make_float4(colors[3 * v], colors[3 * v + 1], colors[3 * v + 2], normals[3 * v]);
      va[2 * v + 1] = make_float4(normals[3 * v + 1], normals[3 * v + 2], 0.f, 0.f);
    }
    MPX_CHECK_CUDA(cudaMalloc(&db->faces4, sizeof(int4) * f4.size()));
    MPX_CHECK_CUDA(cudaMalloc(&db->vattr, sizeof(float4) * va.size()));
    MPX_CHECK_CUDA(cudaMemcpy(db->faces4, f4.data(), sizeof(int4) * f4.size(), cudaMemcpyHostToDevice));
    MPX_CHECK_CUDA(cudaMemcpy(db->vattr, va.data(), sizeof(float4) * va.size(), cudaMemcpyHostToDevice));
  }
  // tiled kernel scratch per CTA slot: range word per triangle, strip lists (a small triangle is at most 65 px tall:
  // <= kTileMaxSpan strips), list of large triangles
  db->tile_words = static_cast<long long>(nf_max) * (2 + kTileMaxSpan);
  MPX_CHECK_CUDA(cudaMalloc(&db->tile_scratch, sizeof(unsigned) * db->tile_words * db->slots));
  *out = db;
  return MPX_OK;
}

int meshdb_set_textures(MeshDb* db, const float* uv, const unsigned char* tex, const int64_t* tex_offsets,
                        const int32_t* tex_dims, const int32_t* tex_modulate) {
  MPX_REQUIRE(db != nullptr && uv != nullptr && tex != nullptr && tex_offsets != nullptr && tex_dims != nullptr,
              "meshdb_set_textures: null argument");
  MPX_REQUIRE(db->tex_info == nullptr, "meshdb_set_textures: textures already set");
  const int n = db->n_meshes;
  std::vector<long long> vo(n + 1);
  MPX_CHECK_CUDA(cudaMemcpy(vo.data(), db->vert_offsets, sizeof(long long) * (n + 1), cudaMemcpyDeviceToHost));
  std::vector<int4> info(n);
  std::vector<long long> offs(n);
  for (int i = 0; i < n; ++i) {
    const int th = tex_dims[2 * i], tw = tex_dims[2 * i + 1];
    MPX_REQUIRE(th >= 0 && tw >= 0 && th <= 16384 && tw <= 16384, "meshdb_set_textures: mesh %d texture %dx%d", i, th, tw);
    MPX_REQUIRE(tex_offsets[i + 1] - tex_offsets[i] == static_cast<int64_t>(th) * tw * 3,
                "meshdb_set_textures: mesh %d texture bytes do not match its size", i);
    info[i] = make_int4(th, tw, tex_modulate ? tex_modulate[i] : 0, 0);
    offs[i] = tex_offsets[i];
  }
  const long long nv = vo[n], bytes = tex_offsets[n];
  MPX_CHECK_CUDA(cudaMalloc(&db->uv, sizeof(float) * 2 * (nv > 0 ? nv : 1)));
  MPX_CHECK_CUDA(cudaMalloc(&db->tex, bytes > 0 ? bytes : 1));
  MPX_CHECK_CUDA(cudaMalloc(&db->tex_offsets, sizeof(long long) * n));
  MPX_CHECK_CUDA(cudaMalloc(&db->tex_info, sizeof(int4) * n));
  MPX_CHECK_CUDA(cudaMemcpy(db->uv, uv, sizeof(float) * 2 * nv, cudaMemcpyHostToDevice));
  {  // texture coordinates into the packed per-vertex attributes
    std::vector<float4> va(2 * (nv > 0 ? nv : 1));
    MPX_CHECK_CUDA(cudaMemcpy(va.data(), db->vattr, sizeof(float4) * 2 * nv, cudaMemcpyDeviceToHost));
    for (long long v = 0; v < nv; ++v) {
      va[2 * v + 1].z = uv[2 * v];
      va[2 * v + 1].w = uv[2 * v + 1];
    }
    MPX_CHECK_CUDA(cudaMemcpy(db->vattr, va.data(), sizeof(float4) * 2 * nv, cudaMemcpyHostToDevice));
  }
  MPX_CHECK_CUDA(cudaMemcpy(db->tex, tex, bytes, cudaMemcpyHostToDevice));
  MPX_CHECK_CUDA(cudaMemcpy(db->tex_offsets, offs.data(), sizeof(long long) * n, cudaMemcpyHostToDevice));
  MPX_CHECK_CUDA(cudaMemcpy(db->tex_info, info.data(), sizeof(int4) * n, cudaMemcpyHostToDevice));
  return MPX_OK;
}

void meshdb_destroy(MeshDb* db) {
  if (!db) return;
  cudaFree(db->uv);
  cudaFree(db->tex);
  cudaFree(db->tex_offsets);
  cudaFree(db->tex_info);
  cudaFree(db->verts);
  cudaFree(db->normals);
  cudaFree(db->colors);
  cudaFree(db->faces);
  cudaFree(db->vert_offsets);
  cudaFree(db->face_offsets);
  cudaFree(db->vtx_cache);
  cudaFree(db->faces4);
  cudaFree(db->vattr);
  cudaFree(db->tile_scratch);
  cudaFree(db->radius);
  delete db;
}

size_t raster_workspace_bytes(int h, int w) {
  return static_cast<size_t>(2 * sm_count()) * h * w * sizeof(unsigned long long);
}

int raster_launch(const MeshDb* db, const int32_t* label_idx, const float* TCO, const float* K, int n_views,
                  int h, int w, unsigned flags, const RasterOut& out, void* workspace, size_t workspace_bytes,
                  cudaStream_t stream) {
  MPX_REQUIRE(db != nullptr, "raster: null mesh database");
  MPX_REQUIRE(h > 0 && w > 0 && h <= 4096 && w <= 4096, "raster: resolution %dx%d unsupported", h, w);
  MPX_REQUIRE(workspace_bytes >= raster_workspace_bytes(h, w), "raster: workspace too small");
  if (out.x) {
    MPX_REQUIRE(h % 2 == 0 && w % 2 == 0, "raster: fused output needs even resolution");
    MPX_REQUIRE(out.ch_per_view == 3 || out.ch_per_view == 4 || out.ch_per_view == 6 || out.ch_per_view == 7,
                "raster: ch_per_view must be 3 (rgb), 4 (+depth), 6 (+normals) or 7 (+normals, depth)");
    MPX_REQUIRE(out.views_per_sample >= 1 &&
                    out.ch_offset + out.views_per_sample * out.ch_per_view <= out.c_pad,
                "raster: channels do not fit c_pad=%d", out.c_pad);
    if (out.crop_images) {
      MPX_REQUIRE(out.views_per_sample == 1, "raster: the fused crop needs one view per sample");
      MPX_REQUIRE(out.crop_c == out.ch_offset && (out.crop_c == 3 || out.crop_c == 4),
                  "raster: fused crop channels (%d) must equal ch_offset (%d)", out.crop_c, out.ch_offset);
      MPX_REQUIRE(out.crop_c + out.ch_per_view <= 16 && (out.c_pad == 16 || out.c_pad == 32),
                  "raster: fused crop layout unsupported");
      MPX_REQUIRE((reinterpret_cast<uintptr_t>(out.x) & 15) == 0, "raster: x must be 16-byte aligned");
    }
  }
  if (n_views == 0) return MPX_OK;
  if (g_scatter && n_views * 8 <= sm_count()) {
    // a handful of views: triangles of a view spread over `parts` CTAs, then a resolve kernel over row strips
    unsigned long long* vis = reinterpret_cast<unsigned long long*>(workspace);
    MPX_CHECK_CUDA(cudaMemsetAsync(vis, 0xFF, static_cast<size_t>(n_views) * h * w * sizeof(unsigned long long), stream));
    int parts = sm_count() / n_views;
    if (parts > 40) parts = 40;  // 10k triangles / (40 * 256 threads) = one triangle per thread
    raster_cover_kernel<<<n_views * parts, kCoverThreads, 0, stream>>>(*db, label_idx, TCO, K, n_views, h, w, vis,
                                                                       parts);
    MPX_CHECK_CUDA(cudaGetLastError());
    int strips = 2 * sm_count() / n_views;
    if (strips > h) strips = h;
    const int rows = (h + strips - 1) / strips;
    strips = (h + rows - 1) / rows;  // no empty strips
    if (db->tex_info != nullptr)
      raster_resolve_kernel<true><<<n_views * strips, kRasterThreads, 0, stream>>>(*db, label_idx, TCO, K, n_views, h, w,
                                                                                  flags, out, vis, strips);
    else
      raster_resolve_kernel<false><<<n_views * strips, kRasterThreads, 0, stream>>>(*db, label_idx, TCO, K, n_views, h, w,
                                                                                   flags, out, vis, strips);
    MPX_CHECK_CUDA(cudaGetLastError());
    g_launches += 2;
    return MPX_OK;
  }
  if (g_tiled && h < 4096 && w < 4096) {
    // rows per strip from the shared memory left for the 64-bit visibility strip with two CTAs per SM
    const bool axis = out.crop_images != nullptr && h + w <= kAxisTableMax;
    const size_t fixed = static_cast<size_t>(kRecFields * kTileBatch + kTileBatch + 1) * sizeof(int) +
                         (axis ? static_cast<size_t>(h + w) * sizeof(AxisW) : 0) + 16;
    const size_t budget = 110 * 1024;
    int R = fixed < budget ? static_cast<int>((budget - fixed) / (sizeof(unsigned long long) * w)) : 0;
    if (R > h) R = h;
    if (R >= kTileMinRows) {
      int n_strips = (h + R - 1) / R;
      R = (h + n_strips - 1) / n_strips;
      n_strips = (h + R - 1) / R;
      if (n_strips <= kTileMaxStrips && R >= kTileMinRows) {
        int groups = 1;
        if (n_views < db->slots) groups = db->slots / n_views;
        if (groups > n_strips) groups = n_strips;
        const long long items = static_cast<long long>(n_views) * groups;
        const int grid = items < db->slots ? static_cast<int>(items) : db->slots;
        const size_t dyn = static_cast<size_t>(R) * w * sizeof(unsigned long long) + fixed;
        auto kern = db->tex_info != nullptr ? raster_tiled_kernel<true> : raster_tiled_kernel<false>;
        MPX_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(dyn)));
        kern<<<grid, kTileThreads, dyn, stream>>>(*db, label_idx, TCO, K, n_views, h, w, flags, out, R, n_strips, groups);
        MPX_CHECK_CUDA(cudaGetLastError());
        ++g_launches;
        return MPX_OK;
      }
    }
  }
  // CTA b of the untiled kernel uses visibility buffer b of the workspace, which holds 2 x sm_count() of them, and vertex
  // cache slot b of the mesh database, which holds db->slots (2 x sm_count() when it was created).  mpx_set_sm_limit can
  // change sm_count() after the database exists, so the grid takes the smaller of the two; the persistent loop covers
  // every (view, strip) item with any grid size.
  const int slots = db->slots < 2 * sm_count() ? db->slots : 2 * sm_count();
  int strips = 1;
  if (n_views < slots) {
    strips = slots / n_views;
    if (strips > 16) strips = 16;
    if (strips > h) strips = h;
  }
  const long long items = static_cast<long long>(n_views) * strips;
  const int grid = items < slots ? static_cast<int>(items) : slots;
  if (db->tex_info != nullptr)
    raster_kernel<true><<<grid, kRasterThreads, 0, stream>>>(*db, label_idx, TCO, K, n_views, h, w, flags, out,
                                                             reinterpret_cast<unsigned long long*>(workspace), strips);
  else
    raster_kernel<false><<<grid, kRasterThreads, 0, stream>>>(*db, label_idx, TCO, K, n_views, h, w, flags, out,
                                                              reinterpret_cast<unsigned long long*>(workspace), strips);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

int raster_scene_launch(const MeshDb* db, int n_views, int n_inst, const int32_t* inst_offsets, const int32_t* inst_label,
                        const float* inst_TCO, const float* inst_color, const float* K, int h, int w, unsigned flags,
                        float* rgb, float* normals, float* depth, int32_t* inst_id, void* workspace,
                        size_t workspace_bytes, cudaStream_t stream) {
  MPX_REQUIRE(db != nullptr, "raster_scene: null mesh database");
  MPX_REQUIRE(n_views >= 0 && n_inst >= 0, "raster_scene: n_views=%d n_inst=%d", n_views, n_inst);
  MPX_REQUIRE(h > 0 && w > 0 && h <= 4096 && w <= 4096, "raster_scene: resolution %dx%d unsupported", h, w);
  MPX_REQUIRE((flags & 4u) == 0, "raster_scene: point lights are not implemented for scenes (only white ambient light)");
  MPX_REQUIRE((flags & ~3u) == 0, "raster_scene: flags 0x%x: only bits 0 (quantise) and 1 (GL normals)", flags);
  MPX_REQUIRE(static_cast<long long>(n_inst) <= static_cast<long long>(kSceneMaxInst) * n_views,
              "raster_scene: %d instances for %d views (at most %d per view)", n_inst, n_views, kSceneMaxInst);
  MPX_REQUIRE(workspace_bytes >= raster_workspace_bytes(h, w), "raster_scene: workspace too small");
  if (n_views == 0) return MPX_OK;
  const int n_cap = n_inst < 1 ? 1 : (n_inst < kSceneMaxInst ? n_inst : kSceneMaxInst);
  MPX_REQUIRE(static_cast<long long>(n_cap) * db->nf_max < (1ll << 31),
              "raster_scene: %d instances of up to %d triangles reach 2^31 scene triangles", n_cap, db->nf_max);
  const size_t smem_cover = scene_smem_bytes(n_cap, false), smem_resolve = scene_smem_bytes(n_cap, true);
  auto resolve = db->tex_info != nullptr ? scene_resolve_kernel<true> : scene_resolve_kernel<false>;
  MPX_CHECK_CUDA(cudaFuncSetAttribute(scene_cover_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem_cover)));
  MPX_CHECK_CUDA(cudaFuncSetAttribute(resolve, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem_resolve)));
  SceneIn in{inst_offsets, inst_label, inst_TCO, inst_color, K, n_inst};
  const size_t npix = static_cast<size_t>(h) * w;
  const int chunk = 2 * sm_count();  // the visibility buffers of raster_workspace_bytes
  // triangles per view if every instance had the largest mesh: about two per cover thread
  const long long tris_per_view = static_cast<long long>((n_inst + n_views - 1) / n_views) * db->nf_max;
  unsigned long long* vis = reinterpret_cast<unsigned long long*>(workspace);
  for (int v0 = 0; v0 < n_views; v0 += chunk) {
    const int nv = n_views - v0 < chunk ? n_views - v0 : chunk;
    MPX_CHECK_CUDA(cudaMemsetAsync(vis, 0xFF, static_cast<size_t>(nv) * npix * sizeof(unsigned long long), stream));
    long long parts = (tris_per_view + 2 * kCoverThreads - 1) / (2 * kCoverThreads);
    const int max_parts = 8 * sm_count() / nv > 1 ? 8 * sm_count() / nv : 1;
    if (parts > max_parts) parts = max_parts;
    if (parts < 1) parts = 1;
    scene_cover_kernel<<<nv * static_cast<int>(parts), kCoverThreads, smem_cover, stream>>>(*db, in, v0, h, w, vis,
                                                                                           static_cast<int>(parts), n_cap);
    MPX_CHECK_CUDA(cudaGetLastError());
    int strips = 2 * sm_count() / nv;
    if (strips < 1) strips = 1;
    if (strips > h) strips = h;
    const int rows = (h + strips - 1) / strips;
    strips = (h + rows - 1) / rows;  // no empty strips
    RasterOut out;
    memset(&out, 0, sizeof(out));
    out.rgb = rgb ? rgb + static_cast<size_t>(v0) * 3 * npix : nullptr;
    out.normals = normals ? normals + static_cast<size_t>(v0) * 3 * npix : nullptr;
    out.depth = depth ? depth + static_cast<size_t>(v0) * npix : nullptr;
    resolve<<<nv * strips, kRasterThreads, smem_resolve, stream>>>(*db, in, v0, h, w, flags, out,
                                                                  inst_id ? inst_id + static_cast<size_t>(v0) * npix : nullptr,
                                                                  vis, strips, n_cap);
    MPX_CHECK_CUDA(cudaGetLastError());
    g_launches += 2;
  }
  return MPX_OK;
}

}  // namespace mpx
