/*
 * tests/scene_ref.c -- CPU restatement of the multi-object scene contract of mpx_raster_render_scene.  TEST
 * INFRASTRUCTURE ONLY: the checker of the CUDA scene renderer; nothing under megapose6d_b200/ uses it.
 *
 * It is compiled together with oracle/raster_ref.c (included below), so every per-vertex, per-triangle and per-fragment
 * step -- projection, 1/256-pixel snapping, exact edge functions, the per-sample near/far test, barycentrics, texture,
 * eye-normal texture, depth -- is the oracle's own code or a line-for-line restatement of its render_view.
 *
 * What it adds (reference: panda3d_renderer/panda3d_scene_renderer.py:139-358 render_scene, several posed objects seen by
 * one camera with one depth test; outputs CameraRenderingData, panda3d_renderer/types.py:43-125):
 *   - view v draws instances inst_offsets[v] .. inst_offsets[v+1]-1; instance i is mesh inst_label[i] at pose
 *     inst_TCO[i] (row-major 4x4, camera frame of that view); every fragment uses its own instance's pose, mesh, vertex
 *     attributes and texture;
 *   - scene triangle index: triangle t of the view's k-th instance has s = (face counts of instances 0..k-1) + t, and
 *     the visibility key is (~bits(1/z) << 32) | s.  The smallest key wins: the nearest fragment, ties to the lower
 *     instance, then to the lower triangle.  A one-instance scene holds exactly the keys of render_view, and therefore
 *     produces exactly its pixels;
 *   - colour override: inst_color [n_inst,3] (may be NULL); when an instance's first component is >= 0 its albedo
 *     (vertex colours and texture) is replaced by that colour before quantisation (Panda3dObjectData.color, alpha 1);
 *   - invalid input: an instance with a non-finite pose or a label outside [0, n_meshes) contributes nothing (and counts
 *     no faces); a view with non-finite K or no instances is all zero with inst_id -1;
 *   - inst_id [n_views,h,w] int32: the instance's index within its view for every covered pixel, -1 for background;
 *   - point lights (flags bit 2) are refused (-3): the reference positions scene lights through node callbacks, and what
 *     they mean for several objects is not defined.
 */
#include "raster_ref.c"

/* camera transform, projection and snapping of one mesh's vertices: render_view's vertex loop */
static void snap_vertices(const float* verts, int nv, const float* R, const float* K, vtx_t* vtx) {
  const float fx = K[0], cx = K[2], fy = K[4], cy = K[5];
  for (int i = 0; i < nv; ++i) {
    const float px = verts[3 * i], py = verts[3 * i + 1], pz = verts[3 * i + 2];
    const float xc = fmaf(R[0], px, fmaf(R[1], py, fmaf(R[2], pz, R[3])));
    const float yc = fmaf(R[4], px, fmaf(R[5], py, fmaf(R[6], pz, R[7])));
    const float zc = fmaf(R[8], px, fmaf(R[9], py, fmaf(R[10], pz, R[11])));
    vtx_t o;
    o.behind = !(zc >= K_PROJ_MIN);
    const float zs = o.behind ? 1.0f : zc;
    const float iz = 1.0f / zs;
    float u = fmaf(fx, xc * iz, cx);
    float v = fmaf(fy, yc * iz, cy);
    u = fminf(fmaxf(u, -K_CLAMP), K_CLAMP);
    v = fminf(fmaxf(v, -K_CLAMP), K_CLAMP);
    if (!(u == u)) { u = 0.f; o.behind = 1; }
    if (!(v == v)) { v = 0.f; o.behind = 1; }
    o.X = (int)lrintf(u * (float)K_SUB);
    o.Y = (int)lrintf(v * (float)K_SUB);
    o.iz = iz;
    vtx[i] = o;
  }
}

typedef struct {
  const float *verts, *normals, *colors;
  const int32_t* faces;
  int nv, nf;
  tex_t tex;
  int textured;
  const float* R;
  const float* color; /* override or NULL */
  vtx_t* vtx;
  int64_t base; /* scene index of its first triangle */
} inst_t;

int raster_ref_render_scene(int n_meshes, const float* verts, const float* normals, const float* colors,
                            const int64_t* vert_offsets, const int32_t* faces, const int64_t* face_offsets,
                            const float* uv, const uint8_t* tex, const int64_t* tex_offsets, const int32_t* tex_dims,
                            const int32_t* tex_modulate, int n_views, const int32_t* inst_offsets,
                            const int32_t* inst_label, const float* inst_TCO, const float* inst_color, const float* K,
                            int h, int w, unsigned flags, float* rgb, float* nrm, float* depth, int32_t* inst_id) {
  if (flags & 4u) return -3;
  const int npix = h * w;
  const int q8 = (flags & 1u) != 0, gl_axes = (flags & 2u) != 0;
  const float dep_a = -0.10101010f;
  const float dep_b = 1.01010101f;
  uint64_t* vis = (uint64_t*)malloc(sizeof(uint64_t) * (npix > 0 ? npix : 1));
  if (!vis) return -1;
  int status = 0;
  for (int view = 0; view < n_views && status == 0; ++view) {
    float* o_rgb = rgb ? rgb + (size_t)3 * npix * view : NULL;
    float* o_nrm = nrm ? nrm + (size_t)3 * npix * view : NULL;
    float* o_dep = depth ? depth + (size_t)npix * view : NULL;
    int32_t* o_id = inst_id ? inst_id + (size_t)npix * view : NULL;
    if (o_rgb) memset(o_rgb, 0, sizeof(float) * 3 * npix);
    if (o_nrm) memset(o_nrm, 0, sizeof(float) * 3 * npix);
    if (o_dep) memset(o_dep, 0, sizeof(float) * npix);
    if (o_id) for (int i = 0; i < npix; ++i) o_id[i] = -1;
    const float* Kv = K + 9 * view;
    int k_ok = 1;
    for (int i = 0; i < 9; ++i) k_ok = k_ok && isfinite(Kv[i]);
    const int lo = inst_offsets[view], n = inst_offsets[view + 1] - lo;
    if (!k_ok || n <= 0) continue;
    inst_t* in = (inst_t*)calloc((size_t)n, sizeof(inst_t));
    if (!in) { status = -1; break; }
    int64_t base = 0;
    for (int k = 0; k < n; ++k) {
      const int i = lo + k;
      const int lab = inst_label[i];
      int ok = lab >= 0 && lab < n_meshes;
      for (int e = 0; e < 16; ++e) ok = ok && isfinite(inst_TCO[16 * i + e]);
      in[k].base = base;
      if (!ok) continue;
      const int64_t vo = vert_offsets[lab], fo = face_offsets[lab];
      in[k].verts = verts + 3 * vo;
      in[k].normals = normals + 3 * vo;
      in[k].colors = colors + 3 * vo;
      in[k].faces = faces + 3 * fo;
      in[k].nv = (int)(vert_offsets[lab + 1] - vo);
      in[k].nf = (int)(face_offsets[lab + 1] - fo);
      in[k].R = inst_TCO + 16 * i;
      in[k].color = (inst_color && inst_color[3 * i] >= 0.f) ? inst_color + 3 * i : NULL;
      if (tex && uv && tex_dims[2 * lab] > 0 && tex_dims[2 * lab + 1] > 0) {
        in[k].textured = 1;
        in[k].tex.uv = uv + 2 * vo;
        in[k].tex.tex = tex + tex_offsets[lab];
        in[k].tex.th = tex_dims[2 * lab];
        in[k].tex.tw = tex_dims[2 * lab + 1];
        in[k].tex.modulate = tex_modulate ? tex_modulate[lab] : 0;
      }
      in[k].vtx = (vtx_t*)malloc(sizeof(vtx_t) * (in[k].nv > 0 ? in[k].nv : 1));
      if (!in[k].vtx) { status = -1; break; }
      snap_vertices(in[k].verts, in[k].nv, in[k].R, Kv, in[k].vtx);
      base += in[k].nf;
    }
    if (status == 0) {
      for (int i = 0; i < npix; ++i) vis[i] = ~(uint64_t)0;
      /* coverage: render_view's loop with the scene index in the key */
      for (int k = 0; k < n; ++k) {
        if (!in[k].vtx) continue;
        for (int tri = 0; tri < in[k].nf; ++tri) {
          const tri_t t = load_tri(in[k].vtx, in[k].faces, tri);
          if (!t.ok) continue;
          const int minx = imin(t.ax, imin(t.bx, t.cx)), maxx = imax(t.ax, imax(t.bx, t.cx));
          const int miny = imin(t.ay, imin(t.by, t.cy)), maxy = imax(t.ay, imax(t.by, t.cy));
          const int j0 = imax(0, -floor_div(-(minx - K_HALF), K_SUB));
          const int j1 = imin(w - 1, floor_div(maxx - K_HALF, K_SUB));
          const int i0 = imax(0, -floor_div(-(miny - K_HALF), K_SUB));
          const int i1 = imin(h - 1, floor_div(maxy - K_HALF, K_SUB));
          const uint32_t s = (uint32_t)(in[k].base + tri);
          for (int i = i0; i <= i1; ++i) {
            for (int j = j0; j <= j1; ++j) {
              float l0, l1, l2, iz;
              if (!tri_sample(&t, j * K_SUB + K_HALF, i * K_SUB + K_HALF, &l0, &l1, &l2, &iz)) continue;
              uint32_t zb;
              memcpy(&zb, &iz, 4);
              const uint64_t key = ((uint64_t)(~zb) << 32) | s;
              if (key < vis[i * w + j]) vis[i * w + j] = key;
            }
          }
        }
      }
      /* resolve: render_view's shading (ambient light) with the winning instance's data */
      for (int pix = 0; pix < npix; ++pix) {
        const uint64_t key = vis[pix];
        if (key == ~(uint64_t)0) continue;
        const int i = pix / w, j = pix - i * w;
        const int64_t s = (int64_t)(key & 0xffffffffu);
        int k = n - 1;
        while (in[k].base > s || !in[k].vtx) --k; /* the last instance with faces starting at or before s */
        const inst_t* I = &in[k];
        const int tri = (int)(s - I->base);
        const tri_t t = load_tri(I->vtx, I->faces, tri);
        float l0, l1, l2, iz;
        tri_sample(&t, j * K_SUB + K_HALF, i * K_SUB + K_HALF, &l0, &l1, &l2, &iz);
        const float z = 1.0f / iz;
        const float b0 = (l0 * t.iza) * z;
        const float b1 = (l1 * t.izb) * z;
        const float b2 = (l2 * t.izc) * z;
        const int ia = I->faces[3 * tri], ib = I->faces[3 * tri + 1], ic = I->faces[3 * tri + 2];
        float col[3], nn[3];
        for (int c = 0; c < 3; ++c) {
          col[c] = fmaf(b0, I->colors[3 * ia + c], fmaf(b1, I->colors[3 * ib + c], b2 * I->colors[3 * ic + c]));
          nn[c] = fmaf(b0, I->normals[3 * ia + c], fmaf(b1, I->normals[3 * ib + c], b2 * I->normals[3 * ic + c]));
        }
        if (I->textured) {
          const float* tuv = I->tex.uv;
          const float tu = fmaf(b0, tuv[2 * ia], fmaf(b1, tuv[2 * ib], b2 * tuv[2 * ic]));
          const float tv = fmaf(b0, tuv[2 * ia + 1], fmaf(b1, tuv[2 * ib + 1], b2 * tuv[2 * ic + 1]));
          float tc[3];
          texture_sample(&I->tex, tu, tv, tc);
          for (int c = 0; c < 3; ++c) col[c] = I->tex.modulate ? tc[c] * col[c] : tc[c];
        }
        if (I->color)
          for (int c = 0; c < 3; ++c) col[c] = I->color[c];
        if (o_rgb) {
          o_rgb[pix] = quant8(col[0], q8);
          o_rgb[npix + pix] = quant8(col[1], q8);
          o_rgb[2 * npix + pix] = quant8(col[2], q8);
        }
        if (o_nrm) {
          const float* R = I->R;
          float ex = fmaf(R[0], nn[0], fmaf(R[1], nn[1], R[2] * nn[2]));
          float ey = fmaf(R[4], nn[0], fmaf(R[5], nn[1], R[6] * nn[2]));
          float ez = fmaf(R[8], nn[0], fmaf(R[9], nn[1], R[10] * nn[2]));
          const float len = sqrtf(fmaf(ex, ex, fmaf(ey, ey, ez * ez)));
          if (len > 0.f) {
            const float inv = 1.0f / len;
            ex = ex * inv; ey = ey * inv; ez = ez * inv;
          }
          const float px_ = ex;
          const float py_ = gl_axes ? -ey : ez;
          const float pz_ = gl_axes ? -ez : -ey;
          o_nrm[pix] = quant8(normal_texture(px_), q8);
          o_nrm[npix + pix] = quant8(normal_texture(py_), q8);
          o_nrm[2 * npix + pix] = quant8(normal_texture(pz_), q8);
        }
        if (o_dep) {
          const float d = fmaf(dep_a, iz, dep_b);
          o_dep[pix] = (d > 0.999f) ? 0.f : z;
        }
        if (o_id) o_id[pix] = k;
      }
    }
    for (int k = 0; k < n; ++k) free(in[k].vtx);
    free(in);
  }
  free(vis);
  return status;
}
