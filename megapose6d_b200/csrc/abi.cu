// extern "C" surface of libmpx.so (declared in include/mpx.h). Thin argument validation + dispatch;
// every entry point enqueues work on the caller's stream and returns without synchronising.
#include <stdarg.h>
#include "mpx_common.cuh"
#include "../../include/mpx.h"

namespace mpx {
long long g_launches = 0;
int g_sm_limit = 0;
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace mpx

using namespace mpx;

#define MPX_NOT_NULL(p) MPX_REQUIRE((p) != nullptr, "%s: argument %s is NULL", __func__, #p)

extern "C" {

int mpx_abi_version(void) { return MPX_ABI_VERSION; }
int mpx_act_dtype(void) { return kActIsFp16 ? 0 : 1; }
const char* mpx_last_error(void) { return g_err; }

long long mpx_launch_count(void) { return g_launches; }
int mpx_set_sm_limit(int n_sms) {
  MPX_REQUIRE(n_sms == 0 || (n_sms >= 16 && n_sms % 2 == 0), "mpx_set_sm_limit: %d is not 0 or an even number >= 16", n_sms);
  g_sm_limit = n_sms;
  return MPX_OK;
}
int mpx_sm_count(void) { return sm_count(); }
int mpx_profile_enable(int on) {
  conv_profile_enable(on);
  return MPX_OK;
}
int mpx_profile_summary(double* conv_ms, double* conv_flops, long long* conv_launches) {
  MPX_NOT_NULL(conv_ms);
  MPX_NOT_NULL(conv_flops);
  MPX_NOT_NULL(conv_launches);
  return conv_profile_summary(conv_ms, conv_flops, conv_launches);
}

// ---- mesh database ----
struct mpx_meshdb {
  MeshDb* db;
};

int mpx_meshdb_create(int n_meshes, const float* h_verts, const float* h_normals, const float* h_colors,
                      const int64_t* h_vert_offsets, const int32_t* h_faces, const int64_t* h_face_offsets,
                      mpx_meshdb** out) {
  MPX_NOT_NULL(h_verts);
  MPX_NOT_NULL(h_normals);
  MPX_NOT_NULL(h_colors);
  MPX_NOT_NULL(h_vert_offsets);
  MPX_NOT_NULL(h_faces);
  MPX_NOT_NULL(h_face_offsets);
  MPX_NOT_NULL(out);
  MeshDb* db = nullptr;
  int rc = meshdb_create(n_meshes, h_verts, h_normals, h_colors, h_vert_offsets, h_faces, h_face_offsets, &db);
  if (rc != MPX_OK) return rc;
  *out = new mpx_meshdb{db};
  return MPX_OK;
}

int mpx_meshdb_destroy(mpx_meshdb* db) {
  if (db) {
    meshdb_destroy(db->db);
    delete db;
  }
  return MPX_OK;
}

int mpx_meshdb_set_textures(mpx_meshdb* db, const float* uv, const uint8_t* tex, const int64_t* tex_offsets,
                            const int32_t* tex_dims, const int32_t* tex_modulate) {
  MPX_NOT_NULL(db);
  return meshdb_set_textures(db->db, uv, tex, tex_offsets, tex_dims, tex_modulate);
}


// ---- rasteriser ----
size_t mpx_raster_workspace_bytes(int h, int w) { return raster_workspace_bytes(h, w); }

int mpx_raster_set_mode(int mode) {
  raster_set_scatter(mode & 1);
  raster_set_tiled(mode & 4);
  return raster_set_red_only(mode & 2);
}

int mpx_raster_render(const mpx_meshdb* db, const int32_t* d_label_idx, const float* d_TCO, const float* d_K,
                      int n_views, int h, int w, uint32_t flags, float* d_rgb, float* d_normals, float* d_depth,
                      void* d_workspace, size_t workspace_bytes, void* stream) {
  MPX_NOT_NULL(db);
  MPX_REQUIRE(n_views >= 0, "mpx_raster_render: n_views < 0");
  if (n_views > 0) {
    MPX_NOT_NULL(d_label_idx);
    MPX_NOT_NULL(d_TCO);
    MPX_NOT_NULL(d_K);
    MPX_NOT_NULL(d_workspace);
  }
  RasterOut out;
  memset(&out, 0, sizeof(out));
  out.rgb = d_rgb;
  out.normals = d_normals;
  out.depth = d_depth;
  return raster_launch(db->db, d_label_idx, d_TCO, d_K, n_views, h, w, flags, out, d_workspace, workspace_bytes,
                       static_cast<cudaStream_t>(stream));
}

int mpx_raster_render_fused(const mpx_meshdb* db, const int32_t* d_label_idx, const float* d_TCO,
                            const float* d_K, int n_views, int views_per_sample, int h, int w, uint32_t flags,
                            void* d_x, int c_pad, int ch_offset, int ch_per_view, const float* d_depth_norm_z,
                            void* d_workspace, size_t workspace_bytes, void* stream) {
  MPX_NOT_NULL(db);
  MPX_NOT_NULL(d_x);
  MPX_REQUIRE(n_views >= 0, "mpx_raster_render_fused: n_views < 0");
  MPX_REQUIRE(views_per_sample >= 1 && n_views % views_per_sample == 0,
              "mpx_raster_render_fused: n_views=%d not a multiple of views_per_sample=%d", n_views,
              views_per_sample);
  if (n_views > 0) {
    MPX_NOT_NULL(d_label_idx);
    MPX_NOT_NULL(d_TCO);
    MPX_NOT_NULL(d_K);
    MPX_NOT_NULL(d_workspace);
  }
  RasterOut out;
  memset(&out, 0, sizeof(out));
  out.x = reinterpret_cast<act_t*>(d_x);
  out.c_pad = c_pad;
  out.ch_offset = ch_offset;
  out.ch_per_view = ch_per_view;
  out.views_per_sample = views_per_sample;
  out.depth_norm_z = d_depth_norm_z;
  out.depth_norm_kind = static_cast<int>((flags >> MPX_RASTER_DEPTH_NORM_SHIFT) & 3u);
  return raster_launch(db->db, d_label_idx, d_TCO, d_K, n_views, h, w, flags, out, d_workspace, workspace_bytes,
                       static_cast<cudaStream_t>(stream));
}

int mpx_render_crop_fused(const mpx_meshdb* db, const int32_t* d_label_idx, const float* d_TCO, const float* d_K,
                          int n, int h, int w, uint32_t flags, const float* d_img_nhwc4, int b, int im_h, int im_w,
                          const int32_t* d_im_idx, const float* d_boxes_crop, int c_in, void* d_x, int c_pad,
                          int ch_per_view, const float* d_depth_norm_z, void* d_workspace, size_t workspace_bytes,
                          void* stream) {
  MPX_NOT_NULL(db);
  MPX_NOT_NULL(d_x);
  MPX_REQUIRE(n >= 0, "mpx_render_crop_fused: n < 0");
  if (n > 0) {
    MPX_NOT_NULL(d_label_idx);
    MPX_NOT_NULL(d_TCO);
    MPX_NOT_NULL(d_K);
    MPX_NOT_NULL(d_img_nhwc4);
    MPX_NOT_NULL(d_boxes_crop);
    MPX_NOT_NULL(d_workspace);
  }
  MPX_REQUIRE(b > 0 && im_h > 0 && im_w > 0, "mpx_render_crop_fused: empty observation");
  RasterOut out;
  memset(&out, 0, sizeof(out));
  out.x = reinterpret_cast<act_t*>(d_x);
  out.c_pad = c_pad;
  out.ch_offset = c_in;
  out.ch_per_view = ch_per_view;
  out.views_per_sample = 1;
  out.depth_norm_z = d_depth_norm_z;
  out.depth_norm_kind = static_cast<int>((flags >> MPX_RASTER_DEPTH_NORM_SHIFT) & 3u);
  out.crop_images = reinterpret_cast<const float4*>(d_img_nhwc4);
  out.crop_b = b;
  out.crop_h = im_h;
  out.crop_w = im_w;
  out.crop_c = c_in;
  out.crop_im_idx = d_im_idx;
  out.crop_boxes = d_boxes_crop;
  return raster_launch(db->db, d_label_idx, d_TCO, d_K, n, h, w, flags, out, d_workspace, workspace_bytes,
                       static_cast<cudaStream_t>(stream));
}

// ---- geometry ----
int mpx_pose_init_autodepth(const float* d_points, int n_pts, const int32_t* d_label_idx, const float* d_bboxes,
                            const float* d_K, const float* d_R, int n, float* d_TCO, void* stream) {
  MPX_REQUIRE(n >= 0, "mpx_pose_init_autodepth: n < 0");
  if (n > 0) {
    MPX_NOT_NULL(d_points);
    MPX_NOT_NULL(d_label_idx);
    MPX_NOT_NULL(d_bboxes);
    MPX_NOT_NULL(d_K);
    MPX_NOT_NULL(d_R);
    MPX_NOT_NULL(d_TCO);
  }
  return pose_init_autodepth(d_points, n_pts, d_label_idx, d_bboxes, d_K, d_R, n, d_TCO,
                             static_cast<cudaStream_t>(stream));
}

int mpx_normalize_T(const float* d_T_in, int n, float* d_T_out, void* stream) {
  MPX_REQUIRE(n >= 0, "mpx_normalize_T: n < 0");
  if (n > 0) {
    MPX_NOT_NULL(d_T_in);
    MPX_NOT_NULL(d_T_out);
  }
  return normalize_T(d_T_in, n, d_T_out, static_cast<cudaStream_t>(stream));
}

int mpx_crop_geometry(const float* d_points, int n_pts, const int32_t* d_label_idx, const float* d_TCO,
                      const float* d_K, const float* d_tCR, int n, float lamb, int im_h, int im_w, int out_h,
                      int out_w, float* d_boxes_rend, float* d_boxes_crop, float* d_K_crop, void* stream) {
  MPX_REQUIRE(n >= 0, "mpx_crop_geometry: n < 0");
  if (n > 0) {
    MPX_NOT_NULL(d_points);
    MPX_NOT_NULL(d_label_idx);
    MPX_NOT_NULL(d_TCO);
    MPX_NOT_NULL(d_K);
    MPX_NOT_NULL(d_tCR);
    MPX_NOT_NULL(d_boxes_rend);
    MPX_NOT_NULL(d_boxes_crop);
    MPX_NOT_NULL(d_K_crop);
  }
  MPX_REQUIRE(im_h > 0 && im_w > 0 && out_h > 0 && out_w > 0, "mpx_crop_geometry: bad sizes");
  return crop_geometry(d_points, n_pts, d_label_idx, d_TCO, d_K, d_tCR, n, lamb, im_h, im_w, out_h, out_w,
                       d_boxes_rend, d_boxes_crop, d_K_crop, static_cast<cudaStream_t>(stream));
}

int mpx_multiview_cameras(const float* d_TCO, const float* d_tCR, int n, const float* h_offsets, int n_extra,
                          float* d_TCV_O, void* stream) {
  MPX_REQUIRE(n >= 0, "mpx_multiview_cameras: n < 0");
  if (n > 0) {
    MPX_NOT_NULL(d_TCO);
    MPX_NOT_NULL(d_tCR);
    MPX_NOT_NULL(d_TCV_O);
  }
  if (n_extra > 0) MPX_NOT_NULL(h_offsets);
  return multiview_cameras(d_TCO, d_tCR, n, h_offsets, n_extra, d_TCV_O, static_cast<cudaStream_t>(stream));
}

int mpx_pose_update(const float* d_TCO, const float* d_K_crop, const float* d_pose9, const float* d_tCR, int n,
                    float* d_TCO_out, void* stream) {
  MPX_REQUIRE(n >= 0, "mpx_pose_update: n < 0");
  if (n > 0) {
    MPX_NOT_NULL(d_TCO);
    MPX_NOT_NULL(d_K_crop);
    MPX_NOT_NULL(d_pose9);
    MPX_NOT_NULL(d_tCR);
    MPX_NOT_NULL(d_TCO_out);
  }
  return pose_update(d_TCO, d_K_crop, d_pose9, d_tCR, n, d_TCO_out, static_cast<cudaStream_t>(stream));
}

int mpx_topk_per_group(const float* d_logits, int n_groups, int m, int k, int32_t* d_idx, void* stream) {
  MPX_REQUIRE(n_groups >= 0 && m >= 0 && k >= 0, "mpx_topk_per_group: negative size");
  if (n_groups > 0 && k > 0) {
    MPX_NOT_NULL(d_logits);
    MPX_NOT_NULL(d_idx);
  }
  return topk_per_group(d_logits, n_groups, m, k, d_idx, static_cast<cudaStream_t>(stream));
}

// ---- crop ----
int mpx_image_to_nhwc4(const float* d_images_nchw, int b, int c, int h, int w, float* d_out_nhwc4, void* stream) {
  MPX_NOT_NULL(d_images_nchw);
  MPX_NOT_NULL(d_out_nhwc4);
  return image_to_nhwc4(d_images_nchw, b, c, h, w, d_out_nhwc4, static_cast<cudaStream_t>(stream));
}

int mpx_roi_align(const float* d_img_nhwc4, int b, int h, int w, const int32_t* d_im_idx, const float* d_boxes,
                  int n, int c, int out_h, int out_w, float* d_out, void* stream) {
  MPX_REQUIRE(n >= 0, "mpx_roi_align: n < 0");
  if (n > 0) {
    MPX_NOT_NULL(d_img_nhwc4);
    MPX_NOT_NULL(d_boxes);
    MPX_NOT_NULL(d_out);
  }
  CropOut out;
  memset(&out, 0, sizeof(out));
  out.nchw = d_out;
  return roi_align_launch(d_img_nhwc4, b, h, w, d_im_idx, d_boxes, n, c, out_h, out_w, out,
                          static_cast<cudaStream_t>(stream));
}

int mpx_roi_align_fused(const float* d_img_nhwc4, int b, int h, int w, const int32_t* d_im_idx,
                        const float* d_boxes, int n, int c, int out_h, int out_w, void* d_x, int c_pad,
                        const float* d_depth_norm_z, int depth_norm_kind, void* stream) {
  MPX_REQUIRE(n >= 0, "mpx_roi_align_fused: n < 0");
  MPX_REQUIRE(depth_norm_kind >= 0 && depth_norm_kind <= 3, "mpx_roi_align_fused: depth_norm_kind=%d", depth_norm_kind);
  if (n > 0) {
    MPX_NOT_NULL(d_img_nhwc4);
    MPX_NOT_NULL(d_boxes);
    MPX_NOT_NULL(d_x);
  }
  MPX_REQUIRE(c <= c_pad, "mpx_roi_align_fused: c=%d > c_pad=%d", c, c_pad);
  CropOut out;
  memset(&out, 0, sizeof(out));
  out.x = reinterpret_cast<act_t*>(d_x);
  out.c_pad = c_pad;
  out.depth_norm_z = d_depth_norm_z;
  out.depth_norm_kind = depth_norm_kind;
  return roi_align_launch(d_img_nhwc4, b, h, w, d_im_idx, d_boxes, n, c, out_h, out_w, out,
                          static_cast<cudaStream_t>(stream));
}

// ---- network ----
size_t mpx_net_input_bytes(int n, int h, int w, int c_pad) {
  return static_cast<size_t>(n) * (h / 2) * (w / 2) * 4 * c_pad * 2;
}

int mpx_conv2d(const void* d_x, int n, int h, int w, int c_in, const void* d_w, const float* d_bias,
                    int c_out, int r, int s, int stride, int pad_lo_h, int pad_lo_w, int pad_hi_h, int pad_hi_w,
                    int relu, const void* d_residual, void* d_out, int block_n, int max_ctas, void* stream) {
  MPX_NOT_NULL(d_x);
  MPX_NOT_NULL(d_w);
  MPX_NOT_NULL(d_bias);
  MPX_NOT_NULL(d_out);
  MPX_REQUIRE(n > 0 && h > 0 && w > 0, "mpx_conv2d: empty input");
  MPX_REQUIRE((reinterpret_cast<uintptr_t>(d_x) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_w) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(d_out) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(d_bias) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(d_residual) & 15) == 0,
              "mpx_conv2d: pointers must be 16-byte aligned");
  ConvDesc d{n, h, w, c_in, c_out, r, s, stride, pad_lo_h, pad_lo_w, pad_hi_h, pad_hi_w, relu & 1, (relu >> 1) & 1, (relu >> 2) & 1};
  return conv_forward(d, d_x, d_w, d_bias, d_residual, d_out, block_n, max_ctas,
                      static_cast<cudaStream_t>(stream));
}

int mpx_conv2d_splitk(const void* d_x, int n, int h, int w, int c_in, const void* d_w, const float* d_bias,
                           int c_out, int r, int s, int stride, int pad_lo_h, int pad_lo_w, int pad_hi_h,
                           int pad_hi_w, int relu, const void* d_residual, void* d_out, int block_n, int splits,
                           void* stream) {
  MPX_NOT_NULL(d_x);
  MPX_NOT_NULL(d_w);
  MPX_NOT_NULL(d_bias);
  MPX_NOT_NULL(d_out);
  MPX_REQUIRE(n > 0 && h > 0 && w > 0, "mpx_conv2d_splitk: empty input");
  MPX_REQUIRE(splits == 0 || splits == 1 || splits == 2 || splits == 4 || splits == 8,
              "mpx_conv2d_splitk: splits=%d must be 0 (heuristic), 1, 2, 4 or 8", splits);
  MPX_REQUIRE(block_n == 64 || block_n == 128 || block_n == 256, "mpx_conv2d_splitk: block_n must be 64|128|256");
  MPX_REQUIRE((reinterpret_cast<uintptr_t>(d_x) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_w) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(d_out) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_bias) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(d_residual) & 15) == 0,
              "mpx_conv2d_splitk: pointers must be 16-byte aligned");
  ConvDesc d{n, h, w, c_in, c_out, r, s, stride, pad_lo_h, pad_lo_w, pad_hi_h, pad_hi_w, relu & 1, (relu >> 1) & 1};
  return conv_forward(d, d_x, d_w, d_bias, d_residual, d_out, block_n, 0, static_cast<cudaStream_t>(stream),
                      splits == 0 ? -1 : splits);
}

int mpx_maxpool3x3s2(const void* d_x, int n, int h, int w, int c, void* d_out, void* stream) {
  MPX_NOT_NULL(d_x);
  MPX_NOT_NULL(d_out);
  return maxpool3x3s2(d_x, n, h, w, c, d_out, static_cast<cudaStream_t>(stream));
}

int mpx_avgpool_linear(const void* d_x, int n, int hw, int c, const float* d_w, const float* d_b, int out_dim,
                       float* d_out, void* stream) {
  MPX_NOT_NULL(d_x);
  MPX_NOT_NULL(d_w);
  MPX_NOT_NULL(d_b);
  MPX_NOT_NULL(d_out);
  return avgpool_linear(d_x, n, hw, c, d_w, d_b, out_dim, d_out, static_cast<cudaStream_t>(stream));
}

struct mpx_net {
  Net* net;
};

int mpx_net_create(int c_pad, int out_dim, const void* const* h_conv_w, const float* const* h_conv_b,
                   int n_convs, const float* d_head_w, const float* d_head_b, mpx_net** out) {
  MPX_NOT_NULL(h_conv_w);
  MPX_NOT_NULL(h_conv_b);
  MPX_NOT_NULL(d_head_w);
  MPX_NOT_NULL(d_head_b);
  MPX_NOT_NULL(out);
  for (int i = 0; i < n_convs; ++i) {
    MPX_REQUIRE(h_conv_w[i] != nullptr && h_conv_b[i] != nullptr, "mpx_net_create: conv %d has a NULL tensor", i);
  }
  Net* net = nullptr;
  int rc = net_create(c_pad, out_dim, h_conv_w, h_conv_b, n_convs, d_head_w, d_head_b, &net);
  if (rc != MPX_OK) return rc;
  *out = new mpx_net{net};
  return MPX_OK;
}

int mpx_net_create_preact(int c_pad, int out_dim, const int32_t* h_layer_blocks, const void* const* h_conv_w,
                          const float* const* h_conv_b, int n_convs, const float* const* h_block_affine, int n_blocks,
                          const float* d_head_w, const float* d_head_b, mpx_net** out) {
  MPX_NOT_NULL(h_layer_blocks);
  MPX_NOT_NULL(h_conv_w);
  MPX_NOT_NULL(h_conv_b);
  MPX_NOT_NULL(h_block_affine);
  MPX_NOT_NULL(d_head_w);
  MPX_NOT_NULL(d_head_b);
  MPX_NOT_NULL(out);
  for (int i = 0; i < n_convs; ++i)
    MPX_REQUIRE(h_conv_w[i] != nullptr && h_conv_b[i] != nullptr, "mpx_net_create_preact: conv %d has a NULL tensor", i);
  for (int i = 0; i < n_blocks; ++i)
    MPX_REQUIRE(h_block_affine[i] != nullptr, "mpx_net_create_preact: block %d has no affine parameters", i);
  int lb[4] = {h_layer_blocks[0], h_layer_blocks[1], h_layer_blocks[2], h_layer_blocks[3]};
  Net* net = nullptr;
  int rc = net_create_preact(c_pad, out_dim, lb, h_conv_w, h_conv_b, n_convs, h_block_affine, n_blocks, d_head_w, d_head_b, &net);
  if (rc != MPX_OK) return rc;
  *out = new mpx_net{net};
  return MPX_OK;
}

int mpx_conv_set_mode(int mode) {
  conv_set_mode(mode);
  return MPX_OK;
}

int mpx_net_set_graphs(int on) {
  net_set_graphs(on);
  return MPX_OK;
}

int mpx_net_destroy(mpx_net* net) {
  if (net) {
    net_destroy(net->net);
    delete net;
  }
  return MPX_OK;
}

size_t mpx_net_workspace_bytes(const mpx_net* net, int n, int h, int w) {
  return net_workspace_bytes(net ? net->net : nullptr, n, h, w);
}

int mpx_net_forward(const mpx_net* net, const void* d_x, int n, int h, int w, float* d_out, void* d_workspace,
                    size_t workspace_bytes, void* stream) {
  MPX_NOT_NULL(net);
  MPX_REQUIRE(n >= 0, "mpx_net_forward: n < 0");
  if (n > 0) {
    MPX_NOT_NULL(d_x);
    MPX_NOT_NULL(d_out);
    MPX_NOT_NULL(d_workspace);
  }
  return net_forward(net->net, d_x, n, h, w, d_out, d_workspace, workspace_bytes,
                     static_cast<cudaStream_t>(stream));
}

}  // extern "C"
