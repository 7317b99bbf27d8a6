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

int mpx_raster_render_scene(const mpx_meshdb* db, int n_views, int n_inst, const int32_t* d_inst_offsets,
                            const int32_t* d_inst_label, const float* d_inst_TCO, const float* d_inst_color,
                            const float* d_K, int h, int w, uint32_t flags, float* d_rgb, float* d_normals,
                            float* d_depth, int32_t* d_inst_id, void* d_workspace, size_t workspace_bytes, void* stream) {
  MPX_NOT_NULL(db);
  MPX_REQUIRE(n_views >= 0 && n_inst >= 0, "mpx_raster_render_scene: n_views=%d n_inst=%d", n_views, n_inst);
  if (n_views > 0) {
    MPX_NOT_NULL(d_inst_offsets);
    MPX_NOT_NULL(d_K);
    MPX_NOT_NULL(d_workspace);
  }
  if (n_inst > 0) {
    MPX_NOT_NULL(d_inst_label);
    MPX_NOT_NULL(d_inst_TCO);
  }
  return raster_scene_launch(db->db, n_views, n_inst, d_inst_offsets, d_inst_label, d_inst_TCO, d_inst_color, d_K, h, w,
                             flags, d_rgb, d_normals, d_depth, d_inst_id, d_workspace, workspace_bytes,
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

// ---- BOP pose errors ----
int mpx_bop_vsd(int n_pairs, int h, int w, const uint16_t* d_depth_test, int n_img, const float* d_depth_scale,
                const double* d_K, const float* d_depth_est, int n_est, const float* d_depth_gt, int n_gt,
                const int32_t* d_est_idx, const int32_t* d_gt_idx, const int32_t* d_img_idx, const double* d_diameter,
                const double* h_taus, int n_taus, float delta, int64_t* d_counts, double* d_err, void* stream) {
  MPX_REQUIRE(n_pairs >= 0, "mpx_bop_vsd: n_pairs=%d < 0", n_pairs);
  MPX_REQUIRE(n_taus >= 1 && n_taus <= MPX_BOP_MAX_TAUS, "mpx_bop_vsd: n_taus=%d not in 1..%d", n_taus, MPX_BOP_MAX_TAUS);
  MPX_NOT_NULL(h_taus);
  if (n_pairs == 0) return MPX_OK;
  MPX_REQUIRE(h > 0 && w > 0 && static_cast<long long>(h) * w < (1ll << 31), "mpx_bop_vsd: bad image size %dx%d", h, w);
  MPX_REQUIRE(n_img > 0 && n_est > 0 && n_gt > 0, "mpx_bop_vsd: n_img=%d n_est=%d n_gt=%d", n_img, n_est, n_gt);
  MPX_NOT_NULL(d_depth_test);
  MPX_NOT_NULL(d_depth_scale);
  MPX_NOT_NULL(d_K);
  MPX_NOT_NULL(d_depth_est);
  MPX_NOT_NULL(d_depth_gt);
  MPX_NOT_NULL(d_est_idx);
  MPX_NOT_NULL(d_gt_idx);
  MPX_NOT_NULL(d_img_idx);
  MPX_NOT_NULL(d_diameter);
  MPX_NOT_NULL(d_counts);
  MPX_NOT_NULL(d_err);
  return bop_vsd(n_pairs, h, w, d_depth_test, n_img, d_depth_scale, d_K, d_depth_est, n_est, d_depth_gt, n_gt, d_est_idx,
                 d_gt_idx, d_img_idx, d_diameter, h_taus, n_taus, delta, d_counts, d_err, static_cast<cudaStream_t>(stream));
}

int mpx_bop_point_errors(int kind, int n_pairs, int n_models, const double* d_pts, const int64_t* d_pt_offsets,
                         long long n_pts_total, const double* d_syms, const int64_t* d_sym_offsets, long long n_syms_total,
                         const int32_t* d_model_idx, const double* d_pose_est, const double* d_pose_gt, const double* d_K,
                         double* d_err, int32_t* d_sym_argmin, void* stream) {
  MPX_REQUIRE(kind >= MPX_BOP_MSSD && kind <= MPX_BOP_ADI, "mpx_bop_point_errors: unknown error kind %d", kind);
  MPX_REQUIRE(n_pairs >= 0, "mpx_bop_point_errors: n_pairs=%d < 0", n_pairs);
  if (n_pairs == 0) return MPX_OK;
  MPX_REQUIRE(n_models >= 1 && n_pts_total >= 0 && n_syms_total >= 0, "mpx_bop_point_errors: n_models=%d", n_models);
  MPX_NOT_NULL(d_pts);
  MPX_NOT_NULL(d_pt_offsets);
  MPX_NOT_NULL(d_model_idx);
  MPX_NOT_NULL(d_pose_est);
  MPX_NOT_NULL(d_pose_gt);
  MPX_NOT_NULL(d_err);
  if (kind == MPX_BOP_MSSD || kind == MPX_BOP_MSPD) {
    MPX_NOT_NULL(d_syms);
    MPX_NOT_NULL(d_sym_offsets);
  }
  if (kind == MPX_BOP_MSPD) MPX_NOT_NULL(d_K);
  return bop_point_errors(kind, n_pairs, n_models, d_pts, d_pt_offsets, n_pts_total,
                          (kind == MPX_BOP_MSSD || kind == MPX_BOP_MSPD) ? d_syms : nullptr, d_sym_offsets, n_syms_total,
                          d_model_idx, d_pose_est, d_pose_gt, d_K, d_err, d_sym_argmin, static_cast<cudaStream_t>(stream));
}

// ---- depth refinement (TEASER++) ----
static bool is_device_ptr(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}
#define MPX_DEVICE(p)                                                                                                 \
  do {                                                                                                                \
    MPX_NOT_NULL(p);                                                                                                  \
    MPX_REQUIRE(is_device_ptr(p), "%s: argument %s is not device memory", __func__, #p);                              \
  } while (0)
#define MPX_DEVICE_OR_NULL(p)                                                                                         \
  do {                                                                                                                \
    if (p) MPX_DEVICE(p);                                                                                             \
  } while (0)

int mpx_teaser_points(int n_pred, int h, int w, const float* d_depth_rendered, const float* d_depth_measured, int n_view,
                      const int32_t* d_view_idx, const float* d_K, int mask_type, float thresh, float* d_src, float* d_tgt,
                      int32_t* d_count, float* d_raw_src, float* d_raw_tgt, void* stream) {
  MPX_REQUIRE(n_pred >= 0, "mpx_teaser_points: n_pred=%d < 0", n_pred);
  MPX_REQUIRE(mask_type == MPX_TEASER_MASK_SIMPLE || mask_type == MPX_TEASER_MASK_THRESHOLD,
              "mpx_teaser_points: unknown mask type %d", mask_type);
  if (n_pred == 0) return MPX_OK;
  MPX_REQUIRE(h > 0 && w > 0 && static_cast<long long>(h) * w < (1ll << 31), "mpx_teaser_points: bad image size %dx%d", h, w);
  MPX_REQUIRE(n_view > 0, "mpx_teaser_points: n_view=%d", n_view);
  MPX_REQUIRE((d_raw_src == nullptr) == (d_raw_tgt == nullptr), "mpx_teaser_points: give both raw clouds or neither");
  MPX_DEVICE(d_depth_rendered);
  MPX_DEVICE(d_depth_measured);
  MPX_DEVICE(d_view_idx);
  MPX_DEVICE(d_K);
  MPX_DEVICE(d_src);
  MPX_DEVICE(d_tgt);
  MPX_DEVICE(d_count);
  MPX_DEVICE_OR_NULL(d_raw_src);
  MPX_DEVICE_OR_NULL(d_raw_tgt);
  return teaser_points(n_pred, h, w, d_depth_rendered, d_depth_measured, d_view_idx, d_K, mask_type, thresh, d_src, d_tgt,
                       d_count, d_raw_src, d_raw_tgt, static_cast<cudaStream_t>(stream));
}

size_t mpx_teaser_fps_workspace_bytes(int n_pred, int cap) {
  return n_pred > 0 && cap > 0 ? teaser_fps_workspace_bytes(n_pred, cap) : 0;
}

int mpx_teaser_fps(int n_pred, int cap, const float* d_src, const float* d_tgt, const int32_t* d_count, int k,
                   int32_t* d_idx, float* d_samp_src, float* d_samp_tgt, void* d_workspace, size_t workspace_bytes,
                   void* stream) {
  MPX_REQUIRE(n_pred >= 0, "mpx_teaser_fps: n_pred=%d < 0", n_pred);
  MPX_REQUIRE(k >= 1 && k <= MPX_TEASER_MAX_POINTS, "mpx_teaser_fps: k=%d not in 1..%d", k, MPX_TEASER_MAX_POINTS);
  if (n_pred == 0) return MPX_OK;
  MPX_REQUIRE(cap > 0, "mpx_teaser_fps: cap=%d", cap);
  MPX_REQUIRE(workspace_bytes >= teaser_fps_workspace_bytes(n_pred, cap), "mpx_teaser_fps: workspace of %zu bytes < %zu",
              workspace_bytes, teaser_fps_workspace_bytes(n_pred, cap));
  MPX_DEVICE(d_src);
  MPX_DEVICE(d_tgt);
  MPX_DEVICE(d_count);
  MPX_DEVICE(d_idx);
  MPX_DEVICE(d_samp_src);
  MPX_DEVICE(d_samp_tgt);
  MPX_DEVICE(d_workspace);
  return teaser_fps(n_pred, cap, d_src, d_tgt, d_count, k, d_idx, d_samp_src, d_samp_tgt, d_workspace,
                    static_cast<cudaStream_t>(stream));
}

int mpx_teaser_graph(int n_pred, int k, const float* d_samp_src, const float* d_samp_tgt, const int32_t* d_m, double bound,
                     uint64_t* d_adj, void* stream) {
  MPX_REQUIRE(n_pred >= 0, "mpx_teaser_graph: n_pred=%d < 0", n_pred);
  MPX_REQUIRE(k >= 1 && k <= MPX_TEASER_MAX_POINTS, "mpx_teaser_graph: k=%d not in 1..%d", k, MPX_TEASER_MAX_POINTS);
  if (n_pred == 0) return MPX_OK;
  MPX_DEVICE(d_samp_src);
  MPX_DEVICE(d_samp_tgt);
  MPX_DEVICE(d_m);
  MPX_DEVICE(d_adj);
  return teaser_graph(n_pred, k, d_samp_src, d_samp_tgt, d_m, bound, reinterpret_cast<unsigned long long*>(d_adj),
                      static_cast<cudaStream_t>(stream));
}

size_t mpx_teaser_clique_workspace_bytes(int n_pred, int k) {
  return n_pred > 0 && k > 0 ? teaser_clique_workspace_bytes(n_pred, k) : 0;
}

int mpx_teaser_max_clique(int n_pred, int k, const uint64_t* d_adj, const int32_t* d_m, long long node_budget,
                          int32_t* d_clique, int32_t* d_clique_size, int32_t* d_status, int64_t* d_nodes,
                          void* d_workspace, size_t workspace_bytes, void* stream) {
  MPX_REQUIRE(n_pred >= 0, "mpx_teaser_max_clique: n_pred=%d < 0", n_pred);
  MPX_REQUIRE(k >= 1 && k <= MPX_TEASER_MAX_POINTS, "mpx_teaser_max_clique: k=%d not in 1..%d", k, MPX_TEASER_MAX_POINTS);
  if (n_pred == 0) return MPX_OK;
  MPX_REQUIRE(workspace_bytes >= teaser_clique_workspace_bytes(n_pred, k),
              "mpx_teaser_max_clique: workspace of %zu bytes < %zu", workspace_bytes,
              teaser_clique_workspace_bytes(n_pred, k));
  MPX_DEVICE(d_adj);
  MPX_DEVICE(d_m);
  MPX_DEVICE(d_clique);
  MPX_DEVICE(d_clique_size);
  MPX_DEVICE(d_status);
  MPX_DEVICE_OR_NULL(d_nodes);
  MPX_DEVICE(d_workspace);
  return teaser_max_clique(n_pred, k, reinterpret_cast<const unsigned long long*>(d_adj), d_m,
                           node_budget > 0 ? node_budget : MPX_TEASER_CLIQUE_NODE_BUDGET, d_clique, d_clique_size,
                           d_status, reinterpret_cast<long long*>(d_nodes), d_workspace, static_cast<cudaStream_t>(stream));
}

int mpx_teaser_solve(int n_pred, int k, const float* d_samp_src, const float* d_samp_tgt, const int32_t* d_m,
                     const int32_t* d_clique, const int32_t* d_clique_size, double noise_bound, double gnc_factor,
                     int max_iterations, double cost_threshold, int min_num_inliers, float* d_poses, float* d_poses_input,
                     double* d_T, int32_t* d_num_inliers, int32_t* d_flags, void* stream) {
  MPX_REQUIRE(n_pred >= 0, "mpx_teaser_solve: n_pred=%d < 0", n_pred);
  MPX_REQUIRE(k >= 1 && k <= MPX_TEASER_MAX_POINTS, "mpx_teaser_solve: k=%d not in 1..%d", k, MPX_TEASER_MAX_POINTS);
  MPX_REQUIRE(noise_bound > 0 && gnc_factor > 1 && max_iterations >= 1,
              "mpx_teaser_solve: noise_bound=%g gnc_factor=%g max_iterations=%d", noise_bound, gnc_factor, max_iterations);
  if (n_pred == 0) return MPX_OK;
  MPX_DEVICE(d_samp_src);
  MPX_DEVICE(d_samp_tgt);
  MPX_DEVICE(d_m);
  MPX_DEVICE(d_clique);
  MPX_DEVICE(d_clique_size);
  MPX_DEVICE(d_poses);
  MPX_DEVICE(d_poses_input);
  MPX_DEVICE(d_T);
  MPX_DEVICE(d_num_inliers);
  MPX_DEVICE(d_flags);
  return teaser_solve(n_pred, k, d_samp_src, d_samp_tgt, d_m, d_clique, d_clique_size, noise_bound, gnc_factor,
                      max_iterations, cost_threshold, min_num_inliers, d_poses, d_poses_input, d_T, d_num_inliers, d_flags,
                      static_cast<cudaStream_t>(stream));
}

// ---- BOP ground-truth annotation (a BOP 2019 group entry point, placed here for the device-pointer checks) ----
int mpx_bop_gt_info(int n_gt, int h, int w, const uint16_t* d_depth_test, int n_img, const float* d_depth_scale,
                    const double* d_K, const float* d_depth_gt_large, const int32_t* d_img_idx, float delta,
                    int64_t* d_counts, int32_t* d_bbox, uint8_t* d_mask, uint8_t* d_mask_visib, void* stream) {
  MPX_REQUIRE(n_gt >= 0, "mpx_bop_gt_info: n_gt=%d < 0", n_gt);
  if (n_gt == 0) return MPX_OK;
  MPX_REQUIRE(h > 0 && w > 0 && 9ll * h * w < (1ll << 31), "mpx_bop_gt_info: bad image size %dx%d", h, w);
  MPX_REQUIRE(n_img > 0, "mpx_bop_gt_info: n_img=%d", n_img);
  MPX_DEVICE(d_depth_test);
  MPX_DEVICE(d_depth_scale);
  MPX_DEVICE(d_K);
  MPX_DEVICE(d_depth_gt_large);
  MPX_DEVICE(d_img_idx);
  MPX_DEVICE(d_counts);
  MPX_DEVICE(d_bbox);
  MPX_DEVICE_OR_NULL(d_mask);
  MPX_DEVICE_OR_NULL(d_mask_visib);
  return bop_gt_info(n_gt, h, w, d_depth_test, n_img, d_depth_scale, d_K, d_depth_gt_large, d_img_idx, delta, d_counts,
                     d_bbox, d_mask, d_mask_visib, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
