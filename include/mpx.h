/*
 * mpx.h -- C ABI of libmpx.so, the H100 (sm_90a) render-and-compare engine behind the MegaPose
 * inference API.  This is the drop-in boundary: plain pointers and sizes, no torch types.
 *
 * Conventions (all entry points):
 *   - return 0 on success, negative on error; the message is available from mpx_last_error()
 *     (thread-local, valid until the next failing call on the same thread);
 *   - pointers named d_* are DEVICE pointers (e.g. torch.Tensor.data_ptr()), h_* are HOST pointers;
 *   - the library never allocates or frees caller tensors; outputs are caller-allocated;
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream);
 *     no entry point synchronises the device;
 *   - poses are row-major 4x4 float32 (TCO: object -> camera, OpenCV camera axes), intrinsics are
 *     row-major 3x3 float32, boxes are (x1, y1, x2, y2) float32 pixels;
 *   - handles (mpx_meshdb, mpx_net) are opaque and owned by the library.
 *
 * Each group cites the reference interface (under /root/reference/src/megapose) that it replaces.
 */
#ifndef MPX_H_
#define MPX_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPX_ABI_VERSION 5

/* ---- library ------------------------------------------------------------------------------ */
int mpx_abi_version(void);
/* 16-bit storage type of weights / activations / the network input tensor ("act16" below): 0 = IEEE fp16 (default: the
 * number format the reference's networks were trained under, training/train_megapose.py:299 torch.cuda.amp.autocast;
 * conversions saturate at +-65504), 1 = bf16 (library built with -DMPX_ACT_BF16).  Accumulation is fp32 in both. */
int mpx_act_dtype(void);
const char* mpx_last_error(void);
/* number of CUDA kernels this library has launched so far in this process (host-side counter) */
long long mpx_launch_count(void);
/* Persistent grids (convolutions, the tiled rasteriser) are sized for mpx_sm_count() SMs: the device's count, or the even
 * limit set here (0 = all).  A limit leaves SMs free for the latency-bound launches of another stream -- the refiner
 * iterations of one frame beside the coarse stage of the next (megapose6d_b200/frame_pipeline.py).  Process-wide; set it
 * before mesh databases are created and before CUDA graphs are captured (both record grid sizes). */
int mpx_set_sm_limit(int n_sms);
int mpx_sm_count(void);
/* measurement aid for bench.py: when enabled every convolution launch is bracketed by CUDA events on
 * its stream; mpx_profile_summary synchronises the device, returns the summed duration (ms), the
 * algorithmic FLOPs (2*M*N*K per launch) and the launch count since enabling, and resets. */
int mpx_profile_enable(int on);
int mpx_profile_summary(double* conv_ms, double* conv_flops, long long* conv_launches);

/* ---- mesh database ---------------------------------------------------------------------------
 * Replaces MeshDataBase / BatchedMeshes (lib3d/rigid_mesh_database.py:57-169) for the point sets
 * and the Panda3D/Assimp model loading (panda3d_renderer/panda3d_scene_renderer.py:195-208) for
 * the triangle meshes.  All meshes of an object dataset are uploaded once.
 *   h_verts   [sum_nv,3] float32, already scaled to metres (RigidObject.scale applied by caller)
 *   h_normals [sum_nv,3] float32 unit vertex normals (object frame)
 *   h_colors  [sum_nv,3] float32 albedo in [0,1]
 *   h_vert_offsets [n_meshes+1] int64 prefix offsets into the vertex arrays
 *   h_faces   [sum_nf,3] int32 vertex indices LOCAL to each mesh
 *   h_face_offsets [n_meshes+1] int64 prefix offsets into h_faces
 */
typedef struct mpx_meshdb mpx_meshdb;
int mpx_meshdb_create(int n_meshes, const float* h_verts, const float* h_normals,
                      const float* h_colors, const int64_t* h_vert_offsets, const int32_t* h_faces,
                      const int64_t* h_face_offsets, mpx_meshdb** out);
int mpx_meshdb_destroy(mpx_meshdb* db);

/* Optional diffuse textures (what Panda3D / Assimp load from the model's material,
 * panda3d_renderer/panda3d_scene_renderer.py:195-208).  Host arrays: h_uv [sum_nv,2] per-vertex texture coordinates
 * (v up), h_tex all RGB8 images back to back (row 0 = top), h_tex_offsets [n+1] byte offsets, h_tex_dims [n,2] =
 * (height, width), (0,0) for an untextured mesh, h_tex_modulate [n] (may be NULL): 1 = multiply the texture with the
 * interpolated vertex colours.  Sampling: repeat wrap, bilinear over texel centres, no mip-mapping.  Call once, after
 * mpx_meshdb_create. */
int mpx_meshdb_set_textures(mpx_meshdb* db, const float* h_uv, const uint8_t* h_tex, const int64_t* h_tex_offsets,
                            const int32_t* h_tex_dims, const int32_t* h_tex_modulate);

/* ---- rasteriser ------------------------------------------------------------------------------
 * Replaces Panda3dBatchRenderer.render (panda3d_renderer/panda3d_batch_renderer.py:217-282) and
 * everything under it (worker_loop :89-150, Panda3dSceneRenderer.render_scene
 * panda3d_scene_renderer.py:298-358, camera model panda3d_renderer/types.py:58-101, depth
 * linearisation and the eye-normal texture panda3d_renderer/utils.py:44-68).
 * One view per (d_label_idx[i], d_TCO[i], d_K[i]); near/far 0.1/10 m; two-sided; black background;
 * non-finite pose or intrinsics => all-zero view (panda3d_batch_renderer.py:109-135).
 */
#define MPX_RASTER_QUANTIZE8 1u      /* round colour/normal channels to k/255 (uint8 read-back)  */
#define MPX_RASTER_NORMALS_GL 2u     /* eye normals in GL Y-up axes instead of Panda Z-up axes  */
#define MPX_RASTER_POINT_LIGHTS 4u   /* rgb lit by make_scene_lights() (ambient 0.1 + six point lights of 0.4 on the object's
                                      * axes at 10 bounding radii, panda3d_scene_renderer.py:104-136) instead of ambient 1.0:
                                      * what models with render_normals=False are fed (models/pose_rigid.py:374-378) */
/* depth normalisation of the fused depth channels (PosePredictor.normalize_depth, models/pose_rigid.py:466-496), applied
 * with d_depth_norm_z[sample] = tCR_z; raster entry points carry it in flags bits 8-9, mpx_roi_align_fused as an argument */
#define MPX_DEPTH_NORM_TCR_SCALE_CLAMP_CENTER 0  /* clamp(depth / z, 0, 2) - 1 (the released RGB-D refiner) */
#define MPX_DEPTH_NORM_TCR_SCALE 1               /* depth / z */
#define MPX_DEPTH_NORM_TCR_CENTER_CLAMP 2        /* clamp(depth - z, -2, 2) */
#define MPX_DEPTH_NORM_NONE 3
#define MPX_RASTER_DEPTH_NORM_SHIFT 8

size_t mpx_raster_workspace_bytes(int h, int w);

/* kernel selection, default 7: bit 0 = batches of at most SMs/8 views (refiner iterations, final scoring) spread
 * the triangles of each view over many CTAs (coverage kernel + resolve kernel) instead of one CTA per
 * (view, row strip); bit 1 = (untiled kernels) visibility through a fire-and-forget 64-bit min reduction instead of
 * read-then-atomic; bit 2 = larger batches use the tiled kernel (triangles binned into screen strips, z-test of a strip in
 * shared memory, candidate fragments dealt out evenly over the threads) instead of one CTA per view with a global
 * visibility buffer.  All combinations produce identical pixels. */
int mpx_raster_set_mode(int mode);

/* contract output: float32 NCHW planes; any of d_rgb [N,3,h,w], d_normals [N,3,h,w],
 * d_depth [N,1,h,w] may be NULL. */
int mpx_raster_render(const mpx_meshdb* db, const int32_t* d_label_idx, const float* d_TCO,
                      const float* d_K, int n_views, int h, int w, uint32_t flags, float* d_rgb,
                      float* d_normals, float* d_depth, void* d_workspace, size_t workspace_bytes,
                      void* stream);

/* fused output: writes act16 channels straight into the network input tensor (see mpx_net):
 * view i belongs to sample i / views_per_sample, view slot v = i % views_per_sample and its
 * channels land at ch_offset + v * ch_per_view: ch_per_view = 3 (rgb), 4 (rgb, depth), 6 (rgb, normals) or
 * 7 (rgb, normals, depth), i.e. what render_normals / render_depth select (models/pose_rigid.py:394-404).
 * d_depth_norm_z [n_samples] (may be NULL = none) applies the depth normalisation selected by flags bits 8-9
 * to the depth channel. */
int mpx_raster_render_fused(const mpx_meshdb* db, const int32_t* d_label_idx, const float* d_TCO,
                            const float* d_K, int n_views, int views_per_sample, int h, int w,
                            uint32_t flags, void* d_x, int c_pad, int ch_offset, int ch_per_view,
                            const float* d_depth_norm_z, void* d_workspace, size_t workspace_bytes,
                            void* stream);

/* multi-object scenes: Panda3dSceneRenderer.render_scene (panda3d_renderer/panda3d_scene_renderer.py:139-358, outputs
 * CameraRenderingData, panda3d_renderer/types.py:43-125).  View v draws instances d_inst_offsets[v] ..
 * d_inst_offsets[v+1]-1 (d_inst_offsets [n_views+1]), instance i = mesh d_inst_label[i] at pose d_inst_TCO[i] [16] in that
 * view's camera frame, under d_K[v] [9], with one shared depth test.  Triangle t of the view's k-th instance has scene
 * index (face counts of instances 0..k-1) + t, and the nearest fragment wins with ties to the lower scene index -- to the
 * lower instance, then the lower triangle: a one-instance scene renders exactly what mpx_raster_render renders.
 * d_inst_color [n_inst,3] (may be NULL): when its first component is >= 0 the instance's albedo (vertex colours and
 * texture) is replaced by that colour (Panda3dObjectData.color).  Outputs (any may be NULL): d_rgb, d_normals
 * [n_views,3,h,w], d_depth [n_views,1,h,w] as mpx_raster_render, d_inst_id [n_views,h,w] int32 = the instance's index
 * within its view, -1 for background.  A non-finite pose or an unknown label: that instance draws nothing; non-finite K
 * or no instances: the view is black with d_inst_id -1.  Malformed device offsets are clamped to [0, n_inst]; a view that
 * still holds more than 1024 instances draws nothing.  Refused before any launch: flags other than bits 0-1 (point lights
 * are not defined for scenes), n_inst > 1024 * n_views, up to 2^31 scene triangles per view, a workspace smaller than
 * mpx_raster_workspace_bytes(h, w).  Views run in chunks of 2 x mpx_sm_count() on `stream`. */
int mpx_raster_render_scene(const mpx_meshdb* db, int n_views, int n_inst, const int32_t* d_inst_offsets,
                            const int32_t* d_inst_label, const float* d_inst_TCO, const float* d_inst_color,
                            const float* d_K, int h, int w, uint32_t flags, float* d_rgb, float* d_normals,
                            float* d_depth, int32_t* d_inst_id, void* d_workspace, size_t workspace_bytes, void* stream);

/* single-view samples (coarse / scoring model, models/pose_rigid.py:634-708): crop + render in one pass.
 * Sample i renders (d_label_idx[i], d_TCO[i], d_K[i] = its crop intrinsics) and crops the observation
 * d_img_nhwc4[d_im_idx[i]] with d_boxes_crop[i] (roi_align as in mpx_roi_align); each pixel's complete channel
 * vector [crop rgb(d) | render rgb, normals(, depth) | zero pad] is stored once.  c_in = 3|4, ch_per_view = 6|7. */
int mpx_render_crop_fused(const mpx_meshdb* db, const int32_t* d_label_idx, const float* d_TCO,
                          const float* d_K, int n, int h, int w, uint32_t flags, const float* d_img_nhwc4,
                          int b, int im_h, int im_w, const int32_t* d_im_idx, const float* d_boxes_crop,
                          int c_in, void* d_x, int c_pad, int ch_per_view, const float* d_depth_norm_z,
                          void* d_workspace, size_t workspace_bytes, void* stream);

/* ---- hypothesis geometry -----------------------------------------------------------------------
 * mpx_pose_init_autodepth: TCO_init_from_boxes_autodepth_with_R (lib3d/cosypose_ops.py:169-218).
 *   d_points [n_labels, n_pts, 3]; d_label_idx, d_bboxes [n,4], d_K [n,9], d_R [n,9] -> d_TCO [n,16]
 */
int mpx_pose_init_autodepth(const float* d_points, int n_pts, const int32_t* d_label_idx,
                            const float* d_bboxes, const float* d_K, const float* d_R, int n,
                            float* d_TCO, void* stream);

/* mpx_normalize_T: normalize_T (lib3d/transform_ops.py:106-119), in-place allowed. */
int mpx_normalize_T(const float* d_T_in, int n, float* d_T_out, void* stream);

/* mpx_crop_geometry: the box/intrinsics part of PosePredictor.crop_inputs and
 * compute_crops_multiview (models/pose_rigid.py:180-303): project_points_robust +
 * boxes_from_uv (lib3d/camera_geometry.py:40-64), deepim_boxes via deepim_crops_robust
 * (lib3d/cropping.py:30-110), get_K_crop_resize (lib3d/camera_geometry.py:67-115).
 *   d_points [n_labels, n_pts, 3] (the deterministic 2000- or 200-point subsets)
 *   d_tCR [n,3]; outputs d_boxes_rend [n,4], d_boxes_crop [n,4], d_K_crop [n,9] */
int mpx_crop_geometry(const float* d_points, int n_pts, const int32_t* d_label_idx,
                      const float* d_TCO, const float* d_K, const float* d_tCR, int n, float lamb,
                      int im_h, int im_w, int out_h, int out_w, float* d_boxes_rend,
                      float* d_boxes_crop, float* d_K_crop, void* stream);

/* mpx_multiview_cameras: make_TCO_multiview (lib3d/multiview.py:165-246), closed form of the
 * Panda3D scene-graph look-at (multiview.py:31-92); float64 internally.
 *   h_offsets [n_extra,3] camera positions wrt camera 0 in units of |tCR|
 *   d_TCV_O [n, 1 + n_extra, 16]: view 0 is TCO itself */
int mpx_multiview_cameras(const float* d_TCO, const float* d_tCR, int n, const float* h_offsets,
                          int n_extra, float* d_TCV_O, void* stream);

/* mpx_pose_update: PosePredictor.update_pose (models/pose_rigid.py:305-312) =
 * compute_rotation_matrix_from_ortho6d (lib3d/rotations.py:25-40) +
 * pose_update_with_reference_point (lib3d/cosypose_ops.py:33-58). */
int mpx_pose_update(const float* d_TCO, const float* d_K_crop, const float* d_pose9,
                    const float* d_tCR, int n, float* d_TCO_out, void* stream);

/* mpx_topk_per_group: top-K by logit per detection, the device-side equivalent of
 * PoseEstimator.filter_pose_estimates (inference/pose_estimator.py:643-667) for the coarse
 * stage.  d_logits [n_groups, m]; d_idx [n_groups, k] int32 indices into m, descending logit,
 * ties broken by lower index. */
int mpx_topk_per_group(const float* d_logits, int n_groups, int m, int k, int32_t* d_idx,
                       void* stream);

/* ---- crop ---------------------------------------------------------------------------------------
 * torchvision.ops.roi_align as called by crop_images (lib3d/cropping.py:113-144): sampling_ratio
 * 4, aligned=False, spatial_scale 1, plus the depth validity masking of the RGB-D branch.
 * mpx_image_to_nhwc4 packs an observation [B,C,H,W] float32 (C = 3|4) to [B,H,W,4] float32 once
 * per frame (channel 3 = depth or 0). */
int mpx_image_to_nhwc4(const float* d_images_nchw, int b, int c, int h, int w, float* d_out_nhwc4,
                       void* stream);
/* contract output: d_out [n, c, out_h, out_w] float32 */
int mpx_roi_align(const float* d_img_nhwc4, int b, int h, int w, const int32_t* d_im_idx,
                  const float* d_boxes, int n, int c, int out_h, int out_w, float* d_out,
                  void* stream);
/* fused output: act16 channels 0..c-1 of the network input tensor; for c == 4 the depth channel is
 * normalised with d_depth_norm_z as in mpx_raster_render_fused. */
int mpx_roi_align_fused(const float* d_img_nhwc4, int b, int h, int w, const int32_t* d_im_idx,
                        const float* d_boxes, int n, int c, int out_h, int out_w, void* d_x,
                        int c_pad, const float* d_depth_norm_z, int depth_norm_kind, void* stream);

/* ---- network -------------------------------------------------------------------------------------
 * ResNet-34 + fc + head of PosePredictor.net_forward (models/pose_rigid.py:314-334) with the
 * backbone of models/torchvision_resnet.py:181-316.  Weights are passed already BN-folded and
 * repacked (see megapose6d_b200/backbone.py): per conv an act16 [C_out, R*S*C_in] matrix and an
 * fp32 bias.
 *
 * Network input tensor ("x"): act16, space-to-depth NHWC [n, H/2, W/2, 4*c_pad] with channel
 * index (dy*2+dx)*c_pad + c, c_pad = the channel count rounded up to a multiple of 16: 16 (coarse, 9 real channels) or
 * 32 (refiner, 27|32) for the released models, up to 256 for configurations with more rendered views.
 */
size_t mpx_net_input_bytes(int n, int h, int w, int c_pad);

/* single convolution (also the unit the parity tests exercise):
 *   d_x [n,H,W,C_in] act16, d_w [C_out, R*S*C_in] act16, d_bias [C_out] fp32,
 *   d_residual / d_out [n,P,Q,C_out] act16 (residual may be NULL)
 *   relu: bit 0 = ReLU; bit 1 = the weights are the space-to-depth form of the 7x7 stem (4x4 taps over C_in = 64,
 *   megapose6d_b200/backbone.py: _stem_s2d; 15 of its 64 (tap, 16-channel) slices are zero by construction);
 *   bit 2 = fused 3x3/s2/p1 max-pool (models/torchvision_resnet.py:197 `self.maxpool` right after the stem's ReLU): d_out is
 *   then the ZEROED [n, (P-1)/2+1, (Q-1)/2+1, C_out] tensor and is max-reduced into; needs bit 0, no residual and
 *   block_n = 0, and returns MPX_ERR_UNSUPPORTED (nothing launched, no error text) otherwise
 *   block_n: 0 = auto, else 64|128|256; max_ctas: 0 = one per SM */
int mpx_conv2d(const void* d_x, int n, int h, int w, int c_in, const void* d_w,
                    const float* d_bias, int c_out, int r, int s, int stride, int pad_lo_h,
                    int pad_lo_w, int pad_hi_h, int pad_hi_w, int relu, const void* d_residual,
                    void* d_out, int block_n, int max_ctas, void* stream);

/* the same convolution with its K loop split over the `splits` (0 = heuristic, 1, 2, 4, 8) CTAs of a thread-block
 * cluster per output tile -- the form the network uses for small batches (refiner iterations: a handful of output
 * tiles, up to 72 serial k-blocks).  The partial tiles are reduced through distributed shared memory in rank order
 * (deterministic).  block_n must be explicit. */
int mpx_conv2d_splitk(const void* d_x, int n, int h, int w, int c_in, const void* d_w,
                           const float* d_bias, int c_out, int r, int s, int stride, int pad_lo_h,
                           int pad_lo_w, int pad_hi_h, int pad_hi_w, int relu, const void* d_residual,
                           void* d_out, int block_n, int splits, void* stream);

/* convolution options, default 8.  One kernel serves every shape (TMA im2col + wgmma, 128-row tiles, 64/128/256-wide
 * tiles chosen from the shape), except that C_out = 64 with at least 2 * mpx_sm_count() 256-pixel tiles (automatic tile
 * width, no K split, no pooled epilogue) runs on a pixel-major kernel: 256 pixels on the wgmma N dimension, two consumer
 * warpgroups taking alternate tiles, the epilogue staged through shared memory and stored by TMA, and the structurally
 * zero k16 steps of the space-to-depth stem (relu bit 1, c_pad 16 or 32) skipped.  The bits:
 *   8   mpx_net_forward splits the K loop of the convolutions after the stem over a thread-block cluster for batches <= 64
 *   512 launch without programmatic dependent launch
 *   262144 / 524288 cap the automatic small-batch K split (bit 3) at 2 / 1 CTAs per tile: less SM time per layer at a higher
 *       latency (set before graphs are captured; the trade for two frames in flight, frame_pipeline.py)
 *   2097152 mpx_net_forward lets the stem's epilogue max-pool (mpx_conv2d relu bit 2) instead of storing the stem output and
 *       running mpx_maxpool3x3s2 on it; the outputs are identical
 *   4194304 (bit 22) never use the pixel-major C_out = 64 kernel (the 128-row kernel serves those convolutions)
 *   8388608 (bit 23) the pixel-major kernel loads its activations by im2col (every input pixel once per filter tap) for
 *       every shape; by default a stride-1 convolution whose padded input row (W + both pads) is at most 256 pixels and
 *       whose C_in is at most 128 loads one band of whole input rows per (filter row, 64 channels) instead and reuses
 *       it over the filter's columns; the outputs are identical
 *   67108864 (bit 26) use the pixel-major C_out = 64 kernel for every convolution it can serve, whatever its size
 * Other bits are accepted and have no effect. */
int mpx_conv_set_mode(int mode);

/* 3x3/s2/p1 max pool, act16 NHWC (torchvision_resnet.py:302) */
int mpx_maxpool3x3s2(const void* d_x, int n, int h, int w, int c, void* d_out, void* stream);

/* global average pool + folded (fc o head) linear: d_x [n, hw, c] act16, d_w [out_dim, c] fp32,
 * d_b [out_dim] fp32 -> d_out [n, out_dim] fp32 */
int mpx_avgpool_linear(const void* d_x, int n, int hw, int c, const float* d_w, const float* d_b,
                       int out_dim, float* d_out, void* stream);

typedef struct mpx_net mpx_net;
/* h_conv_w / h_conv_b: arrays of 36 DEVICE pointers in execution order (stem, then per BasicBlock
 * conv1, conv2, [downsample]); c_pad as above; d_head_w [out_dim,512] fp32, d_head_b [out_dim]. */
int mpx_net_create(int c_pad, int out_dim, const void* const* h_conv_w, const float* const* h_conv_b,
                   int n_convs, const float* d_head_w, const float* d_head_b, mpx_net** out);
/* Pre-activation backbones (WideResNet34 / WideResNet18 of models/wide_resnet.py:29-126, backbone_str "resnet34" /
 * "resnet18", width 1): h_layer_blocks [4] blocks per layer; h_conv_w / h_conv_b: 1 + 2 * blocks + 3 DEVICE pointers in
 * execution order (stem = the 5x5/s2 convolution as 3x3 over the space-to-depth input, bn1 folded; per block conv1 with
 * bn2 folded, conv2 with a zero bias, [bare 1x1 downsample with a zero bias]); h_block_affine: per block a DEVICE pointer
 * to [2, C_in] fp32 (scale, shift of the block's bn1, applied with ReLU to the block input); d_head_w [out_dim, 512] is
 * the head itself (there is no fc). */
int mpx_net_create_preact(int c_pad, int out_dim, const int32_t* h_layer_blocks, const void* const* h_conv_w,
                          const float* const* h_conv_b, int n_convs, const float* const* h_block_affine, int n_blocks,
                          const float* d_head_w, const float* d_head_b, mpx_net** out);
int mpx_net_destroy(mpx_net* net);
/* mpx_net_forward replays a cached CUDA graph per (buffers, shape) after the first call; 0 disables that
 * (every launch is then issued eagerly on the caller's stream). Default: enabled. */
int mpx_net_set_graphs(int on);
size_t mpx_net_workspace_bytes(const mpx_net* net, int n, int h, int w);
/* d_x: network input tensor (see above) for n samples of size h x w; d_out [n, out_dim] fp32 */
int mpx_net_forward(const mpx_net* net, const void* d_x, int n, int h, int w, float* d_out,
                    void* d_workspace, size_t workspace_bytes, void* stream);

/* ---- BOP 2019 pose errors ------------------------------------------------------------------------
 * The pose-error functions of the BOP toolkit (bop_toolkit_lib/pose_error.py: vsd, mssd, mspd, add, adi), vendored by the
 * reference under deps/bop_toolkit_challenge; megapose6d_b200/bop_eval.py drives them.  Lengths are millimetres.
 *
 * mpx_bop_vsd: Visible Surface Discrepancy with the "step" cost and "bop19" visibility.  Pair p compares estimate render
 * d_depth_est[d_est_idx[p]] with ground-truth render d_depth_gt[d_gt_idx[p]] ([n_est|n_gt, h, w] float32 METRES, 0 = no
 * surface, as mpx_raster_render writes them) on test image i = d_img_idx[p]: d_depth_test [n_img, h, w] raw uint16,
 * d_depth_scale [n_img] (test depth in mm = fp32(raw) * fp32(scale)), d_K [n_img, 9] float64.  Renders are shared by every
 * pair that names them.  d_diameter [n_pairs] float64 mm; h_taus [n_taus] (1..MPX_BOP_MAX_TAUS) host float64 tolerances
 * as fractions of the diameter; delta in mm.  Outputs: d_counts [n_pairs, 2 + n_taus] int64 = {union, intersection, pixels
 * of the intersection with |dist_gt - dist_est| / diameter >= tau_k}, d_err [n_pairs, n_taus] float64 =
 * (count_k + union - intersection) / union, 1.0 when the union is empty, NaN for a pair whose indices are out of range.
 * The float64 arithmetic is the toolkit's, in its order, without contraction: the errors are bit-identical to it on the same
 * depth images.  Refused before any launch: n_pairs < 0, empty images, h * w >= 2^31, n_taus out of range, a NULL
 * required pointer. */
#define MPX_BOP_MAX_TAUS 16
int mpx_bop_vsd(int n_pairs, int h, int w, const uint16_t* d_depth_test, int n_img, const float* d_depth_scale,
                const double* d_K, const float* d_depth_est, int n_est, const float* d_depth_gt, int n_gt,
                const int32_t* d_est_idx, const int32_t* d_gt_idx, const int32_t* d_img_idx, const double* d_diameter,
                const double* h_taus, int n_taus, float delta, int64_t* d_counts, double* d_err, void* stream);

/* mpx_bop_point_errors: d_err [n_pairs] float64 of `kind` for pairs of poses of model d_model_idx[p]:
 *   MPX_BOP_MSSD  min over the model's symmetries of the max point distance (mm)
 *   MPX_BOP_MSPD  min over the symmetries of the max distance of the projections under d_K [n_pairs, 9] (px)
 *   MPX_BOP_ADD   mean point distance (identity symmetry only)
 *   MPX_BOP_ADI   mean distance from each point in the gt pose to the nearest point in the estimated pose
 * d_pts [n_pts_total, 3] float64 model points (mm), model m = rows d_pt_offsets[m] .. d_pt_offsets[m+1]-1
 * (d_pt_offsets [n_models+1] int64); d_syms [n_syms_total, 12] float64 symmetry transforms (R row-major, t), model m = rows
 * d_sym_offsets[m] .. d_sym_offsets[m+1]-1 (needed by MSSD / MSPD, the identity included); d_pose_est / d_pose_gt
 * [n_pairs, 12] float64 (R row-major, t in mm).  d_sym_argmin [n_pairs] int32 (may be NULL): index of the minimising
 * symmetry within the model's set, the first one on ties (0 for ADD / ADI).  A pair with an unknown model, no points or
 * no symmetries gets NaN and -1; offsets are clamped to the totals.  Refused before any launch: an unknown kind,
 * n_pairs < 0, n_models < 1, a NULL required pointer. */
#define MPX_BOP_MSSD 0
#define MPX_BOP_MSPD 1
#define MPX_BOP_ADD 2
#define MPX_BOP_ADI 3
int mpx_bop_point_errors(int kind, int n_pairs, int n_models, const double* d_pts, const int64_t* d_pt_offsets,
                         long long n_pts_total, const double* d_syms, const int64_t* d_sym_offsets, long long n_syms_total,
                         const int32_t* d_model_idx, const double* d_pose_est, const double* d_pose_gt, const double* d_K,
                         double* d_err, int32_t* d_sym_argmin, void* stream);

/* mpx_bop_gt_info: the per-gt outputs of the toolkit's scripts/calc_gt_info.py and scripts/calc_gt_masks.py (which the
 * reference's BOPDataset reads as scene_gt_info.json and mask_visib/) for n_gt ground-truth instances of any number of test
 * images, in one pass.  Gt g lies in image i = d_img_idx[g] (d_depth_test [n_img, h, w] raw uint16, d_depth_scale [n_img],
 * d_K [n_img, 9] float64, as mpx_bop_vsd); d_depth_gt_large [n_gt, 3h, 3w] float32 METRES (0 = no surface) is its render
 * alone on the scripts' enlarged canvas, principal point shifted by (w, h), so that the image is the window at (w, h).
 * Depth in mm and the scene_gt_info arithmetic (depth_im_to_dist_im_fast, bop19 visibility against delta in mm) are those
 * of mpx_bop_vsd.  Outputs: d_counts [n_gt, 3] int64 = {px_count_all (canvas), px_count_valid, px_count_visib (image)};
 * d_bbox [n_gt, 8] int32 = {bbox_obj, bbox_visib} as misc.calc_2d_bbox (x, y, x_max - x_min, y_max - y_min), in image
 * coordinates (bbox_obj may be negative), both [-1, -1, -1, -1] unless px_count_visib > 0; d_mask / d_mask_visib
 * [n_gt, h, w] uint8 0/1 (either may be NULL) = calc_gt_masks.py's model-distance > 0 and bop19 visibility, whose distance
 * images come from misc.depth_im_to_dist_im (X d = ((x - cx) d) (1 / fx)): near delta, mask_visib can differ from the
 * visibility that px_count_visib counts.  A gt whose image index is out of range gets counts and boxes of -1 and empty masks.
 * The counts and boxes are integer reductions: they do not depend on the launch shape.  Refused before any launch:
 * n_gt < 0, n_img < 1, empty images, 9 h w >= 2^31, a NULL or non-device required pointer, non-device masks. */
int mpx_bop_gt_info(int n_gt, int h, int w, const uint16_t* d_depth_test, int n_img, const float* d_depth_scale,
                    const double* d_K, const float* d_depth_gt_large, const int32_t* d_img_idx, float delta,
                    int64_t* d_counts, int32_t* d_bbox, uint8_t* d_mask, uint8_t* d_mask_visib, void* stream);

/* ---- depth refinement (TEASER++) ----------------------------------------------------------------------------------
 * Replaces the per-prediction host path of TeaserppRefiner.refine_poses / compute_teaserpp_refinement
 * (inference/teaserpp_refiner.py:53-161, 208-287): meshcat_utils.get_pointcloud, refiner_utils.compute_masks,
 * pytorch3d.ops.sample_farthest_points and teaserpp_python.RobustRegistrationSolver (known correspondences, no scale,
 * GNC-TLS rotation, PMC_EXACT max clique).  megapose6d_b200/teaserpp_refiner.py drives the stages; each is ONE launch for
 * all n_pred predictions of a call.  The arithmetic is the contract stated in DESIGN §4 (parity with the libraries is not
 * pinned).  Sizes: n_pred >= 0, h, w > 0 with h * w < 2^31, 1 <= k <= MPX_TEASER_MAX_POINTS.  Refused before any launch:
 * bad sizes, a NULL required pointer, a required pointer that is not device memory.
 *
 * mpx_teaser_points: prediction p compares d_depth_rendered[p] [n_pred, h, w] with d_depth_measured[d_view_idx[p]]
 * [n_view, h, w] (float32 metres) under d_K[p] [n_pred, 9] float32.  mask_type MPX_TEASER_MASK_SIMPLE (both depths > 0) or
 * MPX_TEASER_MASK_THRESHOLD (also |measured - rendered| <= thresh).  Masked pixels in row-major order go to
 * d_src / d_tgt [n_pred, h * w, 3] float32 (x = fp32((u - cx) * fp32(z / fx)) in float64, likewise y; z), d_count [n_pred]
 * int32 receives the number of masked pixels.  d_raw_src / d_raw_tgt [n_pred, h, w, 3] (may be NULL) receive the
 * unmasked clouds. */
#define MPX_TEASER_MAX_POINTS 1024
#define MPX_TEASER_MASK_SIMPLE 0
#define MPX_TEASER_MASK_THRESHOLD 1
int mpx_teaser_points(int n_pred, int h, int w, const float* d_depth_rendered, const float* d_depth_measured, int n_view,
                      const int32_t* d_view_idx, const float* d_K, int mask_type, float thresh, float* d_src, float* d_tgt,
                      int32_t* d_count, float* d_raw_src, float* d_raw_tgt, void* stream);

/* mpx_teaser_fps: farthest-point sampling of the n = min(d_count[p], cap) points of d_src[p] [n_pred, cap, 3] (one
 * 8-CTA cluster per prediction): index 0, then k - 1 times the arg-max (lowest index on ties) of the running minimum of
 * the fp32 squared distances dx*dx + dy*dy + dz*dz; for n < k the remaining indices are n - 1.  d_idx [n_pred, k] int32
 * (-1 when n == 0); d_samp_src / d_samp_tgt [n_pred, k, 3] float32 receive d_src / d_tgt at those indices (zeros when
 * n == 0).  d_workspace: mpx_teaser_fps_workspace_bytes(n_pred, cap) bytes. */
size_t mpx_teaser_fps_workspace_bytes(int n_pred, int cap);
int mpx_teaser_fps(int n_pred, int cap, const float* d_src, const float* d_tgt, const int32_t* d_count, int k,
                   int32_t* d_idx, float* d_samp_src, float* d_samp_tgt, void* d_workspace, size_t workspace_bytes,
                   void* stream);

/* mpx_teaser_graph: consistency graph of the d_m[p] (0..k) samples of prediction p (d_samp_src / d_samp_tgt
 * [n_pred, k, 3] float32): d_adj [n_pred, k, 16] uint64, bit j % 64 of word j / 64 of row i set when i != j and
 * | ||t_j - t_i|| - ||s_j - s_i|| | <= bound, in float64 without contraction (norm = sqrt((x*x + y*y) + z*z)). */
int mpx_teaser_graph(int n_pred, int k, const float* d_samp_src, const float* d_samp_tgt, const int32_t* d_m, double bound,
                     uint64_t* d_adj, void* stream);

/* mpx_teaser_max_clique: maximum clique of each graph (one CTA per prediction): core numbers by peeling, a greedy clique in
 * core order, then branch and bound with a greedy-colouring bound.  The search expands at most node_budget nodes
 * (<= 0: MPX_TEASER_CLIQUE_NODE_BUDGET); when the budget runs out the best clique found so far is returned and bit 0 of
 * d_status[p] is set.  d_clique [n_pred, k] int32: the clique's vertices in ascending order (then -1), d_clique_size
 * [n_pred] int32, d_status [n_pred] int32 (bit 0: budget exhausted), d_nodes [n_pred] int64 (may be NULL): nodes
 * expanded.  d_workspace: mpx_teaser_clique_workspace_bytes(n_pred, k) bytes. */
#define MPX_TEASER_CLIQUE_NODE_BUDGET 20000
size_t mpx_teaser_clique_workspace_bytes(int n_pred, int k);
int mpx_teaser_max_clique(int n_pred, int k, const uint64_t* d_adj, const int32_t* d_m, long long node_budget,
                          int32_t* d_clique, int32_t* d_clique_size, int32_t* d_status, int64_t* d_nodes,
                          void* d_workspace, size_t workspace_bytes, void* stream);

/* mpx_teaser_solve: for every prediction whose clique has >= 2 vertices: GNC-TLS rotation on the chain TIMs of the clique
 * (TIM bound 2 noise_bound, factor gnc_factor, at most max_iterations, stop on |cost change| < cost_threshold; weighted
 * Kabsch by a float64 Jacobi SVD), per-axis adaptive-voting TLS translation (bound noise_bound), the number of the d_m[p]
 * samples with ||R s + t - t_i|| < noise_bound.  Outputs: d_T [n_pred, 16] float64 (row-major 4x4; identity when the
 * clique is invalid), d_num_inliers [n_pred] int32, d_flags [n_pred] int32 (bit 0 valid, bit 1 accepted).  Accepted
 * (valid and num_inliers >= min_num_inliers): d_poses_input[p] = d_poses[p], then d_poses[p] = fp32(T @ double(d_poses[p]))
 * ([n_pred, 16] float32, updated in place). */
int mpx_teaser_solve(int n_pred, int k, const float* d_samp_src, const float* d_samp_tgt, const int32_t* d_m,
                     const int32_t* d_clique, const int32_t* d_clique_size, double noise_bound, double gnc_factor,
                     int max_iterations, double cost_threshold, int min_num_inliers, float* d_poses, float* d_poses_input,
                     double* d_T, int32_t* d_num_inliers, int32_t* d_flags, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MPX_H_ */
