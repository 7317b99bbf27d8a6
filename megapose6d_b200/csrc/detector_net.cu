// ResNet-50 FPN + RPN head plan of torchvision's Mask R-CNN (torchvision.models.detection: resnet_fpn_backbone("resnet50"),
// FeaturePyramidNetwork with LastLevelMaxPool, RPNHead), the part of the detector whose shapes do not depend on the data.
// The reference runs it through torchvision in fp32 (src/megapose/models/mask_rcnn.py, inference/detector.py:90
// `self.model(images)`); here every convolution is the wgmma convolution of conv_wgmma.cu, in act16 NHWC with fp32
// accumulation and a fused epilogue, and three small kernels move data between them:
//   fpn_input_kernel     fp32 NCHW normalised image batch -> space-to-depth act16 input of the 4x4 stem
//   fpn_resample_kernel  nearest 2x upsampling (FPN top-down path) and the stride-2 subsampling of the pool level
//   fpn_output_kernel    act16 NHWC -> the 15 fp32 NCHW tensors torchvision's stages consume
// After the RoI heads, mask_paste_kernel turns the mask logits of every detection into its image-sized fp32 mask.
#include <cuda.h>
#include <array>
#include <vector>
#include "mpx_common.cuh"

namespace mpx {

// [n, 3, h, w] fp32 -> [n, h/2, w/2, 64] act16, channel (dy*2+dx)*16 + c (c_pad 16, channels 3..15 of each slice zero).
// One thread per space-to-depth pixel: 12 reads, 128 B written.
__global__ void __launch_bounds__(256)
fpn_input_kernel(const float* __restrict__ img, uint4* __restrict__ x, int n, int h, int w) {
  pdl_trigger();
  pdl_wait();
  const int hs = h / 2, ws = w / 2;
  const size_t plane = static_cast<size_t>(h) * w;
  const long long total = static_cast<long long>(n) * hs * ws;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int xs = static_cast<int>(i % ws);
    const long long t = i / ws;
    const int ys = static_cast<int>(t % hs);
    const int b = static_cast<int>(t / hs);
    uint4 o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const float* p = img + static_cast<size_t>(b) * 3 * plane + static_cast<size_t>(2 * ys + dy) * w + 2 * xs + dx;
        o[(dy * 2 + dx) * 2].x = pack_act2(__ldg(p), __ldg(p + plane));
        o[(dy * 2 + dx) * 2].y = pack_act2(__ldg(p + 2 * plane), 0.f);
      }
    }
    uint4* dst = x + i * 8;
#pragma unroll
    for (int k = 0; k < 8; ++k) dst[k] = o[k];
  }
}

// act16 NHWC, 8 channels per thread: up = 1: out[y, x] = in[y / 2, x / 2] (F.interpolate(mode="nearest") to twice the
// size); up = 0: out[y, x] = in[2y, 2x] (F.max_pool2d(kernel 1, stride 2)).  A copy: exact.
__global__ void __launch_bounds__(256)
fpn_resample_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int n, int ho, int wo, int hi, int wi, int c8,
                    int up) {
  pdl_trigger();
  pdl_wait();
  const long long total = static_cast<long long>(n) * ho * wo * c8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cc = static_cast<int>(i % c8);
    long long t = i / c8;
    const int xo = static_cast<int>(t % wo);
    t /= wo;
    const int yo = static_cast<int>(t % ho);
    const int b = static_cast<int>(t / ho);
    const int yi = up ? yo >> 1 : yo << 1, xi = up ? xo >> 1 : xo << 1;
    dst[i] = __ldg(src + ((static_cast<size_t>(b) * hi + yi) * wi + xi) * c8 + cc);
  }
}

// One output tensor: channels c0 .. c0 + nc - 1 of the act16 NHWC src [n, hw, c_src] -> fp32 NCHW dst [n, nc, hw].
struct FpnOutJob {
  const act_t* src;
  float* dst;
  int c_src, c0, nc, hw;
  long long begin;  // first work item; a work item = (image, 8-channel group, pixel), pixel fastest
};
constexpr int kFpnOutputs = 15;  // 5 levels x (features, objectness, deltas)
struct FpnOutParams {
  FpnOutJob job[kFpnOutputs];
  long long total;
};

__global__ void __launch_bounds__(256) fpn_output_kernel(const __grid_constant__ FpnOutParams p) {
  pdl_trigger();
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < p.total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    int j = 0;
    while (j + 1 < kFpnOutputs && i >= p.job[j + 1].begin) ++j;
    const FpnOutJob& jb = p.job[j];
    long long r = i - jb.begin;
    const int pix = static_cast<int>(r % jb.hw);
    r /= jb.hw;
    const int groups = (jb.nc + 7) / 8;
    const int g = static_cast<int>(r % groups);
    const int b = static_cast<int>(r / groups);
    const act_t* s = jb.src + (static_cast<size_t>(b) * jb.hw + pix) * jb.c_src + jb.c0 + 8 * g;
    float* d = jb.dst + (static_cast<size_t>(b) * jb.nc + 8 * g) * jb.hw + pix;
    const int m = jb.nc - 8 * g < 8 ? jb.nc - 8 * g : 8;
    if (m == 8 && ((jb.c_src | jb.c0) & 7) == 0) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(s));
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_act2(u[k]);
        d[static_cast<size_t>(2 * k) * jb.hw] = f.x;
        d[static_cast<size_t>(2 * k + 1) * jb.hw] = f.y;
      }
    } else {
      for (int k = 0; k < m; ++k) d[static_cast<size_t>(k) * jb.hw] = static_cast<float>(s[k]);
    }
  }
}

static unsigned fpn_grid(long long items) {
  long long blocks = (items + 255) / 256;
  const long long cap = static_cast<long long>(sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  return static_cast<unsigned>(blocks > 0 ? blocks : 1);
}

// ---------------------------------------------------------------------------------------------
// Workspace: one act16 NHWC tensor per role, 256-B aligned.  Level l is (h >> l) x (w >> l); the pool level (6) is
// ceil(h5 / 2) x ceil(w5 / 2).  Every tensor of a bottleneck (block input / output, conv1 / conv2 outputs, downsample) is at
// most 256 channels at level 2 or the same bytes deeper, so the scratch tensors are all sized at level 2 x 256.
// ---------------------------------------------------------------------------------------------
enum FpnBuf {
  kBufX, kBufStem, kBufPool0, kBufA, kBufB, kBufT1, kBufT2, kBufDs,
  kBufC2, kBufC3, kBufC4, kBufC5,          // layer1..layer4 outputs
  kBufI0, kBufI1, kBufUp,                  // FPN inner (lateral + top-down) ping-pong, upsampled residual
  kBufP2, kBufP3, kBufP4, kBufP5, kBufP6,  // FPN outputs '0'..'3', 'pool'
  kBufRpn,                                 // RPN 3x3 output (one level at a time)
  kBufH2, kBufH3, kBufH4, kBufH5, kBufH6,  // RPN 1x1 outputs [.., 64]: objectness | deltas | zero
  kBufCount
};

static size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

struct FpnDims {
  int lh[5], lw[5];  // RPN / output levels: 2, 3, 4, 5, pool
};
static FpnDims fpn_dims(int h, int w) {
  FpnDims d;
  for (int l = 0; l < 4; ++l) {
    d.lh[l] = h >> (l + 2);
    d.lw[l] = w >> (l + 2);
  }
  d.lh[4] = (d.lh[3] + 1) / 2;
  d.lw[4] = (d.lw[3] + 1) / 2;
  return d;
}

static size_t fpn_layout(int n, int h, int w, size_t off[kBufCount]) {
  const FpnDims d = fpn_dims(h, w);
  auto lvl = [&](int i, int c) { return static_cast<size_t>(n) * d.lh[i] * d.lw[i] * c * 2; };
  size_t bytes[kBufCount];
  const size_t s1 = static_cast<size_t>(n) * (h / 2) * (w / 2) * 64 * 2;
  bytes[kBufX] = s1;
  bytes[kBufStem] = s1;
  bytes[kBufPool0] = lvl(0, 64);
  for (int b : {kBufA, kBufB, kBufT1, kBufT2, kBufDs, kBufI0, kBufI1, kBufUp, kBufRpn}) bytes[b] = lvl(0, 256);
  bytes[kBufC2] = lvl(0, 256);
  bytes[kBufC3] = lvl(1, 512);
  bytes[kBufC4] = lvl(2, 1024);
  bytes[kBufC5] = lvl(3, 2048);
  for (int l = 0; l < 5; ++l) {
    bytes[kBufP2 + l] = lvl(l, 256);
    bytes[kBufH2 + l] = lvl(l, 64);
  }
  size_t total = 0;
  for (int b = 0; b < kBufCount; ++b) {
    off[b] = total;
    total += align256(bytes[b]);
  }
  return total;
}

size_t fpn_workspace_bytes(int n, int h, int w) {
  size_t off[kBufCount];
  return fpn_layout(n, h, w, off);
}

// ---------------------------------------------------------------------------------------------
// Plan handle and CUDA graph cache (one graph per (buffers, shape), as net.cu's Net)
// ---------------------------------------------------------------------------------------------
struct FpnGraphEntry {
  std::array<const void*, 2 + kFpnOutputs> ptrs;  // images, workspace, 15 outputs
  int n, h, w;
  int warm;  // direct runs seen, then launches per replay
  cudaGraphExec_t exec;
};

struct Fpn {
  std::vector<const void*> conv_w;
  std::vector<const float*> conv_b;
  int n_anchors;
  std::vector<FpnGraphEntry> graphs;
  cudaStream_t side = nullptr;
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
};

int fpn_create(const void* const* conv_w, const float* const* conv_b, int n_convs, int n_anchors, Fpn** out) {
  MPX_REQUIRE(n_convs == kFpnConvs, "fpn: expected %d conv tensors, got %d", kFpnConvs, n_convs);
  MPX_REQUIRE(n_anchors >= 1 && n_anchors <= 12, "fpn: %d anchors per location, must be 1..12", n_anchors);
  Fpn* f = new Fpn();
  f->conv_w.assign(conv_w, conv_w + n_convs);
  f->conv_b.assign(conv_b, conv_b + n_convs);
  f->n_anchors = n_anchors;
  *out = f;
  return MPX_OK;
}

void fpn_destroy(Fpn* f) {
  if (!f) return;
  for (auto& g : f->graphs)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  if (f->ev_in) cudaEventDestroy(f->ev_in);
  if (f->ev_out) cudaEventDestroy(f->ev_out);
  if (f->side) cudaStreamDestroy(f->side);
  delete f;
}

static int fpn_resample(const void* src, void* dst, int n, int ho, int wo, int hi, int wi, int up, cudaStream_t stream) {
  const long long items = static_cast<long long>(n) * ho * wo * 32;
  MPX_CHECK_CUDA(launch_pdl(fpn_resample_kernel, dim3(fpn_grid(items)), dim3(256), 0, stream, 1,
                            reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), n, ho, wo, hi, wi, 32, up));
  ++g_launches;
  return MPX_OK;
}

// Weight order (= execution order): stem; per bottleneck conv1, conv2, [downsample], conv3; FPN lateral 1x1 on C2..C5;
// FPN output 3x3 on levels 2..5; RPN 3x3; RPN merged 1x1 (cls_logits | bbox_pred | zero rows).
static int fpn_forward_direct(const Fpn* f, const float* images, int n, int h, int w, float* const* features,
                              float* const* objectness, float* const* deltas, void* workspace, cudaStream_t stream) {
  size_t off[kBufCount];
  fpn_layout(n, h, w, off);
  uint8_t* base = reinterpret_cast<uint8_t*>(workspace);
  auto buf = [&](int b) -> void* { return base + off[b]; };
  const FpnDims dims = fpn_dims(h, w);
  // small batches: the deep convolutions split their K loop over a cluster, as in mpx_net_forward
  const int sk = ((conv_get_mode() & MPX_CONV_NET_SPLITK) != 0 && n <= 64) ? -1 : 0;
  auto conv = [&](int wi, int H, int W, int c_in, int c_out, int k, int stride, int relu, const void* x,
                  const void* residual, void* out) {
    const int pad = k / 2;
    ConvDesc d{n, H, W, c_in, c_out, k, k, stride, pad, pad, pad, pad, relu, 0};
    return conv_forward(d, x, f->conv_w[wi], f->conv_b[wi], residual, out, 0, 0, stream, sk, 2048);
  };
  int rc;
  MPX_CHECK_CUDA(launch_pdl(fpn_input_kernel, dim3(fpn_grid(static_cast<long long>(n) * (h / 2) * (w / 2))), dim3(256), 0,
                            stream, 1, images, reinterpret_cast<uint4*>(buf(kBufX)), n, h, w));
  ++g_launches;
  {
    // 7x7/s2/p3 stem as the 4x4/s1 convolution (pad 2 low, 1 high) over the space-to-depth input, then ReLU, max-pool
    ConvDesc d{n, h / 2, w / 2, 64, 64, 4, 4, 1, 2, 2, 1, 1, 1, 1};
    rc = conv_forward(d, buf(kBufX), f->conv_w[0], f->conv_b[0], nullptr, buf(kBufStem), 0, 0, stream, 0, 2048);
    if (rc != MPX_OK) return rc;
    rc = maxpool3x3s2(buf(kBufStem), n, h / 2, w / 2, 64, buf(kBufPool0), stream);
    if (rc != MPX_OK) return rc;
  }
  static const int kWidth[4] = {64, 128, 256, 512}, kBlocks[4] = {3, 4, 6, 3};
  int wi = 1;
  void* x = buf(kBufPool0);
  int H = h / 4, W = w / 4, C = 64;
  for (int layer = 0; layer < 4; ++layer) {
    const int width = kWidth[layer];
    for (int blk = 0; blk < kBlocks[layer]; ++blk) {
      const int stride = (blk == 0 && layer > 0) ? 2 : 1;
      const int Ho = H / stride, Wo = W / stride;
      rc = conv(wi++, H, W, C, width, 1, 1, 1, x, nullptr, buf(kBufT1));
      if (rc != MPX_OK) return rc;
      rc = conv(wi++, H, W, width, width, 3, stride, 1, buf(kBufT1), nullptr, buf(kBufT2));
      if (rc != MPX_OK) return rc;
      const void* residual = x;
      if (blk == 0) {
        rc = conv(wi++, H, W, C, 4 * width, 1, stride, 0, x, nullptr, buf(kBufDs));
        if (rc != MPX_OK) return rc;
        residual = buf(kBufDs);
      }
      void* out = blk + 1 == kBlocks[layer] ? buf(kBufC2 + layer) : (x == buf(kBufA) ? buf(kBufB) : buf(kBufA));
      rc = conv(wi++, Ho, Wo, width, 4 * width, 1, 1, 1, buf(kBufT2), residual, out);
      if (rc != MPX_OK) return rc;
      x = out;
      H = Ho;
      W = Wo;
      C = 4 * width;
    }
  }
  // FPN: inner_l = lateral_l(C_l) + nearest_up(inner_{l+1}) (the sum in the lateral convolution's fp32 epilogue),
  // P_l = output_l(inner_l); pool = P5[::2, ::2]
  const int lat0 = wi, out0 = wi + 4, rpn0 = wi + 8;
  static const int kCin[4] = {256, 512, 1024, 2048};
  void* inner[2] = {buf(kBufI0), buf(kBufI1)};
  int cur = 0;
  rc = conv(lat0 + 3, dims.lh[3], dims.lw[3], 2048, 256, 1, 1, 0, buf(kBufC5), nullptr, inner[cur]);
  if (rc != MPX_OK) return rc;
  rc = conv(out0 + 3, dims.lh[3], dims.lw[3], 256, 256, 3, 1, 0, inner[cur], nullptr, buf(kBufP5));
  if (rc != MPX_OK) return rc;
  for (int l = 2; l >= 0; --l) {
    rc = fpn_resample(inner[cur], buf(kBufUp), n, dims.lh[l], dims.lw[l], dims.lh[l + 1], dims.lw[l + 1], 1, stream);
    if (rc != MPX_OK) return rc;
    rc = conv(lat0 + l, dims.lh[l], dims.lw[l], kCin[l], 256, 1, 1, 0, buf(kBufC2 + l), buf(kBufUp), inner[cur ^ 1]);
    if (rc != MPX_OK) return rc;
    cur ^= 1;
    rc = conv(out0 + l, dims.lh[l], dims.lw[l], 256, 256, 3, 1, 0, inner[cur], nullptr, buf(kBufP2 + l));
    if (rc != MPX_OK) return rc;
  }
  rc = fpn_resample(buf(kBufP5), buf(kBufP6), n, dims.lh[4], dims.lw[4], dims.lh[3], dims.lw[3], 0, stream);
  if (rc != MPX_OK) return rc;
  // RPN head on every level: 3x3 + ReLU, then the merged 1x1
  for (int l = 0; l < 5; ++l) {
    rc = conv(rpn0, dims.lh[l], dims.lw[l], 256, 256, 3, 1, 1, buf(kBufP2 + l), nullptr, buf(kBufRpn));
    if (rc != MPX_OK) return rc;
    rc = conv(rpn0 + 1, dims.lh[l], dims.lw[l], 256, 64, 1, 1, 0, buf(kBufRpn), nullptr, buf(kBufH2 + l));
    if (rc != MPX_OK) return rc;
  }
  // the 15 fp32 NCHW outputs
  FpnOutParams p{};
  long long total = 0;
  const int A = f->n_anchors;
  for (int l = 0; l < 5; ++l) {
    const int hw = dims.lh[l] * dims.lw[l];
    const FpnOutJob jobs[3] = {
        {reinterpret_cast<const act_t*>(buf(kBufP2 + l)), features[l], 256, 0, 256, hw, 0},
        {reinterpret_cast<const act_t*>(buf(kBufH2 + l)), objectness[l], 64, 0, A, hw, 0},
        {reinterpret_cast<const act_t*>(buf(kBufH2 + l)), deltas[l], 64, A, 4 * A, hw, 0}};
    for (int k = 0; k < 3; ++k) {
      FpnOutJob& jb = p.job[3 * l + k];
      jb = jobs[k];
      jb.begin = total;
      total += static_cast<long long>(n) * ((jb.nc + 7) / 8) * hw;
    }
  }
  p.total = total;
  MPX_CHECK_CUDA(launch_pdl(fpn_output_kernel, dim3(fpn_grid(total)), dim3(256), 0, stream, 1, p));
  ++g_launches;
  return MPX_OK;
}

int fpn_forward(Fpn* f, const float* images, int n, int h, int w, float* const* features, float* const* objectness,
                float* const* deltas, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  MPX_REQUIRE(workspace_bytes >= fpn_workspace_bytes(n, h, w), "fpn: workspace too small");
  MPX_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "fpn: workspace must be 256-B aligned");
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(stream, &cap);
  if (!net_graphs_enabled() || conv_profile_enabled() || cap != cudaStreamCaptureStatusNone)
    return fpn_forward_direct(f, images, n, h, w, features, objectness, deltas, workspace, stream);
  std::array<const void*, 2 + kFpnOutputs> key;
  key[0] = images;
  key[1] = workspace;
  for (int l = 0; l < 5; ++l) {
    key[2 + l] = features[l];
    key[7 + l] = objectness[l];
    key[12 + l] = deltas[l];
  }
  FpnGraphEntry* e = nullptr;
  for (auto& g : f->graphs)
    if (g.ptrs == key && g.n == n && g.h == h && g.w == w) e = &g;
  if (!e) {
    if (f->graphs.size() >= 32) {
      for (auto& g : f->graphs)
        if (g.exec) cudaGraphExecDestroy(g.exec);
      f->graphs.clear();
    }
    f->graphs.push_back(FpnGraphEntry{key, n, h, w, 0, nullptr});
    e = &f->graphs.back();
  }
  if (e->exec == nullptr) {
    if (e->warm == 0) {  // first sight of this shape: run eagerly (one-time attribute / driver set-up)
      e->warm = 1;
      return fpn_forward_direct(f, images, n, h, w, features, objectness, deltas, workspace, stream);
    }
    if (!f->side) {
      MPX_CHECK_CUDA(cudaStreamCreateWithFlags(&f->side, cudaStreamNonBlocking));
      MPX_CHECK_CUDA(cudaEventCreateWithFlags(&f->ev_in, cudaEventDisableTiming));
      MPX_CHECK_CUDA(cudaEventCreateWithFlags(&f->ev_out, cudaEventDisableTiming));
    }
    cudaGraph_t graph = nullptr;
    MPX_CHECK_CUDA(cudaStreamBeginCapture(f->side, cudaStreamCaptureModeThreadLocal));
    const long long launches_before = g_launches;
    const int rc = fpn_forward_direct(f, images, n, h, w, features, objectness, deltas, workspace, f->side);
    cudaError_t ce = cudaStreamEndCapture(f->side, &graph);
    e->warm = static_cast<int>(g_launches - launches_before);
    g_launches = launches_before;
    if (rc == MPX_OK && ce == cudaSuccess && graph != nullptr) {
      ce = cudaGraphInstantiate(&e->exec, graph, 0);
      if (ce != cudaSuccess) e->exec = nullptr;
    }
    if (graph) cudaGraphDestroy(graph);
    if (e->exec == nullptr) {
      cudaGetLastError();
      net_set_graphs(0);  // eager launches for the rest of the process, as mpx_net_forward does
      return fpn_forward_direct(f, images, n, h, w, features, objectness, deltas, workspace, stream);
    }
  }
  MPX_CHECK_CUDA(cudaEventRecord(f->ev_in, stream));
  MPX_CHECK_CUDA(cudaStreamWaitEvent(f->side, f->ev_in, 0));
  MPX_CHECK_CUDA(cudaGraphLaunch(e->exec, f->side));
  MPX_CHECK_CUDA(cudaEventRecord(f->ev_out, f->side));
  MPX_CHECK_CUDA(cudaStreamWaitEvent(stream, f->ev_out, 0));
  g_launches += e->warm;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------
// Mask inference and pasting: torchvision's maskrcnn_inference (sigmoid, the label's channel), then
// GeneralizedRCNNTransform.postprocess: resize_boxes to the original size and paste_masks_in_image (padding 1).  Each
// step is the fp32 operation torchvision runs, in its order, with the same roundings: the box arithmetic is written with
// explicit round-to-nearest intrinsics (torchvision runs each of those operations as a kernel of its own, so nothing may
// be fused into an FMA), the bilinear weights and sums as ATen's upsample_bilinear2d writes them.
// ---------------------------------------------------------------------------------------------
struct MaskImage {
  float* out;               // [count, 1, H, W]
  int start, count;         // detections start .. start + count - 1 of the batch
  int h, w, H, W;           // transformed (model) size and original size
};
struct MaskPasteParams {
  MaskImage img[kMaskMaxImages];
  int n_images, n_classes, m;
  float scale;              // (m + 2) / m: expand_boxes' scale, rounded to fp32 as torch rounds a Python float operand
};

// grid (pixel blocks, detection); one block pastes a slice of one detection's image-sized mask
__global__ void __launch_bounds__(256)
mask_paste_kernel(const __grid_constant__ MaskPasteParams p, const float* __restrict__ logits,
                  const long long* __restrict__ labels, const float* __restrict__ boxes, float* __restrict__ boxes_out) {
  __shared__ float prob[(kMaskMaxM + 2) * (kMaskMaxM + 2)];  // the zero-padded (m + 2)^2 probabilities
  const int d = blockIdx.y;
  int i = 0;
  while (i + 1 < p.n_images && d >= p.img[i + 1].start) ++i;
  const MaskImage im = p.img[i];
  // resize_boxes: ratio = fp32(new) / fp32(old), then one product per coordinate
  const float rw = __fdiv_rn(static_cast<float>(im.W), static_cast<float>(im.w));
  const float rh = __fdiv_rn(static_cast<float>(im.H), static_cast<float>(im.h));
  const float b0 = __fmul_rn(boxes[4 * d + 0], rw), b1 = __fmul_rn(boxes[4 * d + 1], rh);
  const float b2 = __fmul_rn(boxes[4 * d + 2], rw), b3 = __fmul_rn(boxes[4 * d + 3], rh);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    boxes_out[4 * d + 0] = b0;
    boxes_out[4 * d + 1] = b1;
    boxes_out[4 * d + 2] = b2;
    boxes_out[4 * d + 3] = b3;
  }
  // expand_boxes, then .to(int64) (truncation toward zero)
  const float w_half = __fmul_rn(__fmul_rn(__fsub_rn(b2, b0), 0.5f), p.scale);
  const float h_half = __fmul_rn(__fmul_rn(__fsub_rn(b3, b1), 0.5f), p.scale);
  const float x_c = __fmul_rn(__fadd_rn(b2, b0), 0.5f), y_c = __fmul_rn(__fadd_rn(b3, b1), 0.5f);
  const long long bx0 = static_cast<long long>(__fsub_rn(x_c, w_half));
  const long long bx1 = static_cast<long long>(__fadd_rn(x_c, w_half));
  const long long by0 = static_cast<long long>(__fsub_rn(y_c, h_half));
  const long long by1 = static_cast<long long>(__fadd_rn(y_c, h_half));
  // paste_mask_in_image: the (m + 2)^2 map resized to bw x bh, its pixel (x - bx0, y - by0) lands on image pixel (x, y)
  const long long bw = bx1 - bx0 + 1 > 1 ? bx1 - bx0 + 1 : 1;
  const long long bh = by1 - by0 + 1 > 1 ? by1 - by0 + 1 : 1;
  const long long label = labels[d];
  const bool valid = label >= 0 && label < p.n_classes;
  const int mp = p.m + 2;
  if (valid) {
    const float* src = logits + (static_cast<size_t>(d) * p.n_classes + label) * p.m * p.m;
    for (int k = threadIdx.x; k < mp * mp; k += blockDim.x) {
      const int py = k / mp, px = k % mp;
      float v = 0.f;
      if (py >= 1 && py <= p.m && px >= 1 && px <= p.m) v = 1.0f / (1.0f + expf(-src[(py - 1) * p.m + (px - 1)]));
      prob[k] = v;
    }
  }
  __syncthreads();
  // upsample_bilinear2d, align_corners=False, no scale factors: scale = fp32(in) / out
  const float rheight = static_cast<float>(mp) / static_cast<float>(bh);
  const float rwidth = static_cast<float>(mp) / static_cast<float>(bw);
  const long long hw = static_cast<long long>(im.H) * im.W;
  float* out = im.out + static_cast<size_t>(d - im.start) * hw;
  for (long long k = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; k < hw;
       k += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(k / im.W), x = static_cast<int>(k % im.W);
    float val = 0.f;
    if (valid && x >= bx0 && x <= bx1 && y >= by0 && y <= by1) {
      const int h2 = static_cast<int>(y - by0), w2 = static_cast<int>(x - bx0);
      float h1r = rheight * (h2 + 0.5f) - 0.5f;
      h1r = h1r < 0.f ? 0.f : h1r;
      const int h1 = static_cast<int>(h1r);
      const int h1p = h1 < mp - 1 ? 1 : 0;
      const float h1lambda = h1r - h1, h0lambda = 1.f - h1lambda;
      float w1r = rwidth * (w2 + 0.5f) - 0.5f;
      w1r = w1r < 0.f ? 0.f : w1r;
      const int w1 = static_cast<int>(w1r);
      const int w1p = w1 < mp - 1 ? 1 : 0;
      const float w1lambda = w1r - w1, w0lambda = 1.f - w1lambda;
      const float* r0 = prob + h1 * mp + w1;
      const float* r1 = r0 + h1p * mp;
      val = h0lambda * (w0lambda * r0[0] + w1lambda * r0[w1p]) + h1lambda * (w0lambda * r1[0] + w1lambda * r1[w1p]);
    }
    out[k] = val;
  }
}

int mask_paste(const float* logits, const long long* labels, const float* boxes, int n_masks, int n_classes, int m,
               int n_images, const int* counts, const int* sizes, float* boxes_out, float* const* masks,
               cudaStream_t stream) {
  MaskPasteParams p{};
  p.n_images = n_images;
  p.n_classes = n_classes;
  p.m = m;
  p.scale = static_cast<float>(static_cast<double>(m + 2) / m);
  long long max_hw = 0;
  int start = 0;
  for (int i = 0; i < n_images; ++i) {
    p.img[i] = MaskImage{masks[i], start, counts[i], sizes[4 * i], sizes[4 * i + 1], sizes[4 * i + 2], sizes[4 * i + 3]};
    start += counts[i];
    const long long hw = static_cast<long long>(sizes[4 * i + 2]) * sizes[4 * i + 3];
    if (counts[i] > 0 && hw > max_hw) max_hw = hw;
  }
  if (n_masks == 0) return MPX_OK;
  long long bx = (max_hw + 256 * 8 - 1) / (256 * 8);  // eight pixels per thread
  if (bx < 1) bx = 1;
  mask_paste_kernel<<<dim3(static_cast<unsigned>(bx), static_cast<unsigned>(n_masks)), 256, 0, stream>>>(
      p, logits, labels, boxes, boxes_out);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

}  // namespace mpx
