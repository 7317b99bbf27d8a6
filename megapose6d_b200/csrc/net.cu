// ResNet-34 execution plan around the wgmma convolution: max-pool, pooled linear tail, and the
// fixed 36-convolution schedule of the reference backbone
// (reference: src/megapose/models/torchvision_resnet.py:74-120 BasicBlock, :298-311 forward order;
//  heads: src/megapose/models/pose_rigid.py:120-130, 314-334).
#include <cuda.h>
#include <cstdlib>
#include <vector>
#include "mpx_common.cuh"

namespace mpx {


// ---------------------------------------------------------------------------------------------
// 3x3 / stride 2 / pad 1 max pool on bf16 NHWC; one thread = 8 channels (16 B) of one output pixel
// ---------------------------------------------------------------------------------------------
// one CTA per output row (img, oy): threads walk (ox, channel group) with 32-bit index math only -- the flat
// grid-stride form spent most of its instructions on 64-bit div / mod of the element index
__global__ void __launch_bounds__(512)
maxpool3x3s2_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int n, int h, int w, int c8, int ho, int wo) {
  pdl_trigger();
  pdl_wait();
  const int row_items = wo * c8;
  for (int row = blockIdx.x; row < n * ho; row += gridDim.x) {
    const int img = row / ho, oy = row - img * ho;
    const int iy0 = oy * 2 - 1;
    const uint4* xin = x + static_cast<size_t>(img) * h * w * c8;
    uint4* orow = out + static_cast<size_t>(row) * row_items;
    for (int t = threadIdx.x; t < row_items; t += blockDim.x) {
      const int ox = t / c8, cc = t - ox * c8;
      const int ix0 = ox * 2 - 1;
      float m[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
        const int iy = iy0 + dy;
        if (iy < 0 || iy >= h) continue;
        const uint4* xr = xin + static_cast<size_t>(iy) * w * c8 + cc;
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          const int ix = ix0 + dx;
          if (ix < 0 || ix >= w) continue;
          const uint4 v = __ldg(xr + ix * c8);
          const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = unpack_act2(u[j]);
            m[2 * j] = fmaxf(m[2 * j], f.x);
            m[2 * j + 1] = fmaxf(m[2 * j + 1], f.y);
          }
        }
      }
      uint4 o;
      o.x = pack_act2(m[0], m[1]);
      o.y = pack_act2(m[2], m[3]);
      o.z = pack_act2(m[4], m[5]);
      o.w = pack_act2(m[6], m[7]);
      orow[t] = o;
    }
  }
}

int maxpool3x3s2(const void* x, int n, int h, int w, int c, void* out, cudaStream_t stream) {
  MPX_REQUIRE(c % 8 == 0, "maxpool: C=%d must be a multiple of 8", c);
  const int ho = (h + 2 - 3) / 2 + 1, wo = (w + 2 - 3) / 2 + 1;
  const long long rows = static_cast<long long>(n) * ho;
  if (rows == 0) return MPX_OK;
  MPX_REQUIRE(rows < (1LL << 31), "maxpool: too many rows");
  const int row_items = wo * (c / 8);
  int threads = ((row_items + 31) / 32) * 32;
  if (threads > 512) threads = ((row_items + 1) / 2 + 31) / 32 * 32;  // two passes per row
  if (threads > 512) threads = 512;
  long long blocks = rows;
  const long long cap = static_cast<long long>(sm_count()) * 32;
  if (blocks > cap) blocks = cap;
  MPX_CHECK_CUDA(launch_pdl(maxpool3x3s2_kernel, dim3(static_cast<unsigned>(blocks)), dim3(threads), 0, stream, 1,
                            reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), n, h, w, c / 8, ho, wo));
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------
// per-channel affine + ReLU on a 16-bit NHWC tensor: a = relu(scale[c] * x + shift[c]) -- the pre-activation of the
// WideResNet blocks (relu(bn1(x)), models/wide_resnet.py:53), whose input x is also the block's residual and therefore has to
// stay unactivated.  One thread = 8 channels (16 B); fp32 arithmetic, one rounding.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
affine_relu_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, long long n8, int c8,
                   const float* __restrict__ scale_shift /* [2, C] */) {
  pdl_trigger();
  pdl_wait();
  const float* scale = scale_shift;
  const float* shift = scale_shift + 8 * c8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n8;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % c8) * 8;
    const uint4 v = __ldg(x + i);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_act2(u[j]);
      const float a = fmaxf(fmaf(f.x, __ldg(scale + cg + 2 * j), __ldg(shift + cg + 2 * j)), 0.f);
      const float b = fmaxf(fmaf(f.y, __ldg(scale + cg + 2 * j + 1), __ldg(shift + cg + 2 * j + 1)), 0.f);
      o[j] = pack_act2(a, b);
    }
    out[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

static int affine_relu(const void* x, long long elems, int c, const float* scale_shift, void* out, cudaStream_t stream) {
  MPX_REQUIRE(c % 8 == 0 && elems % c == 0, "affine_relu: C=%d", c);
  if (elems == 0) return MPX_OK;
  const long long n8 = elems / 8;
  long long blocks = (n8 + 255) / 256;
  const long long cap = static_cast<long long>(sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  MPX_CHECK_CUDA(launch_pdl(affine_relu_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, 1,
                            reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), n8, c / 8, scale_shift));
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------
// global average pool + linear (fc and head folded into one [out_dim, C] matrix on the host)
// one CTA (512 threads) per sample: the pixels are split over G = 512 / (C/4) thread groups (each thread sums
// 4 channels over every G-th pixel, fixed order), the groups are combined through shared memory, then one warp per
// output does the dot product with warp-shuffle reductions.  With one sample per launch (refiner) the old
// one-thread-per-4-channels loop over all pixels was a 27 us latency chain.
// ---------------------------------------------------------------------------------------------
constexpr int kPoolThreads = 512;
__global__ void __launch_bounds__(kPoolThreads)
avgpool_linear_kernel(const act_t* __restrict__ x, int hw, int c, const float* __restrict__ w,
                      const float* __restrict__ b, int out_dim, float* __restrict__ out) {
  extern __shared__ float smem_pool[];  // [G][c] partial sums, then [c] pooled
  const int img = blockIdx.x;
  const act_t* xi = x + static_cast<size_t>(img) * hw * c;
  pdl_trigger();
  pdl_wait();
  const int nq = c >> 2;
  const int G = nq >= kPoolThreads ? 1 : kPoolThreads / nq;
  float* part = smem_pool;
  float* pooled = smem_pool + static_cast<size_t>(G) * c;
  const int g = threadIdx.x / nq;
  if (g < G) {
    for (int q = threadIdx.x - g * nq; q < nq; q += kPoolThreads) {  // one pass unless C > 2048
      float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll 4
      for (int p = g; p < hw; p += G) {
        const uint2 v = __ldg(reinterpret_cast<const uint2*>(xi + static_cast<size_t>(p) * c + 4 * q));
        const float2 a = unpack_act2(v.x), d = unpack_act2(v.y);
        s0 += a.x;
        s1 += a.y;
        s2 += d.x;
        s3 += d.y;
      }
      *reinterpret_cast<float4*>(part + static_cast<size_t>(g) * c + 4 * q) = make_float4(s0, s1, s2, s3);
    }
  }
  __syncthreads();
  const float inv = 1.f / static_cast<float>(hw);
  for (int k = threadIdx.x; k < c; k += kPoolThreads) {
    float s = 0.f;
    for (int gg = 0; gg < G; ++gg) s += part[static_cast<size_t>(gg) * c + k];
    pooled[k] = s * inv;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = kPoolThreads >> 5;
  for (int o = warp; o < out_dim; o += nwarps) {
    float acc = 0.f;
    for (int k = lane; k < c; k += 32) acc = fmaf(pooled[k], __ldg(w + static_cast<size_t>(o) * c + k), acc);
    acc = warp_sum(acc);
    if (lane == 0) out[static_cast<size_t>(img) * out_dim + o] = acc + __ldg(b + o);
  }
}

int avgpool_linear(const void* x, int n, int hw, int c, const float* w, const float* b, int out_dim,
                   float* out, cudaStream_t stream) {
  MPX_REQUIRE(c % 4 == 0 && c <= 4096, "avgpool_linear: C=%d unsupported", c);
  if (n == 0) return MPX_OK;
  const int nq = c / 4;
  const int G = nq >= kPoolThreads ? 1 : kPoolThreads / nq;
  const size_t smem = static_cast<size_t>(G + 1) * c * sizeof(float);
  MPX_REQUIRE(smem <= 48 * 1024, "avgpool_linear: C=%d needs %zu bytes of shared memory", c, smem);
  MPX_CHECK_CUDA(launch_pdl(avgpool_linear_kernel, dim3(n), dim3(kPoolThreads), smem, stream, 1,
                            reinterpret_cast<const act_t*>(x), hw, c, w, b, out_dim, out));
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------
// ResNet-34 plan
// ---------------------------------------------------------------------------------------------
// One captured CUDA graph per (buffers, shape): the 38 launches of a forward pass become one graph launch.  For the
// refiner (a handful of samples) the forward pass is launch-latency bound, not throughput bound.
struct GraphEntry {
  const void* x;
  float* out;
  void* ws;
  int n, h, w;
  int warm;  // direct runs seen (the first call of a shape runs eagerly: one-time attribute / driver set-up)
  cudaGraphExec_t exec;
};

struct Net {
  int c_pad;
  int out_dim;
  int preact = 0;            // 1: pre-activation WideResNet blocks (net_create_preact)
  int layer_blocks[4] = {3, 4, 6, 3};
  std::vector<const float*> block_affine;  // preact: per block [2, C_in] fp32 (scale, shift of bn1)
  std::vector<const void*> conv_w;
  std::vector<const float*> conv_b;
  const float* head_w;
  const float* head_b;
  std::vector<GraphEntry> graphs;
  cudaStream_t side = nullptr;  // capture / replay stream (the caller's stream may be the legacy default stream)
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
};

static bool g_use_graphs = true;
void net_set_graphs(int on) { g_use_graphs = on != 0; }

static const int kLayerBlocks[4] = {3, 4, 6, 3};
static const int kLayerWidth[4] = {64, 128, 256, 512};
constexpr int kNumConvs = 36;  // stem + 2 per block (16 blocks) + 3 downsample

int net_create(int c_pad, int out_dim, const void* const* conv_w, const float* const* conv_b,
               int n_convs, const float* head_w, const float* head_b, Net** out) {
  MPX_REQUIRE(c_pad >= 16 && c_pad <= 256 && c_pad % 16 == 0, "net: c_pad=%d must be a multiple of 16 in [16, 256]", c_pad);
  MPX_REQUIRE(n_convs == kNumConvs, "net: expected %d conv tensors, got %d", kNumConvs, n_convs);
  MPX_REQUIRE(out_dim >= 1 && out_dim <= 512, "net: out_dim=%d unsupported", out_dim);
  Net* net = new Net();
  net->c_pad = c_pad;
  net->out_dim = out_dim;
  net->conv_w.assign(conv_w, conv_w + n_convs);
  net->conv_b.assign(conv_b, conv_b + n_convs);
  net->head_w = head_w;
  net->head_b = head_b;
  *out = net;
  return MPX_OK;
}

int net_create_preact(int c_pad, int out_dim, const int* layer_blocks, const void* const* conv_w, const float* const* conv_b,
                      int n_convs, const float* const* block_affine, int n_blocks, const float* head_w, const float* head_b,
                      Net** out) {
  MPX_REQUIRE(c_pad >= 16 && c_pad <= 256 && c_pad % 16 == 0, "net: c_pad=%d must be a multiple of 16 in [16, 256]", c_pad);
  MPX_REQUIRE(out_dim >= 1 && out_dim <= 512, "net: out_dim=%d unsupported", out_dim);
  int blocks = 0;
  for (int l = 0; l < 4; ++l) {
    MPX_REQUIRE(layer_blocks[l] >= 1 && layer_blocks[l] <= 64, "net: layer %d has %d blocks", l + 1, layer_blocks[l]);
    blocks += layer_blocks[l];
  }
  MPX_REQUIRE(n_blocks == blocks && n_convs == 1 + 2 * blocks + 3, "net: expected %d blocks / %d conv tensors, got %d / %d",
              blocks, 1 + 2 * blocks + 3, n_blocks, n_convs);
  Net* net = new Net();
  net->c_pad = c_pad;
  net->out_dim = out_dim;
  net->preact = 1;
  for (int l = 0; l < 4; ++l) net->layer_blocks[l] = layer_blocks[l];
  net->conv_w.assign(conv_w, conv_w + n_convs);
  net->conv_b.assign(conv_b, conv_b + n_convs);
  net->block_affine.assign(block_affine, block_affine + n_blocks);
  net->head_w = head_w;
  net->head_b = head_b;
  *out = net;
  return MPX_OK;
}

void net_destroy(Net* net) {
  if (!net) return;
  for (auto& g : net->graphs)
    if (g.exec) cudaGraphExecDestroy(g.exec);
  if (net->ev_in) cudaEventDestroy(net->ev_in);
  if (net->ev_out) cudaEventDestroy(net->ev_out);
  if (net->side) cudaStreamDestroy(net->side);
  delete net;
}

static size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

size_t net_workspace_bytes(const Net* net, int n, int h, int w) {
  const size_t hs = h / 2, ws = w / 2;
  const size_t stem = align256(static_cast<size_t>(n) * hs * ws * 64 * 2);
  const size_t hp = (hs + 2 - 3) / 2 + 1, wp = (ws + 2 - 3) / 2 + 1;
  const size_t l1 = align256(static_cast<size_t>(n) * hp * wp * 64 * 2);
  return stem + (net != nullptr && net->preact ? 5 : 3) * l1 + 1024;
}

static int net_forward_direct(const Net* net, const void* x, int n, int h, int w, float* out, void* workspace,
                              size_t workspace_bytes, cudaStream_t stream);

int net_forward(const Net* cnet, const void* x, int n, int h, int w, float* out, void* workspace,
                size_t workspace_bytes, cudaStream_t stream) {
  Net* net = const_cast<Net*>(cnet);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(stream, &cap);
  if (!g_use_graphs || conv_profile_enabled() || n == 0 || cap != cudaStreamCaptureStatusNone)
    return net_forward_direct(net, x, n, h, w, out, workspace, workspace_bytes, stream);
  GraphEntry* e = nullptr;
  for (auto& g : net->graphs)
    if (g.x == x && g.out == out && g.ws == workspace && g.n == n && g.h == h && g.w == w) e = &g;
  if (!e) {
    if (net->graphs.size() >= 32) {
      for (auto& g : net->graphs)
        if (g.exec) cudaGraphExecDestroy(g.exec);
      net->graphs.clear();
    }
    net->graphs.push_back(GraphEntry{x, out, workspace, n, h, w, 0, nullptr});
    e = &net->graphs.back();
  }
  if (e->exec == nullptr) {
    if (e->warm == 0) {  // first sight of this shape: run eagerly
      e->warm = 1;
      return net_forward_direct(net, x, n, h, w, out, workspace, workspace_bytes, stream);
    }
    if (!net->side) {
      MPX_CHECK_CUDA(cudaStreamCreateWithFlags(&net->side, cudaStreamNonBlocking));
      MPX_CHECK_CUDA(cudaEventCreateWithFlags(&net->ev_in, cudaEventDisableTiming));
      MPX_CHECK_CUDA(cudaEventCreateWithFlags(&net->ev_out, cudaEventDisableTiming));
    }
    cudaGraph_t graph = nullptr;
    MPX_CHECK_CUDA(cudaStreamBeginCapture(net->side, cudaStreamCaptureModeThreadLocal));
    const long long launches_before = g_launches;
    int rc = net_forward_direct(net, x, n, h, w, out, workspace, workspace_bytes, net->side);
    cudaError_t ce = cudaStreamEndCapture(net->side, &graph);
    e->warm = static_cast<int>(g_launches - launches_before);  // launches per replay
    g_launches = launches_before;
    if (rc != MPX_OK || ce != cudaSuccess || graph == nullptr) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      g_use_graphs = false;  // fall back to eager launches for the rest of the process
      return net_forward_direct(net, x, n, h, w, out, workspace, workspace_bytes, stream);
    }
    ce = cudaGraphInstantiate(&e->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) {
      e->exec = nullptr;
      cudaGetLastError();
      g_use_graphs = false;
      return net_forward_direct(net, x, n, h, w, out, workspace, workspace_bytes, stream);
    }
  }
  MPX_CHECK_CUDA(cudaEventRecord(net->ev_in, stream));
  MPX_CHECK_CUDA(cudaStreamWaitEvent(net->side, net->ev_in, 0));
  MPX_CHECK_CUDA(cudaGraphLaunch(e->exec, net->side));
  MPX_CHECK_CUDA(cudaEventRecord(net->ev_out, net->side));
  MPX_CHECK_CUDA(cudaStreamWaitEvent(stream, net->ev_out, 0));
  g_launches += e->warm;
  return MPX_OK;
}

// Stem convolution + ReLU followed by the 3x3/s2/p1 max-pool.  With mode bit 21 (2097152) the convolution pools in its
// epilogue (max-reductions into the zeroed pooled tensor): the full-resolution stem output -- 2.46 MB per sample at 240x320,
// written once and read once by nothing but the pool -- never exists.  Falls back to the two kernels when the shape is not
// served (the memset is then wasted, nothing else).
static int stem_and_pool(ConvDesc d, const void* x, const void* w, const float* b, void* buf_stem, void* buf_pool,
                         cudaStream_t stream) {
  const int hp = (d.H + 2 - 3) / 2 + 1, wp = (d.W + 2 - 3) / 2 + 1;
  if ((conv_get_mode() & 2097152) != 0 && d.relu) {
    MPX_CHECK_CUDA(cudaMemsetAsync(buf_pool, 0, static_cast<size_t>(d.n_img) * hp * wp * d.C_out * 2, stream));
    d.pool = 1;
    const int rc = conv_forward(d, x, w, b, nullptr, buf_pool, 0, 0, stream);
    if (rc != MPX_ERR_UNSUPPORTED) return rc;
    d.pool = 0;
  }
  const int rc = conv_forward(d, x, w, b, nullptr, buf_stem, 0, 0, stream);
  if (rc != MPX_OK) return rc;
  return maxpool3x3s2(buf_stem, d.n_img, d.H, d.W, d.C_out, buf_pool, stream);
}

// WideResNet (pre-activation) schedule, models/wide_resnet.py:44-58, 106-115: stem 5x5/s2/p2 (a 3x3/s1/p1 convolution over
// the space-to-depth input) + bn1 + relu, max-pool, then per block
//   a = relu(bn1(x)) [affine_relu_kernel];  r = downsample(a) (bare 1x1/s2 convolution) or x;
//   y = relu(bn2(conv1(a))) [bn2 folded into conv1];  x' = conv2(y) + r  [no bias, no ReLU]
// and the spatial mean of the LAST block's raw output into the head (models/pose_rigid.py:323-328).
static int net_forward_preact(const Net* net, const void* x, int n, int h, int w, float* out, void* workspace,
                              cudaStream_t stream) {
  const int hs = h / 2, ws = w / 2;
  const int hp = (hs + 2 - 3) / 2 + 1, wp = (ws + 2 - 3) / 2 + 1;
  uint8_t* base = reinterpret_cast<uint8_t*>(workspace);
  const size_t stem_bytes = align256(static_cast<size_t>(n) * hs * ws * 64 * 2);
  const size_t l1_bytes = align256(static_cast<size_t>(n) * hp * wp * 64 * 2);
  void* buf_stem = base;
  void* bufs[5];
  for (int i = 0; i < 5; ++i) bufs[i] = base + stem_bytes + i * l1_bytes;
  const int sk = ((conv_get_mode() & 8) != 0 && n <= 64) ? -1 : 0;
  int rc;
  {
    ConvDesc d{n, hs, ws, 4 * net->c_pad, 64, 3, 3, 1, 1, 1, 1, 1, 1, 0};
    rc = stem_and_pool(d, x, net->conv_w[0], net->conv_b[0], buf_stem, bufs[0], stream);
    if (rc != MPX_OK) return rc;
  }
  int ci = 1, blk_id = 0;
  int cur = 0;  // buffer holding the block input x
  int H = hp, W = wp, C = 64;
  for (int layer = 0; layer < 4; ++layer) {
    const int width = kLayerWidth[layer];
    for (int blk = 0; blk < net->layer_blocks[layer]; ++blk, ++blk_id) {
      const int stride = (blk == 0 && layer > 0) ? 2 : 1;
      const bool has_ds = (blk == 0 && layer > 0);
      const int ia = (cur + 1) % 5, iy = (cur + 2) % 5, ir = (cur + 3) % 5, io = (cur + 4) % 5;
      const int Ho = conv_out_dim(H, 1, 1, 3, stride), Wo = conv_out_dim(W, 1, 1, 3, stride);
      rc = affine_relu(bufs[cur], static_cast<long long>(n) * H * W * C, C, net->block_affine[blk_id], bufs[ia], stream);
      if (rc != MPX_OK) return rc;
      ConvDesc d1{n, H, W, C, width, 3, 3, stride, 1, 1, 1, 1, 1, 0};
      rc = conv_forward(d1, bufs[ia], net->conv_w[ci], net->conv_b[ci], nullptr, bufs[iy], 0, 0, stream, sk);
      if (rc != MPX_OK) return rc;
      const void* residual = bufs[cur];
      if (has_ds) {
        ConvDesc dd{n, H, W, C, width, 1, 1, stride, 0, 0, 0, 0, 0, 0};
        rc = conv_forward(dd, bufs[ia], net->conv_w[ci + 2], net->conv_b[ci + 2], nullptr, bufs[ir], 0, 0, stream, sk);
        if (rc != MPX_OK) return rc;
        residual = bufs[ir];
      }
      ConvDesc d2{n, Ho, Wo, width, width, 3, 3, 1, 1, 1, 1, 1, 0, 0};
      rc = conv_forward(d2, bufs[iy], net->conv_w[ci + 1], net->conv_b[ci + 1], residual, bufs[io], 0, 0, stream, sk);
      if (rc != MPX_OK) return rc;
      ci += has_ds ? 3 : 2;
      cur = io;
      H = Ho;
      W = Wo;
      C = width;
    }
  }
  return avgpool_linear(bufs[cur], n, H * W, C, net->head_w, net->head_b, net->out_dim, out, stream);
}

// Blocks of layers [layer_from, layer_to) of the post-activation ResNet on `n` images: bufs[cur] holds the input, the
// three buffers rotate as in the reference's BasicBlock (conv1 -> t1; downsample -> t2; conv2 + residual -> out).  Returns the
// buffer holding the result through *result.
struct TrunkState {
  int ci, H, W, C;
};
static int run_layers(const Net* net, int n, int layer_from, int layer_to, void* const bufs[3], int cur, TrunkState& st,
                      int sk, cudaStream_t stream, void** result) {
  int rc;
  void* cur_ptr = bufs[cur];
  for (int layer = layer_from; layer < layer_to; ++layer) {
    const int width = kLayerWidth[layer];
    for (int blk = 0; blk < kLayerBlocks[layer]; ++blk) {
      const int stride = (blk == 0 && layer > 0) ? 2 : 1;
      const bool has_ds = (blk == 0 && layer > 0);
      const int t1 = (cur + 1) % 3, t2 = (cur + 2) % 3;
      const int Ho = conv_out_dim(st.H, 1, 1, 3, stride), Wo = conv_out_dim(st.W, 1, 1, 3, stride);
      // conv1 + bn1 + relu
      ConvDesc d1{n, st.H, st.W, st.C, width, 3, 3, stride, 1, 1, 1, 1, 1};
      rc = conv_forward(d1, bufs[cur], net->conv_w[st.ci], net->conv_b[st.ci], nullptr, bufs[t1], 0, 0, stream, sk);
      if (rc != MPX_OK) return rc;
      ++st.ci;
      const void* residual = bufs[cur];
      int out_buf = t2;
      if (has_ds) {
        // downsample: 1x1/s2 conv + bn (no relu) -> residual; conv_w order: conv1, conv2, downsample
        ConvDesc dd{n, st.H, st.W, st.C, width, 1, 1, stride, 0, 0, 0, 0, 0};
        rc = conv_forward(dd, bufs[cur], net->conv_w[st.ci + 1], net->conv_b[st.ci + 1], nullptr, bufs[t2], 0, 0, stream, sk);
        if (rc != MPX_OK) return rc;
        residual = bufs[t2];
        out_buf = cur;  // block input is dead once conv1 and the downsample have consumed it
      }
      // conv2 + bn2 + residual + relu
      ConvDesc d2{n, Ho, Wo, width, width, 3, 3, 1, 1, 1, 1, 1, 1};
      cur_ptr = bufs[out_buf];
      rc = conv_forward(d2, bufs[t1], net->conv_w[st.ci], net->conv_b[st.ci], residual, cur_ptr, 0, 0, stream, sk);
      if (rc != MPX_OK) return rc;
      st.ci += has_ds ? 2 : 1;
      cur = out_buf;
      st.H = Ho;
      st.W = Wo;
      st.C = width;
    }
  }
  *result = cur_ptr;
  return MPX_OK;
}

static int net_forward_direct(const Net* net, const void* x, int n, int h, int w, float* out, void* workspace,
                              size_t workspace_bytes, cudaStream_t stream) {
  MPX_REQUIRE(h % 2 == 0 && w % 2 == 0, "net: input %dx%d must be even", h, w);
  MPX_REQUIRE(workspace_bytes >= net_workspace_bytes(net, n, h, w), "net: workspace too small");
  MPX_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "net: workspace must be 256-B aligned");
  if (n == 0) return MPX_OK;
  const int hs = h / 2, ws = w / 2;
  const int hp = (hs + 2 - 3) / 2 + 1, wp = (ws + 2 - 3) / 2 + 1;
  uint8_t* base = reinterpret_cast<uint8_t*>(workspace);
  const size_t stem_bytes = align256(static_cast<size_t>(n) * hs * ws * 64 * 2);
  const size_t l1_bytes = align256(static_cast<size_t>(n) * hp * wp * 64 * 2);
  void* buf_stem = base;
  void* bufs[3] = {base + stem_bytes, base + stem_bytes + l1_bytes, base + stem_bytes + 2 * l1_bytes};
  // small batches (refiner iterations, final scoring): layers 2-4 split their K loop over a cluster
  const int sk = ((conv_get_mode() & 8) != 0 && n <= 64) ? -1 : 0;

  if (net->preact) return net_forward_preact(net, x, n, h, w, out, workspace, stream);
  int ci = 0;
  int rc;
  void* res = nullptr;
  // stem: 7x7/s2/p3 conv expressed as 4x4/s1 (pad 2 low, 1 high) over the space-to-depth input
  {
    ConvDesc d{n, hs, ws, 4 * net->c_pad, 64, 4, 4, 1, 2, 2, 1, 1, 1, 1};
    rc = stem_and_pool(d, x, net->conv_w[ci], net->conv_b[ci], buf_stem, bufs[0], stream);
    if (rc != MPX_OK) return rc;
    ++ci;
  }

  TrunkState st{ci, hp, wp, 64};
  rc = run_layers(net, n, 0, 4, bufs, 0, st, sk, stream, &res);
  if (rc != MPX_OK) return rc;
  return avgpool_linear(res, n, st.H * st.W, st.C, net->head_w, net->head_b, net->out_dim, out, stream);
}

}  // namespace mpx
