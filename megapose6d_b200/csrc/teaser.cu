// TEASER++ depth refinement (include/mpx.h: mpx_teaser_*).  One launch per stage for all predictions of a call:
//
//   points  one CTA per prediction: masks, both point clouds, order-preserving compaction (block-wide ballot scan) into the
//           prediction's segment; the count stays on the device.
//   fps     one 8-CTA cluster per prediction: each CTA holds a contiguous slice of the points with their running minima
//           (shared memory, or the workspace when the slice exceeds it); every step is a fused min-update and arg-max,
//           the CTAs' candidates are exchanged through distributed shared memory (double-buffered, one cluster barrier).
//   graph   one thread per (prediction, row, 64-bit word) of the adjacency bitsets, float64 in the oracle's order.
//   clique  one CTA per prediction: core numbers by batch peeling (popc over the bitsets), renumbering by core number
//           into shared memory (k x 16 words, 128 KB for k = 1024), a greedy clique as the lower bound, then one warp runs
//           a bitset branch and bound with a greedy-colouring bound (lane w owns word w) on an explicit stack in the
//           workspace, within a node budget.
//   solve   one CTA per prediction: chain TIMs, GNC-TLS with a float64 Jacobi-SVD Kabsch, per-axis adaptive voting with a
//           bitonic sort of the end points in shared memory, the inlier count and the gated pose update.
#include <cooperative_groups.h>
#include "mpx_common.cuh"
#include "../../include/mpx.h"

namespace cg = cooperative_groups;

namespace mpx {

constexpr int kPtsThreads = 1024;
constexpr int kFpsCluster = 8;
constexpr int kFpsThreads = 512;
constexpr int kFpsSmemPoints = 6144;  // float4 per CTA in shared memory (96 KB: two CTAs per SM)
constexpr int kWords = MPX_TEASER_MAX_POINTS / 64;
constexpr int kCliqueThreads = 512;
constexpr int kSolveThreads = 256;

// ---------------------------------------------------------------------------------------------------------------------
// points and compaction
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kPtsThreads) teaser_points_kernel(
    int hw, int w, const float* __restrict__ rend, const float* __restrict__ meas, const int* __restrict__ view_idx,
    const float* __restrict__ Ks, int mask_type, float thresh, float* __restrict__ src, float* __restrict__ tgt,
    int* __restrict__ count, float* __restrict__ raw_src, float* __restrict__ raw_tgt) {
  const int p = blockIdx.x;
  const float* r_im = rend + static_cast<size_t>(p) * hw;
  const float* m_im = meas + static_cast<size_t>(view_idx[p]) * hw;
  const float* K = Ks + 9 * p;
  const float fx = K[0], cx = K[2], fy = K[4], cy = K[5];
  float* s_out = src + static_cast<size_t>(p) * hw * 3;
  float* t_out = tgt + static_cast<size_t>(p) * hw * 3;
  __shared__ int warp_off[kPtsThreads / 32];
  __shared__ int base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int px0 = 0; px0 < hw; px0 += kPtsThreads) {
    const int px = px0 + threadIdx.x;
    bool keep = false;
    float sx = 0.f, sy = 0.f, sz = 0.f, tx = 0.f, ty = 0.f, tz = 0.f;
    if (px < hw) {
      const int v = px / w, u = px - v * w;
      sz = r_im[px];
      tz = m_im[px];
      keep = tz > 0.f && sz > 0.f;
      if (mask_type == MPX_TEASER_MASK_THRESHOLD) keep = keep && !(fabsf(__fsub_rn(tz, sz)) > thresh);
      const double du = __dadd_rn(static_cast<double>(u), -static_cast<double>(cx));
      const double dv = __dadd_rn(static_cast<double>(v), -static_cast<double>(cy));
      sx = __double2float_rn(__dmul_rn(du, static_cast<double>(__fdiv_rn(sz, fx))));
      sy = __double2float_rn(__dmul_rn(dv, static_cast<double>(__fdiv_rn(sz, fy))));
      tx = __double2float_rn(__dmul_rn(du, static_cast<double>(__fdiv_rn(tz, fx))));
      ty = __double2float_rn(__dmul_rn(dv, static_cast<double>(__fdiv_rn(tz, fy))));
      if (raw_src) {
        float* rs = raw_src + (static_cast<size_t>(p) * hw + px) * 3;
        float* rt = raw_tgt + (static_cast<size_t>(p) * hw + px) * 3;
        rs[0] = sx, rs[1] = sy, rs[2] = sz;
        rt[0] = tx, rt[1] = ty, rt[2] = tz;
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_off[warp] = __popc(bal);
    __syncthreads();
    if (warp == 0) {  // exclusive scan of the warp counts
      const int c = warp_off[lane];
      int incl = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      warp_off[lane] = incl - c;
    }
    __syncthreads();
    if (keep) {
      const size_t i = static_cast<size_t>(base + warp_off[warp] + __popc(bal & ((1u << lane) - 1u)));
      s_out[3 * i] = sx, s_out[3 * i + 1] = sy, s_out[3 * i + 2] = sz;
      t_out[3 * i] = tx, t_out[3 * i + 1] = ty, t_out[3 * i + 2] = tz;
    }
    __syncthreads();
    if (threadIdx.x == kPtsThreads - 1) base += warp_off[warp] + __popc(bal);
    __syncthreads();
  }
  if (threadIdx.x == 0) count[p] = base;
}

int teaser_points(int n_pred, int h, int w, const float* rend, const float* meas, const int* view_idx, const float* K,
                  int mask_type, float thresh, float* src, float* tgt, int* count, float* raw_src, float* raw_tgt,
                  cudaStream_t stream) {
  if (n_pred == 0) return MPX_OK;
  teaser_points_kernel<<<n_pred, kPtsThreads, 0, stream>>>(h * w, w, rend, meas, view_idx, K, mask_type, thresh, src, tgt,
                                                          count, raw_src, raw_tgt);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// farthest-point sampling
// ---------------------------------------------------------------------------------------------------------------------
struct ArgMax {
  float v;
  int i;
};
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }
__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (better(ov, oi, v, i)) v = ov, i = oi;
  }
}

__global__ void __launch_bounds__(kFpsThreads) teaser_fps_kernel(int cap, const float* __restrict__ src,
                                                                 const float* __restrict__ tgt,
                                                                 const int* __restrict__ count, int k,
                                                                 int* __restrict__ idx_out, float* __restrict__ samp_src,
                                                                 float* __restrict__ samp_tgt, float4* __restrict__ ws) {
  extern __shared__ float4 spts[];
  __shared__ ArgMax slot[2];
  __shared__ ArgMax wbest[kFpsThreads / 32];
  __shared__ int s_sel;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = static_cast<int>(cluster.block_rank());
  const int p = blockIdx.x / kFpsCluster;
  const int n = min(count[p], cap);
  const float* P = src + static_cast<size_t>(p) * cap * 3;
  const int chunk = (n + kFpsCluster - 1) / kFpsCluster;
  const int lo = min(n, rank * chunk), hi = min(n, lo + chunk), len = hi - lo;
  float4* pts = len <= kFpsSmemPoints ? spts : ws + static_cast<size_t>(p) * cap + lo;
  const float inf = __int_as_float(0x7f800000);
  for (int i = threadIdx.x; i < len; i += kFpsThreads)
    pts[i] = make_float4(P[3 * (lo + i)], P[3 * (lo + i) + 1], P[3 * (lo + i) + 2], inf);
  int* idx = idx_out + static_cast<size_t>(p) * k;
  int sel = 0;
  const int steps = min(n, k);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  for (int step = 1; step < steps; ++step) {
    const float qx = P[3 * sel], qy = P[3 * sel + 1], qz = P[3 * sel + 2];
    float bv = -inf;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < len; i += kFpsThreads) {
      float4 q = pts[i];
      const float dx = __fsub_rn(q.x, qx), dy = __fsub_rn(q.y, qy), dz = __fsub_rn(q.z, qz);
      const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      q.w = fminf(q.w, d);
      pts[i].w = q.w;
      if (q.w > bv) bv = q.w, bi = lo + i;  // increasing i: the first maximum of this thread is kept
    }
    warp_argmax(bv, bi);
    if (lane == 0) wbest[warp] = ArgMax{bv, bi};
    __syncthreads();
    if (warp == 0) {
      bv = lane < kFpsThreads / 32 ? wbest[lane].v : -inf;
      bi = lane < kFpsThreads / 32 ? wbest[lane].i : 0x7fffffff;
      warp_argmax(bv, bi);
      if (lane == 0) slot[step & 1] = ArgMax{bv, bi};
    }
    cluster.sync();
    if (warp == 0) {
      bv = -inf;
      bi = 0x7fffffff;
      if (lane < kFpsCluster) {
        const ArgMax* r = cluster.map_shared_rank(&slot[step & 1], lane);
        bv = r->v;
        bi = r->i;
      }
      warp_argmax(bv, bi);
      if (lane == 0) s_sel = bi;
    }
    __syncthreads();
    sel = s_sel;
    if (rank == 0 && threadIdx.x == 0) idx[step] = sel;
  }
  cluster.sync();  // no CTA leaves while another may still read its slot
  if (rank == 0) {
    for (int j = threadIdx.x; j < k; j += kFpsThreads) {
      const int i = n == 0 ? -1 : (j == 0 ? 0 : (j < steps ? idx[j] : n - 1));
      // idx[j] for 0 < j < steps was written by this thread's CTA before the barriers above
      if (j == 0 || j >= steps) idx[j] = i;
      float* ss = samp_src + (static_cast<size_t>(p) * k + j) * 3;
      float* st = samp_tgt + (static_cast<size_t>(p) * k + j) * 3;
      const float* T = tgt + static_cast<size_t>(p) * cap * 3;
      for (int c = 0; c < 3; ++c) {
        ss[c] = i < 0 ? 0.f : P[3 * i + c];
        st[c] = i < 0 ? 0.f : T[3 * i + c];
      }
    }
  }
}

size_t teaser_fps_workspace_bytes(int n_pred, int cap) { return sizeof(float4) * static_cast<size_t>(n_pred) * cap; }

int teaser_fps(int n_pred, int cap, const float* src, const float* tgt, const int* count, int k, int* idx,
               float* samp_src, float* samp_tgt, void* ws, cudaStream_t stream) {
  if (n_pred == 0) return MPX_OK;
  const size_t smem = sizeof(float4) * kFpsSmemPoints;
  MPX_CHECK_CUDA(cudaFuncSetAttribute(teaser_fps_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(n_pred * kFpsCluster);
  cfg.blockDim = dim3(kFpsThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kFpsCluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  MPX_CHECK_CUDA(cudaLaunchKernelEx(&cfg, teaser_fps_kernel, cap, src, tgt, count, k, idx, samp_src, samp_tgt,
                                    static_cast<float4*>(ws)));
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// consistency graph
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double norm3_rn(double x, double y, double z) {
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}

__global__ void teaser_graph_kernel(int k, const float* __restrict__ ss, const float* __restrict__ st,
                                    const int* __restrict__ m_all, double bound, unsigned long long* __restrict__ adj) {
  const int p = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = t / kWords, wd = t - i * kWords;
  if (i >= k) return;
  const int m = max(0, min(m_all[p], k));  // the ABI documents 0..k; anything else is clamped
  const float* S = ss + static_cast<size_t>(p) * k * 3;
  const float* T = st + static_cast<size_t>(p) * k * 3;
  unsigned long long bits = 0;
  if (i < m) {
    const double sx = S[3 * i], sy = S[3 * i + 1], sz = S[3 * i + 2];
    const double tx = T[3 * i], ty = T[3 * i + 1], tz = T[3 * i + 2];
    const int j1 = min(m, 64 * wd + 64);
    for (int j = 64 * wd; j < j1; ++j) {
      if (j == i) continue;
      // a = s_j - s_i, b = t_j - t_i; pair (j, i) gives the negated vectors and the same norms, so the graph is symmetric
      const double ax = __dadd_rn(static_cast<double>(S[3 * j]), -sx);
      const double ay = __dadd_rn(static_cast<double>(S[3 * j + 1]), -sy);
      const double az = __dadd_rn(static_cast<double>(S[3 * j + 2]), -sz);
      const double bx = __dadd_rn(static_cast<double>(T[3 * j]), -tx);
      const double by = __dadd_rn(static_cast<double>(T[3 * j + 1]), -ty);
      const double bz = __dadd_rn(static_cast<double>(T[3 * j + 2]), -tz);
      if (fabs(__dadd_rn(norm3_rn(bx, by, bz), -norm3_rn(ax, ay, az))) <= bound) bits |= 1ull << (j - 64 * wd);
    }
  }
  adj[(static_cast<size_t>(p) * k + i) * kWords + wd] = bits;
}

int teaser_graph(int n_pred, int k, const float* ss, const float* st, const int* m, double bound,
                 unsigned long long* adj, cudaStream_t stream) {
  if (n_pred == 0) return MPX_OK;
  const int threads = 256;
  teaser_graph_kernel<<<dim3((k * kWords + threads - 1) / threads, n_pred), threads, 0, stream>>>(k, ss, st, m, bound, adj);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// maximum clique
// ---------------------------------------------------------------------------------------------------------------------
// per-prediction workspace: P bitsets of every search level, then the colour-ordered candidate lists (v | colour << 16)
__host__ __device__ inline size_t clique_ws_words(int k) {
  const size_t kk = static_cast<size_t>(k) + 1;
  return kk * kWords + (kk * (kk + 1) / 2 + 1) / 2;  // uint64 words: level bitsets + uint32 list pool
}

__global__ void __launch_bounds__(kCliqueThreads) teaser_clique_kernel(
    int k, const unsigned long long* __restrict__ adj_all, const int* __restrict__ m_all, long long budget,
    int* __restrict__ clique_out, int* __restrict__ size_out, int* __restrict__ status_out, long long* __restrict__ nodes_out,
    unsigned long long* __restrict__ ws_all) {
  extern __shared__ unsigned long long sadj[];  // [k][kWords], renumbered
  __shared__ int deg[MPX_TEASER_MAX_POINTS], core[MPX_TEASER_MAX_POINTS], perm[MPX_TEASER_MAX_POINTS];
  __shared__ int best_r[MPX_TEASER_MAX_POINTS], cur_r[MPX_TEASER_MAX_POINTS];
  __shared__ int lvl_base[MPX_TEASER_MAX_POINTS + 1], lvl_len[MPX_TEASER_MAX_POINTS + 1];
  __shared__ unsigned long long rem[kWords];
  __shared__ unsigned peel[MPX_TEASER_MAX_POINTS / 32];
  __shared__ int s_k, s_min;
  const int p = blockIdx.x;
  const int m = max(0, min(m_all[p], k));  // the ABI documents 0..k; anything else is clamped
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned long long* A = adj_all + static_cast<size_t>(p) * k * kWords;
  int* cl = clique_out + static_cast<size_t>(p) * k;
  for (int i = tid; i < k; i += kCliqueThreads) cl[i] = -1;
  if (m <= 1) {
    if (tid == 0) {
      if (m == 1) cl[0] = 0;
      size_out[p] = m > 0 ? m : 0;
      status_out[p] = 0;
      if (nodes_out) nodes_out[p] = 0;
    }
    return;
  }
  const int W = (m + 63) / 64;
  // ---- core numbers: peel every remaining vertex of degree <= kc at once
  if (tid < kWords) rem[tid] = tid < W ? (tid == W - 1 && (m & 63) ? (1ull << (m & 63)) - 1 : ~0ull) : 0ull;
  for (int v = tid; v < m; v += kCliqueThreads) {
    int d = 0;
    for (int x = 0; x < W; ++x) d += __popcll(A[v * kWords + x]);
    deg[v] = d;
  }
  if (tid == 0) s_k = 0;
  __syncthreads();
  while (true) {
    int any_left = 0, any_peel = 0;
    for (int v0 = 0; v0 < MPX_TEASER_MAX_POINTS; v0 += kCliqueThreads) {
      const int v = v0 + tid;
      const bool in = v < m && ((rem[v >> 6] >> (v & 63)) & 1ull);
      const bool pl = in && deg[v] <= s_k;
      const unsigned b = __ballot_sync(0xffffffffu, pl);
      if (lane == 0) peel[v >> 5] = b;
      if (pl) core[v] = s_k;
      any_left |= in;
      any_peel |= pl;
    }
    any_left = __syncthreads_or(any_left);
    if (!any_left) break;
    any_peel = __syncthreads_or(any_peel);
    if (!any_peel) {
      if (tid == 0) s_min = 0x7fffffff;
      __syncthreads();
      for (int v = tid; v < m; v += kCliqueThreads)
        if ((rem[v >> 6] >> (v & 63)) & 1ull) atomicMin(&s_min, deg[v]);
      __syncthreads();
      if (tid == 0) s_k = s_min;
      __syncthreads();
      continue;
    }
    if (tid < kWords) rem[tid] &= ~(static_cast<unsigned long long>(peel[2 * tid]) |
                                    (static_cast<unsigned long long>(peel[2 * tid + 1]) << 32));
    __syncthreads();
    for (int v = tid; v < m; v += kCliqueThreads) {
      if (!((rem[v >> 6] >> (v & 63)) & 1ull)) continue;
      int d = 0;
      for (int x = 0; x < W; ++x) d += __popcll(A[v * kWords + x] & rem[x]);
      deg[v] = d;
    }
    __syncthreads();
  }
  // ---- renumber: new index = rank by (core descending, index ascending)
  for (int v = tid; v < m; v += kCliqueThreads) {
    int r = 0;
    const int cv = core[v];
    for (int u = 0; u < m; ++u) r += core[u] > cv || (core[u] == cv && u < v);
    perm[r] = v;
  }
  __syncthreads();
  for (int t = tid; t < m * kWords; t += kCliqueThreads) {
    const int i = t / kWords, x = t - i * kWords;
    unsigned long long bits = 0;
    if (x < W) {
      const unsigned long long* row = A + static_cast<size_t>(perm[i]) * kWords;
      const int j1 = min(m, 64 * x + 64);
      for (int j = 64 * x; j < j1; ++j) {
        const int o = perm[j];
        bits |= ((row[o >> 6] >> (o & 63)) & 1ull) << (j - 64 * x);
      }
    }
    sadj[t] = bits;
  }
  __syncthreads();
  if (warp != 0) return;

  // ---- one warp: lane x < kWords owns word x of every bitset
  const bool own = lane < W;
  unsigned long long* ws = ws_all + static_cast<size_t>(p) * clique_ws_words(k);
  unsigned long long* Pst = ws;                                                  // [(k + 1)][kWords]
  unsigned* pool = reinterpret_cast<unsigned*>(ws + (static_cast<size_t>(k) + 1) * kWords);
  // greedy clique in core order
  int best = 0;
  {
    unsigned long long cand = own ? (lane == W - 1 && (m & 63) ? (1ull << (m & 63)) - 1 : ~0ull) : 0ull;
    while (true) {
      const unsigned bal = __ballot_sync(0xffffffffu, cand != 0ull);
      if (!bal) break;
      const int f = __ffs(bal) - 1;
      const unsigned long long q = __shfl_sync(0xffffffffu, cand, f);
      const int v = 64 * f + __ffsll(static_cast<long long>(q)) - 1;
      if (lane == 0) best_r[best] = v;
      ++best;
      cand &= own ? sadj[v * kWords + lane] : 0ull;
    }
  }
  // candidates: vertices whose core number reaches the lower bound
  unsigned long long P0 = 0ull;
  if (own) {
    for (int b = 0; b < 64; ++b) {
      const int v = 64 * lane + b;
      if (v < m && core[perm[v]] >= best) P0 |= 1ull << b;
    }
  }
  // greedy colouring of P; appends (v, colour) with colour >= kmin to pool[base...], returns the count
  auto colour = [&](unsigned long long U, int kmin, size_t base) -> int {
    int len = 0, col = 0;
    while (__ballot_sync(0xffffffffu, U != 0ull)) {
      ++col;
      unsigned long long Q = U;
      while (true) {
        const unsigned bal = __ballot_sync(0xffffffffu, Q != 0ull);
        if (!bal) break;
        const int f = __ffs(bal) - 1;
        const unsigned long long q = __shfl_sync(0xffffffffu, Q, f);
        const int b = __ffsll(static_cast<long long>(q)) - 1;
        const int v = 64 * f + b;
        if (own) Q &= ~sadj[v * kWords + lane];
        if (lane == f) {
          Q &= ~(1ull << b);
          U &= ~(1ull << b);
        }
        if (col >= kmin) {
          if (lane == 0) pool[base + len] = static_cast<unsigned>(v) | (static_cast<unsigned>(col) << 16);
          ++len;
        }
      }
    }
    return len;
  };
  long long nodes = 1;
  int exhausted = 0;
  int depth = 0;
  if (lane < kWords) Pst[lane] = P0;
  lvl_base[0] = 0;
  const int l0 = colour(P0, best + 1, 0);
  if (lane == 0) lvl_len[0] = l0;
  __syncwarp();
  while (depth >= 0) {
    const int len = lvl_len[depth];
    if (len == 0) {
      --depth;
      continue;
    }
    const unsigned e = pool[lvl_base[depth] + len - 1];
    const int v = static_cast<int>(e & 0xffffu), col = static_cast<int>(e >> 16);
    if (depth + col <= best) {
      --depth;
      continue;
    }
    const unsigned long long Pw = lane < kWords ? Pst[static_cast<size_t>(depth) * kWords + lane] : 0ull;
    const unsigned long long newP = own ? (Pw & sadj[v * kWords + lane]) : 0ull;
    __syncwarp();
    if (lane < kWords) Pst[static_cast<size_t>(depth) * kWords + lane] = (lane == (v >> 6)) ? (Pw & ~(1ull << (v & 63))) : Pw;
    if (lane == 0) {
      lvl_len[depth] = len - 1;
      cur_r[depth] = v;
    }
    __syncwarp();
    if (!__ballot_sync(0xffffffffu, newP != 0ull)) {
      if (depth + 1 > best) {
        best = depth + 1;
        for (int i = lane; i < best; i += 32) best_r[i] = cur_r[i];
        __syncwarp();
      }
      continue;
    }
    if (nodes >= budget) {
      exhausted = 1;
      break;
    }
    ++nodes;
    const size_t nb = static_cast<size_t>(lvl_base[depth]) + len;
    const int nl = colour(newP, best - depth, nb);
    if (nl > 0) {
      if (lane < kWords) Pst[static_cast<size_t>(depth + 1) * kWords + lane] = newP;
      if (lane == 0) {
        lvl_base[depth + 1] = static_cast<int>(nb);
        lvl_len[depth + 1] = nl;
      }
      ++depth;
    }
    __syncwarp();
  }
  // ---- the clique in the original numbering, ascending
  unsigned long long mark = 0ull;
  for (int i = 0; i < best; ++i) {
    const int o = perm[best_r[i]];
    if (lane == (o >> 6)) mark |= 1ull << (o & 63);
  }
  int off = 0;
  for (int x = 0; x < kWords; ++x) {
    const unsigned long long wv = __shfl_sync(0xffffffffu, mark, x);
    for (int b = lane; b < 64; b += 32) {
      if ((wv >> b) & 1ull) cl[off + __popcll(wv & ((1ull << b) - 1ull))] = 64 * x + b;
    }
    off += __popcll(wv);
  }
  if (lane == 0) {
    size_out[p] = best;
    status_out[p] = exhausted;
    if (nodes_out) nodes_out[p] = nodes;
  }
}

size_t teaser_clique_workspace_bytes(int n_pred, int k) { return 8 * clique_ws_words(k) * static_cast<size_t>(n_pred); }

int teaser_max_clique(int n_pred, int k, const unsigned long long* adj, const int* m, long long budget, int* clique,
                      int* size, int* status, long long* nodes, void* ws, cudaStream_t stream) {
  if (n_pred == 0) return MPX_OK;
  const size_t smem = sizeof(unsigned long long) * static_cast<size_t>(k) * kWords;
  MPX_CHECK_CUDA(cudaFuncSetAttribute(teaser_clique_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  teaser_clique_kernel<<<n_pred, kCliqueThreads, smem, stream>>>(k, adj, m, budget, clique, size, status, nodes,
                                                                 static_cast<unsigned long long*>(ws));
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// solve
// ---------------------------------------------------------------------------------------------------------------------
__device__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double r = red[0];
  for (int i = 1; i < kSolveThreads / 32; ++i) r += red[i];
  return r;
}
__device__ double block_max(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double r = red[0];
  for (int i = 1; i < kSolveThreads / 32; ++i) r = fmax(r, red[i]);
  return r;
}

// R = V diag(1, 1, det(V U^T)) U^T for H = U S V^T (row-major 3x3), by one-sided Jacobi on the columns of H
__device__ void kabsch_from_H(const double* H, double* R) {
  double B[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 9; ++i) B[i] = H[i];
  for (int sweep = 0; sweep < 40; ++sweep) {
    bool rotated = false;
    for (int pi = 0; pi < 3; ++pi) {
      const int a = pi == 2 ? 1 : 0, b = pi == 0 ? 1 : 2;
      double al = 0, be = 0, ga = 0;
      for (int r = 0; r < 3; ++r) {
        al += B[3 * r + a] * B[3 * r + a];
        be += B[3 * r + b] * B[3 * r + b];
        ga += B[3 * r + a] * B[3 * r + b];
      }
      if (ga == 0.0 || fabs(ga) <= 1e-15 * sqrt(al * be)) continue;
      rotated = true;
      const double zeta = (be - al) / (2.0 * ga);
      const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
      for (int r = 0; r < 3; ++r) {
        const double x = B[3 * r + a], y = B[3 * r + b];
        B[3 * r + a] = c * x - s * y;
        B[3 * r + b] = s * x + c * y;
        const double vx = V[3 * r + a], vy = V[3 * r + b];
        V[3 * r + a] = c * vx - s * vy;
        V[3 * r + b] = s * vx + c * vy;
      }
    }
    if (!rotated) break;
  }
  double sg[3];
  int ord[3] = {0, 1, 2};
  for (int c = 0; c < 3; ++c) sg[c] = sqrt(B[c] * B[c] + B[3 + c] * B[3 + c] + B[6 + c] * B[6 + c]);
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2 - i; ++j)
      if (sg[ord[j]] < sg[ord[j + 1]]) {
        const int t = ord[j];
        ord[j] = ord[j + 1];
        ord[j + 1] = t;
      }
  double U[3][3], Vs[3][3];  // columns, sorted by singular value
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) Vs[c][r] = V[3 * r + ord[c]];
  const double s0 = sg[ord[0]] > 0 ? sg[ord[0]] : 1.0;
  for (int r = 0; r < 3; ++r) U[0][r] = sg[ord[0]] > 0 ? B[3 * r + ord[0]] / s0 : (r == 0 ? 1.0 : 0.0);
  double u1[3];
  for (int r = 0; r < 3; ++r) u1[r] = B[3 * r + ord[1]];
  double d = u1[0] * U[0][0] + u1[1] * U[0][1] + u1[2] * U[0][2];
  for (int r = 0; r < 3; ++r) u1[r] -= d * U[0][r];
  double nu = sqrt(u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2]);
  if (!(nu > 1e-300)) {  // rank 1: any unit vector orthogonal to U0
    const int ax = fabs(U[0][0]) < 0.9 ? 0 : 1;
    double e[3] = {0, 0, 0};
    e[ax] = 1.0;
    d = U[0][ax];
    for (int r = 0; r < 3; ++r) u1[r] = e[r] - d * U[0][r];
    nu = sqrt(u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2]);
  }
  for (int r = 0; r < 3; ++r) U[1][r] = u1[r] / nu;
  U[2][0] = U[0][1] * U[1][2] - U[0][2] * U[1][1];  // proper U: det(U) = 1
  U[2][1] = U[0][2] * U[1][0] - U[0][0] * U[1][2];
  U[2][2] = U[0][0] * U[1][1] - U[0][1] * U[1][0];
  const double detV = Vs[0][0] * (Vs[1][1] * Vs[2][2] - Vs[1][2] * Vs[2][1]) -
                      Vs[1][0] * (Vs[0][1] * Vs[2][2] - Vs[0][2] * Vs[2][1]) +
                      Vs[2][0] * (Vs[0][1] * Vs[1][2] - Vs[0][2] * Vs[1][1]);
  const double dd = detV < 0 ? -1.0 : 1.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      R[3 * i + j] = Vs[0][i] * U[0][j] + Vs[1][i] * U[1][j] + dd * Vs[2][i] * U[2][j];
}

struct Ev {
  double x;
  int key;  // (leaving << 11) | index; +inf padding sorts last
};
__device__ __forceinline__ bool ev_less(const Ev& a, const Ev& b) {
  return a.x < b.x || (a.x == b.x && a.key < b.key);
}

__global__ void __launch_bounds__(kSolveThreads) teaser_solve_kernel(
    int k, const float* __restrict__ ss, const float* __restrict__ st, const int* __restrict__ m_all,
    const int* __restrict__ clique_all, const int* __restrict__ csize, double noise_bound, double gnc_factor, int max_it,
    double cost_thr, int min_inliers, float* __restrict__ poses, float* __restrict__ poses_input, double* __restrict__ T_out,
    int* __restrict__ n_in_out, int* __restrict__ flags_out) {
  extern __shared__ double dsm[];  // a [k][3], b [k][3], wgt [k], r2 [k], then the end points [2k]
  double(*a)[3] = reinterpret_cast<double(*)[3]>(dsm);
  double(*b)[3] = reinterpret_cast<double(*)[3]>(dsm + 3 * k);
  double* wgt = dsm + 6 * k;
  double* r2 = dsm + 7 * k;
  Ev* ev = reinterpret_cast<Ev*>(dsm + 8 * k);
  __shared__ double red[kSolveThreads / 32];
  __shared__ double Rs[9], ts[3];
  const int p = blockIdx.x, tid = threadIdx.x;
  const int m = max(0, min(m_all[p], k)), mc = min(csize[p], m);
  const int* c = clique_all + static_cast<size_t>(p) * k;
  const float* S = ss + static_cast<size_t>(p) * k * 3;
  const float* Tg = st + static_cast<size_t>(p) * k * 3;
  double* Tp = T_out + 16 * p;
  if (mc <= 1) {
    if (tid < 16) Tp[tid] = (tid % 5 == 0) ? 1.0 : 0.0;
    if (tid == 0) {
      n_in_out[p] = 0;
      flags_out[p] = 0;
    }
    return;
  }
  for (int i = tid; i < mc; i += kSolveThreads) {
    const int i0 = c[i], i1 = c[i + 1 < mc ? i + 1 : 0];
    for (int d = 0; d < 3; ++d) {
      a[i][d] = __dadd_rn(static_cast<double>(S[3 * i1 + d]), -static_cast<double>(S[3 * i0 + d]));
      b[i][d] = __dadd_rn(static_cast<double>(Tg[3 * i1 + d]), -static_cast<double>(Tg[3 * i0 + d]));
    }
    wgt[i] = 1.0;
  }
  __syncthreads();
  // ---- rotation: GNC-TLS
  const double nb = 2.0 * noise_bound, nb2 = nb * nb;
  double mu = 1.0, prev_cost = 0.0;
  for (int it = 0; it < max_it; ++it) {
    double h[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = tid; i < mc; i += kSolveThreads)
      for (int r = 0; r < 3; ++r)
        for (int q = 0; q < 3; ++q) h[3 * r + q] += wgt[i] * a[i][r] * b[i][q];
    double H[9];
    for (int e = 0; e < 9; ++e) H[e] = block_sum(h[e], red);
    if (tid == 0) kabsch_from_H(H, Rs);
    __syncthreads();
    double mx = 0.0;
    for (int i = tid; i < mc; i += kSolveThreads) {
      double d2 = 0.0;
      for (int r = 0; r < 3; ++r) {
        const double e = b[i][r] - (Rs[3 * r] * a[i][0] + Rs[3 * r + 1] * a[i][1] + Rs[3 * r + 2] * a[i][2]);
        d2 += e * e;
      }
      r2[i] = d2;
      mx = fmax(mx, d2);
    }
    if (it == 0) {
      mu = 1.0 / (2.0 * block_max(mx, red) / nb2 - 1.0);
      if (mu <= 0) break;
    }
    const double th1 = (mu + 1.0) / mu * nb2, th2 = mu / (mu + 1.0) * nb2;
    double cs = 0.0;
    __syncthreads();
    for (int i = tid; i < mc; i += kSolveThreads) {
      cs += wgt[i] * r2[i];
      const double q = r2[i];
      wgt[i] = q > th1 ? 0.0 : (q < th2 ? 1.0 : sqrt(nb2 * mu * (mu + 1.0) / q) - mu);
    }
    const double cost = block_sum(cs, red);
    mu *= gnc_factor;
    if (fabs(cost - prev_cost) < cost_thr) break;
    prev_cost = cost;
  }
  __syncthreads();
  double R[9];
  for (int e = 0; e < 9; ++e) R[e] = Rs[e];
  // ---- translation: adaptive voting per axis on t_c - R s_c
  int n_ev = 1;
  while (n_ev < 2 * mc) n_ev <<= 1;
  const double b2 = noise_bound * noise_bound;
  for (int ax = 0; ax < 3; ++ax) {
    for (int e = tid; e < n_ev; e += kSolveThreads) {
      if (e < 2 * mc) {
        const int i = e >> 1, leave = e & 1, ci = c[i];
        const double x = static_cast<double>(Tg[3 * ci + ax]) -
                         (R[3 * ax] * S[3 * ci] + R[3 * ax + 1] * S[3 * ci + 1] + R[3 * ax + 2] * S[3 * ci + 2]);
        if (!leave) r2[i] = x;  // the axis' values (the residuals are no longer needed)
        ev[e] = Ev{leave ? __dadd_rn(x, noise_bound) : __dadd_rn(x, -noise_bound), (leave << 11) | i};
      } else {
        ev[e] = Ev{__longlong_as_double(0x7ff0000000000000ll), 0x7fffffff};
      }
    }
    __syncthreads();
    for (int sz = 2; sz <= n_ev; sz <<= 1) {
      for (int st2 = sz >> 1; st2 > 0; st2 >>= 1) {
        for (int e = tid; e < n_ev; e += kSolveThreads) {
          const int o = e ^ st2;
          if (o > e) {
            const bool up = (e & sz) == 0;
            if (ev_less(ev[o], ev[e]) == up) {
              const Ev t = ev[e];
              ev[e] = ev[o];
              ev[o] = t;
            }
          }
        }
        __syncthreads();
      }
    }
    if (tid == 0) {
      double sx = 0.0, sx2 = 0.0, bestv = 0.0, best_cost = __longlong_as_double(0x7ff0000000000000ll);
      int n = 0;
      for (int e = 0; e < 2 * mc; ++e) {
        const int key = ev[e].key, i = key & 2047;
        const double x = r2[i];
        if (key >> 11) {
          sx = __dadd_rn(sx, -x);
          sx2 = __dadd_rn(sx2, -__dmul_rn(x, x));
          --n;
        } else {
          sx = __dadd_rn(sx, x);
          sx2 = __dadd_rn(sx2, __dmul_rn(x, x));
          ++n;
        }
        if (n > 0) {
          const double est = __ddiv_rn(sx, static_cast<double>(n));
          const double cost = __dadd_rn(__dadd_rn(sx2, -__dmul_rn(sx, est)), __dmul_rn(static_cast<double>(mc - n), b2));
          if (cost < best_cost) best_cost = cost, bestv = est;
        }
      }
      ts[ax] = bestv;
    }
    __syncthreads();
  }
  const double t0 = ts[0], t1 = ts[1], t2 = ts[2];
  // ---- inliers among all samples
  double cnt = 0.0;
  for (int i = tid; i < m; i += kSolveThreads) {
    const double sx = S[3 * i], sy = S[3 * i + 1], sz = S[3 * i + 2];
    const double dx = (R[0] * sx + R[1] * sy + R[2] * sz) + t0 - static_cast<double>(Tg[3 * i]);
    const double dy = (R[3] * sx + R[4] * sy + R[5] * sz) + t1 - static_cast<double>(Tg[3 * i + 1]);
    const double dz = (R[6] * sx + R[7] * sy + R[8] * sz) + t2 - static_cast<double>(Tg[3 * i + 2]);
    cnt += sqrt(dx * dx + dy * dy + dz * dz) < noise_bound ? 1.0 : 0.0;
  }
  const int n_in = static_cast<int>(block_sum(cnt, red));
  if (tid == 0) {
    const double T[16] = {R[0], R[1], R[2], t0, R[3], R[4], R[5], t1, R[6], R[7], R[8], t2, 0, 0, 0, 1};
    for (int e = 0; e < 16; ++e) Tp[e] = T[e];
    const bool acc = n_in >= min_inliers;
    n_in_out[p] = n_in;
    flags_out[p] = 1 | (acc ? 2 : 0);
    if (acc) {
      float* P = poses + 16 * p;
      double in[16];
      for (int e = 0; e < 16; ++e) {
        in[e] = static_cast<double>(P[e]);
        poses_input[16 * p + e] = P[e];
      }
      for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
          P[4 * i + j] = static_cast<float>(T[4 * i] * in[j] + T[4 * i + 1] * in[4 + j] + T[4 * i + 2] * in[8 + j] +
                                            T[4 * i + 3] * in[12 + j]);
    }
  }
}

int teaser_solve(int n_pred, int k, const float* ss, const float* st, const int* m, const int* clique, const int* csize,
                 double noise_bound, double gnc_factor, int max_it, double cost_thr, int min_inliers, float* poses,
                 float* poses_input, double* T, int* n_in, int* flags, cudaStream_t stream) {
  if (n_pred == 0) return MPX_OK;
  int n_ev = 1;
  while (n_ev < 2 * k) n_ev <<= 1;
  const size_t smem = sizeof(double) * 8 * k + sizeof(Ev) * n_ev;
  MPX_CHECK_CUDA(cudaFuncSetAttribute(teaser_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  teaser_solve_kernel<<<n_pred, kSolveThreads, smem, stream>>>(k, ss, st, m, clique, csize, noise_bound, gnc_factor, max_it,
                                                            cost_thr, min_inliers, poses, poses_input, T, n_in, flags);
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  return MPX_OK;
}

}  // namespace mpx
