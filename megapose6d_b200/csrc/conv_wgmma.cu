// Implicit-GEMM convolution for sm_90a: TMA im2col (activations) + TMA tiled (weights) -> 128B-swizzled shared memory ->
// wgmma (act16 x act16 -> fp32 register accumulators) -> fused epilogue (folded-BN bias, residual add, ReLU, optionally the
// stem's 3x3/s2 max-pool) -> act16 NHWC.
//
// Replaces the cuDNN convolutions issued by every nn.Conv2d + BatchNorm2d + ReLU (+ residual) of the
// reference backbone (reference: src/megapose/models/torchvision_resnet.py:74-120 BasicBlock.forward,
// :298-311 ResNet._forward_impl).
//
// GEMM view:  D[M, N] = A[M, K] * B[N, K]^T
//   M = n_img * P * Q output pixels (flattened NHW, what TMA im2col walks natively)
//   N = C_out
//   K = R * S * C_in, ordered (r, s, c);  one K-block = 64 channels of one filter tap
//
// Persistent, warp-specialised CTA (384 threads, one CTA per SM):
//   warpgroup 0    : TMA producer (one thread)
//   warpgroups 1, 2: consumers; each issues wgmma.m64nNk16 for 64 of the tile's 128 rows and runs the epilogue of those
//                    rows straight from its register accumulator
// Pipeline: a ring of shared-memory stages with full (TMA -> wgmma) and empty (wgmma -> TMA) mbarriers; the producer
// runs ahead into the next tile while the consumers finish the epilogue of the current one.
#include <cuda.h>
#include <vector>
#include "mpx_common.cuh"

namespace mpx {

#ifdef MPX_ACT_BF16
#define kTmaActType CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
#define MPX_WGMMA_AB "bf16.bf16"
#else
#define kTmaActType CU_TENSOR_MAP_DATA_TYPE_FLOAT16
#define MPX_WGMMA_AB "f16.f16"
#endif

// ---------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must trap, not hang the GPU.  No printf here: a function call inside the consumers' wgmma
// pipeline makes ptxas serialise every wgmma.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 8000000000LL) __trap();  // ~4 s at 2 GHz
  }
}

__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_im2col_4d(void* smem, const CUtensorMap* map, uint64_t* bar, int c, int w, int h,
                                                   int n, uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};" ::"r"(smem_u32(smem)),
      "l"(map), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
      : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D[64, N] (+)= A[64, 16] * B[N, 16]^T, both operands K-major in shared memory; `accumulate` = 0 overwrites D.
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." MPX_WGMMA_AB " "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32." MPX_WGMMA_AB " "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32." MPX_WGMMA_AB " "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
template <int BLOCK_N>
__device__ __forceinline__ void wgmma_tile(float (&d)[BLOCK_N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BLOCK_N == 64) wgmma_m64n64k16(d, da, db, accumulate);
  else if constexpr (BLOCK_N == 128) wgmma_m64n128k16(d, da, db, accumulate);
  else wgmma_m64n256k16(d, da, db, accumulate);
}

// K-major, 128-byte-swizzled operand tile (rows of 64 act16 = 128 B, 8-row groups 1024 B apart), as TMA writes it with
// CU_TENSOR_MAP_SWIZZLE_128B.  wgmma descriptor: start>>4 [0,14), LBO>>4 [16,30) (unused for swizzled K-major),
// SBO>>4 [32,46) = 1024 B, layout type [62,64) = 1 (128-byte swizzle).
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(64) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the 256 consumer threads only (the producer warpgroup does not take part)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// 3x3 / stride-2 / pad-1 max-pool epilogue: (ReLU'd, >= 0) output values are max-reduced into every pooled pixel whose
// window contains them, four channels (two lanes' value pairs) per reduction.  The maximum is exact and order-independent
// and the pooled tensor is zeroed before the launch, so the result equals maxpool3x3s2_kernel applied to the stored
// convolution.
__device__ __forceinline__ void red_max_act4(act_t* dst, uint32_t lo, uint32_t hi) {
#ifdef MPX_ACT_BF16
  asm volatile("red.global.max.noftz.v2.bf16x2 [%0], {%1, %2};" ::"l"(dst), "r"(lo), "r"(hi) : "memory");
#else
  asm volatile("red.global.max.noftz.v2.f16x2 [%0], {%1, %2};" ::"l"(dst), "r"(lo), "r"(hi) : "memory");
#endif
}

// ---------------------------------------------------------------------------------------------
// optional per-launch timing (bench.py roofline): CUDA events around every conv launch
// ---------------------------------------------------------------------------------------------
struct ProfileSlot {
  cudaEvent_t e0, e1;
  double flops;
};
static bool g_profile = false;
static std::vector<ProfileSlot> g_slots;
static size_t g_slots_used = 0;

static ProfileSlot* profile_begin(cudaStream_t stream) {
  if (!g_profile) return nullptr;
  if (g_slots_used == g_slots.size()) {
    ProfileSlot s;
    if (cudaEventCreate(&s.e0) != cudaSuccess || cudaEventCreate(&s.e1) != cudaSuccess) return nullptr;
    s.flops = 0;
    g_slots.push_back(s);
  }
  ProfileSlot* slot = &g_slots[g_slots_used++];
  cudaEventRecord(slot->e0, stream);
  return slot;
}
static void profile_end(ProfileSlot* slot, cudaStream_t stream, double flops) {
  if (!slot) return;
  slot->flops = flops;
  cudaEventRecord(slot->e1, stream);
}
bool conv_profile_enabled() { return g_profile; }
void conv_profile_enable(int on) {
  g_profile = on != 0;
  g_slots_used = 0;
}
// Synchronises the device; sums the recorded launches since conv_profile_enable(1) and resets.
int conv_profile_summary(double* total_ms, double* total_flops, long long* launches) {
  MPX_CHECK_CUDA(cudaDeviceSynchronize());
  double ms = 0, fl = 0;
  for (size_t i = 0; i < g_slots_used; ++i) {
    float t = 0.f;
    MPX_CHECK_CUDA(cudaEventElapsedTime(&t, g_slots[i].e0, g_slots[i].e1));
    ms += t;
    fl += g_slots[i].flops;
  }
  *total_ms = ms;
  *total_flops = fl;
  *launches = static_cast<long long>(g_slots_used);
  g_slots_used = 0;
  return MPX_OK;
}

// kernel-selection bits, see include/mpx.h (mpx_conv_set_mode)
static int g_conv_mode = 8;
int conv_get_mode() { return g_conv_mode; }
void conv_set_mode(int mode) { g_conv_mode = mode; }

struct ConvParams {
  int M_total;  // n_img * P * Q
  int P, Q;     // output height / width
  int C_out;
  int S;         // filter width (taps are ordered r-major)
  int stride;
  int pad_h, pad_w;  // lower padding
  int cblocks;       // C_in / 64
  int num_k_blocks;  // R * S * cblocks
  int m_tiles, n_tiles;
  int relu;
  int pool;                 // 1: max-pool epilogue into `out` = the zeroed [n, (P-1)/2+1, (Q-1)/2+1, C_out] tensor
  const float* bias;        // [C_out] folded BN shift
  const act_t* residual;    // [M_total, C_out] or nullptr
  act_t* out;               // [M_total, C_out]
  // split-K: the `splits` (1, 2, 4 or 8) CTAs of a cluster share one output tile, each accumulating a contiguous
  // range of k-blocks; reduction through distributed shared memory (see splitk_reduce_slice)
  int splits;
};

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kATileBytes = kBlockM * kBlockK * 2;  // 16 KiB
constexpr int kThreads = 384;

template <int BLOCK_N>
struct ConvCfg {
  static constexpr int kBTileBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = kATileBytes + kBTileBytes;
  static constexpr int kStages = (BLOCK_N == 256) ? 4 : (BLOCK_N == 128 ? 6 : 8);  // 192 KiB of stages
  static constexpr int kSmemBytes =
      kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/ + 2048 /*bias, C_out <= 512*/;
  // split-K: fp32 partial tile parked in the drained stages; +16 B per row keeps the row-owner stores conflict-free
  static constexpr int kParkPitch = BLOCK_N * 4 + 16;
  static_assert(kBlockM * kParkPitch <= kStages * kStageBytes, "split-K tile does not fit the pipeline stages");
};

// ---------------------------------------------------------------------------------------------
// Split-K over a thread-block cluster (small batches: a handful of output tiles, up to 72 serial k-blocks that a single
// CTA would walk alone).  The S CTAs of a cluster compute the same output tile over disjoint k-ranges; each parks its
// fp32 accumulator tile in its own shared memory (the drained pipeline stages), the cluster synchronises, and CTA `rank`
// finishes rows [rank*128/S, (rank+1)*128/S): it sums the S partial rows through distributed shared memory in rank order
// (deterministic), applies bias / residual / ReLU and stores act16.  No global scratch, no second kernel.
// ---------------------------------------------------------------------------------------------
template <int NCOLS>
__device__ __forceinline__ void splitk_reduce_slice(uint32_t tile_smem, int splits, int rank, long long m0, int M_total,
                                                    int C_out, int n0, act_t* __restrict__ out,
                                                    const act_t* __restrict__ residual, const float* bias_s, int relu,
                                                    int tid, int nthreads) {
  constexpr int kVecPerRow = NCOLS / 4;
  const int rows_per = kBlockM / splits;
  for (int u = tid; u < rows_per * kVecPerRow; u += nthreads) {
    const int r = rank * rows_per + u / kVecPerRow;
    const int c = (u % kVecPerRow) * 4;
    const long long m = m0 + r;
    if (m >= M_total) continue;
    const uint32_t local = tile_smem + static_cast<uint32_t>(r * ConvCfg<NCOLS>::kParkPitch + c * 4);
    float4 part[8];
#pragma unroll
    for (int sp = 0; sp < 8; ++sp) {
      if (sp < splits) {
        uint32_t remote;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(sp));
        asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(part[sp].x), "=f"(part[sp].y), "=f"(part[sp].z), "=f"(part[sp].w)
                     : "r"(remote)
                     : "memory");
      }
    }
    float4 a = part[0];
#pragma unroll
    for (int sp = 1; sp < 8; ++sp)
      if (sp < splits) { a.x += part[sp].x; a.y += part[sp].y; a.z += part[sp].z; a.w += part[sp].w; }
    const float4 b4 = *reinterpret_cast<const float4*>(bias_s + c);
    float f[4] = {a.x + b4.x, a.y + b4.y, a.z + b4.z, a.w + b4.w};
    const size_t off = static_cast<size_t>(m) * C_out + n0 + c;
    if (residual != nullptr) {
      const uint2 rr = __ldg(reinterpret_cast<const uint2*>(residual + off));
      const float2 t0 = unpack_act2(rr.x), t1 = unpack_act2(rr.y);
      f[0] += t0.x; f[1] += t0.y; f[2] += t1.x; f[3] += t1.y;
    }
    if (relu) {
#pragma unroll
      for (int j = 0; j < 4; ++j) f[j] = fmaxf(f[j], 0.f);
    }
    uint2 o;
    o.x = pack_act2(f[0], f[1]);
    o.y = pack_act2(f[2], f[3]);
    *reinterpret_cast<uint2*>(out + off) = o;
  }
}

// ---------------------------------------------------------------------------------------------
// The convolution kernel
// ---------------------------------------------------------------------------------------------
// wgmma accumulator layout of m64nNk16 (fp32): thread t of the warpgroup holds, for j in [0, N/8), the column pair
// 8j + 2 (t % 4) + {0, 1} of row 16 (t / 32) + (t % 32) / 4 in d[4j], d[4j+1] and of the row 8 below in d[4j+2], d[4j+3].
template <int BLOCK_N>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                  const ConvParams p) {
  using Cfg = ConvCfg<BLOCK_N>;
  constexpr int kStages = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kATileBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;
  float* bias_s = reinterpret_cast<float*>(bars + 32);  // [C_out] folded-BN bias, read by broadcast in the epilogue

  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);  // warpgroup, warp-uniform
  const int total_tiles = p.m_tiles * p.n_tiles * p.splits;        // work items: (tile, k-split)
  for (int i = threadIdx.x; i < p.C_out; i += blockDim.x) bias_s[i] = p.bias[i];

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  pdl_trigger();
  __syncthreads();
  pdl_wait();  // activations / residual of the previous kernel are complete from here on

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int pq = p.P * p.Q;
      for (int item = blockIdx.x; item < total_tiles; item += gridDim.x) {
        const int tile = item / p.splits;
        const int split = item - tile * p.splits;
        const int kb_begin = split * p.num_k_blocks / p.splits;
        const int kb_end = (split + 1) * p.num_k_blocks / p.splits;
        const int m_tile = tile / p.n_tiles;
        const int n_tile = tile - m_tile * p.n_tiles;
        const int m0 = m_tile * kBlockM;
        const int img = m0 / pq;
        const int rem = m0 - img * pq;
        const int p0 = rem / p.Q;
        const int q0 = rem - p0 * p.Q;
        const int base_w = q0 * p.stride - p.pad_w;
        const int base_h = p0 * p.stride - p.pad_h;
        int tap = kb_begin / p.cblocks, cb = kb_begin - tap * p.cblocks;
        for (int kb = kb_begin; kb < kb_end; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          const int r = tap / p.S;
          const int s = tap - r * p.S;
          tma_load_im2col_4d(smem_a + stage * kATileBytes, &map_a, &full_bar[stage], cb * kBlockK, base_w, base_h, img,
                             static_cast<uint16_t>(s), static_cast<uint16_t>(r));
          tma_load_2d(smem_b + stage * Cfg::kBTileBytes, &map_b, &full_bar[stage], kb * kBlockK, n_tile * BLOCK_N);
          if (++cb == p.cblocks) {
            cb = 0;
            ++tap;
          }
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
  } else {
    // ===================== consumers: wgmma + epilogue =====================
    const int half = wg - 1;  // rows [64 * half, 64 * half + 64) of the tile
    const int t = threadIdx.x & 127;
    const int lane = threadIdx.x & 31;
    const int row_lo = half * 64 + (t >> 5) * 16 + (lane >> 2);  // and row_lo + 8
    const int col = 2 * (lane & 3);
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < total_tiles; item += gridDim.x) {
      const int tile = item / p.splits;
      const int split = item - tile * p.splits;
      const int kb_begin = split * p.num_k_blocks / p.splits;
      const int kb_end = (split + 1) * p.num_k_blocks / p.splits;
      const int m_tile = tile / p.n_tiles;
      const int n_tile = tile - m_tile * p.n_tiles;
      float acc[BLOCK_N / 2];
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
      int prev_stage = -1;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t da = make_sw128_desc(smem_u32(smem_a + stage * kATileBytes + half * 64 * 128));
        const uint64_t db = make_sw128_desc(smem_u32(smem_b + stage * Cfg::kBTileBytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k)  // 16 act16 = 32 B inside the swizzle atom: +2 in the (addr >> 4) field
          wgmma_tile<BLOCK_N>(acc, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k), 1u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage can be refilled
        if (prev_stage >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        }
        prev_stage = stage;
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1u;
        }
      }
      wgmma_wait<0>();
      if (prev_stage >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      }
      const long long m0 = static_cast<long long>(m_tile) * kBlockM;
      const int n0 = n_tile * BLOCK_N;
      if (p.splits > 1) {
        // one item per CTA: park the fp32 partial tile in the (drained) pipeline stages
        consumers_sync();  // the other consumer warpgroup's MMAs have retired too
        const uint32_t park = smem_u32(smem);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t rbase = park + static_cast<uint32_t>((row_lo + 8 * h) * Cfg::kParkPitch + col * 4);
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j)
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(rbase + static_cast<uint32_t>(32 * j)),
                         "f"(acc[4 * j + 2 * h]), "f"(acc[4 * j + 2 * h + 1])
                         : "memory");
        }
        continue;
      }
      const int pq = p.P * p.Q;
      const int pp = (p.P - 1) / 2 + 1, pq2 = (p.Q - 1) / 2 + 1;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long m = m0 + row_lo + 8 * h;
        const bool valid = m < p.M_total;  // uniform over the 4 lanes of a row
        const size_t off = static_cast<size_t>(valid ? m : 0) * p.C_out + n0 + col;
        const act_t* res_row = (valid && p.residual) ? p.residual + off : nullptr;
        uint32_t packed[BLOCK_N / 8];
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const float2 b = *reinterpret_cast<const float2*>(bias_s + n0 + 8 * j + col);
          float f0 = acc[4 * j + 2 * h] + b.x;
          float f1 = acc[4 * j + 2 * h + 1] + b.y;
          if (res_row) {
            const float2 r = unpack_act2(__ldg(reinterpret_cast<const uint32_t*>(res_row + 8 * j)));
            f0 += r.x;
            f1 += r.y;
          }
          if (p.relu) {
            f0 = fmaxf(f0, 0.f);
            f1 = fmaxf(f1, 0.f);
          }
          packed[j] = pack_act2(f0, f1);
        }
        if (!p.pool) {
          if (valid) {
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) *reinterpret_cast<uint32_t*>(p.out + off + 8 * j) = packed[j];
          }
          continue;
        }
        uint32_t nb[BLOCK_N / 8];  // the odd lane's pair: channels col + 2, col + 3 for the even lane
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) nb[j] = __shfl_xor_sync(0xffffffffu, packed[j], 1);
        if (!valid || (lane & 1) != 0) continue;
        const int img = static_cast<int>(m / pq);
        const int rem = static_cast<int>(m - static_cast<long long>(img) * pq);
        const int y = rem / p.Q, x = rem - y * p.Q;
        // pooled rows / columns whose 3x3 window (2k-1 .. 2k+1) contains y / x
        const int py0 = y >> 1, py1 = ((y & 1) && ((y + 1) >> 1) < pp) ? (y + 1) >> 1 : py0;
        const int px0 = x >> 1, px1 = ((x & 1) && ((x + 1) >> 1) < pq2) ? (x + 1) >> 1 : px0;
        for (int py = py0; py <= py1; ++py) {
          for (int px = px0; px <= px1; ++px) {
            act_t* dst = p.out + ((static_cast<size_t>(img) * pp + py) * pq2 + px) * p.C_out + n0 + col;
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) red_max_act4(dst + 8 * j, packed[j], nb[j]);
          }
        }
      }
    }
  }

  __syncthreads();
  if (p.splits > 1) {
    cluster_sync_all();  // every CTA of the cluster has parked its partial tile
    const int item = blockIdx.x;
    const int tile = item / p.splits;
    const int m_tile = tile / p.n_tiles;
    const int n_tile = tile - m_tile * p.n_tiles;
    const int n0 = n_tile * BLOCK_N;
    splitk_reduce_slice<BLOCK_N>(smem_u32(smem), p.splits, static_cast<int>(cluster_ctarank()),
                                 static_cast<long long>(m_tile) * kBlockM, p.M_total, p.C_out, n0, p.out, p.residual,
                                 bias_s + n0, p.relu, threadIdx.x, blockDim.x);
    cluster_sync_all();  // peers may still be reading this CTA's shared memory
  }
}

// ---------------------------------------------------------------------------------------------
// Host side: tensor maps + launch
// ---------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                     const cuuint64_t*, const cuuint64_t*, const int*, const int*,
                                     cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion,
                                     CUtensorMapFloatOOBfill);

static PFN_encodeTiled g_encode_tiled = nullptr;
static PFN_encodeIm2col g_encode_im2col = nullptr;

// libcuda is reached through the runtime so the library loads (and its symbols can be listed) on a
// machine without a driver.
static int load_driver_entry_points() {
  if (g_encode_tiled && g_encode_im2col) return MPX_OK;
  cudaDriverEntryPointQueryResult q;
  void* f = nullptr;
  MPX_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q));
  MPX_REQUIRE(f != nullptr && q == cudaDriverEntryPointSuccess,
              "cuTensorMapEncodeTiled not available from the driver");
  g_encode_tiled = reinterpret_cast<PFN_encodeTiled>(f);
  f = nullptr;
  MPX_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &f, cudaEnableDefault, &q));
  MPX_REQUIRE(f != nullptr && q == cudaDriverEntryPointSuccess,
              "cuTensorMapEncodeIm2col not available from the driver");
  g_encode_im2col = reinterpret_cast<PFN_encodeIm2col>(f);
  return MPX_OK;
}

template <int BLOCK_N>
static int launch_conv(const CUtensorMap& ma, const CUtensorMap& mb, const ConvParams& p, cudaStream_t stream,
                       int max_ctas) {
  using Cfg = ConvCfg<BLOCK_N>;
  static bool attr_set = false;
  if (!attr_set) {
    MPX_CHECK_CUDA(cudaFuncSetAttribute(conv_wgmma_kernel<BLOCK_N>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        Cfg::kSmemBytes));
    attr_set = true;
  }
  int grid = p.m_tiles * p.n_tiles * p.splits;
  const int cap = max_ctas > 0 ? max_ctas : sm_count();
  ProfileSlot* slot = profile_begin(stream);
  // split-K: one work item per CTA, the k-splits of a tile form a cluster
  if (p.splits == 1 && grid > cap) grid = cap;
  MPX_CHECK_CUDA(launch_pdl(conv_wgmma_kernel<BLOCK_N>, dim3(grid), dim3(kThreads), Cfg::kSmemBytes, stream, p.splits,
                            ma, mb, p));
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  profile_end(slot, stream, 2.0 * p.M_total * p.C_out * p.num_k_blocks * kBlockK);
  return MPX_OK;
}

int conv_out_dim(int in, int pad_lo, int pad_hi, int k, int stride) {
  return (in + pad_lo + pad_hi - k) / stride + 1;
}

// x: [n_img, H, W, C_in] act16; w: [C_out, R*S*C_in] act16 ((r,s,c) ordered); bias fp32 [C_out];
// residual/out: [n_img, P, Q, C_out] act16.
int conv_forward(const ConvDesc& d, const void* x, const void* w, const float* bias,
                 const void* residual, void* out, int block_n_override, int max_ctas,
                 cudaStream_t stream, int splitk) {
  MPX_REQUIRE(d.C_in % 64 == 0 && d.C_in >= 64, "conv: C_in=%d must be a multiple of 64", d.C_in);
  MPX_REQUIRE(d.C_out % 64 == 0 && d.C_out <= 512, "conv: C_out=%d must be a multiple of 64, at most 512", d.C_out);
  MPX_REQUIRE(d.stride == 1 || d.stride == 2, "conv: stride %d unsupported", d.stride);
  MPX_REQUIRE(d.R >= 1 && d.R <= 8 && d.S >= 1 && d.S <= 8, "conv: filter %dx%d unsupported", d.R, d.S);
  // the pooled epilogue needs non-negative values (ReLU) and no residual; refused without an error text otherwise
  if (d.pool && (!d.relu || residual != nullptr || block_n_override != 0 || splitk != 0)) return MPX_ERR_UNSUPPORTED;
  int rc = load_driver_entry_points();
  if (rc != MPX_OK) return rc;

  const int P = conv_out_dim(d.H, d.pad_lo_h, d.pad_hi_h, d.R, d.stride);
  const int Q = conv_out_dim(d.W, d.pad_lo_w, d.pad_hi_w, d.S, d.stride);
  MPX_REQUIRE(P > 0 && Q > 0, "conv: empty output");
  const long long M_total = static_cast<long long>(d.n_img) * P * Q;
  MPX_REQUIRE(M_total > 0 && M_total < (1LL << 31), "conv: M=%lld out of range", M_total);

  int block_n = block_n_override;
  if (block_n <= 0) {
    // wide tiles amortise the activation loads; with only a handful of output tiles (refiner: one sample) the
    // conv is bound by the serial K loop of a single tile instead, so narrower tiles spread it over more SMs
    const long long m_tiles_est = (M_total + kBlockM - 1) / kBlockM;
    block_n = d.C_out >= 256 ? 256 : d.C_out;
    while (block_n > 64 && m_tiles_est * (d.C_out / block_n) < 32) block_n /= 2;
  }
  MPX_REQUIRE((block_n == 64 || block_n == 128 || block_n == 256) && d.C_out % block_n == 0,
              "conv: BLOCK_N=%d invalid for C_out=%d", block_n, d.C_out);

  // --- activation map (im2col). Dims are innermost-first: {C, W, H, N}.
  CUtensorMap map_a, map_b;
  {
    cuuint64_t dims[4] = {static_cast<cuuint64_t>(d.C_in), static_cast<cuuint64_t>(d.W),
                          static_cast<cuuint64_t>(d.H), static_cast<cuuint64_t>(d.n_img)};
    cuuint64_t strides[3] = {static_cast<cuuint64_t>(d.C_in) * 2,
                             static_cast<cuuint64_t>(d.W) * d.C_in * 2,
                             static_cast<cuuint64_t>(d.H) * d.W * d.C_in * 2};
    // Bounding box of the filter's *base* pixel (CUTLASS: lower = -pad_lo,
    // upper = pad_hi - (filter-1)*dilation; cutlass/conv/collective/detail.hpp).
    int lower[2] = {-d.pad_lo_w, -d.pad_lo_h};
    int upper[2] = {d.pad_hi_w - (d.S - 1), d.pad_hi_h - (d.R - 1)};
    cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(d.stride), static_cast<cuuint32_t>(d.stride), 1};
    CUresult r = g_encode_im2col(&map_a, kTmaActType, 4, const_cast<void*>(x),
                                 dims, strides, lower, upper, /*channelsPerPixel=*/kBlockK,
                                 /*pixelsPerColumn=*/kBlockM, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MPX_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeIm2col failed (%d)", static_cast<int>(r));
    // Driver quirk (<= 13.1) for im2col maps over tensors smaller than 128 KiB: same fix-up as
    // cute/atom/copy_traits_sm90_im2col.hpp.
    int drv = 0;
    cudaDriverGetVersion(&drv);
    const size_t bytes = static_cast<size_t>(d.n_img) * d.H * d.W * d.C_in * 2;
    if (drv <= 13010 && bytes < 131072) {
      reinterpret_cast<uint64_t*>(&map_a)[1] &= ~(1ull << 21);
    }
  }
  {
    const cuuint64_t K_total = static_cast<cuuint64_t>(d.R) * d.S * d.C_in;
    cuuint64_t dims[2] = {K_total, static_cast<cuuint64_t>(d.C_out)};
    cuuint64_t strides[1] = {K_total * 2};
    cuuint32_t box[2] = {kBlockK, static_cast<cuuint32_t>(block_n)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode_tiled(&map_b, kTmaActType, 2, const_cast<void*>(w), dims,
                                strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MPX_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", static_cast<int>(r));
  }

  ConvParams p{};
  p.M_total = static_cast<int>(M_total);
  p.P = P;
  p.Q = Q;
  p.C_out = d.C_out;
  p.S = d.S;
  p.stride = d.stride;
  p.pad_h = d.pad_lo_h;
  p.pad_w = d.pad_lo_w;
  p.cblocks = d.C_in / kBlockK;
  p.num_k_blocks = d.R * d.S * p.cblocks;
  p.m_tiles = static_cast<int>((M_total + kBlockM - 1) / kBlockM);
  p.n_tiles = d.C_out / block_n;
  p.relu = d.relu;
  p.pool = d.pool;
  p.bias = bias;
  p.residual = reinterpret_cast<const act_t*>(residual);
  p.out = reinterpret_cast<act_t*>(out);
  p.splits = 1;
  if (splitk != 0) {
    // Few output tiles and a long K loop (deep layers at batch 1: one 80-row tile, 72 k-blocks): split K over a cluster.
    const int tiles = p.m_tiles * p.n_tiles;
    const int sms = max_ctas > 0 ? max_ctas : sm_count();
    int want = splitk > 0 ? splitk : 1;
    if (splitk < 0 && tiles * 2 <= sms && p.num_k_blocks >= 8) {
      want = p.num_k_blocks / 4;
      if (want > sms / tiles) want = sms / tiles;
    }
    // bits 18 / 19 of the mode cap the automatic split at 2 / 1: fewer, longer CTAs -- less SM time per layer at a higher
    // latency, the better trade when another frame's kernels fill the device beside this one (frame_pipeline.py)
    const int cap = (splitk < 0 && (g_conv_mode & 524288)) ? 1 : ((splitk < 0 && (g_conv_mode & 262144)) ? 2 : 8);
    int splits = 1;
    while (splits * 2 <= want && splits * 2 <= cap && splits * 2 <= p.num_k_blocks) splits *= 2;
    p.splits = splits;
  }

  switch (block_n) {
    case 64:
      return launch_conv<64>(map_a, map_b, p, stream, max_ctas);
    case 128:
      return launch_conv<128>(map_a, map_b, p, stream, max_ctas);
    default:
      return launch_conv<256>(map_a, map_b, p, stream, max_ctas);
  }
}

}  // namespace mpx
