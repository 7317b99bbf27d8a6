// Implicit-GEMM convolution for sm_90a: TMA im2col (activations) + TMA tiled (weights) -> 128B-swizzled shared memory ->
// wgmma (act16 x act16 -> fp32 register accumulators) -> fused epilogue (folded-BN bias, residual add, ReLU) -> act16 NHWC.
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
__device__ __forceinline__ void wgmma_m64n160k16(float (&d)[80], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %82, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n160k16.f32." MPX_WGMMA_AB " "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, %80, %81, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
template <int BLOCK_N>
__device__ __forceinline__ void wgmma_tile(float (&d)[BLOCK_N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BLOCK_N == 64) wgmma_m64n64k16(d, da, db, accumulate);
  else if constexpr (BLOCK_N == 128) wgmma_m64n128k16(d, da, db, accumulate);
  else if constexpr (BLOCK_N == 160) wgmma_m64n160k16(d, da, db, accumulate);
  else wgmma_m64n256k16(d, da, db, accumulate);
}

// K-major, 128-byte-swizzled operand tile (rows of 64 act16 = 128 B, 8-row groups 1024 B apart), as TMA writes it with
// CU_TENSOR_MAP_SWIZZLE_128B.  wgmma descriptor: start>>4 [0,14), LBO>>4 [16,30) (unused for swizzled K-major),
// SBO>>4 [32,46) = 1024 B, layout type [62,64) = 1 (128-byte swizzle).  The swizzle is applied to the absolute shared
// address on sm_90a, so a tile may also start a whole number of 128-byte rows past a 1024-byte boundary (the band B
// operand of conv64_wgmma_kernel) with the base-offset field [49,52) left at 0: measured on an H100, where setting that
// field to (start >> 7) & 7 misreads every odd row shift.
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
static int g_conv_mode = MPX_CONV_NET_SPLITK;
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
  // launches with C_out > 512 (the detector's layer3 / layer4, up to 2048) stage C_out * 4 B of bias instead
  static int smem_bytes(int c_out) { return c_out <= 512 ? kSmemBytes : kSmemBytes - 2048 + 4 * c_out; }
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
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long m = m0 + row_lo + 8 * h;
        const bool valid = m < p.M_total;  // uniform over the 4 lanes of a row
        const size_t off = static_cast<size_t>(valid ? m : 0) * p.C_out + n0 + col;
        if (!valid) continue;
        const act_t* res_row = p.residual ? p.residual + off : nullptr;
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
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) *reinterpret_cast<uint32_t*>(p.out + off + 8 * j) = packed[j];
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
// C_out = 64: pixel-major kernel with ping-pong consumers and a TMA epilogue
// ---------------------------------------------------------------------------------------------
// D^T[64 ch, N px] = W[64, K] * X[N px, K]^T: the weights are the wgmma A operand (one 64 x 64 box per k-block), the
// activations the B operand, so each k16 step is one m64nNk16 -- 4 KB of operand reads per 262144 MACs at N = 256
// instead of 4 KB per 65536 with 64-wide tiles.  Two producers fill the B operand:
//   im2col (kBandN = 0): a tile is 256 consecutive output pixels of the flattened NHW space; per k-block two 128-pixel
//     im2col boxes fill one 256-row tile, so every input pixel is loaded once per filter tap.
//   band (kBandN = 160 or 256, stride 1): a tile is `band_rows` whole output rows of one image.  Output pixel (j, q) of
//     the tile is column j * Wp + q of a padded-width pixel space, Wp = Q + S - 1 = the padded input width, so tap (r, s)
//     reads band pixel column + s of filter row r's band: the input rows p0 + r - pad_h .. + band_rows - 1, every padded
//     column, loaded by one tiled TMA box per (filter row, cblock) with the padding zero-filled by the tensor map.  Tap s
//     takes its B operand s rows (s * 128 B) into the band; columns q >= Q and rows past the tile are computed and dropped.
//     The bands have a ring of their own (a tile holds `cblocks` of them at once: the (r, s, cblock, k) sum order of
//     every output stays that of the im2col producer); the weights keep the per-k-block ring.
// Warpgroup 0 is the TMA producer; warpgroups 1 and 2 take alternate tiles of the CTA's persistent sequence, so one runs
// its epilogue while the other issues MMAs.  The epilogue goes through a per-warpgroup staging tile: the residual is
// TMA-loaded into it while the mainloop runs, the result is written over it in place and TMA-stored (rows >= M_total, or
// for band tiles rows >= P, are clipped by the tensor map).
constexpr int kC64Pixels = 256;
constexpr int kC64Stages = 4;
constexpr int kC64ActBytes = kC64Pixels * kBlockK * 2;  // 32 KiB
constexpr int kC64WBytes = 64 * kBlockK * 2;            // 8 KiB
constexpr int kC64StageBytes = kC64ActBytes + kC64WBytes;
constexpr int kC64StagingBytes = kC64Pixels * 64 * 2;   // 32 KiB per consumer warpgroup
// band producer: up to 3 band slots, then the weights (all k-blocks resident, or a ring of 8 stages), then the two
// staging tiles; with the ring, the same 224 KiB as the im2col producer's stages and staging tiles
constexpr int kC64BandSlots = 3;
constexpr int kC64BandWStages = 8;
static_assert(kC64BandSlots * kC64ActBytes + kC64BandWStages * kC64WBytes == kC64Stages * kC64StageBytes,
              "conv64: the band producer's ring layout is the im2col producer's");
constexpr int kC64SmemBytes = 227 * 1024;
// stages / bands / weights / staging tiles in the first kC64BufferBytes, then 256 B of barriers and 256 B of bias
constexpr int kC64BufferBytes = kC64SmemBytes - 1024 /*align slack*/ - 256 /*barriers*/ - 256 /*bias*/;
static_assert(kC64Stages * kC64StageBytes + 2 * kC64StagingBytes <= kC64BufferBytes, "conv64: shared memory budget");

struct Conv64Params {
  int M_total, P, Q, S, stride, pad_h, pad_w, cblocks, num_k_blocks, m_tiles;
  int band_w, band_rows, tiles_per_img;  // band producer: Wp, output rows per tile, tiles per image
  // band producer layout (bytes, multiples of 1024): band_slots slots of slot_bytes at 0, the weights at w_off (every
  // k-block when w_resident, else a ring of kC64BandWStages), the two staging tiles of staging_bytes at staging_off
  int band_slots, slot_bytes, w_resident, w_off, staging_off, staging_bytes;
  int relu;
  int has_residual;
  const float* bias;
};

__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* smem, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(map),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// the 128 threads of consumer warpgroup `cw` (named barriers 2 and 3)
__device__ __forceinline__ void warpgroup_sync(int cw) { asm volatile("bar.sync %0, 128;" ::"r"(2 + cw) : "memory"); }
// mainloop hand-off between the consumer warpgroups (named barriers 4 and 5: 128 arrive + 128 wait)
__device__ __forceinline__ void mainloop_turn_wait(int cw) { asm volatile("bar.sync %0, 256;" ::"r"(4 + cw) : "memory"); }
__device__ __forceinline__ void mainloop_turn_pass(int cw) { asm volatile("bar.arrive %0, 256;" ::"r"(5 - cw) : "memory"); }

// Space-to-depth 7x7 stem (megapose6d_b200/backbone.py: _stem_s2d): weight column (r, s, (dy*2+dx)*c_pad + c) holds the 7x7
// tap (2r+dy-1, 2s+dx-1), zero when that lies outside 0..6.  Bit k of the result: k16 step k of k-block kb multiplies a
// slice that is not structurally zero.  c_pad = 16 * cblocks, so step k covers channels 16 (4 cb + k) .. + 15, all in slice
// (4 cb + k) / cblocks.
__host__ __device__ __forceinline__ uint32_t stem_live_steps(int kb, int cblocks, int S) {
  const int tap = kb / cblocks, cb = kb - tap * cblocks;
  const int r = tap / S, s = tap - r * S;
  uint32_t live = 0;
  for (int k = 0; k < 4; ++k) {
    const int slice = (4 * cb + k) / cblocks;
    const int ky = 2 * r + (slice >> 1) - 1, kx = 2 * s + (slice & 1) - 1;
    if (ky >= 0 && ky <= 6 && kx >= 0 && kx <= 6) live |= 1u << k;
  }
  return live;
}

// One k-block's MMAs as one chain: the k16 steps whose bit is set in `live`, between a fence and a commit.  `live` must fold
// to a constant at every call site: a wgmma behind a run-time branch makes ptxas end each branch with its own commit and
// add a dummy group at the join, so the next wgmma_wait<1> drains the tensor pipe every k-block.
template <int N>
__device__ __forceinline__ void wgmma_kblock(uint32_t live, float (&acc)[N / 2], uint64_t da, uint64_t db) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < kBlockK / 16; ++k)  // 16 act16 = 32 B inside the swizzle atom: +2 per step in the (addr >> 4) field
    if (live & (1u << k)) wgmma_tile<N>(acc, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k), 1u);
  wgmma_commit();
}

// kStemCblocks = 0: every k16 step is issued.  1 or 2: the weights are the space-to-depth stem's (relu bit 1, 4x4 taps,
// c_pad = 16 * kStemCblocks), its 16 * kStemCblocks k-blocks are unrolled so that stem_live_steps folds to a constant per
// k-block, and the structurally zero k16 steps are not issued.
// kBandN = 0: the im2col producer; 160 or 256: the band producer with an m64n{kBandN}k16 chain per k16 step.
template <int kStemCblocks, int kBandN>
__global__ void __launch_bounds__(kThreads, 1)
conv64_wgmma_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                    const __grid_constant__ CUtensorMap map_res, const __grid_constant__ CUtensorMap map_out,
                    const Conv64Params p) {
  constexpr bool kBand = kBandN > 0;
  constexpr int kN = kBand ? kBandN : kC64Pixels;            // wgmma N = accumulator columns per tile
  constexpr int kStages = kBand ? kC64BandWStages : kC64Stages;  // ring of k-blocks (im2col: activations + weights)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_x = smem;  // im2col: kStages activation tiles; band: p.band_slots bands
  uint8_t* smem_w = smem + (kBand ? p.w_off : kC64Stages * kC64ActBytes);
  uint8_t* staging = smem + (kBand ? p.staging_off : kC64Stages * kC64StageBytes);
  const int staging_bytes = kBand ? p.staging_bytes : kC64StagingBytes;
  const int slot_bytes = kBand ? p.slot_bytes : kC64ActBytes;
  const bool w_resident = kBand && p.w_resident;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kC64BufferBytes);
  uint64_t* full_bar = bars;            // [kStages]
  uint64_t* empty_bar = bars + 8;       // [kStages]
  uint64_t* res_bar = bars + 16;        // [2], one per consumer warpgroup
  uint64_t* band_full = bars + 18;      // [kC64BandSlots]
  uint64_t* band_empty = bars + 21;     // [kC64BandSlots]
  uint64_t* w_bar = bars + 24;          // resident weights
  float* bias_s = reinterpret_cast<float*>(bars + 32);

  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);
  const int nk = p.num_k_blocks;
  for (int i = threadIdx.x; i < 64; i += blockDim.x) bias_s[i] = p.bias[i];
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_out) : "memory");
    if (p.has_residual) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_res) : "memory");
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);  // one arrive per warp of the consuming warpgroup
    }
    if constexpr (kBand) {
      for (int i = 0; i < kC64BandSlots; ++i) {
        mbar_init(&band_full[i], 1);
        mbar_init(&band_empty[i], 4);
      }
      mbar_init(w_bar, 1);
    }
    mbar_init(&res_bar[0], 1);
    mbar_init(&res_bar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  pdl_trigger();
  __syncthreads();
  pdl_wait();

  if (wg == 0) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      if constexpr (kBand) {
        // per k-block (r, s, cb) in K order: the band of (r, cb) before its first tap (s = 0), then the weights
        int slot = 0;
        uint32_t slot_phase = 0;
        const uint32_t band_bytes = static_cast<uint32_t>(p.band_w * p.band_rows) * 128u;
        if (w_resident) {  // every k-block's weights once, for all of this CTA's tiles
          mbar_expect_tx(w_bar, static_cast<uint32_t>(nk) * kC64WBytes);
          for (int kb = 0; kb < nk; ++kb)
            tma_load_2d(smem_w + kb * kC64WBytes, &map_w, w_bar, kb * kBlockK, 0);
        }
        for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x) {
          const int img = tile / p.tiles_per_img;
          const int p0 = (tile - img * p.tiles_per_img) * p.band_rows;
          int r = 0, s = 0, cb = 0;
          for (int kb = 0; kb < nk; ++kb) {
            if (s == 0) {
              mbar_wait(&band_empty[slot], slot_phase ^ 1u);
              mbar_expect_tx(&band_full[slot], band_bytes);
              tma_load_4d(smem_x + slot * slot_bytes, &map_x, &band_full[slot], cb * kBlockK, -p.pad_w,
                          p0 + r - p.pad_h, img);
              if (++slot == p.band_slots) {
                slot = 0;
                slot_phase ^= 1u;
              }
            }
            if (!w_resident) {
              mbar_wait(&empty_bar[stage], phase ^ 1u);
              mbar_expect_tx(&full_bar[stage], kC64WBytes);
              tma_load_2d(smem_w + stage * kC64WBytes, &map_w, &full_bar[stage], kb * kBlockK, 0);
              if (++stage == kStages) {
                stage = 0;
                phase ^= 1u;
              }
            }
            if (++cb == p.cblocks) {
              cb = 0;
              if (++s == p.S) {
                s = 0;
                ++r;
              }
            }
          }
        }
      } else {
        const int pq = p.P * p.Q;
        for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x) {
          int base_w[2], base_h[2], img[2];
          const int m0 = tile * kC64Pixels;
          const bool second = m0 + kBlockM < p.M_total;  // a half past the last pixel is not loaded: its columns are clipped
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int m = m0 + hh * kBlockM;
            img[hh] = m / pq;
            const int rem = m - img[hh] * pq;
            const int p0 = rem / p.Q;
            base_w[hh] = (rem - p0 * p.Q) * p.stride - p.pad_w;
            base_h[hh] = p0 * p.stride - p.pad_h;
          }
          const uint32_t bytes = (second ? kC64ActBytes : kC64ActBytes / 2) + kC64WBytes;
          int tap = 0, cb = 0;
          for (int kb = 0; kb < nk; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            mbar_expect_tx(&full_bar[stage], bytes);
            const int r = tap / p.S;
            const int s = tap - r * p.S;
            uint8_t* dst = smem_x + stage * kC64ActBytes;
            tma_load_im2col_4d(dst, &map_x, &full_bar[stage], cb * kBlockK, base_w[0], base_h[0], img[0],
                               static_cast<uint16_t>(s), static_cast<uint16_t>(r));
            if (second)
              tma_load_im2col_4d(dst + kATileBytes, &map_x, &full_bar[stage], cb * kBlockK, base_w[1], base_h[1], img[1],
                                 static_cast<uint16_t>(s), static_cast<uint16_t>(r));
            tma_load_2d(smem_w + stage * kC64WBytes, &map_w, &full_bar[stage], kb * kBlockK, 0);
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
    }
  } else {
    // ===================== consumers: wgmma + staged epilogue =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;
    const int t = threadIdx.x & 127;
    const int lane = threadIdx.x & 31;
    const int q = lane >> 2;
    // after the lane ^ 4 exchange this thread holds channels (c, c + 1) + 8 h of pixel column 8 j + px
    const int c = 16 * (t >> 5) + (q & ~1);
    const int px = 2 * (lane & 3) + (q & 1);
    const bool odd = (q & 1) != 0;
    uint8_t* stage_buf = staging + cw * staging_bytes;
    if (w_resident) mbar_wait(w_bar, 0);
    const int bands_per_tile = nk / p.S;  // R * cblocks
    int local = 0;
    for (int i = cw, tile = blockIdx.x + cw * gridDim.x; tile < p.m_tiles; i += 2, tile += 2 * gridDim.x, ++local) {
      const int m0 = tile * kC64Pixels;
      const int img = kBand ? tile / p.tiles_per_img : 0;
      const int p0 = kBand ? (tile - img * p.tiles_per_img) * p.band_rows : 0;
      if (p.has_residual && t == 0) {
        bulk_wait_read_all();  // the previous tile's store has read the staging tile
        if constexpr (kBand) {
          mbar_expect_tx(&res_bar[cw], static_cast<uint32_t>(p.band_rows * p.Q) * 128u);
          tma_load_4d(stage_buf, &map_res, &res_bar[cw], 0, 0, p0, img);
        } else {
          mbar_expect_tx(&res_bar[cw], kC64StagingBytes);
          tma_load_2d(stage_buf, &map_res, &res_bar[cw], 0, m0);
        }
      }
      // stage / phase from the CTA's k-block counter (both warpgroups' tiles, in tile order); unsigned, since only the
      // counter modulo 2 * kStages matters and that survives wrap-around at 2^32.  The band ring's slot and phase come
      // from the CTA's band counter the same way (64-bit: 3 slots do not divide 2^32).
      const uint32_t g = static_cast<uint32_t>(i) * static_cast<uint32_t>(nk);
      int stage = static_cast<int>(g % kStages);
      uint32_t phase = (g / kStages) & 1u;
      const uint64_t gb0 = static_cast<uint64_t>(i) * static_cast<uint64_t>(bands_per_tile);
      const int slot0 = kBand ? static_cast<int>(gb0 % static_cast<uint64_t>(p.band_slots)) : 0;
      const uint32_t slot_phase0 = kBand ? static_cast<uint32_t>(gb0 / static_cast<uint64_t>(p.band_slots)) & 1u : 0u;
      float acc[kN / 2];
#pragma unroll
      for (int j = 0; j < kN / 2; ++j) acc[j] = 0.f;
      // The mainloops take turns: this one starts once the other warpgroup has waited on every full barrier of the
      // previous tile, so no waiter is ever more than one phase behind a barrier (parity waits cannot tell phases 0 and 2
      // apart).  One arrive per following tile, so no arrival is left pending at exit.
      if (i > 0) mainloop_turn_wait(cw);
      int prev_stage = -1, prev_slot = -1;
      // k-block (r, s, cb); the band producer's B operand is (r, cb)'s band shifted by s pixel rows
      auto kblock = [&](uint32_t live, int kb, int r, int s, int cb) {
        uint64_t db;
        int slot = -1;
        if constexpr (kBand) {
          const int u = slot0 + r * p.cblocks + cb;  // band r * cblocks + cb of the tile
          slot = u % p.band_slots;
          if (s == 0) mbar_wait(&band_full[slot], slot_phase0 ^ (static_cast<uint32_t>(u / p.band_slots) & 1u));
          db = make_sw128_desc(smem_u32(smem_x + slot * slot_bytes) + static_cast<uint32_t>(s) * 128u);
        } else {
          db = make_sw128_desc(smem_u32(smem_x + stage * kC64ActBytes));
        }
        uint32_t wa;
        if (w_resident) {
          wa = smem_u32(smem_w + kb * kC64WBytes);
        } else {
          mbar_wait(&full_bar[stage], phase);
          wa = smem_u32(smem_w + stage * kC64WBytes);
        }
        wgmma_kblock<kN>(live, acc, make_sw128_desc(wa), db);
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its weights (and a band it used last) can go
        __syncwarp();
        if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        if (prev_slot >= 0 && lane == 0) mbar_arrive(&band_empty[prev_slot]);
        prev_slot = (kBand && s == p.S - 1) ? slot : -1;
        if (!w_resident) {
          prev_stage = stage;
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      };
      if constexpr (kStemCblocks > 0) {
#pragma unroll
        for (int kb = 0; kb < 16 * kStemCblocks; ++kb)
          kblock(stem_live_steps(kb, kStemCblocks, 4), kb, kb / (4 * kStemCblocks), (kb / kStemCblocks) % 4,
                 kb % kStemCblocks);
      } else {
        int r = 0, s = 0, cb = 0;
#pragma unroll 1
        for (int kb = 0; kb < nk; ++kb) {
          kblock(0xFu, kb, r, s, cb);
          if (++cb == p.cblocks) {
            cb = 0;
            if (++s == p.S) {
              s = 0;
              ++r;
            }
          }
        }
      }
      if (tile + static_cast<int>(gridDim.x) < p.m_tiles) mainloop_turn_pass(cw);
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) {
        if (prev_stage >= 0) mbar_arrive(&empty_bar[prev_stage]);
        if (prev_slot >= 0) mbar_arrive(&band_empty[prev_slot]);
      }

      if (t == 0) bulk_wait_read_all();
      warpgroup_sync(cw);
      if (p.has_residual) mbar_wait(&res_bar[cw], static_cast<uint32_t>(local) & 1u);
      const uint32_t sbase = smem_u32(stage_buf);
      const float2 bias2[2] = {*reinterpret_cast<const float2*>(bias_s + c), *reinterpret_cast<const float2*>(bias_s + c + 8)};
      // band tiles: column n = 8 j + px is output pixel (row, col) = (n / Wp, n % Wp) of the tile, staged at row * Q + col
      // when col < Q and row < the tile's rows; im2col tiles stage column n at n
      const int rows = kBand ? min(p.band_rows, p.P - p0) : 0;
      int prow = 0, pcol = px;
#pragma unroll
      for (int j = 0; j < kN / 8; ++j) {
        if constexpr (kBand) {
          while (pcol >= p.band_w) {  // Wp may be below 8
            pcol -= p.band_w;
            ++prow;
          }
        }
        const bool keep = !kBand || (pcol < p.Q && prow < rows);
        const int srow = kBand ? prow * p.Q + pcol : 8 * j + px;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          const float other = __shfl_xor_sync(0xffffffffu, odd ? v0 : v1, 4);
          float f0 = (odd ? other : v0) + bias2[h].x;
          float f1 = (odd ? v1 : other) + bias2[h].y;
          const int chunk = (c + 8 * h) >> 3;
          const uint32_t addr = sbase + static_cast<uint32_t>(srow * 128 + ((chunk ^ (srow & 7)) << 4) + ((c & 7) << 1));
          if (keep) {
            if (p.has_residual) {
              uint32_t rr;
              asm volatile("ld.shared.b32 %0, [%1];" : "=r"(rr) : "r"(addr) : "memory");
              const float2 r = unpack_act2(rr);
              f0 += r.x;
              f1 += r.y;
            }
            if (p.relu) {
              f0 = fmaxf(f0, 0.f);
              f1 = fmaxf(f1, 0.f);
            }
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_act2(f0, f1)) : "memory");
          }
        }
        pcol += 8;
      }
      fence_proxy_async_smem();
      warpgroup_sync(cw);
      if (t == 0) {
        if constexpr (kBand) tma_store_4d(&map_out, stage_buf, 0, 0, p0, img);
        else tma_store_2d(&map_out, stage_buf, 0, m0);
        bulk_commit();
      }
    }
    if (t == 0) bulk_wait_all();
  }
}

// ---------------------------------------------------------------------------------------------
// C_out = 128 .. 512: ping-pong consumers that each own a whole 128 x 128 tile, and a TMA epilogue
// ---------------------------------------------------------------------------------------------
// The producer is conv_wgmma_kernel<128>'s (one 128 x 64 im2col box and one 128 x 64 weight box per k-block; items in
// (m-tile, n-tile) order, n fastest, so consecutive items reuse the activation box from L2).  Warpgroups 1 and 2 take
// alternate items of the CTA's persistent sequence: per k16 step one warpgroup issues two m64n128k16 (rows 0-63 and 64-127)
// with the same B descriptor, 128 fp32 accumulators per thread, and hands the mainloop to the other warpgroup when its
// last k-block is issued, so one runs its epilogue while the other keeps the tensor pipe busy.  Epilogue as in
// conv64_wgmma_kernel: the residual is TMA-loaded into the warpgroup's staging tile (two 128 x 64 boxes, 128B swizzle)
// while the mainloop runs, bias + residual + ReLU + conversion overwrite it in place, and two TMA stores write it out
// (rows >= M_total clipped by the tensor map).  Every output's k16 sum order is that of conv_wgmma_kernel.
constexpr int kPPStages = 4;
constexpr int kPPStageBytes = 2 * kATileBytes;            // 16 KiB activations + 16 KiB weights
constexpr int kPPStagingBytes = kBlockM * 128 * 2;        // 32 KiB per consumer warpgroup
constexpr int kPPBufferBytes = kPPStages * kPPStageBytes + 2 * kPPStagingBytes;
constexpr int kPPSmemBytes = kPPBufferBytes + 1024 /*align slack*/ + 256 /*barriers*/ + 2048 /*bias, C_out <= 512*/;

struct ConvPPParams {
  int P, Q, S, stride, pad_h, pad_w, cblocks, num_k_blocks, m_tiles, n_tiles;
  int relu;
  int has_residual;
  const float* bias;
};

__global__ void __launch_bounds__(kThreads, 1)
convpp_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                    const __grid_constant__ CUtensorMap map_res, const __grid_constant__ CUtensorMap map_out,
                    const ConvPPParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kPPStages * kATileBytes;
  uint8_t* staging = smem + kPPStages * kPPStageBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kPPBufferBytes);
  uint64_t* full_bar = bars;       // [kPPStages]
  uint64_t* empty_bar = bars + 8;  // [kPPStages]
  uint64_t* res_bar = bars + 16;   // [2], one per consumer warpgroup
  float* bias_s = reinterpret_cast<float*>(bars + 32);

  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);
  const int nk = p.num_k_blocks;
  const int items = p.m_tiles * p.n_tiles;
  for (int i = threadIdx.x; i < 128 * p.n_tiles; i += blockDim.x) bias_s[i] = p.bias[i];
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_out) : "memory");
    if (p.has_residual) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_res) : "memory");
    for (int i = 0; i < kPPStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);  // one arrive per warp of the consuming warpgroup
    }
    mbar_init(&res_bar[0], 1);
    mbar_init(&res_bar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  pdl_trigger();
  __syncthreads();
  pdl_wait();

  if (wg == 0) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int pq = p.P * p.Q;
      for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const int m_tile = item / p.n_tiles;
        const int n_tile = item - m_tile * p.n_tiles;
        const int m0 = m_tile * kBlockM;
        const int img = m0 / pq;
        const int rem = m0 - img * pq;
        const int p0 = rem / p.Q;
        const int q0 = rem - p0 * p.Q;
        const int base_w = q0 * p.stride - p.pad_w;
        const int base_h = p0 * p.stride - p.pad_h;
        int tap = 0, cb = 0;
        for (int kb = 0; kb < nk; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          mbar_expect_tx(&full_bar[stage], kPPStageBytes);
          const int r = tap / p.S;
          const int s = tap - r * p.S;
          tma_load_im2col_4d(smem_a + stage * kATileBytes, &map_a, &full_bar[stage], cb * kBlockK, base_w, base_h, img,
                             static_cast<uint16_t>(s), static_cast<uint16_t>(r));
          tma_load_2d(smem_b + stage * kATileBytes, &map_b, &full_bar[stage], kb * kBlockK, n_tile * 128);
          if (++cb == p.cblocks) {
            cb = 0;
            ++tap;
          }
          if (++stage == kPPStages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
  } else {
    // ===================== consumers: wgmma + staged epilogue =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;
    const int t = threadIdx.x & 127;
    const int lane = threadIdx.x & 31;
    const int row0 = 16 * (t >> 5) + (lane >> 2);  // + 64 mh + 8 h: the accumulator rows of this thread
    const int col = 2 * (lane & 3);                 // + 8 j: its column pair
    uint8_t* stage_buf = staging + cw * kPPStagingBytes;
    int local = 0;
    for (int i = cw, item = blockIdx.x + cw * gridDim.x; item < items; i += 2, item += 2 * gridDim.x, ++local) {
      const int m_tile = item / p.n_tiles;
      const int n0 = (item - m_tile * p.n_tiles) * 128;
      const int m0 = m_tile * kBlockM;
      if (p.has_residual && t == 0) {
        bulk_wait_read_all();  // the previous item's store has read the staging tile
        mbar_expect_tx(&res_bar[cw], kPPStagingBytes);
        tma_load_2d(stage_buf, &map_res, &res_bar[cw], n0, m0);
        tma_load_2d(stage_buf + kPPStagingBytes / 2, &map_res, &res_bar[cw], n0 + 64, m0);
      }
      // stage / phase from the CTA's k-block counter (both warpgroups' items, in item order), as in conv64_wgmma_kernel
      const uint32_t g = static_cast<uint32_t>(i) * static_cast<uint32_t>(nk);
      int stage = static_cast<int>(g % kPPStages);
      uint32_t phase = (g / kPPStages) & 1u;
      float acc0[64], acc1[64];  // rows 0-63 / 64-127 of the tile
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        acc0[j] = 0.f;
        acc1[j] = 0.f;
      }
      // mainloop hand-off: see conv64_wgmma_kernel
      if (i > 0) mainloop_turn_wait(cw);
      int prev_stage = -1;
#pragma unroll 1
      for (int kb = 0; kb < nk; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t da = make_sw128_desc(smem_u32(smem_a + stage * kATileBytes));
        const uint64_t db = make_sw128_desc(smem_u32(smem_b + stage * kATileBytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {  // 64 rows of 128 B = 8 KiB: +512 in the (addr >> 4) field
          wgmma_m64n128k16(acc0, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k), 1u);
          wgmma_m64n128k16(acc1, da + static_cast<uint64_t>(512 + 2 * k), db + static_cast<uint64_t>(2 * k), 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage can be refilled
        __syncwarp();
        if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == kPPStages) {
          stage = 0;
          phase ^= 1u;
        }
      }
      if (item + static_cast<int>(gridDim.x) < items) mainloop_turn_pass(cw);
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

      if (t == 0) bulk_wait_read_all();
      warpgroup_sync(cw);
      if (p.has_residual) mbar_wait(&res_bar[cw], static_cast<uint32_t>(local) & 1u);
      // staging tile: box c / 64 holds channels n0 + 64 (c / 64) .., row m at 128 m, 16-byte chunk k of the row at
      // (k ^ (m & 7)) * 16 (128B swizzle); a warp's 8 rows x 4 lanes hit 32 distinct banks
      const uint32_t sbase = smem_u32(stage_buf);
#pragma unroll
      for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = 64 * mh + row0 + 8 * h;
          const uint32_t rbase = sbase + static_cast<uint32_t>(row * 128 + col * 2);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const float2 b = *reinterpret_cast<const float2*>(bias_s + n0 + 8 * j + col);
            const float v0 = mh ? acc1[4 * j + 2 * h] : acc0[4 * j + 2 * h];
            const float v1 = mh ? acc1[4 * j + 2 * h + 1] : acc0[4 * j + 2 * h + 1];
            float f0 = v0 + b.x;
            float f1 = v1 + b.y;
            const uint32_t addr = rbase + static_cast<uint32_t>((j >> 3) * (kPPStagingBytes / 2) +
                                                                (((j & 7) ^ (row & 7)) << 4));
            if (p.has_residual) {
              uint32_t rr;
              asm volatile("ld.shared.b32 %0, [%1];" : "=r"(rr) : "r"(addr) : "memory");
              const float2 r = unpack_act2(rr);
              f0 += r.x;
              f1 += r.y;
            }
            if (p.relu) {
              f0 = fmaxf(f0, 0.f);
              f1 = fmaxf(f1, 0.f);
            }
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_act2(f0, f1)) : "memory");
          }
        }
      }
      fence_proxy_async_smem();
      warpgroup_sync(cw);
      if (t == 0) {
        tma_store_2d(&map_out, stage_buf, n0, m0);
        tma_store_2d(&map_out, stage_buf + kPPStagingBytes / 2, n0 + 64, m0);
        bulk_commit();
      }
    }
    if (t == 0) bulk_wait_all();
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
  const int smem = Cfg::smem_bytes(p.C_out);
  static int attr_bytes = 0;  // the largest dynamic shared-memory size set on this instantiation so far
  if (smem > attr_bytes) {
    MPX_CHECK_CUDA(cudaFuncSetAttribute(conv_wgmma_kernel<BLOCK_N>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_bytes = smem;
  }
  int grid = p.m_tiles * p.n_tiles * p.splits;
  const int cap = max_ctas > 0 ? max_ctas : sm_count();
  ProfileSlot* slot = profile_begin(stream);
  // split-K: one work item per CTA, the k-splits of a tile form a cluster
  if (p.splits == 1 && grid > cap) grid = cap;
  MPX_CHECK_CUDA(launch_pdl(conv_wgmma_kernel<BLOCK_N>, dim3(grid), dim3(kThreads), smem, stream, p.splits,
                            ma, mb, p));
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  profile_end(slot, stream, 2.0 * p.M_total * p.C_out * p.num_k_blocks * kBlockK);
  return MPX_OK;
}

int conv_out_dim(int in, int pad_lo, int pad_hi, int k, int stride) {
  return (in + pad_lo + pad_hi - k) / stride + 1;
}

// im2col map of the activations, 128-pixel boxes of 64 channels.  Dims are innermost-first: {C, W, H, N}.
static int encode_im2col_map(CUtensorMap* map, const ConvDesc& d, const void* x) {
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
  CUresult r = g_encode_im2col(map, kTmaActType, 4, const_cast<void*>(x),
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
    reinterpret_cast<uint64_t*>(map)[1] &= ~(1ull << 21);
  }
  return MPX_OK;
}

// row-major [rows, cols] act16 matrix, (box_cols x box_rows) boxes, 128B swizzle
static int encode_2d_map(CUtensorMap* map, const void* ptr, cuuint64_t cols, cuuint64_t rows, int box_cols, int box_rows,
                         CUtensorMapL2promotion promo) {
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode_tiled(map, kTmaActType, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, promo,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MPX_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", static_cast<int>(r));
  return MPX_OK;
}

// [n, H, W, C] act16 tensor, (64 x box_w x box_h x 1) boxes, 128B swizzle; out-of-range elements are zero-filled on load
// and clipped on store
static int encode_nhwc_map(CUtensorMap* map, const void* ptr, int n, int H, int W, int C, int box_w, int box_h) {
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H),
                        static_cast<cuuint64_t>(n)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(C) * 2, static_cast<cuuint64_t>(W) * C * 2,
                           static_cast<cuuint64_t>(H) * W * C * 2};
  cuuint32_t box[4] = {static_cast<cuuint32_t>(kBlockK), static_cast<cuuint32_t>(box_w), static_cast<cuuint32_t>(box_h),
                       1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_encode_tiled(map, kTmaActType, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MPX_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", static_cast<int>(r));
  return MPX_OK;
}

// The band producer serves stride 1 when one padded input row (Wp = W + both pads = Q + S - 1 pixels) fits a TMA box
// dimension and a ring slot, and a tile's cblocks bands leave a slot free for the producer to run ahead.
static bool conv64_band_fits(const ConvDesc& d) {
  const int wp = d.W + d.pad_lo_w + d.pad_hi_w;
  return d.stride == 1 && wp <= kC64Pixels && d.C_in / kBlockK <= kC64BandSlots - 1;
}

// Shared-memory layout of the band producer.  Every tile reuses the same weights, so when all k-blocks fit beside at least
// cblocks + 1 band slots and the two staging tiles (each sized to the tile), they are loaded once per CTA and stay
// resident: the stem's 128 KB and layer1's 72 KB would otherwise be refetched from L2 for every tile, more bytes than its
// bands.  Otherwise the weights go through a ring of 8 stages beside 3 slots of 32 KB.  A tap's B operand may read up to
// (N + S - 2) pixels past its slot's start for columns that are dropped; those reads must stay inside the layout.
static void conv64_band_layout(Conv64Params& p, int band_n, int S) {
  auto round1k = [](int b) { return (b + 1023) & ~1023; };
  const int slot = round1k(p.band_w * p.band_rows * 128);
  const int staging = round1k(p.band_rows * p.Q * 128);
  const int weights = p.num_k_blocks * kC64WBytes;
  const int reach = (band_n + S - 2) * 128 + 128;
  for (int slots = kC64BandSlots; slots >= p.cblocks + 1; --slots) {
    const int end = slots * slot + weights + 2 * staging;
    if (end <= kC64BufferBytes && (slots - 1) * slot + reach <= kC64BufferBytes) {
      p.band_slots = slots;
      p.slot_bytes = slot;
      p.w_resident = 1;
      p.w_off = slots * slot;
      p.staging_off = p.w_off + weights;
      p.staging_bytes = staging;
      return;
    }
  }
  p.band_slots = kC64BandSlots;
  p.slot_bytes = kC64ActBytes;
  p.w_resident = 0;
  p.w_off = kC64BandSlots * kC64ActBytes;
  p.staging_off = p.w_off + kC64BandWStages * kC64WBytes;
  p.staging_bytes = kC64StagingBytes;
}

static int conv64_forward(const ConvDesc& d, const void* x, const void* w, const float* bias, const void* residual,
                          void* out, int M_total, int P, int Q, int cap, cudaStream_t stream) {
  const int K_total = d.R * d.S * d.C_in;
  Conv64Params p{};
  p.M_total = M_total;
  p.P = P;
  p.Q = Q;
  p.S = d.S;
  p.stride = d.stride;
  p.pad_h = d.pad_lo_h;
  p.pad_w = d.pad_lo_w;
  p.cblocks = d.C_in / kBlockK;
  p.num_k_blocks = d.R * d.S * p.cblocks;
  p.relu = d.relu;
  p.has_residual = residual != nullptr;
  p.bias = bias;
  const bool band = conv64_band_fits(d) && (g_conv_mode & MPX_CONV_FORCE_IM2COL) == 0;
  int band_n = 0;
  CUtensorMap map_x, map_w, map_res, map_out;
  int rc;
  if (band) {
    p.band_w = d.W + d.pad_lo_w + d.pad_hi_w;
    p.band_rows = kC64Pixels / p.band_w < P ? kC64Pixels / p.band_w : P;
    p.tiles_per_img = (P + p.band_rows - 1) / p.band_rows;
    p.m_tiles = d.n_img * p.tiles_per_img;
    // the columns a tile's MMAs must cover: its last row ends (band_rows - 1) * Wp + Q columns in
    band_n = (p.band_rows - 1) * p.band_w + Q <= 160 ? 160 : 256;
    conv64_band_layout(p, band_n, d.S);
    rc = encode_nhwc_map(&map_x, x, d.n_img, d.H, d.W, d.C_in, p.band_w, p.band_rows);
    if (rc != MPX_OK) return rc;
    rc = encode_nhwc_map(&map_out, out, d.n_img, P, Q, 64, Q, p.band_rows);
    if (rc != MPX_OK) return rc;
    map_res = map_out;
    if (residual != nullptr) {
      rc = encode_nhwc_map(&map_res, residual, d.n_img, P, Q, 64, Q, p.band_rows);
      if (rc != MPX_OK) return rc;
    }
  } else {
    p.m_tiles = (M_total + kC64Pixels - 1) / kC64Pixels;
    rc = encode_im2col_map(&map_x, d, x);
    if (rc != MPX_OK) return rc;
    rc = encode_2d_map(&map_out, out, 64, M_total, 64, kC64Pixels, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
    if (rc != MPX_OK) return rc;
    map_res = map_out;
    if (residual != nullptr) {
      rc = encode_2d_map(&map_res, residual, 64, M_total, 64, kC64Pixels, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
      if (rc != MPX_OK) return rc;
    }
  }
  rc = encode_2d_map(&map_w, w, K_total, 64, kBlockK, 64, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc != MPX_OK) return rc;
  // the coarse / scoring (c_pad 16) and refiner (c_pad 32) stems skip their zero slices; wider c_pad issues every step
  const int stem_cblocks = (d.s2d_stem && d.R == 4 && d.S == 4 && p.cblocks <= 2) ? p.cblocks : 0;
  long long live_steps = 0;  // k16 steps per tile
  for (int kb = 0; kb < p.num_k_blocks; ++kb)
    live_steps += __builtin_popcount(stem_cblocks ? stem_live_steps(kb, p.cblocks, p.S) : 0xFu);

  typedef void (*Conv64Kernel)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, Conv64Params);
  // [stem cblocks][im2col, band n160, band n256]
  static const Conv64Kernel kernels[3][3] = {
      {conv64_wgmma_kernel<0, 0>, conv64_wgmma_kernel<0, 160>, conv64_wgmma_kernel<0, 256>},
      {conv64_wgmma_kernel<1, 0>, conv64_wgmma_kernel<1, 160>, conv64_wgmma_kernel<1, 256>},
      {conv64_wgmma_kernel<2, 0>, conv64_wgmma_kernel<2, 160>, conv64_wgmma_kernel<2, 256>}};
  static bool attr_set = false;
  if (!attr_set) {
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b)
        MPX_CHECK_CUDA(cudaFuncSetAttribute(kernels[a][b], cudaFuncAttributeMaxDynamicSharedMemorySize, kC64SmemBytes));
    attr_set = true;
  }
  const int grid = p.m_tiles < cap ? p.m_tiles : cap;
  ProfileSlot* slot = profile_begin(stream);
  const Conv64Kernel kernel = kernels[stem_cblocks][band_n == 0 ? 0 : (band_n == 160 ? 1 : 2)];
  MPX_CHECK_CUDA(launch_pdl(kernel, dim3(grid), dim3(kThreads), kC64SmemBytes, stream, 1, map_x, map_w, map_res, map_out,
                            p));
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  profile_end(slot, stream, 2.0 * M_total * 64 * live_steps * 16);
  return MPX_OK;
}

static int convpp_forward(const ConvDesc& d, const void* x, const void* w, const float* bias, const void* residual,
                          void* out, int M_total, int P, int Q, int cap, cudaStream_t stream) {
  ConvPPParams p{};
  p.P = P;
  p.Q = Q;
  p.S = d.S;
  p.stride = d.stride;
  p.pad_h = d.pad_lo_h;
  p.pad_w = d.pad_lo_w;
  p.cblocks = d.C_in / kBlockK;
  p.num_k_blocks = d.R * d.S * p.cblocks;
  p.m_tiles = (M_total + kBlockM - 1) / kBlockM;
  p.n_tiles = d.C_out / 128;
  p.relu = d.relu;
  p.has_residual = residual != nullptr;
  p.bias = bias;
  CUtensorMap map_a, map_b, map_res, map_out;
  int rc = encode_im2col_map(&map_a, d, x);
  if (rc != MPX_OK) return rc;
  rc = encode_2d_map(&map_b, w, static_cast<cuuint64_t>(p.num_k_blocks) * kBlockK, d.C_out, kBlockK, 128,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc != MPX_OK) return rc;
  rc = encode_2d_map(&map_out, out, d.C_out, M_total, 64, kBlockM, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
  if (rc != MPX_OK) return rc;
  map_res = map_out;
  if (residual != nullptr) {
    rc = encode_2d_map(&map_res, residual, d.C_out, M_total, 64, kBlockM, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
    if (rc != MPX_OK) return rc;
  }
  static bool attr_set = false;
  if (!attr_set) {
    MPX_CHECK_CUDA(cudaFuncSetAttribute(convpp_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPPSmemBytes));
    attr_set = true;
  }
  const int items = p.m_tiles * p.n_tiles;
  const int grid = items < cap ? items : cap;
  ProfileSlot* slot = profile_begin(stream);
  MPX_CHECK_CUDA(launch_pdl(convpp_wgmma_kernel, dim3(grid), dim3(kThreads), kPPSmemBytes, stream, 1, map_a, map_b,
                            map_res, map_out, p));
  MPX_CHECK_CUDA(cudaGetLastError());
  ++g_launches;
  profile_end(slot, stream, 2.0 * M_total * d.C_out * p.num_k_blocks * kBlockK);
  return MPX_OK;
}

// x: [n_img, H, W, C_in] act16; w: [C_out, R*S*C_in] act16 ((r,s,c) ordered); bias fp32 [C_out];
// residual/out: [n_img, P, Q, C_out] act16.
int conv_forward(const ConvDesc& d, const void* x, const void* w, const float* bias,
                 const void* residual, void* out, int block_n_override, int max_ctas,
                 cudaStream_t stream, int splitk, int max_c_out) {
  MPX_REQUIRE(d.C_in % 64 == 0 && d.C_in >= 64, "conv: C_in=%d must be a multiple of 64", d.C_in);
  MPX_REQUIRE(max_c_out <= 2048, "conv: C_out limit %d above 2048", max_c_out);
  MPX_REQUIRE(d.C_out % 64 == 0 && d.C_out <= max_c_out, "conv: C_out=%d must be a multiple of 64, at most %d", d.C_out,
              max_c_out);
  MPX_REQUIRE(d.stride == 1 || d.stride == 2, "conv: stride %d unsupported", d.stride);
  MPX_REQUIRE(d.R >= 1 && d.R <= 8 && d.S >= 1 && d.S <= 8, "conv: filter %dx%d unsupported", d.R, d.S);
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
    // conv is bound by the serial K loop of a single tile instead, so narrower tiles spread it over more SMs.
    // Start from the widest tile that divides C_out (C_out = 192, 320, 448: 64; 384: 128); halving keeps dividing it.
    const long long m_tiles_est = (M_total + kBlockM - 1) / kBlockM;
    block_n = d.C_out % 256 == 0 ? 256 : (d.C_out % 128 == 0 ? 128 : 64);
    while (block_n > 64 && m_tiles_est * (d.C_out / block_n) < 32) block_n /= 2;
  }
  MPX_REQUIRE((block_n == 64 || block_n == 128 || block_n == 256) && d.C_out % block_n == 0,
              "conv: BLOCK_N=%d invalid for C_out=%d", block_n, d.C_out);

  // C_out = 64 with enough 256-pixel tiles to give every CTA at least two (one per consumer warpgroup): the pixel-major
  // kernel.  MPX_CONV_NEVER_C64 never takes it, MPX_CONV_FORCE_C64 takes it whatever the size.  It loads its activations
  // by filter-row band where conv64_band_fits, by im2col otherwise (or under MPX_CONV_FORCE_IM2COL).
  const bool aligned = (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(residual) & 15) == 0;
  const long long tiles256 = (M_total + kC64Pixels - 1) / kC64Pixels;
  const int cap = max_ctas > 0 ? max_ctas : sm_count();
  if (d.C_out == 64 && block_n_override == 0 && splitk <= 0 && aligned && (g_conv_mode & MPX_CONV_NEVER_C64) == 0 &&
      ((g_conv_mode & MPX_CONV_FORCE_C64) != 0 || tiles256 >= 2LL * cap)) {
    // a heuristic K split (splitk < 0) only applies below 2 * SMs / 4 128-row tiles, far under this kernel's threshold;
    // with MPX_CONV_FORCE_C64 a shape it would split stays on the 128-row kernel
    const long long m_tiles128 = (M_total + kBlockM - 1) / kBlockM;
    const int nkb = d.R * d.S * (d.C_in / kBlockK);
    if (!(splitk < 0 && m_tiles128 * 2 <= cap && nkb >= 8))
      return conv64_forward(d, x, w, bias, residual, out, static_cast<int>(M_total), P, Q, cap, stream);
  }

  // C_out = 128 with at least two 128 x 128 tiles per CTA: the ping-pong kernel.  C_out = 256 and 512 keep the 128 x 256
  // tiles of the 128-row kernel by default: a 128-wide tile fills 32 KB of shared memory per 128 x 128 x 64 block where
  // those fill 48 KB per twice the work, and on an H100 that costs the 3x3 convolutions of layers 3 and 4 more than the
  // overlapped epilogue gains (DESIGN 3.1).  MPX_CONV_NEVER_PP never takes it, MPX_CONV_FORCE_PP takes it for every C_out
  // it serves (multiples of 128 up to 512), whatever the size, except for a shape the small-batch heuristic splits over K.
  const long long m_tiles = (M_total + kBlockM - 1) / kBlockM;
  if (d.C_out % 128 == 0 && d.C_out <= 512 && block_n_override == 0 && splitk <= 0 && aligned &&
      (g_conv_mode & MPX_CONV_NEVER_PP) == 0 &&
      ((g_conv_mode & MPX_CONV_FORCE_PP) != 0 || (d.C_out == 128 && m_tiles >= 2LL * cap))) {
    const int nkb = d.R * d.S * (d.C_in / kBlockK);
    if (!(splitk < 0 && m_tiles * (d.C_out / block_n) * 2 <= cap && nkb >= 8))
      return convpp_forward(d, x, w, bias, residual, out, static_cast<int>(M_total), P, Q, cap, stream);
  }

  // --- activation map (im2col): 128-pixel boxes of 64 channels
  CUtensorMap map_a, map_b;
  rc = encode_im2col_map(&map_a, d, x);
  if (rc != MPX_OK) return rc;
  rc = encode_2d_map(&map_b, w, static_cast<cuuint64_t>(d.R) * d.S * d.C_in, d.C_out, kBlockK, block_n,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc != MPX_OK) return rc;

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
    // MPX_CONV_SPLITK_CAP2 / _CAP1 cap the automatic split at 2 / 1: fewer, longer CTAs -- less SM time per layer at a
    // higher latency, the better trade when another frame's kernels fill the device beside this one (frame_pipeline.py)
    const int cap = (splitk < 0 && (g_conv_mode & MPX_CONV_SPLITK_CAP1))
                        ? 1
                        : ((splitk < 0 && (g_conv_mode & MPX_CONV_SPLITK_CAP2)) ? 2 : 8);
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
