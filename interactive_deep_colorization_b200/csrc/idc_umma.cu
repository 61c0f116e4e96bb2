// wgmma engine: implicit-GEMM convolution on the Hopper tensor cores (sm_90a).
//
//   D[128 pixels x BN couts] (FP32, registers) += A[128 x 64] (smem, K-major, SW128) * B[BN x 64]^T
//
// * A tiles are gathered by TMA straight from the NHWC activation planes: one 4-D box
//   {64 ch, wbox, hbox, 1 image} per filter tap, shifted by the tap offset; out-of-bounds
//   pixels are zero-filled by TMA (= the reference's zero padding), the `::2` decimation
//   (model.py:149-151) and the output-parity views of the transposed convs are expressed as
//   tensor-map strides, so no im2col / decimated copy ever exists in HBM.
// * 1e-3 ab parity needs ~22 mantissa bits (SURVEY 7.3): activations and weights are stored as
//   FP16 hi + lo planes and every product is issued as 3 MMAs (hi*hi + hi*lo + lo*hi).
//   IDC_FLAG_FAST_FP16 drops the lo planes (1 MMA).
// * The tensor core's FP32 accumulation is not round-to-nearest, so a long K summed entirely inside it drifts.
//   Accumulation is therefore CHUNKED: wgmma sums `chunk_kb` k-blocks (12 MMAs each, the 8 small cross terms
//   first) into a fresh register accumulator, which is then added into the tile's FP32 accumulator with
//   round-to-nearest CUDA-core adds.
// * warp roles: warpgroup 0 = TMA producer (warp 0; the other three idle and give their registers away),
//   warpgroups 1-2 = MMA + accumulate + epilogue, each owning 64 of the tile's 128 pixel rows (one m64 wgmma per
//   K step).  Persistent grid = min(work items, #SM).
// * also in this file: deterministic split-K for launches that cannot fill the machine (the CTA's own pieces never
//   leave its registers) and conv1_1_umma_kernel (model1.0 as one padded k-block whose operand rows the threads
//   write themselves).
#include <stdio.h>
#include <stdlib.h>

#include "idc_internal.h"

namespace idc {

constexpr int kBM = 128;        // pixels per tile (two m64 wgmma row blocks)
constexpr int kBK = 64;         // channels per k-block (128 bytes of FP16 = one SW128 row)
constexpr int kThreads = 384;   // producer warpgroup + 2 MMA / epilogue warpgroups
constexpr int kProdRegs = 40;   // setmaxnreg budgets: the producer warpgroup gives its registers to the math warpgroups
constexpr int kMathRegs = 232;
constexpr int kMathThreads = 256;

struct UmmaParams {
  const CUtensorMap* amaps;  // device array, [view][hi, lo]
  const int4* kblk;          // [ncls][nkb] : {map index (hi), c0, dy, dx}
  int nkb, ncls;
  int chunk_kb;              // k-blocks accumulated inside the tensor core per chunk (>=1)
  int split_k;               // >1: K is split over `split_k` CTAs per tile (small-batch latency path)
  float* ws;                 // split-K partial sums [work item][BN/2 registers][256 threads] FP32
  int* counters;             // split-K arrival counters [tile] (self-resetting)
  int n_img, tiles_y, tiles_x, n_tiles_n, total_tiles;
  int hbox, wbox, wshift;
  int Hl, Wl, cout_pad;
  const float* bias;   // bias / descale
  const float* scale;  // bn_scale * descale
  const float* shift;
  const float* gadd;   // [n_img][gadd_ld] or null
  int gadd_ld;
  float gadd_mult;     // output buffer's storage scale 2^S_out, applied to the global-hints vector
  int act;
  __half* out_hi;
  __half* out_lo;
  int Hout, Wout, Cout, os;
  float* out_f32;      // logits [M][out_ld] or null
  int out_ld;
  const float* wout;   // fused head weights [2][128] or null
  const float* bout;
  float* out_ab;
  float out_mult;
  int* err;
  unsigned* range;     // the context's range word: range_bit is set when a stored value exceeds FP16's 65504
  unsigned range_bit;
  int n_amaps;         // entries of `amaps` (prefetched in the prologue)
  int max_ctas;        // host side only: grid cap for side-branch launches
  int img0;            // first image of this launch (n_img = img0 + images of the launch): idc_forward_host
                       // runs the last op in image chunks so that the D2H of a chunk overlaps the next one
};

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok;
}
// Bounded wait: a protocol bug becomes an error code + trap instead of a hung GPU.
__device__ __noinline__ void mbar_timeout(int* err, int code) {
  if (err) {
    atomicExch(err, code);
    __threadfence_system();
  }
  __trap();
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* err, int code) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 6000000000LL) mbar_timeout(err, code);
  }
}

// one lane of a converged warp (warp-uniform control flow keeps descriptors / addresses in uniform
// registers; a role wrapped in `if (lane == 0)` makes ptxas re-broadcast every operand per instruction)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}

// ---- clusters of two CTAs (pairs) ----
__device__ __forceinline__ void tma_load_2d_mc(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1) {
  // the box lands at the same shared-memory offset in both CTAs of the cluster and signals both CTAs' `bar`
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "h"((uint16_t)3)
      : "memory");
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
__device__ __forceinline__ void mbar_arrive_remote(uint32_t local_bar, uint32_t rank) {   // the same barrier in CTA `rank`
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(local_bar), "r"(rank)
      : "memory");
}

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization attribute may
// start while its predecessor is still running; everything that depends on the predecessor's output sits behind
// pdl_wait().  Every thread of every kernel of a forward executes pdl_wait() before it exits, so "kernel k is
// complete" implies "kernels 0..k-1 are complete" (completion stays transitive along the chain).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

// ---- wgmma (warpgroup MMA): D[64 x N] (registers) += A[64 x 16] (smem) * B[N x 16]^T (smem), both K-major ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// The accumulator registers are tied to the asm statements ("+f"); after wgmma_wait they are plain registers again.
template <int R>
__device__ __forceinline__ void wgmma_reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

template <int BN>
__device__ __forceinline__ void wgmma_bn(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (BN == 128) wgmma_n128(d, adesc, bdesc, accumulate);
  else wgmma_n64(d, adesc, bdesc, accumulate);
}

// K-major, 128-byte-swizzled operand tile: rows of 64 FP16 (128 B), 8-row swizzle atoms 1024 B apart (SBO);
// LBO unused for a single K atom.  sm_90 wgmma descriptor: layout type 1 (SWIZZLE_128B) in bits 62-63.
// Advancing the start address by 32 B (2 units) selects the next K=16 slice inside the swizzle atom.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr, uint32_t sbo = 1024u) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);  // start address
  d |= (uint64_t)1 << 16;                       // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(sbo >> 4) << 32;              // stride byte offset (pitch of the 8-row groups)
  d |= (uint64_t)1 << 62;                       // SWIZZLE_128B
  return d;
}

// two floats -> packed f16x2 (low half = a), saturating to +-65504 instead of inf (one F2FP instruction)
__device__ __forceinline__ uint32_t pack_f16x2_sat(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// hi = f16(a, b); lo = f16(a - hi, b - hi)
__device__ __forceinline__ uint32_t lo_f16x2(float a, float b, uint32_t hw) {
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw));
  return pack_f16x2_sat(a - hf.x, b - hf.y);
}
// Range check of the FP16 stores: a running max of |h| over packed pairs (two calls fuse into one VHMNMX), and whether
// it reached 65504, FP16's largest value: the value rounded to it (|v| >= 65488) or saturated there (|v| > 65504).
__device__ __forceinline__ uint32_t habs_max2(uint32_t m, uint32_t w) {
  const __half2 r = __hmax2(*reinterpret_cast<const __half2*>(&m), __habs2(*reinterpret_cast<const __half2*>(&w)));
  return *reinterpret_cast<const uint32_t*>(&r);
}
__device__ __forceinline__ bool f16_top(uint32_t m) {     // m: a habs_max2 result (sign bits clear)
  return ((m & 0xFFFFu) >= kF16MaxBits) | ((m >> 16) >= kF16MaxBits);
}

__device__ __forceinline__ void split_h(float v, __half& hi, __half& lo) {
  v = fminf(fmaxf(v, -65504.f), 65504.f);
  hi = __float2half_rn(v);
  lo = __float2half_rn(v - __half2float(hi));
}

// Register fragment of one m64nN wgmma accumulator, thread t of the warpgroup (warp wi = t / 32, lane l):
// register i holds row 16*wi + l/4 + 8*((i >> 1) & 1), column 8*(i >> 2) + 2*(l & 3) + (i & 1).
__device__ __forceinline__ int frag_col(int i, int lane) { return 8 * (i >> 2) + 2 * (lane & 3) + (i & 1); }

// HALO (stride-1 3x3 layers): instead of one TMA box per filter tap, ONE halo tile of 18 rows x 10 pixels per
// 64-channel input group serves all 9 taps of a 16-row x 8-pixel M-tile -- the wgmma A descriptor starts at the
// pixel-shifted window (start = slot + ((dy+1)*10 + dx+1)*128 B, SBO = 10*128 B: one 8-pixel image row per core-matrix
// group; the 128-byte swizzle is a function of the absolute shared-memory address, so the base-offset field stays 0 --
// the halo tests fail with it set to the start's row phase).  The stage ring then holds weight tiles only.
constexpr int kHaloW = 10, kHaloH = 18;
constexpr int kHaloPlane = (kHaloW * kHaloH * 128 + 1023) / 1024 * 1024;   // 23040 -> 23552


template <int BN, int MT, int CG, bool SPLIT, bool HALO>
struct SmemPlan {
  static constexpr int kABytes = MT * kBM * kBK * 2;            // MT M-tiles of 128 pixels x 64 ch FP16 (16 KB each)
  static constexpr int kAStage = HALO ? 0 : kABytes;            // A bytes inside a ring stage (one plane)
  static constexpr int kBBytes = BN * kBK * 2;                  // the whole weight tile (pairs: half of it multicast by each CTA)
  static constexpr int kStageBytes = (SPLIT ? 2 : 1) * (kAStage + kBBytes);
  static constexpr int kHaloSlot = (SPLIT ? 2 : 1) * kHaloPlane;
  static constexpr int kHaloBytes = HALO ? 2 * kHaloSlot : 0;   // two halo slots (double buffered)
  static constexpr int kOutRow = 64 * 2 + 16;                   // epilogue staging: 64 FP16 columns + 16 B pad per row
  static constexpr int kOutWarp = 16 * kOutRow;                 // one warp's 16 rows
  static constexpr int kOutStage = 8 * kOutWarp;
  static constexpr int kTail = 3 * BN * 4 + 272 * 4 + 256;      // epi vecs, head, barriers
  static constexpr int kBudget = 232448 - 1024 - kTail - kOutStage - kHaloBytes;   // 227 KB opt-in limit minus alignment slack
  static constexpr int kStages = kBudget / kStageBytes >= 4 ? 4 : kBudget / kStageBytes;
  static constexpr int kTotal = kStages * kStageBytes + kHaloBytes + kOutStage + kTail + 1024;
  static_assert(kStages >= 2, "need at least a double-buffered operand ring");
  static_assert(MT * BN <= 128, "register budget: chunk + tile accumulators of MT*BN columns per math thread pair");
  static_assert(!HALO || MT == 1, "halo tiles are single 16x8-pixel M-tiles");
  static_assert(CG == 1 || CG == 2, "clusters of one or two CTAs");
};

// ------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------
// CG == 2 (pairs): a cluster of two CTAs works on two M-tiles (pixel tiles 2*pair and 2*pair + 1) of the same n-tile and
// K range; each CTA loads its own A tile and HALF of the weight tile, multicast into both CTAs' shared memory, so the
// weight tile crosses L2 -> SM once per pair.  A ring stage is refilled only when the MMA warps of BOTH CTAs have
// released it (each math warp arrives on the stage's `empty` barrier in both CTAs).  An odd number of M-tiles leaves
// one dummy tile (image index past the batch: loads zero-filled or ignored, nothing stored).
template <int BN, int MT, int CG, bool SPLIT, bool HALO>
__global__ void __launch_bounds__(kThreads, 1)
umma_conv_kernel(const __grid_constant__ CUtensorMap bmap_hi, const __grid_constant__ CUtensorMap bmap_lo,
                 const __grid_constant__ UmmaParams p) {
  using SP = SmemPlan<BN, MT, CG, SPLIT, HALO>;
  constexpr int STAGES = SP::kStages;
  constexpr int R = BN / 2;                                       // accumulator registers per thread and M-tile half
  constexpr bool PAIR = CG == 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_halo = smem + STAGES * SP::kStageBytes;             // HALO: 2 slots x {hi, lo} planes, 1024-aligned
  uint8_t* s_out = s_halo + SP::kHaloBytes;
  float* s_bias = reinterpret_cast<float*>(s_out + SP::kOutStage);
  float* s_scale = s_bias + BN;
  float* s_shift = s_scale + BN;
  float* s_head = s_shift + BN;                                   // [2][128] + bias[2] (+pad)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_head + 272);   // [STAGES] TMA -> MMA
  uint64_t* empty_bar = full_bar + 4;                               // [STAGES] MMA warps (of both CTAs) -> TMA
  uint64_t* afull_bar = full_bar + 8;                               // [2] HALO: halo TMA -> MMA
  uint64_t* aempty_bar = full_bar + 10;                             // [2] HALO: MMA warps -> halo TMA

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t cta_rank = PAIR ? cluster_ctarank() : 0u;

  // ---- one-time setup ----
  if (p.wout) {
    for (int i = threadIdx.x; i < 256; i += kThreads) s_head[i] = p.wout[i];
    if (threadIdx.x < 2) s_head[256 + threadIdx.x] = p.bout[threadIdx.x];
  }
  if (threadIdx.x == 32) {                          // descriptors are input-independent: fetch them during the prologue
    prefetch_tmap(&bmap_hi);
    if (SPLIT) prefetch_tmap(&bmap_lo);
    for (int i = 0; i < p.n_amaps; ++i) prefetch_tmap(p.amaps + i);
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), 8 * CG);   // one arrive per MMA warp of every CTA the stage's weights went to
    }
    if (HALO)
      for (int a = 0; a < 2; ++a) {
        mbar_init(smem_u32(&afull_bar[a]), 1);
        mbar_init(smem_u32(&aempty_bar[a]), 8);
      }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (PAIR) cluster_sync_all(); else __syncthreads();   // pairs: the peer's barriers exist before anything arrives on them
  pdl_launch_dependents();                          // the next kernel of the forward may start its own prologue
  pdl_wait();                                       // activations of the previous layer are complete and visible

  const int tiles_per_img = p.tiles_y * p.tiles_x;
  const int S = p.split_k;
  const int n_items = p.total_tiles * S;
  const int w0 = blockIdx.x / CG, wstep = gridDim.x / CG;

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProdRegs));
    if (warp == 0) {
      // =============================== TMA producer ===============================
      int stage = 0;
      uint32_t phase = 0;
      uint32_t hcount = 0;                               // HALO: halo loads issued (slot = hcount & 1)
      for (int w = w0; w < n_items; w += wstep) {
        const int tile = w / S, ks = w - tile * S;
        const int kbeg = (ks * p.nkb) / S, kend = ((ks + 1) * p.nkb) / S;
        // tile order: n-tile fastest, then output-parity class, then spatial tile, then image -- CTAs that
        // run together share the A tile (all n-tiles) and the source rows (all 4 classes of an up-layer).
        // Pairs: `tile` counts M-tile PAIRS; this CTA takes M-tile 2*pair + rank.
        int r = tile;
        const int nt = r % p.n_tiles_n;
        r /= p.n_tiles_n;
        const int cls = r % p.ncls;
        r /= p.ncls;
        if (PAIR) r = 2 * r + (int)cta_rank;
        const int img_rel = r / tiles_per_img;
        r -= img_rel * tiles_per_img;
        const int img = p.img0 + img_rel;
        const int y0 = (r / p.tiles_x) * (p.hbox * MT), x0 = (r % p.tiles_x) * p.wbox;
        const int brow = cls * p.cout_pad + nt * BN + (int)cta_rank * (BN / CG);
        const int4* kb = p.kblk + cls * p.nkb;                // read-only table in global memory (L1-resident)
        for (int k = kbeg; k < kend; ++k) {
          if (HALO && k % 9 == 0) {                            // k-block i = (input group i / 9, tap i % 9)
            const uint32_t slot = hcount & 1, hphase = (hcount >> 1) & 1;
            ++hcount;
            mbar_wait(smem_u32(&aempty_bar[slot]), hphase ^ 1, p.err, 6);
            if (elect_one()) {
              const uint32_t fa = smem_u32(&afull_bar[slot]);
              const uint32_t sh = smem_u32(s_halo + slot * SP::kHaloSlot);
              const int c0 = (k / 9) * kBK;
              mbar_expect_tx(fa, (SPLIT ? 2 : 1) * kHaloW * kHaloH * 128);
              tma_load_4d(sh, p.amaps, fa, c0, x0 - 1, y0 - 1, img);
              if (SPLIT) tma_load_4d(sh + kHaloPlane, p.amaps + 1, fa, c0, x0 - 1, y0 - 1, img);
            }
            __syncwarp();
          }
          mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1, p.err, 1);
          if (elect_one()) {
            const uint32_t fb = smem_u32(&full_bar[stage]);
            const int4 e = __ldg(kb + k);
            const uint32_t sa = smem_u32(smem + stage * SP::kStageBytes);
            const uint32_t sb = sa + (SPLIT ? 2 : 1) * SP::kAStage + cta_rank * (BN / CG) * 128;
            const int kcol = HALO ? e.y : k * kBK;
            mbar_expect_tx(fb, SP::kStageBytes);                // pairs: the peer's multicast half lands here too
            if (!HALO) {
              const CUtensorMap* am = p.amaps + e.x;
              tma_load_4d(sa, am, fb, e.y, x0 + e.w, y0 + e.z, img);
              if (SPLIT) tma_load_4d(sa + SP::kABytes, am + 1, fb, e.y, x0 + e.w, y0 + e.z, img);
            }
            if (PAIR) {
              tma_load_2d_mc(sb, &bmap_hi, fb, kcol, brow);
              if (SPLIT) tma_load_2d_mc(sb + SP::kBBytes, &bmap_lo, fb, kcol, brow);
            } else {
              tma_load_2d(sb, &bmap_hi, fb, kcol, brow);
              if (SPLIT) tma_load_2d(sb + SP::kBBytes, &bmap_lo, fb, kcol, brow);
            }
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ====================== MMA + accumulate + epilogue (2 warpgroups) ======================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kMathRegs));
    const int et = threadIdx.x - 128;                 // 0..255
    const int wg = et >> 7;                           // which half of the tile's rows (MT*64 rows each)
    const int wi = (et >> 5) & 3;                     // warp inside the warpgroup: rows 16*wi .. 16*wi+15 of a 64-row block
    const uint32_t wbuf = smem_u32(s_out) + (uint32_t)(et >> 5) * SP::kOutWarp;
    auto release = [&](uint64_t* bar) {               // one arrive per warp, on this CTA's barrier and (pairs) the peer's
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(smem_u32(bar));
        if (PAIR) mbar_arrive_remote(smem_u32(bar), cta_rank ^ 1u);
      }
    };
    int stage = 0;
    uint32_t phase = 0;
    uint32_t hcount = 0;                              // HALO: halo tiles consumed
    int staged_key = -1;
    bool sat = false;                                 // a value this thread stored reached FP16's largest value
    for (int w = w0; w < n_items; w += wstep) {
      const int tile = w / S, ks = w - tile * S;
      const int kbeg = (ks * p.nkb) / S, kend = ((ks + 1) * p.nkb) / S;
      int r = tile;
      const int nt = r % p.n_tiles_n;
      r /= p.n_tiles_n;
      const int cls = r % p.ncls;
      r /= p.ncls;
      if (PAIR) r = 2 * r + (int)cta_rank;
      const int img_rel = r / tiles_per_img;
      r -= img_rel * tiles_per_img;
      const int img = p.img0 + img_rel;
      const int ty0 = (r / p.tiles_x) * (p.hbox * MT), tx0 = (r % p.tiles_x) * p.wbox;
      const int n0 = nt * BN;
      // stage this tile's per-channel epilogue vectors -- only when they change (n-tile, or image when a
      // global-hints vector is added); for the single-n-tile layers that is once per kernel
      const int vkey = p.gadd ? (img * p.n_tiles_n + nt) : nt;
      if (vkey != staged_key) {
        asm volatile("bar.sync 1, 256;" ::: "memory");      // previous tile's readers are done
        for (int i = et; i < BN; i += kMathThreads) {
          s_bias[i] = p.bias[n0 + i];
          s_scale[i] = p.scale[n0 + i];
          // pairs: the dummy tile of an odd tile count has img == n_img -> clamp (its rows are never stored)
          const int gi = img < p.n_img ? img : p.n_img - 1;
          s_shift[i] = p.shift[n0 + i] + (p.gadd ? p.gadd[(size_t)gi * p.gadd_ld + n0 + i] * p.gadd_mult : 0.f);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        staged_key = vkey;
      }

      float acc[MT][R];
#pragma unroll
      for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int j = 0; j < R; ++j) acc[m][j] = 0.f;
      for (int k0 = kbeg; k0 < kend; k0 += p.chunk_kb) {
        const int k1 = (k0 + p.chunk_kb < kend) ? k0 + p.chunk_kb : kend;
        float part[MT][R];
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
          for (int j = 0; j < R; ++j) part[m][j] = 0.f;
        int prev = -1;
        for (int k = k0; k < k1; ++k) {
          uint32_t hslot = 0;
          if (HALO) {
            if (k % 9 == 0) {
              mbar_wait(smem_u32(&afull_bar[hcount & 1]), (hcount >> 1) & 1, p.err, 7);
              ++hcount;
            }
            hslot = (hcount - 1) & 1;
          }
          mbar_wait(smem_u32(&full_bar[stage]), phase, p.err, 3);
          const uint32_t st0 = smem_u32(smem + stage * SP::kStageBytes);
          const uint32_t sb = st0 + (SPLIT ? 2 : 1) * SP::kAStage;
          const uint64_t b_hi = make_sw128_desc(sb), b_lo = make_sw128_desc(sb + SP::kBBytes);
          uint32_t ha = 0;                                   // HALO: this tap's window (this warpgroup's 8 image rows)
          if (HALO) {
            const int4 e = __ldg(p.kblk + k);
            ha = smem_u32(s_halo + hslot * SP::kHaloSlot) + (uint32_t)((e.z + wg * 8) * kHaloW + e.w) * 128u;
          }
          wgmma_fence();
#pragma unroll
          for (int m = 0; m < MT; ++m) {
            const uint32_t sa = st0 + (uint32_t)(wg * MT + m) * (64 * 128);
            const uint64_t a_hi = HALO ? make_sw128_desc(ha, kHaloW * 128) : make_sw128_desc(sa);
            const uint64_t a_lo = HALO ? make_sw128_desc(ha + kHaloPlane, kHaloW * 128) : make_sw128_desc(sa + SP::kABytes);
            uint32_t first = (k == k0) ? 0u : 1u;            // first MMA of a chunk overwrites the chunk accumulator
            if (SPLIT) {
              // the 8 small cross terms first (accumulator still tiny -> their truncation is harmless),
              // then the 4 dominant hi*hi terms
#pragma unroll
              for (int kk = 0; kk < kBK / 16; ++kk) {
                const uint64_t adv = (uint64_t)(kk * 2);   // 16 FP16 = 32 bytes = 2 descriptor units
                wgmma_bn<BN>(part[m], a_lo + adv, b_hi + adv, first);
                wgmma_bn<BN>(part[m], a_hi + adv, b_lo + adv, 1u);
                first = 1u;
              }
            }
#pragma unroll
            for (int kk = 0; kk < kBK / 16; ++kk) {
              const uint64_t adv = (uint64_t)(kk * 2);
              wgmma_bn<BN>(part[m], a_hi + adv, b_hi + adv, first);
              first = 1u;
            }
          }
          wgmma_commit();
          if (HALO && k % 9 == 8) {                          // last tap of the group: the halo slot is free once it retires
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_u32(&aempty_bar[hslot]));
          }
          if (prev >= 0) {                                   // the previous k-block's MMAs have retired: free its stage
            wgmma_wait<1>();
            release(&empty_bar[prev]);
          }
          prev = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int m = 0; m < MT; ++m) wgmma_reg_fence(part[m]);
        release(&empty_bar[prev]);
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
          for (int j = 0; j < R; ++j) acc[m][j] += part[m][j];   // FP32 round-to-nearest
      }

      // ---- split-K (MT == 1, single CTAs): park the partial tile in the workspace, wait until all S slices of this
      //      tile have arrived (they are co-resident: work items <= #SMs by construction), then every CTA reduces and
      //      finishes ITS share of the 32-column pieces (piece % S == ks), adding the other slices to its own in
      //      slice order (deterministic).  Arrive/depart counters reset themselves for the next launch / graph replay.
      //      Register i belongs to piece i / 16 (columns 8*(i/4) ..); the layout [item][register][thread] keeps
      //      every park / fetch instruction one coalesced 1 KB line. ----
      if (S > 1) {
        float* wp = p.ws + (size_t)w * R * kMathThreads + et;
#pragma unroll
        for (int i = 0; i < R; ++i)
          if ((i >> 4) % S != ks) __stcg(wp + (size_t)i * kMathThreads, acc[0][i]);
        __threadfence();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (et == 0) {
          int* cnt = p.counters + 2 * tile;
          atomicAdd(cnt, 1);
          const long long t0 = clock64();
          int seen;
          do {
            asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(cnt) : "memory");
            if (seen < S && clock64() - t0 > 6000000000LL) mbar_timeout(p.err, 5);
          } while (seen < S);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        for (int q = 0; q < S; ++q) {
          if (q == ks) continue;
          const float* rp = p.ws + (size_t)(tile * S + q) * R * kMathThreads + et;
#pragma unroll
          for (int i = 0; i < R; ++i)
            if ((i >> 4) % S == ks) acc[0][i] += __ldcg(rp + (size_t)i * kMathThreads);
        }
      }

      // ---- epilogue: v = act(acc + bias) * scale + shift on the register fragment, one 64-row block at a time ----
      const float neg_slope = p.act == ACT_RELU ? 0.f : (p.act == ACT_LEAKY02 ? 0.2f : 1.f);
      unsigned own = ~0u;                               // the 32-column pieces this work item stores (split-K: 1 in S)
      if (S > 1) {
        own = 0u;
#pragma unroll
        for (int pc = 0; pc < BN / 32; ++pc) own |= (pc % S == ks ? 1u : 0u) << pc;
      }
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        const int blk = (wg * MT + m) * 64;             // first tile row of this 64-row block
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const int c = frag_col(i, lane);
          // one branch-free form for none / ReLU / LeakyReLU(0.2): max(t, slope*t) with slope = 1 / 0 / 0.2
          const float t = acc[m][i] + s_bias[c];
          acc[m][i] = fmaf(fmaxf(t, neg_slope * t), s_scale[c], s_shift[c]);
        }
        int ry[2], rx[2];
        bool ok[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int rr = blk + wi * 16 + (lane >> 2) + 8 * h;
          ry[h] = ty0 + (rr >> p.wshift);
          rx[h] = tx0 + (rr & (p.wbox - 1));
          ok[h] = ry[h] < p.Hl && rx[h] < p.Wl && img < p.n_img;
        }
        if (p.wout) {
          // fused model_out: conv1x1(128->2) + tanh, x110 (model.py:108-109,175); a pixel's 128 columns live in the
          // 4 lanes of a quad
          float h0[2] = {0.f, 0.f}, h1[2] = {0.f, 0.f};
#pragma unroll
          for (int i = 0; i < R; ++i) {
            const int c = frag_col(i, lane), h = (i >> 1) & 1;
            h0[h] = fmaf(acc[m][i], s_head[c], h0[h]);
            h1[h] = fmaf(acc[m][i], s_head[128 + c], h1[h]);
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
              h0[h] += __shfl_xor_sync(0xffffffffu, h0[h], o);
              h1[h] += __shfl_xor_sync(0xffffffffu, h1[h], o);
            }
            if ((lane & 3) == 0 && ok[h]) {
              const size_t HW = (size_t)p.Hl * p.Wl;
              const size_t o = (size_t)img * 2 * HW + (size_t)ry[h] * p.Wl + rx[h];
              p.out_ab[o] = tanhf(h0[h] + s_head[256]) * p.out_mult;    // out_mult = 110 (model.py:175) or 100 (Caffe spec)
              p.out_ab[o + HW] = tanhf(h1[h] + s_head[257]) * p.out_mult;
            }
          }
        } else if (p.out_f32) {
#pragma unroll
          for (int i = 0; i < R; i += 2) {
            const int h = (i >> 1) & 1;
            if ((S > 1 && (i >> 4) % S != ks) || !ok[h]) continue;   // another CTA of the split finishes this piece
            float* o = p.out_f32 + ((size_t)(img * p.Hl + ry[h]) * p.Wl + rx[h]) * p.out_ld + n0 + frag_col(i, lane);
            *reinterpret_cast<float2*>(o) = make_float2(acc[m][i], acc[m][i + 1]);
          }
        } else {
          // FP16 hi / lo planes: the warp's 16 rows x 64 columns go through a private smem tile (rows padded by 16 B:
          // conflict-free both ways) so that each store instruction writes 16-byte chunks of 4 whole pixel rows
          // instead of 4-byte pieces of 8.
          __half* prow[4];
          const int rl0 = lane >> 3, ch = lane & 7;          // read side: rows rl0 + 4*it, 16-byte chunk ch
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const int rr = blk + wi * 16 + rl0 + 4 * it;
            const int yy = ty0 + (rr >> p.wshift), xx = tx0 + (rr & (p.wbox - 1));
            const bool v = yy < p.Hl && xx < p.Wl && img < p.n_img;
            prow[it] = v ? p.out_hi + ((size_t)(img * p.Hout + yy * p.os + (cls >> 1)) * p.Wout + xx * p.os + (cls & 1)) * p.Cout +
                               n0 + ch * 8
                         : nullptr;
          }
          const ptrdiff_t lo_delta = SPLIT ? p.out_lo - p.out_hi : 0;
          // range check: max |hi| per row half and 32-column piece over the packed hi words (one VHMNMX per four
          // values); only the rows and pieces this CTA stores count
          uint32_t hmax[2][BN / 32] = {};
#pragma unroll
          for (int sl = 0; sl < BN / 64; ++sl) {              // 64-column slabs = registers 32*sl .. 32*sl+31
            if (S > 1 && ((2 * sl) % S != ks) && ((2 * sl + 1) % S != ks)) continue;
#pragma unroll
            for (int plane = 0; plane < (SPLIT ? 2 : 1); ++plane) {
#pragma unroll
              for (int i = 32 * sl; i < 32 * sl + 32; i += 2) {
                const uint32_t hw = pack_f16x2_sat(acc[m][i], acc[m][i + 1]);
                if (plane == 0) hmax[(i >> 1) & 1][i >> 4] = habs_max2(hmax[(i >> 1) & 1][i >> 4], hw);
                const uint32_t v = plane == 0 ? hw : lo_f16x2(acc[m][i], acc[m][i + 1], hw);
                const int rl = (lane >> 2) + 8 * ((i >> 1) & 1), cl = frag_col(i, lane) - 64 * sl;
                st_shared_u32(wbuf + rl * SP::kOutRow + cl * 2, v);
              }
              __syncwarp();
#pragma unroll
              for (int it = 0; it < 4; ++it) {
                const uint4 v = ld_shared_v4(wbuf + (rl0 + 4 * it) * SP::kOutRow + ch * 16);
                const int piece = (64 * sl + ch * 8) >> 5;
                if (prow[it] && (S == 1 || piece % S == ks))
                  *reinterpret_cast<uint4*>(prow[it] + (plane ? lo_delta : 0) + 64 * sl) = v;
              }
              __syncwarp();
            }
          }
          uint32_t top = 0u;                               // over the rows and pieces this thread stores
#pragma unroll
          for (int pc = 0; pc < BN / 32; ++pc) {
            const bool mine = (own >> pc) & 1u;
            top = habs_max2(top, (mine & ok[0]) ? hmax[0][pc] : 0u);
            top = habs_max2(top, (mine & ok[1]) ? hmax[1][pc] : 0u);
          }
          sat |= f16_top(top);
        }
      }
      if (S > 1) {
        asm volatile("bar.sync 1, 256;" ::: "memory");          // all of this CTA's workspace reads are done
        if (et == 0) {
          int* cnt = p.counters + 2 * tile;
          if (atomicAdd(cnt + 1, 1) == S - 1) { cnt[0] = 0; cnt[1] = 0; __threadfence(); }
        }
      }
    }
    if (__any_sync(0xffffffffu, sat) && lane == 0) atomicOr(p.range, p.range_bit);   // saturation is never silent
  }
  // pairs: the peer may still multicast into / arrive on this CTA's shared memory until it has consumed its last stage
  if (PAIR) cluster_sync_all();
}

// ------------------------------------------------------------------------------------------
// conv1_1 on the tensor cores: the input pack cat(L/100, ab/110, mask - maskcent) (model.py:142-148) + model1.0
// (4 -> 64, 3x3, ReLU; model.py:13-14) as ONE padded k-block.  K = 9 taps x 4 channels = 36 -> 48 (three K=16 steps).
// There is no 16-byte granule to aim a TMA box at (a tap contributes 4 channels = 8 bytes), so the 128 threads of a CTA
// (one warpgroup) gather and normalise their pixel's 36 inputs themselves, split them into FP16 hi / lo (x 2^6, like
// kInExp) and write their row of the two K-major SWIZZLE_128B operand tiles directly; the 64 x 48 weight tile
// (hi / lo, pre-swizzled by conv1_1_pack_kernel) stays in shared memory for the life of the CTA.  9 wgmmas per 64-row
// half (lo*hi, hi*lo, hi*hi per K step) replace 2304 FFMAs per pixel.  4 CTAs per SM hide each other's gather / MMA /
// epilogue phases (no intra-CTA pipeline).
// ------------------------------------------------------------------------------------------
constexpr int kC11K = 48;                       // padded K (3 MMA steps of 16)
constexpr int kC11PackBytes = 2 * 8192 + 2 * 64 * 4;   // [B hi | B lo] smem images + bias' + scale'
constexpr int kC11Smem = 2 * 16384 + kC11PackBytes + 1024;   // A hi/lo, pack, alignment slack

__device__ __forceinline__ uint32_t sw128_off(int row, int chunk) {   // byte offset of a 16-byte chunk in a K-major SW128 tile
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4));
}

// one thread per output channel: power-of-two scale so the largest weight lands in [256, 512), hi/lo split, swizzled
// smem image of the [64 cout][48 k] tile (k = tap * 4 + cin, zero beyond 36), bias' = bias * 2^kInExp * 2^e,
// scale' = 2^(s_out - kInExp - e) (s_out: a1_1's storage exponent)
__global__ void conv1_1_pack_kernel(const float* __restrict__ w36x64, const float* __restrict__ bias, int s_out,
                                    uint8_t* __restrict__ out) {
  const int co = threadIdx.x;
  if (co >= 64) return;
  float mx = 0.f;
  for (int k = 0; k < 36; ++k) mx = fmaxf(mx, fabsf(w36x64[k * 64 + co]));
  int e = 0;
  if (mx > 0.f) { int ex; frexpf(mx, &ex); e = 9 - ex; }        // mx * 2^e in [256, 512)
  const float sc = ldexpf(1.f, e);
  __half* bh = reinterpret_cast<__half*>(out);
  __half* bl = reinterpret_cast<__half*>(out + 8192);
  for (int k = 0; k < 64; ++k) {
    const float v = k < 36 ? w36x64[k * 64 + co] * sc : 0.f;
    __half hi, lo;
    split_h(v, hi, lo);
    const uint32_t o = (sw128_off(co, k >> 3) >> 1) + (k & 7);
    bh[o] = hi; bl[o] = lo;
  }
  float* vec = reinterpret_cast<float*>(out + 16384);
  vec[co] = bias[co] * kInScale * sc;
  vec[64 + co] = ldexpf(1.f, s_out - kInExp - e);
}

template <bool SPLIT>
__global__ void __launch_bounds__(128, 4)
conv1_1_umma_kernel(const uint8_t* __restrict__ pack, const float* __restrict__ L, const float* __restrict__ ab,
                    const float* __restrict__ mask, float maskcent, int N, int H, int Wd, __half* __restrict__ ohi,
                    __half* __restrict__ olo, unsigned* range, unsigned out_bit) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_ahi = smem;                       // [128 px][64 k] FP16, K-major SW128 (16 KB); reused as the store staging
  uint8_t* s_alo = smem + 16384;
  uint8_t* s_pack = smem + 32768;              // B hi (8 KB) | B lo (8 KB) | bias' | scale'
  const float* s_vec = reinterpret_cast<const float*>(s_pack + 16384);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kRow = 64 * 2 + 16;            // staging row pitch (16 B pad: conflict-free both ways)

  {
    const uint4* src = reinterpret_cast<const uint4*>(pack);
    uint4* dst = reinterpret_cast<uint4*>(s_pack);
    for (int i = threadIdx.x; i < kC11PackBytes / 16; i += 128) dst[i] = __ldg(src + i);
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the weight tile is read by the tensor core (async proxy)
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  const size_t HW = (size_t)H * Wd, total = (size_t)N * HW;
  const int ntiles = (int)((total + 127) / 128);
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const size_t pix = (size_t)tile * 128 + threadIdx.x;
    const bool live = pix < total;
    const size_t pixc = live ? pix : 0;
    const int n = (int)(pixc / HW);
    const int r = (int)(pixc - (size_t)n * HW);
    const int y = r / Wd, x = r - y * Wd;
    // ---- gather + normalise + split: this thread's row of the A tiles (k = tap * 4 + channel) ----
    float in[kC11K];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int iy = y + ky - 1, ix = x + kx - 1;
        const bool ok = live && iy >= 0 && iy < H && ix >= 0 && ix < Wd;
        const size_t o = (size_t)iy * Wd + ix;
        const int t = (ky * 3 + kx) * 4;
        // zero padding applies to the concatenated, normalised input (model.py:148 then Conv2d pad)
        const float l = ok ? __ldg(L + (size_t)n * HW + o) : 0.f;
        const float a = ok ? __ldg(ab + (size_t)n * 2 * HW + o) : 0.f;
        const float b = ok ? __ldg(ab + (size_t)n * 2 * HW + HW + o) : 0.f;
        const float m = ok ? __ldg(mask + (size_t)n * HW + o) - maskcent : 0.f;
        const float ql = l * 0.01f, qa = a * (1.0f / 110.0f), qb = b * (1.0f / 110.0f);
        in[t + 0] = fmaf(fmaf(-ql, 100.0f, l), 0.01f, ql);                    // x / 100, correctly rounded (cf. div_corrected)
        in[t + 1] = fmaf(fmaf(-qa, 110.0f, a), 1.0f / 110.0f, qa);
        in[t + 2] = fmaf(fmaf(-qb, 110.0f, b), 1.0f / 110.0f, qb);
        in[t + 3] = m;
      }
#pragma unroll
    for (int k = 36; k < kC11K; ++k) in[k] = 0.f;
    // an input (|ab| > 110 * 1023, say) saturates the packed operand; every input pixel is the centre tap (k = 16..19)
    // of exactly one output pixel, its own, so checking the centre taps checks every input once
    uint32_t hin = 0u;
#pragma unroll
    for (int j = 0; j < kC11K / 8; ++j) {
      uint32_t hw[4], lw[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float v0 = in[8 * j + 2 * q] * kInScale, v1 = in[8 * j + 2 * q + 1] * kInScale;
        hw[q] = pack_f16x2_sat(v0, v1);
        if (8 * j + 2 * q >= 16 && 8 * j + 2 * q < 20) hin = habs_max2(hin, hw[q]);
        lw[q] = lo_f16x2(v0, v1, hw[q]);
      }
      const uint32_t o = sw128_off(threadIdx.x, j);
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(smem_u32(s_ahi) + o), "r"(hw[0]), "r"(hw[1]), "r"(hw[2]),
                   "r"(hw[3]) : "memory");
      if (SPLIT)
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(smem_u32(s_alo) + o), "r"(lw[0]), "r"(lw[1]), "r"(lw[2]),
                     "r"(lw[3]) : "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> tensor-core reads
    __syncthreads();
    // ---- 2 x 9 wgmmas (one per 64-row half): the small cross terms first, then hi*hi (as in umma_conv_kernel) ----
    float acc[2][32];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[m][i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const uint64_t a_hi = make_sw128_desc(smem_u32(s_ahi) + m * 8192), a_lo = make_sw128_desc(smem_u32(s_alo) + m * 8192);
      const uint64_t b_hi = make_sw128_desc(smem_u32(s_pack)), b_lo = make_sw128_desc(smem_u32(s_pack) + 8192);
      uint32_t first = 0u;
      if (SPLIT) {
#pragma unroll
        for (int kk = 0; kk < kC11K / 16; ++kk) {
          const uint64_t adv = (uint64_t)(kk * 2);
          wgmma_n64(acc[m], a_lo + adv, b_hi + adv, first);
          wgmma_n64(acc[m], a_hi + adv, b_lo + adv, 1u);
          first = 1u;
        }
      }
#pragma unroll
      for (int kk = 0; kk < kC11K / 16; ++kk) {
        const uint64_t adv = (uint64_t)(kk * 2);
        wgmma_n64(acc[m], a_hi + adv, b_hi + adv, first);
        first = 1u;
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(acc[0]);
    wgmma_reg_fence(acc[1]);
    // ---- epilogue: relu(acc + bias') * scale' = 2^S(a1_1) * relu(conv + b) -> hi / lo -> coalesced stores ----
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int c = frag_col(i, lane);
        acc[m][i] = fmaxf(acc[m][i] + s_vec[c], 0.f) * s_vec[64 + c];
      }
    __syncthreads();        // every warpgroup MMA has read the operand tiles: reuse them as per-warp staging
    const uint32_t wbuf = smem_u32(s_ahi) + warp * (2 * 16 * kRow);   // rows 16*warp (+64 for m = 1) of the tile
    uint32_t hmax[2][2] = {};                         // [m][row half]: max |hi| of the stored values
#pragma unroll
    for (int plane = 0; plane < (SPLIT ? 2 : 1); ++plane) {
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const uint32_t hw = pack_f16x2_sat(acc[m][i], acc[m][i + 1]);
          if (plane == 0) hmax[m][(i >> 1) & 1] = habs_max2(hmax[m][(i >> 1) & 1], hw);
          const uint32_t v = plane == 0 ? hw : lo_f16x2(acc[m][i], acc[m][i + 1], hw);
          const int rl = m * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
          st_shared_u32(wbuf + rl * kRow + frag_col(i, lane) * 2, v);
        }
      __syncwarp();
      __half* gbase = plane == 0 ? ohi : olo;
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rl = it * 4 + (lane >> 3), c = lane & 7;
        const size_t px = (size_t)tile * 128 + (rl >> 4) * 64 + warp * 16 + (rl & 15);
        const uint4 v = ld_shared_v4(wbuf + rl * kRow + c * 16);
        if (px < total) *reinterpret_cast<uint4*>(gbase + px * 64 + c * 8) = v;
      }
      __syncwarp();
    }
    {                                                 // saturation is never silent
      // rows of the tile that hold pixels, relative to this thread's first fragment row
      const int rows_left = (int)min(total - (size_t)tile * 128, (size_t)128) - (warp * 16 + (lane >> 2));
      uint32_t top = 0u;
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int h = 0; h < 2; ++h) top = habs_max2(top, m * 64 + 8 * h < rows_left ? hmax[m][h] : 0u);
      const unsigned bits = (__any_sync(0xffffffffu, live & f16_top(hin)) ? 1u << kRangeInputBit : 0u) |
                            (__any_sync(0xffffffffu, f16_top(top)) ? out_bit : 0u);
      if (bits && lane == 0) atomicOr(range, bits);
    }
    __syncthreads();        // staging read by every warp before the next tile's operand rows overwrite it
  }
}

cudaError_t conv1_1_umma_pack(Ctx* c) {
  if (!c->w11_umma.get()) {
    cudaError_t e = cudaMalloc(c->w11_umma.put(), kC11PackBytes);
    if (e != cudaSuccess) return e;
  }
  conv1_1_pack_kernel<<<1, 64>>>(c->w11, c->b11, c->bufs[c->buf_index.at("a1_1")].exp, c->w11_umma.get());
  cudaError_t e = cudaGetLastError();
  return e != cudaSuccess ? e : cudaDeviceSynchronize();
}

cudaError_t launch_conv1_1_umma(Ctx* c, int n, const float* L, const float* ab, const float* mask, float maskcent,
                                cudaStream_t st, int img0) {
  const ActBuf& o = c->bufs[c->buf_index.at("a1_1")];
  const size_t HW = (size_t)o.H * o.W, npix = (size_t)n * HW, ooff = (size_t)img0 * HW * o.C;
  const int ntiles = (int)((npix + 127) / 128);
  const int grid = ntiles < 4 * c->num_sms ? ntiles : 4 * c->num_sms;
  L += img0 * HW; ab += img0 * 2 * HW; mask += img0 * HW;
  static unsigned long long attr_devs = 0;
  if (c->dev >= 64 || !(attr_devs & (1ull << c->dev))) {
    cudaError_t e = cudaFuncSetAttribute(conv1_1_umma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kC11Smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(conv1_1_umma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kC11Smem);
    if (e != cudaSuccess) return e;
    if (c->dev < 64) attr_devs |= 1ull << c->dev;
  }
  __half* hi = static_cast<__half*>(o.p0.get()) + ooff;
  __half* lo = o.p1.get() ? static_cast<__half*>(o.p1.get()) + ooff : nullptr;
  const unsigned out_bit = 1u << c->buf_index.at("a1_1");
  cudaError_t e = lo ? launch_k(c, conv1_1_umma_kernel<true>, dim3(grid), dim3(128), (size_t)kC11Smem, st, c->w11_umma.get(), L, ab, mask,
                                maskcent, n, o.H, o.W, hi, lo, c->d_range, out_bit)
                     : launch_k(c, conv1_1_umma_kernel<false>, dim3(grid), dim3(128), (size_t)kC11Smem, st, c->w11_umma.get(), L, ab, mask,
                                maskcent, n, o.H, o.W, hi, lo, c->d_range, out_bit);
  c->launch_count++;
  return e;
}

// ------------------------------------------------------------------------------------------
// host side: tensor maps + launch plan
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

struct UmmaPlan {
  DevMem<CUtensorMap> d_amaps;
  DevMem<int4> d_kblk;
  CUtensorMap bmap_hi, bmap_lo;
  UmmaParams prm{};
  int num_sms = 132;
  int dev = 0;
  int mt = 1;               // M-tiles (128 pixels each) per CTA tile
  int cg = 1;               // 2: pairs (clusters of two CTAs sharing the weight tile)
  int split_k = 1;
  bool halo = false;        // one halo tile per input-channel group instead of one TMA box per tap (stride-1 3x3 layers)
  size_t ws_floats = 0;
  int ws_tiles = 0;
};

struct ViewKey {
  int src, s, qy, qx;
  bool operator==(const ViewKey& o) const { return src == o.src && s == o.s && qy == o.qy && qx == o.qx; }
};

static int floordiv2(int v) { return v >= 0 ? v / 2 : -((-v + 1) / 2); }

template <int BN, int MT, int CG, bool SPLIT, bool HALO = false>
static cudaError_t launch_inst(const UmmaPlan& pl, const UmmaParams& prm, cudaStream_t st, bool pdl) {
  using SP = SmemPlan<BN, MT, CG, SPLIT, HALO>;
  static unsigned long long attr_devs = 0;       // the opt-in is per device: one bit per device ordinal
  if (pl.dev >= 64 || !(attr_devs & (1ull << pl.dev))) {
    cudaError_t e = cudaFuncSetAttribute(umma_conv_kernel<BN, MT, CG, SPLIT, HALO>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         SP::kTotal);
    if (e != cudaSuccess) return e;
    if (pl.dev < 64) attr_devs |= 1ull << pl.dev;
  }
  const long items = (long)prm.total_tiles * prm.split_k;
  int grid = items * CG < pl.num_sms ? (int)items * CG : (pl.num_sms / CG) * CG;
  if (prm.max_ctas > 0 && grid > prm.max_ctas) grid = prm.max_ctas;   // persistent loop: any grid size covers all tiles
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = SP::kTotal;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  int na = 0;
  if (CG > 1) {
    at[na].id = cudaLaunchAttributeClusterDimension;
    at[na].val.clusterDim.x = CG; at[na].val.clusterDim.y = 1; at[na].val.clusterDim.z = 1;
    ++na;
  }
  if (pdl) {   // may start while the previous kernel of the forward drains (see pdl_wait in the kernel)
    at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = at;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, umma_conv_kernel<BN, MT, CG, SPLIT, HALO>, pl.bmap_hi, pl.bmap_lo, prm);
}

int umma_plan_op(Ctx* c, ConvOp& op) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) { c->err = "cuTensorMapEncodeTiled entry point not available"; return IDC_ERR_CUDA; }
  op.umma_plan.reset();
  std::unique_ptr<UmmaPlan, UmmaPlanFree> pl(new UmmaPlan());   // installed on the op once complete
  pl->num_sms = c->num_sms;
  pl->dev = c->dev;
  // tile geometry: 128 output columns where the layer allows it (the chunk and tile accumulators of a 128 x 128 tile
  // take 128 of a math thread's 232 registers; 256 columns would not fit), 64 otherwise
  op.bn_tile = (op.cout_pad % 128 == 0) ? 128 : 64;
  if (op.cout_pad % op.bn_tile) { c->err = "cout not tileable: " + op.name; return IDC_ERR_ARG; }
  if (op.fuse_out_head && op.cout_pad != 128) { c->err = "fused model_out needs 128 columns: " + op.name; return IDC_ERR_ARG; }
  int best = 1 << 30;
  for (int wb = 128; wb >= 8; wb >>= 1) {
    const int hb = kBM / wb;
    const int t = ceil_div(op.Wl, wb) * ceil_div(op.Hl, hb);
    if (t < best) { best = t; op.wbox = wb; op.hbox = hb; }
  }
  // HALO: stride-1 3x3 convs of one source with 128 output columns per tile load one 18x10-pixel halo tile per 64 input
  // channels instead of one box per tap, when the launch fills the machine.  Option halo=0 turns it off, =3 forces it
  // on every eligible op (also 64 columns, also tiny launches).
  {
    const int mode = c->opt.halo;
    bool ok = mode >= 1 && !c->fast && op.ncls == 1 && op.ntaps == 9;
    unsigned seen = 0;
    for (int t = 0; ok && t < op.ntaps; ++t) {
      const Tap& tp = op.taps[0][t];
      if (tp.src != op.taps[0][0].src || op.src[tp.src].s != 1 || tp.ty < -1 || tp.ty > 1 || tp.tx < -1 || tp.tx > 1) ok = false;
      else seen |= 1u << ((tp.ty + 1) * 3 + tp.tx + 1);
    }
    if (ok && (seen != 0x1FFu || op.src[op.taps[0][0].src].cin % kBK)) ok = false;
    if (ok && !(op.bn_tile == 128 || (mode >= 3 && op.bn_tile == 64))) ok = false;
    if (ok) {   // only launches that fill the machine
      const long T = (long)c->max_n * ceil_div(op.Hl, 16) * ceil_div(op.Wl, 8) * (op.cout_pad / op.bn_tile);
      if (T < 2L * pl->num_sms && mode < 3) ok = false;
    }
    pl->halo = ok;
    if (ok) { op.wbox = 8; op.hbox = 16; }
  }
  // Two M-tiles per CTA tile (one 256-pixel TMA box, two wgmma row blocks per warpgroup sharing each weight tile) for the
  // 64-column layers when the launch still fills the machine at the ctx's max batch.  The register budget allows it
  // only at 64 columns: option mt=2 on a 128-column layer runs it with 64-column tiles.
  pl->mt = 1;
  if (op.bn_tile == 64 && !pl->halo && !op.fuse_out_head) {
    const long tiles2 = (long)op.ncls * c->max_n * ceil_div(op.Hl, 2 * op.hbox) * ceil_div(op.Wl, op.wbox) *
                        (op.cout_pad / op.bn_tile);
    if (tiles2 >= 2L * pl->num_sms) pl->mt = 2;
  }
  {
    const int v = c->opt.mt;
    if (!pl->halo && v == 1) pl->mt = 1;
    if (!pl->halo && v == 2 && !op.fuse_out_head) { pl->mt = 2; op.bn_tile = 64; }
  }
  // pairs for launches that give every SM >= 2 tiles (option pairs: 0 = never, the default, 1 = those launches, 2 = always).
  // Measured on an H100 (400 W limit) at 64 x 256^2: 72.4 ms per forward with pairs on the large launches, 59.7 ms without -- the
  // halved weight traffic does not pay for coupling both CTAs' MMA warps to every stage refill.
  pl->cg = 1;
  {
    const long tiles_mt = (long)op.ncls * c->max_n * ceil_div(op.Hl, op.hbox * pl->mt) * ceil_div(op.Wl, op.wbox) *
                          (op.cout_pad / op.bn_tile);
    const int mode = c->opt.pairs;
    if (!c->fast && (mode >= 2 || (mode == 1 && tiles_mt >= 2L * pl->num_sms))) pl->cg = 2;
  }
  const int nkb = op.K / kBK;
  // split-K for launches that cannot fill the machine even at the ctx's max batch (interactive path): K is cut into S
  // slices per tile, all work items co-resident.
  {
    const int ty = ceil_div(op.Hl, op.hbox * pl->mt), tx = ceil_div(op.Wl, op.wbox), ntn = op.cout_pad / op.bn_tile;
    const long T = (long)op.ncls * c->max_n * ty * tx * ntn;
    const bool eligible = nkb >= 8 && !op.fuse_out_head && pl->mt == 1 && pl->cg == 1 && !pl->halo;
    int S = 1;
    if (T * 2 <= pl->num_sms && eligible) {
      S = (int)(pl->num_sms / T);
      if (S > nkb / 4) S = nkb / 4;
      if (S > op.bn_tile / 32) S = op.bn_tile / 32;      // one 32-column piece per CTA at least
      if (S < 1) S = 1;
    }
    {                                                      // experiments; must keep all work items co-resident
      const int v = c->opt.split_k;
      if (eligible && v >= 1 && v <= nkb && v <= op.bn_tile / 32 && T * v <= pl->num_sms) S = v;
    }
    pl->split_k = S;
    pl->ws_tiles = (int)T;
    pl->ws_floats = S > 1 ? (size_t)T * S * kBM * op.bn_tile : 0;
    if (pl->ws_floats > c->splitk_ws_floats) c->splitk_ws_floats = pl->ws_floats;
    if (S > 1 && pl->ws_tiles > c->splitk_max_tiles) c->splitk_max_tiles = pl->ws_tiles;
  }
  // views + k-block table
  std::vector<ViewKey> views;
  std::vector<int4> kblk((size_t)op.ncls * nkb);
  if (pl->halo) {
    // k-block i = (input group i / 9, tap i % 9); entry = {-, K column of the weight tile, dy + 1, dx + 1}
    const int src = op.taps[0][0].src, groups = op.src[src].cin / kBK;
    views.push_back(ViewKey{src, 1, 0, 0});
    for (int i = 0; i < nkb; ++i) {
      const int g = i / 9, t = i % 9;
      kblk[i] = make_int4(0, (t * groups + g) * kBK, op.taps[0][t].ty + 1, op.taps[0][t].tx + 1);
    }
  }
  for (int cls = 0; cls < op.ncls && !pl->halo; ++cls) {
    int kb = 0;
    for (int t = 0; t < op.ntaps; ++t) {
      const Tap& tp = op.taps[cls][t];
      const int s = op.src[tp.src].s;
      ViewKey vk{tp.src, s, 0, 0};
      int dy = tp.ty, dx = tp.tx;
      if (s == 2) {
        vk.qy = ((tp.ty % 2) + 2) % 2; vk.qx = ((tp.tx % 2) + 2) % 2;
        dy = floordiv2(tp.ty); dx = floordiv2(tp.tx);
      }
      int vi = -1;
      for (size_t i = 0; i < views.size(); ++i)
        if (views[i] == vk) vi = (int)i;
      if (vi < 0) { views.push_back(vk); vi = (int)views.size() - 1; }
      const int cin = op.src[tp.src].cin;
      if (cin % kBK) { c->err = "cin not a multiple of 64: " + op.name; return IDC_ERR_ARG; }
      for (int c0 = 0; c0 < cin; c0 += kBK) kblk[(size_t)cls * nkb + kb++] = make_int4(vi * 2, c0, dy, dx);
    }
    if (kb != nkb) { c->err = "k-block count mismatch: " + op.name; return IDC_ERR_ARG; }
  }
  // A tensor maps
  std::vector<CUtensorMap> amaps(views.size() * 2);
  for (size_t i = 0; i < views.size(); ++i) {
    const ViewKey& vk = views[i];
    const ActBuf& b = c->bufs[op.src[vk.src].buf];
    const int Hv = (b.H - vk.qy + vk.s - 1) / vk.s, Wv = (b.W - vk.qx + vk.s - 1) / vk.s;
    for (int part = 0; part < 2; ++part) {
      char* base = (char*)(part == 0 ? b.p0.get() : b.p1.get());
      if (!base) { amaps[i * 2 + part] = amaps[i * 2]; continue; }  // fast mode: lo unused
      base += ((size_t)vk.qy * b.W + vk.qx) * b.C * sizeof(__half);
      cuuint64_t dims[4] = {(cuuint64_t)b.C, (cuuint64_t)Wv, (cuuint64_t)Hv, (cuuint64_t)c->max_n};
      cuuint64_t strides[3] = {(cuuint64_t)vk.s * b.C * 2, (cuuint64_t)vk.s * b.W * b.C * 2,
                               (cuuint64_t)b.H * b.W * b.C * 2};
      cuuint32_t box[4] = {(cuuint32_t)kBK, (cuuint32_t)(pl->halo ? kHaloW : op.wbox),
                           (cuuint32_t)(pl->halo ? kHaloH : op.hbox * pl->mt), 1};
      cuuint32_t estr[4] = {1, 1, 1, 1};
      CUresult r = enc(&amaps[i * 2 + part], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) {
        char msg[256];
        snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled(A) failed (%d) for op %s view %zu", (int)r, op.name.c_str(), i);
        c->err = msg;
        return IDC_ERR_CUDA;
      }
    }
  }
  // B tensor maps: [ncls*cout_pad rows][K] FP16, K-major
  for (int part = 0; part < 2; ++part) {
    cuuint64_t dims[2] = {(cuuint64_t)op.K, (cuuint64_t)op.ncls * op.cout_pad};
    cuuint64_t strides[1] = {(cuuint64_t)op.K * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)(op.bn_tile / pl->cg)};   // pairs: each CTA loads half of the weight tile
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(part == 0 ? &pl->bmap_hi : &pl->bmap_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                     part == 0 ? (void*)op.w_hi : (void*)op.w_lo, dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      char msg[256];
      snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled(B) failed (%d) for op %s", (int)r, op.name.c_str());
      c->err = msg;
      return IDC_ERR_CUDA;
    }
  }
  if (cudaMalloc(pl->d_amaps.put(), amaps.size() * sizeof(CUtensorMap)) != cudaSuccess ||
      cudaMalloc(pl->d_kblk.put(), kblk.size() * sizeof(int4)) != cudaSuccess ||
      cudaMemcpy(pl->d_amaps.get(), amaps.data(), amaps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(pl->d_kblk.get(), kblk.data(), kblk.size() * sizeof(int4), cudaMemcpyHostToDevice) != cudaSuccess) {
    c->err = "uploading the launch plan failed in umma_plan_op: " + op.name;
    return IDC_ERR_CUDA;
  }

  UmmaParams& q = pl->prm;
  q.amaps = pl->d_amaps.get(); q.n_amaps = (int)amaps.size(); q.kblk = pl->d_kblk.get(); q.nkb = nkb; q.ncls = op.ncls;
  {
    // chunk_kb: k-blocks summed inside the tensor core before the FP32 round-to-nearest add.  1 is the most
    // accurate; the Cout <= 128 layers have short K (few chunks per tile to amortise the tile epilogue) and use 2.
    const int natural = (op.cout_pad % 256 == 0) ? 256 : (op.cout_pad % 192 == 0) ? 192 : (op.cout_pad % 128 == 0) ? 128 : 64;
    int g = c->fast ? 4 : (natural <= 128 ? 2 : 1);
    if (c->opt.chunk_kb >= 1) g = c->opt.chunk_kb;
    q.chunk_kb = g;
  }
  q.tiles_y = ceil_div(op.Hl, op.hbox * pl->mt); q.tiles_x = ceil_div(op.Wl, op.wbox);
  q.n_tiles_n = op.cout_pad / op.bn_tile;
  q.hbox = op.hbox; q.wbox = op.wbox;
  q.wshift = 0;
  while ((1 << q.wshift) < op.wbox) q.wshift++;
  q.Hl = op.Hl; q.Wl = op.Wl; q.cout_pad = op.cout_pad;
  q.bias = op.epi.bias; q.scale = op.epi.scale; q.shift = op.epi.shift;
  q.gadd = nullptr; q.gadd_ld = 512; q.gadd_mult = op.out_buf >= 0 ? ldexpf(1.f, c->bufs[op.out_buf].exp) : 1.f;
  q.act = op.epi.act;
  if (op.out_f32) {
    q.out_f32 = op.out_f32_ptr; q.out_ld = op.cout_pad;
  } else if (op.out_buf >= 0) {
    const ActBuf& ob = c->bufs[op.out_buf];
    q.out_hi = (__half*)ob.p0.get(); q.out_lo = (__half*)ob.p1.get();
    q.Hout = ob.H; q.Wout = ob.W; q.Cout = ob.C; q.os = op.os;
  }
  if (op.fuse_out_head) { q.wout = c->wout; q.bout = c->bout; }
  q.err = c->d_err;
  q.range = c->d_range; q.range_bit = op.out_buf >= 0 ? 1u << op.out_buf : 0u;
  q.img0 = 0;
  op.umma_plan = std::move(pl);
  return IDC_OK;
}

void UmmaPlanFree::operator()(UmmaPlan* p) const { delete p; }

bool umma_op_uses_split_k(const ConvOp& op) {
  return op.umma_plan && op.umma_plan->split_k > 1;
}

cudaError_t umma_run_op(Ctx* c, ConvOp& op, int n, float* out_ab_fused, float out_mult, cudaStream_t st, int img0,
                        int max_ctas) {
  const UmmaPlan* pl = op.umma_plan.get();
  if (!pl) return cudaErrorInvalidValue;
  UmmaParams prm = pl->prm;
  prm.max_ctas = (max_ctas > 0 && pl->split_k == 1) ? (max_ctas / pl->cg) * pl->cg : 0;   // split-K needs all items co-resident
  prm.img0 = img0;
  prm.n_img = img0 + n;
  if (img0 && pl->split_k > 1) return cudaErrorInvalidValue;   // image chunks are a large-batch feature
  const int m_tiles = n * prm.tiles_y * prm.tiles_x;
  prm.total_tiles = op.ncls * (pl->cg == 2 ? (m_tiles + 1) / 2 : m_tiles) * prm.n_tiles_n;
  prm.gadd = (op.epi.gadd && c->gadd_active) ? c->gvec.get() : nullptr;
  prm.out_ab = out_ab_fused;
  prm.split_k = pl->split_k;
  prm.ws = c->splitk_ws.get();
  prm.counters = c->splitk_counters.get();
  if (pl->split_k > 1 && (!prm.ws || !prm.counters)) return cudaErrorInvalidValue;
  prm.out_mult = out_mult;
  if (op.fuse_out_head && !out_ab_fused) return cudaErrorInvalidValue;
  c->launch_count++;
  const bool pdl = pdl_take(c);
  const bool split = !c->fast;
  if (pl->halo) {
    if (!split) return cudaErrorInvalidValue;
    switch (op.bn_tile * 10 + pl->cg) {
      case 641: return launch_inst<64, 1, 1, true, true>(*pl, prm, st, pdl);
      case 642: return launch_inst<64, 1, 2, true, true>(*pl, prm, st, pdl);
      case 1281: return launch_inst<128, 1, 1, true, true>(*pl, prm, st, pdl);
      case 1282: return launch_inst<128, 1, 2, true, true>(*pl, prm, st, pdl);
      default: return cudaErrorInvalidValue;
    }
  }
#define IDC_LAUNCH(BN_, MT_, CG_) \
  return split ? launch_inst<BN_, MT_, CG_, true>(*pl, prm, st, pdl) : launch_inst<BN_, MT_, CG_, false>(*pl, prm, st, pdl)
  switch (op.bn_tile * 100 + pl->mt * 10 + pl->cg) {
    case 6411: IDC_LAUNCH(64, 1, 1);
    case 6421: IDC_LAUNCH(64, 2, 1);
    case 12811: IDC_LAUNCH(128, 1, 1);
    case 6412: return launch_inst<64, 1, 2, true>(*pl, prm, st, pdl);     // pairs: parity (split) operands only
    case 6422: return launch_inst<64, 2, 2, true>(*pl, prm, st, pdl);
    case 12812: return launch_inst<128, 1, 2, true>(*pl, prm, st, pdl);
    default: break;
  }
#undef IDC_LAUNCH
  return cudaErrorInvalidValue;
}

}  // namespace idc
