// Internal declarations shared by the translation units of libidc_b200.so.
// Layout vocabulary follows the reference network (model.py): blocks model1..model10,
// activations conv1_2 ... conv10_2, hints, bins.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/idc_b200.h"

namespace idc {

// ---- owners of CUDA handles ----
// Move-only; the destructor releases the handle.  Readers take the raw handle with get(); put() releases the current
// handle and returns the address a cudaMalloc* / cuda*Create call writes the new one to.  HostMem also owns mapped
// cudaHostAlloc blocks; their device alias is a plain pointer kept beside the owner.
template <typename H, auto Release>
class Owner {
 public:
  Owner() = default;
  Owner(Owner&& o) noexcept { std::swap(h_, o.h_); }
  Owner& operator=(Owner&& o) noexcept { std::swap(h_, o.h_); return *this; }
  ~Owner() { reset(); }
  H get() const { return h_; }
  H* put() { reset(); return &h_; }
  void reset() { if (h_) Release(h_); h_ = nullptr; }
  H release() { H h = h_; h_ = nullptr; return h; }   // the caller frees it (e.g. stream-ordered, cudaFreeAsync)
 private:
  H h_ = nullptr;
};
template <typename T> using DevMem = Owner<T*, cudaFree>;
template <typename T> using HostMem = Owner<T*, cudaFreeHost>;
using Stream = Owner<cudaStream_t, cudaStreamDestroy>;
using Event = Owner<cudaEvent_t, cudaEventDestroy>;
using GraphExec = Owner<cudaGraphExec_t, cudaGraphExecDestroy>;

constexpr int kMaxTaps = 34;  // up-layer: 4 deconv + 9 shortcut taps; Caffe hyper-column: 4x4 deconv + 2x9 conv taps
constexpr int kMaxSrc = 6;
constexpr int kMaxCls = 4;    // output parity classes of a stride-2 transposed conv

enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_LEAKY02 = 2 };

// wgmma engine: buffer b is stored as FP16 hi/lo planes of (value * 2^S_b), one exponent per buffer (ActBuf::exp),
// chosen from the weights when they are packed (DESIGN §3): S_b = kActExpRef - ceil(log2 est_b), where est_b is a
// magnitude estimate of the buffer propagated through the plan from the weights alone.  It puts the estimate in
// (2^(kActExpRef-1), 2^kActExpRef], far below FP16's 65504 and far above the range where the lo plane goes subnormal.
// The output of a conv without a BatchNorm also has a bound (1-norms instead of 2-norms); S_b is lowered where needed
// to keep the bound at or below 2^kActExpBound.
// A buffer whose largest |a| on sample inputs was measured (idc_set_act_range) takes S_b = kActExpCal - ceil(log2 max_abs)
// instead: a measured maximum needs less headroom than an estimate that BatchNorm outputs exceed by orders of magnitude.
// A network whose exponents fall outside [kActExpMin, kActExpMax] is refused (the per-channel weight exponent, clamped
// to +-24, could not absorb the shift exactly any more).
constexpr int kActExpRef = 7;
constexpr int kActExpBound = 11;
constexpr int kActExpCal = 10;
constexpr int kActExpMin = -24, kActExpMax = 24;
// Every FP16 activation store whose hi part reaches 65504, FP16's largest value (|v| >= 65488; above 65504 the value
// saturates there), sets bit `buffer index` of the context's range word; the packed conv1_1 input uses bit
// kRangeInputBit.
constexpr unsigned kRangeInputBit = 31;
constexpr unsigned kF16MaxBits = 0x7BFFu;   // 65504
// conv1_1's packed input (L/100, ab/110, mask - maskcent: |x| <= ~1 by construction) is split at this fixed exponent
constexpr int kInExp = 6;
constexpr float kInScale = 64.0f;   // 2^kInExp

// One filter tap of a gather-GEMM convolution.  For logical output pixel (y, x) the tap reads
// source pixel (y*s + ty, x*s + tx) of source `src`; out-of-range pixels read zero
// (= the reference's zero padding).  (ky, kx) is the kernel index used for weight packing.
struct Tap {
  int src;  // 0 = main source, 1 = shortcut source
  int ky, kx;
  int ty, tx;
};

// Activation buffer.  SIMT engine: p0 = float [N,H,W,C].  wgmma engine: p0/p1 = __half
// hi/lo planes, each [N,H,W,C]; value = (hi + lo) * 2^-exp.
struct ActBuf {
  std::string name;
  int H = 0, W = 0, C = 0;
  int exp = 0;   // wgmma engine: storage exponent S_b (0 on the SIMT engine, whose planes are FP32 values)
  DevMem<void> p0, p1;
};

// Per-output-channel epilogue vectors (device, fp32[cout_pad]).
//   v = act(acc + bias) * scale + shift (+ gadd[n][c])
// wgmma engine: weights are pre-scaled per output channel by a power of two 2^e (so the FP16 lo
// term stays normal); bias is stored as bias*2^e and scale as scale*2^-e, which is exact and leaves
// the formula unchanged because ReLU / LeakyReLU are positively homogeneous.
struct Epilogue {
  float* bias = nullptr;
  float* scale = nullptr;  // BN gamma / sqrt(var + eps)   (1 when no BN)
  float* shift = nullptr;  // BN beta - mean * scale        (0 when no BN)
  int act = ACT_NONE;
  bool has_bn = false;
  bool gadd = false;  // add global-hints vector [N, cout] (row a15)
};

struct SrcDesc {
  int buf = -1;  // index into Ctx::bufs
  int s = 1;     // logical->source pixel stride (2 = read the ::2 decimation / the skip tensor)
  int cin = 0;
};

enum OpKind { OP_CONV = 0, OP_UP = 1, OP_CLASS = 2, OP_HYPER = 3 };

struct UmmaPlan;                                                 // idc_umma.cu
struct UmmaPlanFree { void operator()(UmmaPlan* p) const; };

struct ConvOp {
  std::string name;
  int kind = OP_CONV;
  std::string wkey[kMaxSrc];  // state_dict keys, one per source (main conv / deconv, shortcut conv, ...)
  bool src_deconv[kMaxSrc] = {false, false, false, false, false, false};  // source s is a ConvTranspose2d (IOHW weights)
  int src_k[kMaxSrc] = {3, 3, 3, 3, 3, 3};   // kernel size of source s's filter (3, 4 for the transposed convs, 1)
  std::string bnkey;
  int nsrc = 1;
  SrcDesc src[kMaxSrc];
  int ncls = 1;
  int ntaps = 0;                 // taps per class
  Tap taps[kMaxCls][kMaxTaps];
  int Hl = 0, Wl = 0;            // logical output grid (per class)
  int out_buf = -1;
  int os = 1;                    // output pixel = (y*os + cls/2, x*os + cls%2)
  int cout = 0, cout_pad = 0;
  int K = 0;                     // sum over taps of cin(src)
  Epilogue epi;
  bool fuse_out_head = false;    // wgmma engine: model_out (128->2, tanh*110) in the epilogue
  bool out_f32 = false;          // store FP32 [M][cout_pad] instead of an activation (class logits)
  float* out_f32_ptr = nullptr;  // where (ctx->logits or ctx->logits313)
  // packed weights
  float* w_simt = nullptr;       // [ncls][K][cout_pad] fp32
  __half* w_hi = nullptr;        // [ncls*cout_pad][K] fp16 (x wscale)
  __half* w_lo = nullptr;
  // wgmma launch plan (filled by umma_plan_op)
  int bn_tile = 0, hbox = 0, wbox = 0;
  std::unique_ptr<UmmaPlan, UmmaPlanFree> umma_plan;
  double flops_per_image = 0;
};

// conv1_1 weights as a kernel parameter (constant bank): [36][64] with k = tap*4 + cin, then bias
struct Conv11Weights {
  float w[36 * 64];
  float b[64];
};

// Plan-time options (idc_set_option).  -1 = automatic.  They replace the IDC_* environment switches of
// round 1: a C ABI that is embedded in someone else's process must not read process-global state.
struct Options {
  int halo = 1;           // halo-tile A operand: 0 off, 1 = 128-column stride-1 3x3 layers that fill the machine, 3 = every eligible op
  int pairs = 0;          // clusters of 2 CTAs sharing the weight tile: 0 never (default: measured slower), 1 = launches that
                          // give every SM >= 2 tiles, 2 = always
  int mt = -1;            // M-tiles per CTA tile (1 / 2; 2 runs with 64-column tiles)
  int chunk_kb = -1;      // k-blocks summed inside the tensor core before the FP32 round-to-nearest add
  int split_k = -1;       // K slices per tile on launches that cannot fill the machine
  int host_pipe = 1;      // idc_forward_host: chunked copy/compute overlap for batches >= 8
  int pdl = 1;            // programmatic dependent launch between the kernels of a forward
  int conv1_1_umma = 1;   // model1.0 on the tensor cores (one padded k-block); 0 = the FP32 CUDA-core kernel
  int side_dist = 1;      // batch <= 4: run the dist head (class + softmax) on a side stream next to levels 9-10
  int tanh_scale = 110;   // regression head: tanh * 110 (model.py:175); the Caffe deploy nets use 100 (SURVEY q4)
};

struct HostTensor {
  std::vector<float> data;
  std::vector<int64_t> dims;
};

// Resources a context creates at first use, one group at a time.  A group is built into a local and moved into the
// context only when every allocation in it succeeded, so the context holds it whole or not at all.
// idc_forward_host / idc_set_image.  Every device region has a page-locked host twin of the same size (d_in / h_in,
// d_out / h_out, d_rgb / h_rgb, d_small / h_small, AbqStaging; the hint block is the same kind of pair): a copy through
// pageable caller memory goes between a device address and the host address at the same offset in its twin.
//   d_in    [L | ab | mask | glob] packed for the call's n; idc_set_image leaves L at its head
//   d_out   ab of the eager path, then the dist at max_n * 2HW (idc_fetch_dist, idc_ab_reccs, idc_dist_negentropy)
//   d_rgb   rgb of the eager path;  d_small  [ab | rgb | quantised ab] packed for n, the outputs of the click graph
struct HostStaging {
  DevMem<float> d_in, d_out; HostMem<float> h_in, h_out;
  DevMem<uint8_t> d_rgb; HostMem<uint8_t> h_rgb;
  DevMem<char> d_small; HostMem<char> h_small;
};
struct AbqStaging { DevMem<double> d_abq; HostMem<double> h_abq; };   // quantised ab (row a11) of the eager path
// idc_set_hints: [kHintHdrBytes header (int count) | IDC_MAX_HINTS x idc_hint], pinned host + device copy
struct HintBlock { HostMem<char> h_hints; DevMem<char> d_hints; };
// idc_set_click: the clicked pixel's pmf + K colour suggestions ride on a side branch of the click graph
struct ClickBlock {
  HostMem<int> h_click; int* d_click = nullptr;   // {img, y4, x4, K, seq} in mapped host memory, read when the graph runs
  DevMem<char> d_clickout; HostMem<char> h_clickout;   // [8-int header | 544 floats pmf | the picked suggestions]
};
// dist head off the critical path: class + softmax run on s_side next to decoder levels 9-10; the announced click's
// pmf + suggestions run on s_click, next to the full-map softmax
struct SideBranch { Stream s_side, s_click; Event ev_fork, ev_join, ev_click[2]; };
// idc_forward_host pipeline (large batches): H2D of image chunk k+1 overlaps conv1_1 of chunk k, D2H of ab
// chunk k overlaps the last op of chunk k+1
struct HostPipeStreams { Stream s_in, s_out; Event ev_in[8], ev_out[8]; };

struct Ctx {
  int dev = 0;
  int num_sms = 0;                           // of dev, read once by idc_create
  int max_n = 0, H = 0, W = 0;
  unsigned flags = 0;
  Options opt;
  bool simt = false, fast = false, dist = false, glob = false;
  std::map<std::string, HostTensor> raw;
  std::vector<ActBuf> bufs;
  std::map<std::string, int> buf_index;
  std::vector<ConvOp> ops;
  // weight arena
  DevMem<char> arena;
  size_t arena_bytes = 0;
  int* act_exp = nullptr;         // [bufs.size()] storage exponents, in the arena so that adopting ranks read them too
  std::map<std::string, int> act_exp_override;   // idc_set_option("act_exp.<buffer>"): applied at the next pack
  std::map<std::string, double> act_range;       // idc_set_act_range: measured largest |a| per buffer, applied at the next pack
  DevMem<unsigned> d_absmax;                     // idc_act_absmax result word (bit pattern of the maximum), made at first use
  bool weights_ready = false;     // adopted and planned: forwards may run
  bool weights_adopted = false;   // idc_adopt_weights succeeded and no tensor was loaded since: option changes re-plan
  // conv1_1 (4->64) + regression head + misc small weights (device fp32)
  float* w11 = nullptr;   // [36][64]  k = tap*4 + cin
  float* b11 = nullptr;   // [64]
  Conv11Weights h_w11;    // host copy passed by value to conv1_1_kernel
  DevMem<uint8_t> w11_umma;   // conv1_1_umma_kernel: swizzled hi/lo weight tile + bias' / scale' (device, derived)
  float* wout = nullptr;  // [2][128]
  float* bout = nullptr;  // [2]
  // global hints MLP (device fp32)
  float* gw[4] = {nullptr, nullptr, nullptr, nullptr};      // [cout][cin]
  float* gb[4] = {nullptr, nullptr, nullptr, nullptr};
  float* gscale[4] = {nullptr, nullptr, nullptr, nullptr};
  float* gshift[4] = {nullptr, nullptr, nullptr, nullptr};
  DevMem<float> gvec;   // [max_n][512]
  DevMem<float> gtmp;   // [2][max_n][512]
  // workspace
  DevMem<float> logits;      // [max_n*(H/4)*(W/4)][cout_pad(529)]
  DevMem<float> logits313;   // Caffe-spec head: [max_n*(H/4)*(W/4)][320]
  bool caffe313 = false;
  DevMem<float> pts313;      // [313][2] ab bin centres (device)
  // split-K workspace of the wgmma engine (sized by umma_plan_op, allocated after planning)
  DevMem<float> splitk_ws; size_t splitk_ws_floats = 0;
  DevMem<int> splitk_counters; int splitk_max_tiles = 0;
  bool dbg_graph_timing = false; // experiments: events around the click graph launch (idc_debug_graph_timing)
  Event dbg_ev[2];
  float dbg_graph_ms = 0.f;
  HostMem<int> h_err;          // [0] watchdog flag, [1] range word (mapped pinned host memory: survives a device trap)
  int* d_err = nullptr;
  unsigned* d_range = nullptr; // device alias of h_err[1]: bit b = a store into buffer b saturated
  std::unique_ptr<HostStaging> stage;
  std::unique_ptr<AbqStaging> abq;
  Stream own_stream;
  std::unique_ptr<HostPipeStreams> pipe;
  std::unique_ptr<SideBranch> side;
  int image_n = 0;                           // idc_set_image: this many L planes are resident at the head of d_in
  std::unique_ptr<HintBlock> hints;
  int graph_captures = 0;                    // click-graph instantiations (idc_graph_captures)
  // CUDA graph cache for the batch-1 latency path
  GraphExec graph_exec;
  const void* graph_ptrs[8] = {nullptr};
  float graph_maskcent = 0.f;
  int launch_count = 0;
  int graph_launches = 0;
  bool chain = false;           // the previous operation on the forward's stream was a kernel of this forward (PDL)
  bool gadd_active = false;     // a global-hints vector was supplied to this forward
  int last_n = 0;
  DevMem<char> d_reccs_batch;   // colour-suggestion scratch (ReccsScratch) of idc_ab_reccs and the batched calls
  int reccs_batch_q = 0;        // the query count it holds room for
  DevMem<float> d_negent;       // idc_dist_negentropy result, (H/4)*(W/4) floats
  DevMem<float> d_dist313;      // idc_caffe313_dist_pixel result, 320 floats
  bool dist_resident = false;   // keep the dist of the last forward_host on the device (idc_fetch_dist)
  int dist_valid_n = 0;
  bool click_mode = false;
  std::unique_ptr<ClickBlock> click;
  bool click_served = false;    // h_clickout holds the answer for the click in its header
  // per-op profiling
  bool profiling = false;
  std::vector<std::vector<Event>> prof_runs;   // one event list per profiled forward
  std::vector<Event> prof_pool;
  std::string err;
};

// ---- engine entry points (idc_simt.cu / idc_umma.cu / idc_heads.cu) ----
cudaError_t simt_run_op(Ctx* c, ConvOp& op, int n, cudaStream_t st);
int umma_plan_op(Ctx* c, ConvOp& op);              // builds tensor maps; returns IDC_* code
cudaError_t umma_run_op(Ctx* c, ConvOp& op, int n, float* out_ab_fused, float out_mult, cudaStream_t st, int img0 = 0,
                        int max_ctas = 0);   // max_ctas > 0: cap the persistent grid (side-branch launches)
bool umma_op_uses_split_k(const ConvOp& op);

cudaError_t launch_conv1_1(Ctx* c, int n, const float* L, const float* ab, const float* mask,
                           float maskcent, cudaStream_t st, int img0 = 0);   // L/ab/mask: full arrays; images img0..img0+n
cudaError_t launch_conv1_1_umma(Ctx* c, int n, const float* L, const float* ab, const float* mask, float maskcent,
                                cudaStream_t st, int img0 = 0);              // the same layer on the tensor cores
cudaError_t conv1_1_umma_pack(Ctx* c);                                       // weight tile for it, from the arena (device)
// hint block of idc_set_hints: a 16-byte header {count, 0, 0, 0}, then IDC_MAX_HINTS idc_hint entries.  It always
// travels whole, so the copy is the same graph node whatever the count.
constexpr size_t kHintHdrBytes = 16;
constexpr size_t kHintBlockBytes = kHintHdrBytes + (size_t)IDC_MAX_HINTS * sizeof(idc_hint);
// rasterise the hint block (device) into the ab [n,2,H,W] / mask [n,1,H,W] planes conv1_1 reads (c may be null:
// idc_hint_raster, outside a forward)
cudaError_t launch_hint_raster(Ctx* c, int n, int H, int W, const char* hints_dev, float* ab, float* mask,
                               cudaStream_t st);
cudaError_t launch_gamut(double L, int gamut_size, int D, int A, uint8_t* rgb, uint8_t* mask, cudaStream_t st);
cudaError_t launch_out_head(Ctx* c, int n, float* out_ab, cudaStream_t st);   // SIMT / KEEP_CONV10 path
cudaError_t launch_softmax529(Ctx* c, int n, float* out_dist, cudaStream_t st);
cudaError_t launch_lab2rgb(Ctx* c, int n, int h, int w, const float* L, float l_offset, const float* ab,
                           uint8_t* rgb, cudaStream_t st, double* abq = nullptr);   // c may be null (stand-alone call)
cudaError_t launch_decode313(Ctx* c, int n, float T, float* out_ab, cudaStream_t st);
cudaError_t launch_dist313_pixel(Ctx* c, int img, int y, int x, float S, float* out313_dev, cudaStream_t st);
cudaError_t launch_dist313_map(Ctx* c, int n, float S, float* out_dev, cudaStream_t st);
cudaError_t launch_negentropy(int n, int bins, int hw, const float* dist, float* out, cudaStream_t st);
cudaError_t launch_click_pmf(Ctx* c, const int* click_dev, int n_img, int* out_hdr, float* out_pmf, cudaStream_t st);
// Colour suggestions for q pmfs on the device, the one path of every entry point.  Row i of pmf starts at pmf + i * 529,
// its bins bin_stride floats apart; pts_dev [529][2]; res q * n_init * (3K+2) doubles for every restart.  Writes each
// row's picked restart: centers [q][K][2], conf [q][K] (may be null), iters [q] (may be null).  dyn (the click header
// of click_pmf_kernel): K = dyn[3], and nothing is written unless dyn[7] is set and 1 <= K <= 32.
cudaError_t launch_reccs(const float* pmf, size_t bin_stride, int q, const float* pts_dev, int K, int max_iter,
                         int n_init, double* res, float* centers, float* conf, int32_t* iters, cudaStream_t st,
                         const int* dyn = nullptr);
// The k-means points: the caller's [529][2] pts, or (pts null) the PyTorch wrapper's gamut grid
// (data/colorize_image.py:283, quirk q3): bin i = (g[i % 23], g[i / 23]), g = -110, -100, ..., 110.
inline void reccs_points(const float* pts, float* out) {
  for (int i = 0; i < 529; ++i) {
    out[2 * i] = pts ? pts[2 * i] : -110.f + 10.f * (i % 23);
    out[2 * i + 1] = pts ? pts[2 * i + 1] : -110.f + 10.f * (i / 23);
  }
}
// The suggestion scratch for q queries (reccs_batch_scratch_bytes(q)): the k-means points, the [q][529] pmfs, then
// kReccsMaxInit rows of kReccsRes doubles per query for every restart.
constexpr int kReccsMaxInit = 16, kReccsRes = 3 * 32 + 2;   // restarts per query, doubles per restart (at K = 32)
constexpr size_t kReccsBatchPtsBytes = 4352;                 // 529 x 2 floats, rounded up to 256 bytes
inline size_t reccs_batch_pmf_bytes(int q) { return ((size_t)q * 529 * sizeof(float) + 255) / 256 * 256; }
inline size_t reccs_batch_scratch_bytes(int q) {
  return kReccsBatchPtsBytes + reccs_batch_pmf_bytes(q) + (size_t)q * kReccsMaxInit * kReccsRes * sizeof(double);
}
struct ReccsScratch {
  float* pts; float* pmf; double* res;
  ReccsScratch(char* s, int q)
      : pts(reinterpret_cast<float*>(s)), pmf(reinterpret_cast<float*>(s + kReccsBatchPtsBytes)),
        res(reinterpret_cast<double*>(s + kReccsBatchPtsBytes + reccs_batch_pmf_bytes(q))) {}
};
// idc_ab_reccs_batch on the device: queries [q][3] (img, y4, x4, HOST memory, checked by the caller), pts [529][2]
// (HOST memory, or null), scratch a ReccsScratch for q.  The pmfs go to pmf_out when given (else to the scratch).
// Stream-ordered: the queries and points reach the device as kernel parameters.
cudaError_t launch_reccs_batch(Ctx* c, int q, const int32_t* queries, const float* pts, int K, int max_iter, int n_init,
                               char* scratch, float* centers, float* conf, int32_t* iters, float* pmf_out,
                               cudaStream_t st);
// idc_caffe313_reccs_batch on the device: the same scratch and outputs, queries (img, y, x) at full resolution, the pmf
// of each query dist_ab_S of the 313-bin logits (zero-padded to 529), the points the context's pts313 (zero-padded)
cudaError_t launch_caffe313_reccs_batch(Ctx* c, int q, const int32_t* queries, float S, int K, int max_iter, int n_init,
                                        char* scratch, float* centers, float* conf, int32_t* iters, float* pmf_out,
                                        cudaStream_t st);
cudaError_t launch_global_stats(int h, int w, const uint8_t* rgb, const float* pts, float* out316, cudaStream_t st);
cudaError_t launch_rgb2lab(int n, int h, int w, const uint8_t* rgb, double* lab, cudaStream_t st);
cudaError_t launch_render_planes(const double* ab, int ab_order, int ab_f32, const double* mask, int mask_f32, int l_mode,
                                 const double* L, int hin, int win, int H, int W, uint8_t* rgb, cudaStream_t st);
cudaError_t launch_resize_linear_u8(const uint8_t* src, int hs, int ws, uint8_t* dst, int hd, int wd, cudaStream_t st);
cudaError_t launch_cubic_lab2rgb(const double* ab, int hin, int win, const double* L, int H, int W, uint8_t* rgb,
                                 cudaStream_t st);
// batched photos (idc_photos.cu); table: n <= IDC_MAX_PHOTOS entries, checked by the caller
cudaError_t launch_photo_prep(int n, const idc_photo* table, const uint8_t* src, int X, float* L_mc, uint8_t* rgb,
                              cudaStream_t st);
cudaError_t launch_photo_render(int n, const idc_photo* table, const uint8_t* src, int X, const double* lab, uint8_t* out,
                                cudaStream_t st);
cudaError_t launch_rgb_sse(int n, size_t hw3, const uint8_t* a, const uint8_t* b, int64_t* sse, cudaStream_t st);
// hint blocks of `stride` bytes (>= kHintHdrBytes, a multiple of 4), checked by the caller
cudaError_t launch_hint_fill_mean(int n_blocks, int levels, int X, const double* lab, char* blocks, size_t stride,
                                  cudaStream_t st);
// n in [1, 65535], h and w multiples of 4 in [4, IDC_MAX_PHOTO_X], checked by the caller
cudaError_t launch_global_stats_batch(int n, int h, int w, const uint8_t* rgb, const float* pts, float* out,
                                      cudaStream_t st);
// colorization by optimization (idc_levin.cu); arguments checked by the caller (levin_check in idc_api.cu)
size_t levin_workspace_bytes(int n, int h, int w);
cudaError_t launch_levin_weights(int n, int h, int w, const double* lab, double* wts, cudaStream_t st);
cudaError_t launch_levin_solve(int n, int levels, int h, int w, const double* wts, const float* ab_hint,
                               const float* mask, double tol, int max_iter, float* out_ab, int32_t* iters,
                               double* relres, void* workspace, cudaStream_t st);
cudaError_t launch_global_mlp(Ctx* c, int n, const float* glob, cudaStream_t st);
cudaError_t launch_act_to_nchw(Ctx* c, const ActBuf& b, int n, float* out, cudaStream_t st);
cudaError_t launch_nchw_to_act(Ctx* c, const ActBuf& b, int n, const float* in, cudaStream_t st);
// *out_bits (device) = the bit pattern of max |a| over the first n images of b, in stored units (value * 2^b.exp)
cudaError_t launch_act_absmax(Ctx* c, const ActBuf& b, int n, unsigned* out_bits, cudaStream_t st);

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Programmatic dependent launch bookkeeping: a kernel may carry the programmatic-stream-serialization attribute
// only when the operation enqueued right before it on the same stream is another kernel of this forward (every
// kernel of the library executes griddepcontrol.wait, so completion stays transitive along the chain).
inline bool pdl_take(Ctx* c) {
  const bool r = c && c->opt.pdl && !c->simt && c->chain;
  if (c) c->chain = true;
  return r;
}
inline void pdl_break(Ctx* c) { if (c) c->chain = false; }

#ifdef __CUDACC__
// Lab -> sRGB uint8, float64 math like the reference's numpy/skimage path: skimage 0.13 color.lab2rgb (lab2xyz +
// xyz2rgb), clip, *255, truncating cast (data/colorize_image.py:27).  Every render and the display step end here.
__device__ __forceinline__ double lab_finv(double t) {
  return t > 0.2068966 ? t * t * t : (t - 16.0 / 116.0) / 7.787;
}
__device__ __forceinline__ double srgb_gamma(double c) {
  return c > 0.0031308 ? 1.055 * pow(c, 1.0 / 2.4) - 0.055 : 12.92 * c;
}
__device__ __forceinline__ void lab_to_rgb_u8(double l, double a, double b, uint8_t* out) {
  const double fy = (l + 16.0) / 116.0;
  const double fx = a / 500.0 + fy;
  double fz = fy - b / 200.0;
  if (fz < 0.0) fz = 0.0;
  const double X = lab_finv(fx) * 0.95047, Y = lab_finv(fy) * 1.0, Z = lab_finv(fz) * 1.08883;
  // inverse of the sRGB->XYZ matrix used by skimage (xyz_from_rgb), float64
  double R = 3.240481343200526 * X + -1.5371515162713185 * Y + -0.4985363261688878 * Z;
  double G = -0.9692549499965682 * X + 1.8759900014898907 * Y + 0.04155592655829284 * Z;
  double B = 0.05564663913517716 * X + -0.20404133836651123 * Y + 1.0573110696453443 * Z;
  R = srgb_gamma(R); G = srgb_gamma(G); B = srgb_gamma(B);
  out[0] = (uint8_t)(fmin(fmax(R, 0.0), 1.0) * 255.0);
  out[1] = (uint8_t)(fmin(fmax(G, 0.0), 1.0) * 255.0);
  out[2] = (uint8_t)(fmin(fmax(B, 0.0), 1.0) * 255.0);
}

// sRGB uint8 -> Lab, float64 like skimage 0.13 color.rgb2lab (data/colorize_image.py:31-36): rgb2lab_kernel, the gamut
// map and the batched photo prep / render read a pixel through this one sequence.
__device__ __forceinline__ double srgb_inv_gamma(double c) {
  return c > 0.04045 ? pow((c + 0.055) / 1.055, 2.4) : c / 12.92;
}
__device__ __forceinline__ double lab_f(double t) { return t > 0.008856 ? cbrt(t) : 7.787 * t + 16.0 / 116.0; }
__device__ __forceinline__ void rgb_u8_to_lab(const uint8_t* px, double& l, double& a, double& b) {
  const double R = srgb_inv_gamma(px[0] / 255.0), G = srgb_inv_gamma(px[1] / 255.0), B = srgb_inv_gamma(px[2] / 255.0);
  const double X = (0.412453 * R + 0.357580 * G + 0.180423 * B) / 0.95047;
  const double Y = (0.212671 * R + 0.715160 * G + 0.072169 * B) / 1.0;
  const double Z = (0.019334 * R + 0.119193 * G + 0.950227 * B) / 1.08883;
  const double fx = lab_f(X), fy = lab_f(Y), fz = lab_f(Z);
  l = 116.0 * fy - 16.0;
  a = 500.0 * (fx - fy);
  b = 200.0 * (fy - fz);
}

// One 4x4 cell (cy, cx) of the global-hints statistics (global_stats.prototxt) of the uint8 RGB image img, w pixels
// wide: the cell's ab is the float64 row-major sum of its 16 pixels (rgb_u8_to_lab) from -0.0 / 16, rounded once to
// float32, and its bin the first minimum of the float32 ((a - pa)^2 + (b - pb)^2) over the 313 centres with every
// operation rounded separately (numpy's order, no FMA).  The 16 pixels' skimage HSV saturation is added to sat in the
// same order.  global_stats_kernel and global_stats_batch_kernel both call it, so they bin every cell alike.
__device__ __forceinline__ int stats_cell(const uint8_t* __restrict__ img, int w, int cy, int cx, const float2* bins,
                                          double& sat) {
  double sa = -0.0, sb = -0.0;
  for (int dy = 0; dy < 4; ++dy) {
    const uint8_t* row = img + ((size_t)(cy * 4 + dy) * w + cx * 4) * 3;
    for (int dx = 0; dx < 4; ++dx) {
      const uint8_t* px = row + dx * 3;
      double l, a, b;
      rgb_u8_to_lab(px, l, a, b);
      sa = __dadd_rn(sa, a);
      sb = __dadd_rn(sb, b);
      // skimage rgb2hsv: S = (max - min) / max of the /255 values, 0 where max = 0
      const double r8 = px[0] / 255.0, g8 = px[1] / 255.0, b8 = px[2] / 255.0;
      const double mx = fmax(r8, fmax(g8, b8)), mn = fmin(r8, fmin(g8, b8));
      sat = __dadd_rn(sat, mx > 0.0 ? __ddiv_rn(__dsub_rn(mx, mn), mx) : 0.0);
    }
  }
  const float a = __double2float_rn(__ddiv_rn(sa, 16.0)), b = __double2float_rn(__ddiv_rn(sb, 16.0));
  int best = 0;
  float bd = 0.f;
  for (int k = 0; k < 313; ++k) {
    const float da = __fsub_rn(a, bins[k].x), db = __fsub_rn(b, bins[k].y);
    const float d = __fadd_rn(__fmul_rn(da, da), __fmul_rn(db, db));
    if (k == 0 || d < bd) { bd = d; best = k; }
  }
  return best;
}

// OpenCV's source coordinate of output d, (float)((d + 0.5) * scale - 0.5) (modules/imgproc/src/resize.cpp), with the
// multiply and the subtract rounded separately as on the host (nvcc would fuse them).
__device__ __forceinline__ float cv_src_coord(int d, double scale) {
  return __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
}

// OpenCV resize, INTER_LINEAR, CV_8U (modules/imgproc/src/resize.cpp: resizeGeneric_ with HResizeLinear / VResizeLinear,
// INTER_RESIZE_COEF_BITS = 11).  x axis: fx is zeroed when the 2-tap window leaves the image; y axis: the coefficients
// are kept and the ROW INDICES are clipped instead.
__device__ __forceinline__ void cv_lin_coef(int d, double scale, int ssize, bool clamp_f, int& s, int& c0, int& c1) {
  float f = cv_src_coord(d, scale);
  s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (clamp_f) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= ssize - 1) { f = 0.f; s = ssize - 1; }
  }
  c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  c1 = __float2int_rn(__fmul_rn(f, 2048.f));
}

// cv::resize's scale of one axis, 1 / (dsize / ssize) as it computes it
__host__ __device__ __forceinline__ double cv_scale(int ssize, int dsize) { return 1.0 / ((double)dsize / (double)ssize); }

// One output pixel (dy, dx) of that resize from the uint8 RGB image src [hs,ws,3]: the exact-2x decimation (area2) is
// routed to the 2x2 area average as cv::resize does; otherwise the 11-bit fixed-point bilinear sum.
__device__ __forceinline__ void cv_resize_linear_px(const uint8_t* __restrict__ src, int hs, int ws, int dy, int dx,
                                                    double scale_y, double scale_x, bool area2, uint8_t* o) {
  if (area2) {
    const uint8_t* p = src + ((size_t)(2 * dy) * ws + 2 * dx) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = (uint8_t)((p[c] + p[3 + c] + p[(size_t)ws * 3 + c] + p[(size_t)ws * 3 + 3 + c] + 2) >> 2);
    return;
  }
  int sx, a0, a1, sy, b0, b1;
  cv_lin_coef(dx, scale_x, ws, true, sx, a0, a1);
  cv_lin_coef(dy, scale_y, hs, false, sy, b0, b1);
  const int x1 = sx + 1 < ws ? sx + 1 : ws - 1;
  const int y0 = sy < 0 ? 0 : (sy > hs - 1 ? hs - 1 : sy);
  const int y1 = sy + 1 < 0 ? 0 : (sy + 1 > hs - 1 ? hs - 1 : sy + 1);
  const uint8_t* r0 = src + (size_t)y0 * ws * 3;
  const uint8_t* r1 = src + (size_t)y1 * ws * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int S0 = r0[sx * 3 + c] * a0 + r0[x1 * 3 + c] * a1;
    const int S1 = r1[sx * 3 + c] * a0 + r1[x1 * 3 + c] * a1;
    const int v = (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2;
    o[c] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
  }
}

// One axis of scipy.ndimage.zoom(order 0 / 1, mode='constant', cval=0, grid_mode=False) as scipy 1.18 evaluates it
// (ni_interpolation.c NI_ZoomShift): output o samples c = o * ratio, ratio = (n_in-1)/(n_out-1) rounded to float64
// first; c > n_in-1 (the ratio rounded up) is outside the input and reads cval.  Order 0 takes floor(c + 0.5); order 1
// blends floor(c) and the next sample with w0 = 1 - t, w1 = 1 - w0 (scipy's weights; w1 = 0 at c = n_in-1).
// The ratio of one axis: np.divide(n_in - 1, n_out - 1), and 1 where n_out == 1 (scipy's zoom factor for a length-1
// output axis).
__host__ __device__ __forceinline__ double zoom_ratio(int n_in, int n_out) {
  return n_out > 1 ? (double)(n_in - 1) / (double)(n_out - 1) : 1.0;
}
struct ZoomTap {
  int i0, i1;
  double w0, w1;
  bool inside;
};
__device__ __forceinline__ ZoomTap zoom_tap(int o, double ratio, int n_in, int order) {
  ZoomTap t;
  const double c = __dmul_rn((double)o, ratio);
  t.inside = c <= (double)(n_in - 1);
  if (order == 0) {
    t.i0 = t.i1 = min((int)floor(__dadd_rn(c, 0.5)), n_in - 1);
    t.w0 = 1.0;
    t.w1 = 0.0;
  } else {
    const double f = floor(c);
    t.i0 = min((int)f, n_in - 1);
    t.i1 = min(t.i0 + 1, n_in - 1);
    t.w0 = __dsub_rn(1.0, __dsub_rn(c, f));
    t.w1 = __dsub_rn(1.0, t.w0);
  }
  return t;
}

// One plane zoomed at (ty, tx).  Order 1 adds the four taps in scipy's order, (v * wy) * wx each, no FMA, so the value
// equals scipy's bit for bit; order 0 is the sample itself.
__device__ __forceinline__ double zoom_sample(const double* __restrict__ p, int win, const ZoomTap& ty, const ZoomTap& tx,
                                              int order) {
  if (!(ty.inside && tx.inside)) return 0.0;
  const double v00 = __ldg(p + (size_t)ty.i0 * win + tx.i0);
  if (order == 0) return v00;
  const double v01 = __ldg(p + (size_t)ty.i0 * win + tx.i1);
  const double v10 = __ldg(p + (size_t)ty.i1 * win + tx.i0);
  const double v11 = __ldg(p + (size_t)ty.i1 * win + tx.i1);
  double s = __dmul_rn(__dmul_rn(v00, ty.w0), tx.w0);
  s = __dadd_rn(s, __dmul_rn(__dmul_rn(v01, ty.w0), tx.w1));
  s = __dadd_rn(s, __dmul_rn(__dmul_rn(v10, ty.w1), tx.w0));
  return __dadd_rn(s, __dmul_rn(__dmul_rn(v11, ty.w1), tx.w1));
}

__device__ __forceinline__ void pdl_prologue_done() {   // small kernels: let the successor start, then wait for the predecessor
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(Ctx* c, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                            Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_take(c) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#endif

}  // namespace idc
