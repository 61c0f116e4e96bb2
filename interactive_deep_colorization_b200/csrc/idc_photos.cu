// Batched photos: both ends of the automatic-colorization loop (load_image -> net_forward -> get_img_fullres,
// data/colorize_image.py:52-66, :123-131) for a batch of photos of any sizes, one launch per batch each.
//   photo_prep_kernel    one thread per pixel of the X x X network grid per photo: cv2's 8-bit INTER_LINEAR resize of
//                        the photo's own source (cv_resize_linear_px), rgb_u8_to_lab, L - 50 -> the forward's L input
//   photo_render_kernel  one thread per full-resolution pixel of every photo: L from the pixel's own source RGB, ab
//                        zoomed from the photo's quantised output_ab (zoom_tap / zoom_sample), lab_to_rgb_u8
//   rgb_sse_kernel       exact int64 sum of squared differences per image (get_result_PSNR before its float64 tail)
//   hint_fill_mean_kernel  one thread per hint of a batch of hint blocks: the mean ground-truth ab under the hint's
//                        rectangle (a simulated user revealing points of the photo's own colours)
//   global_stats_batch_kernel  one CTA per network-size image: the global-hints statistics (313-bin histogram of the
//                        4x4-pooled ab, mean HSV saturation) of a batch, deterministic and independent of the batch
// The per-pixel arithmetic is the one of resize_linear_u8_kernel, rgb2lab_kernel and render_planes_kernel (the device
// functions in idc_internal.h), so every photo equals the single-image path bit for bit.
#include <algorithm>

#include "idc_internal.h"

namespace idc {

// The photo table travels as a kernel parameter (constant bank): 2 KB at IDC_MAX_PHOTOS, read uniformly by a block.
struct PhotoTable {
  idc_photo p[IDC_MAX_PHOTOS];
};

// Photo of flattened pixel i: the last entry with off <= i (offsets ascend), or -1 before the first photo.
__device__ __forceinline__ int photo_of(const PhotoTable& t, int n, int64_t i) {
  int lo = 0, hi = n - 1, r = -1;
  while (lo <= hi) {
    const int mid = (lo + hi) >> 1;
    if (t.p[mid].off <= i) { r = mid; lo = mid + 1; } else { hi = mid - 1; }
  }
  return r;
}

__global__ void __launch_bounds__(256) photo_prep_kernel(const __grid_constant__ PhotoTable t, const uint8_t* __restrict__ src,
                                                         int X, float* __restrict__ L_mc, uint8_t* __restrict__ rgb) {
  const int p = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= X * X) return;
  const idc_photo ph = t.p[p];
  const int dy = i / X, dx = i - dy * X;
  uint8_t px[3];
  cv_resize_linear_px(src + (size_t)ph.off * 3, ph.h, ph.w, dy, dx, cv_scale(ph.h, X), cv_scale(ph.w, X),
                      ph.w == 2 * X && ph.h == 2 * X, px);
  double l, a, b;
  rgb_u8_to_lab(px, l, a, b);
  const size_t o = (size_t)p * X * X + i;
  L_mc[o] = __double2float_rn(__dsub_rn(l, 50.0));   // img_lab / l_norm - l_mean / l_norm with l_norm 1, l_mean 50
  if (rgb) {
    rgb[o * 3 + 0] = px[0];
    rgb[o * 3 + 1] = px[1];
    rgb[o * 3 + 2] = px[2];
  }
}

// src and out may be the same buffer: a thread reads its own source pixel before it writes it, and nothing else.
__global__ void __launch_bounds__(256) photo_render_kernel(const __grid_constant__ PhotoTable t, int n, int64_t total,
                                                           const uint8_t* src, int X, const double* __restrict__ lab,
                                                           uint8_t* out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int p = photo_of(t, n, i);
  if (p < 0) return;
  const idc_photo ph = t.p[p];
  const int64_t r = i - ph.off;
  if (r >= (int64_t)ph.h * ph.w) return;             // a gap between two photos
  const int y = (int)(r / ph.w), x = (int)(r - (int64_t)y * ph.w);
  double l, a0, b0;
  rgb_u8_to_lab(src + i * 3, l, a0, b0);
  const double* ab = lab + ((size_t)p * 3 + 1) * X * X;
  const ZoomTap ty = zoom_tap(y, zoom_ratio(X, ph.h), X, 1), tx = zoom_tap(x, zoom_ratio(X, ph.w), X, 1);
  const double a = zoom_sample(ab, X, ty, tx, 1);
  const double b = zoom_sample(ab + (size_t)X * X, X, ty, tx, 1);
  lab_to_rgb_u8(l, a, b, out + i * 3);
}

// grid (chunks, n): each block sums its slice of image blockIdx.y in int64 and adds it to sse[img] (integer adds, so
// the order does not matter and the result is exact)
__global__ void __launch_bounds__(256) rgb_sse_kernel(size_t hw3, const uint8_t* __restrict__ a, const uint8_t* __restrict__ b,
                                                      unsigned long long* __restrict__ sse) {
  __shared__ unsigned long long s_warp[8];
  const int img = blockIdx.y;
  const uint8_t* pa = a + (size_t)img * hw3;
  const uint8_t* pb = b + (size_t)img * hw3;
  unsigned long long acc = 0;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < hw3; j += (size_t)gridDim.x * blockDim.x) {
    const int d = (int)pa[j] - (int)pb[j];
    acc += (unsigned long long)(d * d);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long s = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += s_warp[w];
    atomicAdd(sse + img, s);
  }
}

// grid (chunks, n_blocks): thread i of column b sets hint i of block b to the mean of planes 1-2 of photo b / levels of
// lab over the hint's rectangle clipped to X x X, summed in float64 in row-major order and rounded once to float32.
// The sums start at -0.0, the identity of IEEE addition, so they equal a sequential sum from the first pixel bit for
// bit (signed zeros included).  A hint whose clipped rectangle is empty gets (0, 0); the raster skips it anyway.
constexpr int kFillThreads = 128;

__global__ void __launch_bounds__(kFillThreads) hint_fill_mean_kernel(int levels, int X, const double* __restrict__ lab,
                                                                      char* __restrict__ blocks, size_t stride, int cap) {
  char* blk = blocks + (size_t)blockIdx.y * stride;
  const int count = min(max(*reinterpret_cast<const int*>(blk), 0), cap);   // as the raster reads it, within the stride
  const int i = blockIdx.x * kFillThreads + threadIdx.x;
  if (i >= count) return;
  idc_hint* h = reinterpret_cast<idc_hint*>(blk + kHintHdrBytes) + i;
  const int y0 = max(h->y0, 0), x0 = max(h->x0, 0), y1 = min(h->y1, X - 1), x1 = min(h->x1, X - 1);
  float a = 0.f, b = 0.f;
  if (y0 <= y1 && x0 <= x1) {
    const size_t XX = (size_t)X * X;
    const double* pa = lab + ((size_t)(blockIdx.y / levels) * 3 + 1) * XX;
    const double* pb = pa + XX;
    double sa = -0.0, sb = -0.0;
    for (int y = y0; y <= y1; ++y) {
      for (int x = x0; x <= x1; ++x) {
        sa = __dadd_rn(sa, pa[(size_t)y * X + x]);
        sb = __dadd_rn(sb, pb[(size_t)y * X + x]);
      }
    }
    const double cnt = (double)((int64_t)(y1 - y0 + 1) * (x1 - x0 + 1));
    a = __double2float_rn(__ddiv_rn(sa, cnt));
    b = __double2float_rn(__ddiv_rn(sb, cnt));
  }
  h->a = a;
  h->b = b;
}

// grid n, one CTA per image: global_stats.prototxt (rgb2lab -> 4x4 average pool of ab -> nearest of the 313 bins ->
// global average; mean HSV saturation) for image blockIdx.x of rgb [n,h,w,3].  Thread t takes cells t, t + T, ...,
// each through stats_cell (idc_internal.h), the routine of the single-image global_stats_kernel.  Bin counts are
// integer shared-memory atomics; the saturation partials are reduced in a fixed tree.  Nothing depends on n or on
// where the image sits in the batch, so a row is identical bit for bit in any batch and on every run.
constexpr int kStatsThreads = 512;

__global__ void __launch_bounds__(kStatsThreads, 1) global_stats_batch_kernel(int h, int w, const uint8_t* __restrict__ rgb,
                                                                           const float* __restrict__ pts,
                                                                           float* __restrict__ out) {
  __shared__ int count[313];
  __shared__ float2 bins[313];
  __shared__ double s_warp[kStatsThreads / 32];
  for (int k = threadIdx.x; k < 313; k += kStatsThreads) {
    count[k] = 0;
    bins[k] = make_float2(pts[2 * k], pts[2 * k + 1]);
  }
  __syncthreads();
  const uint8_t* img = rgb + (size_t)blockIdx.x * h * w * 3;
  const int w4 = w / 4, cells = (h / 4) * w4;
  double sat = 0.0;
  for (int c = threadIdx.x; c < cells; c += kStatsThreads) {
    const int cy = c / w4, cx = c - cy * w4;
    atomicAdd(&count[stats_cell(img, w, cy, cx, bins, sat)], 1);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sat = __dadd_rn(sat, __shfl_xor_sync(0xffffffffu, sat, o));
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = sat;
  __syncthreads();
  float* o = out + (size_t)blockIdx.x * 316;
  for (int k = threadIdx.x; k < 313; k += kStatsThreads)
    o[k] = __double2float_rn(__ddiv_rn((double)count[k], (double)cells));
  if (threadIdx.x == 0) {
    double t = s_warp[0];
    for (int i = 1; i < kStatsThreads / 32; ++i) t = __dadd_rn(t, s_warp[i]);
    o[313] = 1.f;
    o[314] = __double2float_rn(__ddiv_rn(t, (double)h * w));
    o[315] = 1.f;
  }
}

static PhotoTable make_table(int n, const idc_photo* table) {
  PhotoTable t{};
  for (int i = 0; i < n; ++i) t.p[i] = table[i];
  return t;
}

cudaError_t launch_photo_prep(int n, const idc_photo* table, const uint8_t* src, int X, float* L_mc, uint8_t* rgb,
                              cudaStream_t st) {
  const dim3 grid((unsigned)((X * X + 255) / 256), (unsigned)n);
  photo_prep_kernel<<<grid, 256, 0, st>>>(make_table(n, table), src, X, L_mc, rgb);
  return cudaGetLastError();
}

cudaError_t launch_photo_render(int n, const idc_photo* table, const uint8_t* src, int X, const double* lab, uint8_t* out,
                                cudaStream_t st) {
  const int64_t total = table[n - 1].off + (int64_t)table[n - 1].h * table[n - 1].w;
  photo_render_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(make_table(n, table), n, total, src, X, lab, out);
  return cudaGetLastError();
}

cudaError_t launch_rgb_sse(int n, size_t hw3, const uint8_t* a, const uint8_t* b, int64_t* sse, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(sse, 0, (size_t)n * sizeof(int64_t), st);
  if (e != cudaSuccess) return e;
  const dim3 grid((unsigned)std::min<size_t>((hw3 + 255) / 256, 64), (unsigned)n);
  rgb_sse_kernel<<<grid, 256, 0, st>>>(hw3, a, b, reinterpret_cast<unsigned long long*>(sse));
  return cudaGetLastError();
}

cudaError_t launch_hint_fill_mean(int n_blocks, int levels, int X, const double* lab, char* blocks, size_t stride,
                                  cudaStream_t st) {
  const int cap = (int)std::min<size_t>((stride - kHintHdrBytes) / sizeof(idc_hint), IDC_MAX_HINTS);
  if (cap == 0) return cudaSuccess;                      // blocks without room for a hint: nothing to fill
  const dim3 grid((unsigned)((cap + kFillThreads - 1) / kFillThreads), (unsigned)n_blocks);
  hint_fill_mean_kernel<<<grid, kFillThreads, 0, st>>>(levels, X, lab, blocks, stride, cap);
  return cudaGetLastError();
}

cudaError_t launch_global_stats_batch(int n, int h, int w, const uint8_t* rgb, const float* pts, float* out,
                                      cudaStream_t st) {
  global_stats_batch_kernel<<<(unsigned)n, kStatsThreads, 0, st>>>(h, w, rgb, pts, out);
  return cudaGetLastError();
}

}  // namespace idc
