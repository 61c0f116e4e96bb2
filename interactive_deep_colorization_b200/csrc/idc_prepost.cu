// Row f1 (SURVEY 8f): the image-load side of the wrapper on the GPU.
//   resize_linear_u8_kernel   cv2.resize(im, (Xd, Xd)) of `load_image` (data/colorize_image.py:52-66): OpenCV's 8-bit
//                             INTER_LINEAR is FIXED-POINT arithmetic (11-bit coefficients, 22-bit products); the kernel
//                             restates it integer for integer, so the result is bit-identical to cv2 (including the
//                             exact-2x shortcut to area averaging and the different border rules of the two axes).
//   cubic_lab2rgb_kernel      the GUI's display step (ui/gui_draw.py:280-283): cv2.resize(ab, win, INTER_CUBIC) of the
//                             float64 ab planes, concatenated with the window-size L, skimage lab2rgb, clip, x255,
//                             truncating cast -- one kernel, float64 like the host path.
// The Lab -> RGB step is lab_to_rgb_u8 (idc_internal.h), the one idc_heads.cu's renders use.
#include "idc_internal.h"

namespace idc {

// cv_src_coord, cv_lin_coef and cv_resize_linear_px live in idc_internal.h, shared with the batched photo prep.
__global__ void resize_linear_u8_kernel(const uint8_t* __restrict__ src, int hs, int ws, uint8_t* __restrict__ dst,
                                        int hd, int wd, double scale_y, double scale_x, int area2) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)hd * wd) return;
  const int dy = (int)(i / wd), dx = (int)(i - (size_t)dy * wd);
  cv_resize_linear_px(src, hs, ws, dy, dx, scale_y, scale_x, area2 != 0, dst + i * 3);
}

cudaError_t launch_resize_linear_u8(const uint8_t* src, int hs, int ws, uint8_t* dst, int hd, int wd, cudaStream_t st) {
  const double scale_x = cv_scale(ws, wd), scale_y = cv_scale(hs, hd);
  const int area2 = (ws == 2 * wd && hs == 2 * hd) ? 1 : 0;
  const size_t tot = (size_t)hd * wd;
  resize_linear_u8_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(src, hs, ws, dst, hd, wd, scale_y, scale_x, area2);
  return cudaGetLastError();
}

// OpenCV interpolateCubic (A = -0.75) in float32, each operation rounded on its own in OpenCV's order (nvcc would
// contract the polynomial into FMAs); taps s-1 .. s+2 with clipped indices
__device__ __forceinline__ void cv_cubic_coef(int d, double scale, int& s, float (&w)[4]) {
  const float f = cv_src_coord(d, scale);
  s = (int)floorf(f);
  const float x = __fsub_rn(f, (float)s);
  const float A = -0.75f, A5 = 5 * A, A8 = 8 * A, A4 = 4 * A, A2 = A + 2, A3 = A + 3;   // exact in float32
  const float x1 = __fadd_rn(x, 1.f), y = __fsub_rn(1.f, x);
  w[0] = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x1), A5), x1), A8), x1), A4);
  w[1] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A2, x), A3), x), x), 1.f);
  w[2] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A2, y), A3), y), y), 1.f);
  w[3] = __fsub_rn(__fsub_rn(__fsub_rn(1.f, w[0]), w[1]), w[2]);
}

// cv2's float64 INTER_CUBIC (HResizeCubic, then VResizeCubic): per source row the four products v * wx summed left to
// right, then the four rows weighted by wy the same way; every product and sum rounded on its own, so the resized ab
// equals cv2's bit for bit (tests/cubic_ref.py)
__global__ void cubic_lab2rgb_kernel(const double* __restrict__ ab, int hin, int win, const double* __restrict__ L,
                                     int H, int W, double scale_y, double scale_x, uint8_t* __restrict__ rgb) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)H * W) return;
  const int dy = (int)(i / W), dx = (int)(i - (size_t)dy * W);
  int sx, sy;
  float wx[4], wy[4];
  cv_cubic_coef(dx, scale_x, sx, wx);
  cv_cubic_coef(dy, scale_y, sy, wy);
  int xs[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) xs[k] = min(max(sx - 1 + k, 0), win - 1);
  double v[2];
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const double* p = ab + (size_t)c * hin * win;
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double* r = p + (size_t)min(max(sy - 1 + j, 0), hin - 1) * win;
      double row = __dmul_rn(r[xs[0]], (double)wx[0]);
#pragma unroll
      for (int k = 1; k < 4; ++k) row = __dadd_rn(row, __dmul_rn(r[xs[k]], (double)wx[k]));
      const double t = __dmul_rn(row, (double)wy[j]);
      acc = j == 0 ? t : __dadd_rn(acc, t);
    }
    v[c] = acc;
  }
  lab_to_rgb_u8(L[i], v[0], v[1], rgb + i * 3);
}

cudaError_t launch_cubic_lab2rgb(const double* ab, int hin, int win, const double* L, int H, int W, uint8_t* rgb,
                                 cudaStream_t st) {
  const double scale_x = 1.0 / ((double)W / win), scale_y = 1.0 / ((double)H / hin);
  const size_t tot = (size_t)H * W;
  cubic_lab2rgb_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(ab, hin, win, L, H, W, scale_y, scale_x, rgb);
  return cudaGetLastError();
}

}  // namespace idc
