// Colorization by optimization (Levin, Lischinski & Weiss 2004) on the hint planes of a reveal sweep: the classical
// baseline the network's reveal curve is compared against (DESIGN.md §4b).
//   levin_weights_kernel  one thread per pixel: the 8 normalised affinities w_pq of pixel p to its 3 x 3 neighbours,
//                         from Y = L / 100 of the photo's float64 Lab, 0 for a neighbour outside the image
//   levin_solve_kernel    one CTA per image, both ab channels in lockstep: FP64 BiCGSTAB from u = 0 on the system
//                         reduced to the free (unhinted) pixels, (I - W_ff) u_f = W_fh c_h, iterating on the device
//                         until each channel's true relative residual is below tol or max_iter is spent
// Every sum runs in a fixed order that depends only on the image size, so an image's result does not depend on where it
// sits in a batch or on the batch's other images.
#include <algorithm>

#include "idc_internal.h"

namespace idc {

// neighbour k of pixel (y, x) is (y + kDy[k], x + kDx[k]): the 3 x 3 window in row-major order without its centre
__constant__ int kLevinDy[8] = {-1, -1, -1, 0, 0, 1, 1, 1};
__constant__ int kLevinDx[8] = {-1, 0, 1, -1, 1, -1, 0, 1};
constexpr double kLn001 = -4.605170185988091;       // float64 ln(0.01), as numpy gives it
constexpr double kLevinVarScale = 0.6;
constexpr double kLevinSigmaFloor = 2e-6;

// Each operation rounded on its own (no FMA contraction), in the order tests/levin_ref.py evaluates it.
__global__ void __launch_bounds__(256) levin_weights_kernel(int h, int w, const double* __restrict__ lab,
                                                            double* __restrict__ wts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = h * w;
  if (i >= hw) return;
  const int y = i / w, x = i - y * w;
  const double* L = lab + (size_t)blockIdx.y * 3 * hw;
  const double yp = __ddiv_rn(L[i], 100.0);
  double g[8];
  bool in[8];
  double sum = yp, cnt = 1.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int yy = y + kLevinDy[k], xx = x + kLevinDx[k];
    in[k] = yy >= 0 && yy < h && xx >= 0 && xx < w;
    g[k] = in[k] ? __ddiv_rn(L[yy * w + xx], 100.0) : 0.0;
    if (in[k]) { sum = __dadd_rn(sum, g[k]); cnt = __dadd_rn(cnt, 1.0); }
  }
  // population variance of the window (neighbours and p): mean first, then the squared deviations in the same order
  const double mean = __ddiv_rn(sum, cnt);
  double dev = __dmul_rn(__dsub_rn(yp, mean), __dsub_rn(yp, mean));
  double m = INFINITY;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (!in[k]) continue;
    const double e = __dsub_rn(g[k], mean);
    dev = __dadd_rn(dev, __dmul_rn(e, e));
    const double d = __dsub_rn(g[k], yp);
    m = fmin(m, __dmul_rn(d, d));
  }
  double s = __dmul_rn(kLevinVarScale, __ddiv_rn(dev, cnt));
  s = fmax(s, __ddiv_rn(-m, kLn001));                 // the closest neighbour keeps at least 0.01 before normalising
  s = fmax(s, kLevinSigmaFloor);
  double e[8], tot = 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const double d = __dsub_rn(g[k], yp);
    e[k] = in[k] ? exp(__ddiv_rn(-__dmul_rn(d, d), s)) : 0.0;
    tot = __dadd_rn(tot, e[k]);
  }
  double* o = wts + (size_t)blockIdx.y * 8 * hw + i;
#pragma unroll
  for (int k = 0; k < 8; ++k) o[(size_t)k * hw] = __ddiv_rn(e[k], tot);
}

// ---- the batched solver ----
constexpr int kLevinThreads = 512;
constexpr int kLevinWarps = kLevinThreads / 32;
constexpr int kLevinVecs = 6;      // per channel: u, r (s in place), rhat, p, v, t

size_t levin_workspace_bytes(int n, int h, int w) {
  return (size_t)n * 2 * kLevinVecs * h * w * sizeof(double);
}

// Sum of K per-thread values over the CTA, in a fixed order: a shuffle tree within each warp, then warp 0 adds the
// warps' sums in a second tree.  Every thread gets the result.
template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K], double (*red)[kLevinWarps]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] = __dadd_rn(v[k], __shfl_down_sync(0xffffffffu, v[k], o));
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) red[k][warp] = v[k];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double t = lane < kLevinWarps ? red[k][lane] : 0.0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t = __dadd_rn(t, __shfl_down_sync(0xffffffffu, t, o));
      if (lane == 0) red[k][0] = t;                    // lanes read their slots before the first shuffle
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = red[k][0];
  __syncthreads();                                     // red is reused by the next reduction
}

struct LevinImage {
  const double* wts;      // [8][hw] of the image's photo
  const float* hint;      // ab_hint [2][hw]
  const float* mask;      // [hw]
  int h, w, hw;
};

// (A x)_p = x_p - sum_q w_pq x_q over free p, for x that is 0 on hinted pixels (so the hinted columns drop out)
__device__ __forceinline__ double levin_apply(const LevinImage& im, const double* x, int i, int y, int xcol) {
  double acc = 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int yy = y + kLevinDy[k], xx = xcol + kLevinDx[k];
    if (yy >= 0 && yy < im.h && xx >= 0 && xx < im.w)
      acc = __dadd_rn(acc, __dmul_rn(im.wts[(size_t)k * im.hw + i], x[yy * im.w + xx]));
  }
  return __dsub_rn(x[i], acc);
}

// b_p = sum over hinted q of w_pq c_q, for free p
__device__ __forceinline__ double levin_rhs(const LevinImage& im, int c, int i, int y, int xcol) {
  double acc = 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int yy = y + kLevinDy[k], xx = xcol + kLevinDx[k];
    if (yy >= 0 && yy < im.h && xx >= 0 && xx < im.w) {
      const int q = yy * im.w + xx;
      if (im.mask[q] > 0.f)
        acc = __dadd_rn(acc, __dmul_rn(im.wts[(size_t)k * im.hw + i], (double)im.hint[(size_t)c * im.hw + q]));
    }
  }
  return acc;
}

// grid n, one CTA per image.  Channel c's vectors live at ws + ((img * 2 + c) * kLevinVecs + v) * hw.  Vectors are 0 on
// hinted pixels throughout: only free pixels are ever written.  The global vectors are read by other threads of the CTA
// after __syncthreads, so they are plain (coherent) loads, never the read-only path.
__global__ void __launch_bounds__(kLevinThreads, 1) levin_solve_kernel(int levels, int h, int w,
                                                                      const double* __restrict__ wts,
                                                                      const float* __restrict__ ab_hint,
                                                                      const float* __restrict__ mask, double tol,
                                                                      int max_iter, float* __restrict__ out_ab,
                                                                      int* __restrict__ iters_out,
                                                                      double* __restrict__ relres_out, double* ws) {
  __shared__ double red[4][kLevinWarps];
  const int img = blockIdx.x;
  const int hw = h * w;
  LevinImage im;
  im.wts = wts + (size_t)(img / levels) * 8 * hw;
  im.hint = ab_hint + (size_t)img * 2 * hw;
  im.mask = mask + (size_t)img * hw;
  im.h = h;
  im.w = w;
  im.hw = hw;
  double* vec[2][kLevinVecs];
#pragma unroll
  for (int c = 0; c < 2; ++c) {
#pragma unroll
    for (int v = 0; v < kLevinVecs; ++v) vec[c][v] = ws + ((size_t)(img * 2 + c) * kLevinVecs + v) * hw;
  }
  enum { U = 0, R = 1, RH = 2, P = 3, V = 4, T = 5 };

  // u = 0, r = rhat = b, p = v = t = 0; ||b||^2 per channel
  double nb[2] = {0.0, 0.0};
  for (int i = threadIdx.x; i < hw; i += kLevinThreads) {
    const int y = i / w, x = i - y * w;
    const bool free_px = !(im.mask[i] > 0.f);
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const double b = free_px ? levin_rhs(im, c, i, y, x) : 0.0;
      vec[c][U][i] = 0.0;
      vec[c][R][i] = b;
      vec[c][RH][i] = b;
      vec[c][P][i] = 0.0;
      vec[c][V][i] = 0.0;
      vec[c][T][i] = 0.0;
      nb[c] = __dadd_rn(nb[c], __dmul_rn(b, b));
    }
  }
  block_sum<2>(nb, red);                               // also orders the initialisation before the first iteration
  double bnorm[2], rho[2], alpha[2], omega[2], res[2];
  bool active[2];
  int it[2] = {0, 0};
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    bnorm[c] = sqrt(nb[c]);
    rho[c] = alpha[c] = omega[c] = 1.0;
    res[c] = bnorm[c] > 0.0 ? 1.0 : 0.0;
    active[c] = bnorm[c] > 0.0;                        // b = 0 (no hint reaches a free pixel): u = 0 exactly
  }
  double rho_new[2] = {nb[0], nb[1]};                  // (rhat, r) with rhat = r = b

  while (active[0] || active[1]) {
    // p = r + beta (p - omega v); a channel whose (rhat, r) vanished restarts below through the true residual
    double beta[2];
    bool breakdown[2] = {false, false};
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      if (!active[c]) continue;
      ++it[c];
      breakdown[c] = rho_new[c] == 0.0;
      beta[c] = __dmul_rn(__ddiv_rn(rho_new[c], rho[c]), __ddiv_rn(alpha[c], omega[c]));
      rho[c] = rho_new[c];
    }
    const bool go0 = active[0] && !breakdown[0], go1 = active[1] && !breakdown[1];
    for (int i = threadIdx.x; i < hw; i += kLevinThreads) {
      if (im.mask[i] > 0.f) continue;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        if (!(c ? go1 : go0)) continue;
        vec[c][P][i] = __dadd_rn(vec[c][R][i], __dmul_rn(beta[c], __dsub_rn(vec[c][P][i], __dmul_rn(omega[c], vec[c][V][i]))));
      }
    }
    __syncthreads();
    // v = A p; (rhat, v)
    double d[2] = {0.0, 0.0};
    for (int i = threadIdx.x; i < hw; i += kLevinThreads) {
      if (im.mask[i] > 0.f) continue;
      const int y = i / w, x = i - y * w;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        if (!(c ? go1 : go0)) continue;
        const double v = levin_apply(im, vec[c][P], i, y, x);
        vec[c][V][i] = v;
        d[c] = __dadd_rn(d[c], __dmul_rn(vec[c][RH][i], v));
      }
    }
    block_sum<2>(d, red);
    bool go[2] = {go0, go1};
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      if (!go[c]) continue;
      if (d[c] == 0.0) { breakdown[c] = true; go[c] = false; continue; }
      alpha[c] = __ddiv_rn(rho[c], d[c]);
    }
    // s = r - alpha v, in place of r
    for (int i = threadIdx.x; i < hw; i += kLevinThreads) {
      if (im.mask[i] > 0.f) continue;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        if (!go[c]) continue;
        vec[c][R][i] = __dsub_rn(vec[c][R][i], __dmul_rn(alpha[c], vec[c][V][i]));
      }
    }
    __syncthreads();
    // t = A s; (t, s), (t, t)
    double q[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < hw; i += kLevinThreads) {
      if (im.mask[i] > 0.f) continue;
      const int y = i / w, x = i - y * w;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        if (!go[c]) continue;
        const double t = levin_apply(im, vec[c][R], i, y, x);
        vec[c][T][i] = t;
        q[2 * c] = __dadd_rn(q[2 * c], __dmul_rn(t, vec[c][R][i]));
        q[2 * c + 1] = __dadd_rn(q[2 * c + 1], __dmul_rn(t, t));
      }
    }
    block_sum<4>(q, red);
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      if (!go[c]) continue;
      // t = 0 means s = 0 (A is non-singular on the reachable pixels): the step u + alpha p is exact
      omega[c] = q[2 * c + 1] > 0.0 ? __ddiv_rn(q[2 * c], q[2 * c + 1]) : 0.0;
    }
    // u += alpha p + omega s; r = s - omega t; (rhat, r), (r, r)
    double e[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < hw; i += kLevinThreads) {
      if (im.mask[i] > 0.f) continue;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        if (!go[c]) continue;
        const double s = vec[c][R][i];
        vec[c][U][i] = __dadd_rn(vec[c][U][i], __dadd_rn(__dmul_rn(alpha[c], vec[c][P][i]), __dmul_rn(omega[c], s)));
        const double r = __dsub_rn(s, __dmul_rn(omega[c], vec[c][T][i]));
        vec[c][R][i] = r;
        e[2 * c] = __dadd_rn(e[2 * c], __dmul_rn(vec[c][RH][i], r));
        e[2 * c + 1] = __dadd_rn(e[2 * c + 1], __dmul_rn(r, r));
      }
    }
    block_sum<4>(e, red);
    // A channel whose recursive residual is below tol, that broke down (a zero (rhat, r), (rhat, v) or omega) or that
    // spent max_iter checks its TRUE residual b - A u: below tol it stops; otherwise it restarts from u with
    // r = rhat = the true residual, or stops unconverged at max_iter.
    bool check[2];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      check[c] = false;
      if (!active[c]) continue;
      if (go[c]) rho_new[c] = e[2 * c];
      check[c] = !go[c] || omega[c] == 0.0 || sqrt(e[2 * c + 1]) <= tol * bnorm[c] || it[c] >= max_iter;
    }
    if (check[0] || check[1]) {
      double tr[2] = {0.0, 0.0};
      for (int i = threadIdx.x; i < hw; i += kLevinThreads) {
        if (im.mask[i] > 0.f) continue;
        const int y = i / w, x = i - y * w;
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          if (!check[c]) continue;
          const double r = __dsub_rn(levin_rhs(im, c, i, y, x), levin_apply(im, vec[c][U], i, y, x));
          vec[c][T][i] = r;                            // staged: r and rhat are still read by other threads
          tr[c] = __dadd_rn(tr[c], __dmul_rn(r, r));
        }
      }
      block_sum<2>(tr, red);
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        if (!check[c]) continue;
        res[c] = __ddiv_rn(sqrt(tr[c]), bnorm[c]);
        if (res[c] <= tol || it[c] >= max_iter) {
          active[c] = false;
          check[c] = false;
        } else {
          rho[c] = alpha[c] = omega[c] = 1.0;
          rho_new[c] = tr[c];
        }
      }
      if (check[0] || check[1]) {                      // restarts: r = rhat = the true residual, p = v = 0
        for (int i = threadIdx.x; i < hw; i += kLevinThreads) {
          if (im.mask[i] > 0.f) continue;
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            if (!check[c]) continue;
            const double r = vec[c][T][i];
            vec[c][R][i] = r;
            vec[c][RH][i] = r;
            vec[c][P][i] = 0.0;
            vec[c][V][i] = 0.0;
          }
        }
        __syncthreads();
      }
    }
  }

  // u on free pixels, the hint on hinted ones
  for (int i = threadIdx.x; i < hw; i += kLevinThreads) {
    const bool hinted = im.mask[i] > 0.f;
#pragma unroll
    for (int c = 0; c < 2; ++c)
      out_ab[((size_t)img * 2 + c) * hw + i] = hinted ? im.hint[(size_t)c * hw + i] : __double2float_rn(vec[c][U][i]);
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      iters_out[img * 2 + c] = it[c];
      relres_out[img * 2 + c] = res[c];
    }
  }
}

cudaError_t launch_levin_weights(int n, int h, int w, const double* lab, double* wts, cudaStream_t st) {
  const dim3 grid((unsigned)((h * w + 255) / 256), (unsigned)n);
  levin_weights_kernel<<<grid, 256, 0, st>>>(h, w, lab, wts);
  return cudaGetLastError();
}

cudaError_t launch_levin_solve(int n, int levels, int h, int w, const double* wts, const float* ab_hint,
                               const float* mask, double tol, int max_iter, float* out_ab, int32_t* iters,
                               double* relres, void* workspace, cudaStream_t st) {
  levin_solve_kernel<<<(unsigned)n, kLevinThreads, 0, st>>>(levels, h, w, wts, ab_hint, mask, tol, max_iter, out_ab,
                                                            iters, relres, static_cast<double*>(workspace));
  return cudaGetLastError();
}

}  // namespace idc
