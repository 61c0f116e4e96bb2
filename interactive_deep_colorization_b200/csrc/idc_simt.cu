// FP32 CUDA-core engine: generic gather-GEMM convolution (3x3 / dilated / decimated-input /
// transposed-conv parity classes + fused shortcut) with the fused epilogue
//     v = act(acc + bias) * bn_scale + bn_shift (+ global-hints vector).
// Exact-FP32 reference engine of the product (IDC_FLAG_ENGINE_SIMT); the wgmma engine in
// idc_umma.cu computes the same ops from the same tap tables.
// Reference semantics: nn.Conv2d / nn.ConvTranspose2d / nn.BatchNorm2d(eval) / ReLU as wired in
// /root/reference/models/pytorch/model.py:13-102,149-165.
#include "idc_internal.h"

namespace idc {

struct SimtParams {
  const float* src[kMaxSrc];
  int sH[kMaxSrc], sW[kMaxSrc], sC[kMaxSrc], ss[kMaxSrc];
  int ntaps;
  int tsrc[kMaxTaps], tty[kMaxTaps], ttx[kMaxTaps], tk0[kMaxTaps];
  const float* w;  // [K][cout_pad]
  int K, cout_pad, cout;
  int N, Hl, Wl;
  float* out;
  int Hout, Wout, os, oy0, ox0, out_ld;
  const float* bias;
  const float* scale;
  const float* shift;
  const float* gadd;
  int act;
};

constexpr int BM = 64, BN = 64, BK = 16;

__global__ void __launch_bounds__(256) simt_conv_kernel(const SimtParams p) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN];
  const int tid = threadIdx.x;
  const int M = p.N * p.Hl * p.Wl;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  // A-loader coordinates
  const int pm = tid >> 2, cq = tid & 3;
  const int m = m0 + pm;
  const bool mvalid = m < M;
  int img = 0, y = 0, x = 0;
  if (mvalid) {
    img = m / (p.Hl * p.Wl);
    int r = m - img * p.Hl * p.Wl;
    y = r / p.Wl;
    x = r - y * p.Wl;
  }
  const int kb = tid >> 4, nq = tid & 15;
  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int t = 0; t < p.ntaps; ++t) {
    const int s = p.tsrc[t];
    const int iy = y * p.ss[s] + p.tty[t], ix = x * p.ss[s] + p.ttx[t];
    const bool inb = mvalid && iy >= 0 && iy < p.sH[s] && ix >= 0 && ix < p.sW[s];
    const int C = p.sC[s];
    const float* ap = p.src[s] + ((size_t)(img * p.sH[s] + iy) * p.sW[s] + ix) * C + cq * 4;
    const float* wp = p.w + (size_t)(p.tk0[t] + kb) * p.cout_pad + n0 + nq * 4;
    for (int c0 = 0; c0 < C; c0 += BK) {
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      if (inb) a = __ldg(reinterpret_cast<const float4*>(ap + c0));
      float4 b = __ldg(reinterpret_cast<const float4*>(wp + (size_t)c0 * p.cout_pad));
      As[cq * 4 + 0][pm] = a.x;
      As[cq * 4 + 1][pm] = a.y;
      As[cq * 4 + 2][pm] = a.z;
      As[cq * 4 + 3][pm] = a.w;
      *reinterpret_cast<float4*>(&Bs[kb][nq * 4]) = b;
      __syncthreads();
#pragma unroll
      for (int k = 0; k < BK; ++k) {
        const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
        const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
        const float a4[4] = {av.x, av.y, av.z, av.w};
        const float b4[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a4[i], b4[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
  // epilogue
  const int co0 = n0 + tx * 4;
  float bias[4], sc[4], sh[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    bias[j] = p.bias[co0 + j];
    sc[j] = p.scale[co0 + j];
    sh[j] = p.shift[co0 + j];
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int mm = m0 + ty * 4 + i;
    if (mm >= M) continue;
    const int im = mm / (p.Hl * p.Wl);
    const int r = mm - im * p.Hl * p.Wl;
    const int yy = r / p.Wl, xx = r - yy * p.Wl;
    const int oy = yy * p.os + p.oy0, ox = xx * p.os + p.ox0;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float t = acc[i][j] + bias[j];
      if (p.act == ACT_RELU) t = fmaxf(t, 0.f);
      else if (p.act == ACT_LEAKY02) t = t > 0.f ? t : 0.2f * t;
      t = t * sc[j] + sh[j];
      if (p.gadd) t += p.gadd[(size_t)im * p.cout + co0 + j];
      v[j] = t;
    }
    float* op = p.out + ((size_t)(im * p.Hout + oy) * p.Wout + ox) * p.out_ld + co0;
    *reinterpret_cast<float4*>(op) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

cudaError_t simt_run_op(Ctx* c, ConvOp& op, int n, cudaStream_t st) {
  for (int cls = 0; cls < op.ncls; ++cls) {
    SimtParams p{};
    for (int s = 0; s < op.nsrc; ++s) {
      const ActBuf& b = c->bufs[op.src[s].buf];
      p.src[s] = static_cast<const float*>(b.p0.get());
      p.sH[s] = b.H; p.sW[s] = b.W; p.sC[s] = b.C; p.ss[s] = op.src[s].s;
    }
    p.ntaps = op.ntaps;
    int k0 = 0;
    for (int t = 0; t < op.ntaps; ++t) {
      const Tap& tp = op.taps[cls][t];
      p.tsrc[t] = tp.src; p.tty[t] = tp.ty; p.ttx[t] = tp.tx; p.tk0[t] = k0;
      k0 += op.src[tp.src].cin;
    }
    p.K = op.K; p.cout_pad = op.cout_pad; p.cout = op.cout;
    p.w = op.w_simt + (size_t)cls * op.K * op.cout_pad;
    p.N = n; p.Hl = op.Hl; p.Wl = op.Wl;
    if (op.out_f32) {
      p.out = op.out_f32_ptr; p.Hout = op.Hl; p.Wout = op.Wl; p.os = 1; p.oy0 = 0; p.ox0 = 0;
      p.out_ld = op.cout_pad;
    } else {
      const ActBuf& ob = c->bufs[op.out_buf];
      p.out = static_cast<float*>(ob.p0.get()); p.Hout = ob.H; p.Wout = ob.W; p.os = op.os;
      p.oy0 = cls >> 1; p.ox0 = cls & 1; p.out_ld = ob.C;
    }
    p.bias = op.epi.bias; p.scale = op.epi.scale; p.shift = op.epi.shift;
    p.gadd = (op.epi.gadd && c->gadd_active) ? c->gvec.get() : nullptr;
    p.act = op.epi.act;
    const int M = n * op.Hl * op.Wl;
    dim3 grid(ceil_div(M, BM), op.cout_pad / BN);
    simt_conv_kernel<<<grid, 256, 0, st>>>(p);
    c->launch_count++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace idc
