// C ABI of libidc_b200.so (include/idc_b200.h): context, layer plan, weight packing, forward.
// The plan restates the wiring of SIGGRAPHGenerator.forward
// (/root/reference/models/pytorch/model.py:134-175) as a list of gather-GEMM ops; both engines
// (idc_simt.cu FP32 CUDA cores, idc_umma.cu wgmma) execute the same list.
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cmath>

#include "idc_internal.h"

using namespace idc;

struct idc_ctx : public idc::Ctx {};

namespace {

int fail(Ctx* c, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (c) c->err = buf;
  return code;
}

#define CUDA_TRY(c, expr)                                                                         \
  do {                                                                                            \
    cudaError_t e__ = (expr);                                                                     \
    if (e__ != cudaSuccess)                                                                       \
      return fail(c, IDC_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

constexpr float kBnEps = 1e-5f;  // nn.BatchNorm2d default (SURVEY q7)

int add_buf(Ctx* c, const char* name, int H, int W, int C) {
  ActBuf b;
  b.name = name; b.H = H; b.W = W; b.C = C;
  c->bufs.push_back(std::move(b));
  c->buf_index[name] = (int)c->bufs.size() - 1;
  return (int)c->bufs.size() - 1;
}

// 3x3 conv (optionally dilated, optionally reading the ::2 decimation of its source)
void add_conv(Ctx* c, const char* name, const char* wkey, const char* in, int s, int dil, const char* out, int act,
              const char* bnkey, bool gadd = false) {
  ConvOp op;
  op.name = name; op.kind = OP_CONV; op.wkey[0] = wkey; op.bnkey = bnkey ? bnkey : "";
  const ActBuf& ib = c->bufs[c->buf_index.at(in)];
  const ActBuf& ob = c->bufs[c->buf_index.at(out)];
  op.nsrc = 1;
  op.src[0].buf = c->buf_index.at(in); op.src[0].s = s; op.src[0].cin = ib.C;
  op.ncls = 1; op.ntaps = 9;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      Tap& t = op.taps[0][ky * 3 + kx];
      t.src = 0; t.ky = ky; t.kx = kx; t.ty = s * (ky - 1) * dil; t.tx = s * (kx - 1) * dil;
    }
  op.Hl = ob.H; op.Wl = ob.W; op.out_buf = c->buf_index.at(out); op.os = 1;
  op.cout = ob.C; op.cout_pad = ob.C; op.K = 9 * ib.C;
  op.epi.act = act; op.epi.has_bn = bnkey != nullptr; op.epi.gadd = gadd;
  op.flops_per_image = 2.0 * op.Hl * op.Wl * (double)op.cout * op.K;
  c->ops.push_back(std::move(op));
}

// ConvTranspose2d(4x4, s2, p1) of `lo` + Conv2d(3x3) of the skip tensor, summed, then ReLU
// (model.py:156-157,162-165: modelNup(x) + modelKshortN(skip), followed by modelN[0] = ReLU).
void add_up(Ctx* c, const char* name, const char* dkey, const char* lo, const char* skey, const char* skip,
            const char* out) {
  ConvOp op;
  op.name = name; op.kind = OP_UP; op.wkey[0] = dkey; op.wkey[1] = skey;
  op.src_deconv[0] = true; op.src_k[0] = 4;
  const ActBuf& lb = c->bufs[c->buf_index.at(lo)];
  const ActBuf& sb = c->bufs[c->buf_index.at(skip)];
  const ActBuf& ob = c->bufs[c->buf_index.at(out)];
  op.nsrc = 2;
  op.src[0].buf = c->buf_index.at(lo); op.src[0].s = 1; op.src[0].cin = lb.C;
  op.src[1].buf = c->buf_index.at(skip); op.src[1].s = 2; op.src[1].cin = sb.C;
  op.ncls = 4; op.ntaps = 13;
  for (int cls = 0; cls < 4; ++cls) {
    const int py = cls >> 1, px = cls & 1;
    // oy = 2*iy - 1 + ky  =>  parity 0: (ky=1, iy=y), (ky=3, iy=y-1); parity 1: (ky=0, iy=y+1), (ky=2, iy=y)
    const int kys[2][2] = {{1, 3}, {0, 2}};
    const int tys[2][2] = {{0, -1}, {1, 0}};
    int t = 0;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        Tap& tp = op.taps[cls][t++];
        tp.src = 0; tp.ky = kys[py][a]; tp.kx = kys[px][b]; tp.ty = tys[py][a]; tp.tx = tys[px][b];
      }
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) {
        Tap& tp = op.taps[cls][t++];
        tp.src = 1; tp.ky = ky; tp.kx = kx; tp.ty = py + ky - 1; tp.tx = px + kx - 1;
      }
  }
  op.Hl = lb.H; op.Wl = lb.W; op.out_buf = c->buf_index.at(out); op.os = 2;
  op.cout = ob.C; op.cout_pad = ob.C; op.K = 4 * lb.C + 9 * sb.C;
  op.epi.act = ACT_RELU;
  op.flops_per_image = 2.0 * 4 * op.Hl * op.Wl * (double)op.cout * op.K;
  c->ops.push_back(std::move(op));
}

void build_plan(Ctx* c) {
  const int H = c->H, W = c->W;
  add_buf(c, "a1_1", H, W, 64); add_buf(c, "conv1_2", H, W, 64);
  add_buf(c, "a2_1", H / 2, W / 2, 128); add_buf(c, "conv2_2", H / 2, W / 2, 128);
  add_buf(c, "a3_1", H / 4, W / 4, 256); add_buf(c, "a3_2", H / 4, W / 4, 256); add_buf(c, "conv3_3", H / 4, W / 4, 256);
  const char* n8[] = {"a4_1", "a4_2", "conv4_3", "a5_1", "a5_2", "conv5_3", "a6_1", "a6_2", "conv6_3",
                      "a7_1", "a7_2", "conv7_3"};
  for (const char* nm : n8) add_buf(c, nm, H / 8, W / 8, 512);
  add_buf(c, "a8_1", H / 4, W / 4, 256); add_buf(c, "a8_2", H / 4, W / 4, 256); add_buf(c, "conv8_3", H / 4, W / 4, 256);
  add_buf(c, "a9_1", H / 2, W / 2, 128); add_buf(c, "conv9_3", H / 2, W / 2, 128);
  add_buf(c, "a10_1", H, W, 128);
  const bool keep10 = c->simt || (c->flags & IDC_FLAG_KEEP_CONV10);
  if (keep10) add_buf(c, "conv10_2", H, W, 128);

  // model1 (conv1_1 is the fused pack+conv kernel in idc_heads.cu)            model.py:13-17
  add_conv(c, "c1_2", "model1.2", "a1_1", 1, 1, "conv1_2", ACT_RELU, "model1.4");
  // model2 on conv1_2[:, :, ::2, ::2]                                        model.py:149, 21-25
  add_conv(c, "c2_1", "model2.0", "conv1_2", 2, 1, "a2_1", ACT_RELU, nullptr);
  add_conv(c, "c2_2", "model2.2", "a2_1", 1, 1, "conv2_2", ACT_RELU, "model2.4");
  // model3                                                                   model.py:150, 29-35
  add_conv(c, "c3_1", "model3.0", "conv2_2", 2, 1, "a3_1", ACT_RELU, nullptr);
  add_conv(c, "c3_2", "model3.2", "a3_1", 1, 1, "a3_2", ACT_RELU, nullptr);
  add_conv(c, "c3_3", "model3.4", "a3_2", 1, 1, "conv3_3", ACT_RELU, "model3.6");
  // model4 (+ global-hints vector added to conv4_3norm, deploy_nodist.prototxt:501-527)  model.py:151, 39-45
  add_conv(c, "c4_1", "model4.0", "conv3_3", 2, 1, "a4_1", ACT_RELU, nullptr);
  add_conv(c, "c4_2", "model4.2", "a4_1", 1, 1, "a4_2", ACT_RELU, nullptr);
  add_conv(c, "c4_3", "model4.4", "a4_2", 1, 1, "conv4_3", ACT_RELU, "model4.6", c->glob);
  // model5, model6 (dilation 2), model7                                       model.py:48-72
  add_conv(c, "c5_1", "model5.0", "conv4_3", 1, 2, "a5_1", ACT_RELU, nullptr);
  add_conv(c, "c5_2", "model5.2", "a5_1", 1, 2, "a5_2", ACT_RELU, nullptr);
  add_conv(c, "c5_3", "model5.4", "a5_2", 1, 2, "conv5_3", ACT_RELU, "model5.6");
  add_conv(c, "c6_1", "model6.0", "conv5_3", 1, 2, "a6_1", ACT_RELU, nullptr);
  add_conv(c, "c6_2", "model6.2", "a6_1", 1, 2, "a6_2", ACT_RELU, nullptr);
  add_conv(c, "c6_3", "model6.4", "a6_2", 1, 2, "conv6_3", ACT_RELU, "model6.6");
  add_conv(c, "c7_1", "model7.0", "conv6_3", 1, 1, "a7_1", ACT_RELU, nullptr);
  add_conv(c, "c7_2", "model7.2", "a7_1", 1, 1, "a7_2", ACT_RELU, nullptr);
  add_conv(c, "c7_3", "model7.4", "a7_2", 1, 1, "conv7_3", ACT_RELU, "model7.6");
  // decoder level 8                                                          model.py:156-157, 75-83
  add_up(c, "up8", "model8up.0", "conv7_3", "model3short8.0", "conv3_3", "a8_1");
  add_conv(c, "c8_2", "model8.1", "a8_1", 1, 1, "a8_2", ACT_RELU, nullptr);
  add_conv(c, "c8_3", "model8.3", "a8_2", 1, 1, "conv8_3", ACT_RELU, "model8.5");
  // class head on conv8_3 (dist only)                                        model.py:105, 160
  if (c->dist) {
    ConvOp op;
    op.name = "class"; op.kind = OP_CLASS; op.wkey[0] = "model_class.0";
    const ActBuf& ib = c->bufs[c->buf_index.at("conv8_3")];
    op.nsrc = 1; op.src[0].buf = c->buf_index.at("conv8_3"); op.src[0].s = 1; op.src[0].cin = ib.C;
    op.ncls = 1; op.ntaps = 1;
    op.taps[0][0] = Tap{0, 0, 0, 0, 0};
    op.Hl = ib.H; op.Wl = ib.W; op.out_buf = -1; op.os = 1;
    op.cout = 529; op.cout_pad = 576; op.K = ib.C; op.out_f32 = true; op.src_k[0] = 1;
    op.flops_per_image = 2.0 * op.Hl * op.Wl * 529.0 * op.K;
    c->ops.push_back(std::move(op));
  }
  // Caffe-spec 313-bin head (row a14): hyper-column = conv3x3(conv3_3) + sum_l deconv4x4s2(conv{4..7}_3) +
  // conv3x3(conv8_3) -> ReLU (deploy_nopred.prototxt:651-763), then pred_313 = conv1x1 384->313 (:765-775)
  if (c->caffe313) {
    add_buf(c, "hyper", H / 4, W / 4, 384);
    ConvOp op;
    op.name = "hyper"; op.kind = OP_HYPER;
    const char* dsrc[4] = {"conv4_3", "conv5_3", "conv6_3", "conv7_3"};
    const char* dkey[4] = {"caffe.conv4_pred", "caffe.conv5_pred", "caffe.conv6_pred", "caffe.conv7_pred"};
    op.nsrc = 6;
    for (int s = 0; s < 4; ++s) {
      op.src[s].buf = c->buf_index.at(dsrc[s]); op.src[s].s = 1; op.src[s].cin = 512;
      op.wkey[s] = dkey[s]; op.src_deconv[s] = true; op.src_k[s] = 4;
    }
    op.src[4].buf = c->buf_index.at("conv3_3"); op.src[4].s = 2; op.src[4].cin = 256; op.wkey[4] = "caffe.conv3_pred";
    op.src[5].buf = c->buf_index.at("conv8_3"); op.src[5].s = 2; op.src[5].cin = 256; op.wkey[5] = "caffe.conv8_pred";
    op.ncls = 4; op.ntaps = 34;
    for (int cls = 0; cls < 4; ++cls) {
      const int py = cls >> 1, px = cls & 1;
      const int kys[2][2] = {{1, 3}, {0, 2}};
      const int tys[2][2] = {{0, -1}, {1, 0}};
      int t = 0;
      for (int s = 0; s < 4; ++s)
        for (int a = 0; a < 2; ++a)
          for (int b = 0; b < 2; ++b)
            op.taps[cls][t++] = Tap{s, kys[py][a], kys[px][b], tys[py][a], tys[px][b]};
      for (int s = 4; s < 6; ++s)
        for (int ky = 0; ky < 3; ++ky)
          for (int kx = 0; kx < 3; ++kx) op.taps[cls][t++] = Tap{s, ky, kx, py + ky - 1, px + kx - 1};
    }
    op.Hl = H / 8; op.Wl = W / 8; op.out_buf = c->buf_index.at("hyper"); op.os = 2;
    op.cout = 384; op.cout_pad = 384; op.K = 4 * 4 * 512 + 2 * 9 * 256;
    op.epi.act = ACT_RELU;
    op.flops_per_image = 2.0 * 4 * op.Hl * op.Wl * 384.0 * op.K;
    c->ops.push_back(std::move(op));

    ConvOp pr;
    pr.name = "pred313"; pr.kind = OP_CLASS; pr.wkey[0] = "caffe.pred_313"; pr.src_k[0] = 1;
    pr.nsrc = 1; pr.src[0].buf = c->buf_index.at("hyper"); pr.src[0].s = 1; pr.src[0].cin = 384;
    pr.ncls = 1; pr.ntaps = 1; pr.taps[0][0] = Tap{0, 0, 0, 0, 0};
    pr.Hl = H / 4; pr.Wl = W / 4; pr.out_buf = -1; pr.os = 1;
    pr.cout = 313; pr.cout_pad = 320; pr.K = 384; pr.out_f32 = true;
    pr.flops_per_image = 2.0 * pr.Hl * pr.Wl * 313.0 * pr.K;
    c->ops.push_back(std::move(pr));
  }
  // level 9                                                                  model.py:162-163, 86-93
  add_up(c, "up9", "model9up.0", "conv8_3", "model2short9.0", "conv2_2", "a9_1");
  add_conv(c, "c9_2", "model9.1", "a9_1", 1, 1, "conv9_3", ACT_RELU, "model9.3");
  // level 10                                                                 model.py:164-165, 96-102
  add_up(c, "up10", "model10up.0", "conv9_3", "model1short10.0", "conv1_2", "a10_1");
  if (keep10) {
    add_conv(c, "c10_2", "model10.1", "a10_1", 1, 1, "conv10_2", ACT_LEAKY02, nullptr);
  } else {
    // conv10_2 never leaves the SM: model_out (1x1 128->2, tanh, x110) runs in the epilogue
    add_buf(c, "conv10_2_virtual", 0, 0, 128);
    ConvOp op;
    op.name = "c10_2"; op.kind = OP_CONV; op.wkey[0] = "model10.1";
    const ActBuf& ib = c->bufs[c->buf_index.at("a10_1")];
    op.nsrc = 1; op.src[0].buf = c->buf_index.at("a10_1"); op.src[0].s = 1; op.src[0].cin = ib.C;
    op.ncls = 1; op.ntaps = 9;
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) op.taps[0][ky * 3 + kx] = Tap{0, ky, kx, ky - 1, kx - 1};
    op.Hl = ib.H; op.Wl = ib.W; op.out_buf = -1; op.os = 1;
    op.cout = 128; op.cout_pad = 128; op.K = 9 * ib.C;
    op.epi.act = ACT_LEAKY02; op.fuse_out_head = true;
    op.flops_per_image = 2.0 * op.Hl * op.Wl * 128.0 * op.K;
    c->ops.push_back(std::move(op));
  }
}

// ---------------------------------------------------------------------------------------------
// weight arena
// ---------------------------------------------------------------------------------------------
struct ArenaLayout {
  size_t off = 0;
  template <typename T>
  size_t take(size_t count) {
    off = (off + 255) & ~size_t(255);
    size_t o = off;
    off += count * sizeof(T);
    return o;
  }
};

const char* kGlobKeys[4] = {"glob.0", "glob.1", "glob.2", "glob.3"};

// Assigns arena offsets to every packed tensor (deterministic: same on every rank).
size_t layout_arena(Ctx* c, char* base) {
  ArenaLayout L;
  auto P = [&](size_t o) { return base ? base + o : nullptr; };
  c->w11 = (float*)P(L.take<float>(36 * 64));
  c->b11 = (float*)P(L.take<float>(64));
  c->wout = (float*)P(L.take<float>(256));
  c->bout = (float*)P(L.take<float>(4));
  c->act_exp = (int*)P(L.take<int>(c->bufs.size()));
  for (auto& op : c->ops) {
    op.epi.bias = (float*)P(L.take<float>(op.cout_pad));
    op.epi.scale = (float*)P(L.take<float>(op.cout_pad));
    op.epi.shift = (float*)P(L.take<float>(op.cout_pad));
    const size_t nw = (size_t)op.ncls * op.K * op.cout_pad;
    if (c->simt) {
      op.w_simt = (float*)P(L.take<float>(nw));
    } else {
      op.w_hi = (__half*)P(L.take<__half>(nw));
      op.w_lo = (__half*)P(L.take<__half>(nw));
    }
  }
  if (c->glob) {
    for (int l = 0; l < 4; ++l) {
      const int cin = l == 0 ? 316 : 512;
      c->gw[l] = (float*)P(L.take<float>((size_t)512 * cin));
      c->gb[l] = (float*)P(L.take<float>(512));
      c->gscale[l] = (float*)P(L.take<float>(512));
      c->gshift[l] = (float*)P(L.take<float>(512));
    }
  }
  return (L.off + 255) & ~size_t(255);
}

const HostTensor* find(Ctx* c, const std::string& key) {
  auto it = c->raw.find(key);
  return it == c->raw.end() ? nullptr : &it->second;
}

bool check_dims(const HostTensor* t, std::initializer_list<int64_t> d) {
  if (!t || t->dims.size() != d.size()) return false;
  size_t i = 0;
  for (int64_t v : d)
    if (t->dims[i++] != v) return false;
  return true;
}

void split_f16(float v, __half& hi, __half& lo) {
  hi = __float2half_rn(v);
  lo = __float2half_rn(v - __half2float(hi));
}

// BN(eval) -> y = x*scale + shift   (model.py:17.. ; F.batch_norm with running stats)
void fold_bn(const HostTensor& g, const HostTensor& b, const HostTensor& m, const HostTensor& v, int C, float* scale,
             float* shift) {
  for (int i = 0; i < C; ++i) {
    const double s = (double)g.data[i] / sqrt((double)v.data[i] + (double)kBnEps);
    scale[i] = (float)s;
    shift[i] = (float)((double)b.data[i] - (double)m.data[i] * s);
  }
}

// ref - ceil(log2 est), or ref for est = 0
int exp_below(int ref, double est) {
  if (!(est > 0.0)) return ref;
  int ex = 0;
  const double f = frexp(est, &ex);          // est = f * 2^ex, f in [0.5, 1): ceil(log2 est) = ex, or ex - 1 at f = 0.5
  return ref - (f == 0.5 ? ex - 1 : ex);
}

// Storage exponent of buffer b from its magnitude estimate est and, for the outputs of convs without a BatchNorm, its
// bound (DESIGN §3): the act_exp.<name> override, else kActExpCal - ceil(log2 max_abs) where a range was measured
// (idc_set_act_range), else S_b = min(kActExpRef - ceil(log2 est_b), kActExpBound - ceil(log2 bound_b)).
// bound < 0: none.  Writes it to the arena table and the buffer; fails, naming the buffer, outside the range.
int set_act_exp(Ctx* c, int* table, int b, double est, double bound) {
  ActBuf& buf = c->bufs[b];
  int s = 0;
  if (!c->simt) {
    auto ov = c->act_exp_override.find(buf.name);
    auto rg = c->act_range.find(buf.name);
    if (ov != c->act_exp_override.end()) {
      s = ov->second;
    } else if (rg != c->act_range.end()) {
      s = exp_below(kActExpCal, rg->second);
    } else {     // only this branch needs the estimate: a checkpoint whose estimate overflows can still be calibrated
      if (!std::isfinite(est) || !std::isfinite(bound))
        return fail(c, IDC_ERR_ARG, "activation %s: magnitude estimate %g / bound %g is not finite", buf.name.c_str(), est, bound);
      s = exp_below(kActExpRef, est);
      if (bound >= 0.0) s = std::min(s, exp_below(kActExpBound, bound));
    }
    if (s < kActExpMin || s > kActExpMax)
      return fail(c, IDC_ERR_UNSUPPORTED,
                  "activation %s: storage exponent %d (magnitude estimate %g, bound %g) is outside the supported range [%d, %d]",
                  buf.name.c_str(), s, est, bound, kActExpMin, kActExpMax);
  }
  table[b] = s;
  buf.exp = s;
  return IDC_OK;
}

double sumsq(const float* p, size_t n) {
  double a = 0.0;
  for (size_t i = 0; i < n; ++i) a += (double)p[i] * (double)p[i];
  return a;
}

double sumabs(const float* p, size_t n) {
  double a = 0.0;
  for (size_t i = 0; i < n; ++i) a += fabs((double)p[i]);
  return a;
}

int pack_weights(Ctx* c, char* host) {
  // translate device pointers (already laid out relative to c->arena) to host staging pointers
  auto H = [&](void* dev) { return host + ((char*)dev - c->arena.get()); };
  // magnitude estimates of the buffers, in plan order (FP64): conv output channel co of an op reading sources s is
  // sum_s ||W_s[co]||_2 * est(s) + |bias_co|; a BatchNorm output restarts from its statistics,
  // |gamma| * sqrt(var + mean^2) / sqrt(var + eps) + |beta|; the buffer's estimate is the max over its channels.
  // Outputs of convs without a BatchNorm also get a bound: the max over channels and output-parity classes of
  // sum_s ||W_s[co, class]||_1 * bound(s) + |bias_co|, with bound = est at a BatchNorm output and 1 for the packed
  // conv1_1 input; it holds whenever the BatchNorm outputs stay within their estimates.  Every power-of-two rescaling of
  // the network that computes the same function scales estimate and bound by the same power.
  int* act_exp = (int*)H(c->act_exp);
  std::vector<double> est(c->bufs.size(), 0.0), bound(c->bufs.size(), 0.0);
  // conv1_1: [36][64], k = (ky*3+kx)*4 + cin                                       model.py:13
  {
    const HostTensor* w = find(c, "model1.0.weight");
    const HostTensor* b = find(c, "model1.0.bias");
    if (!check_dims(w, {64, 4, 3, 3}) || !check_dims(b, {64})) return fail(c, IDC_ERR_KEY, "missing/bad model1.0.*");
    float* dst = (float*)H(c->w11);
    for (int co = 0; co < 64; ++co)
      for (int ci = 0; ci < 4; ++ci)
        for (int t = 0; t < 9; ++t) dst[(t * 4 + ci) * 64 + co] = w->data[((size_t)co * 4 + ci) * 9 + t];
    memcpy(H(c->b11), b->data.data(), 64 * sizeof(float));
    const int a11 = c->buf_index.at("a1_1");
    for (int co = 0; co < 64; ++co) {    // the packed input planes count as magnitude 1
      const float* wc = w->data.data() + (size_t)co * 36;
      est[a11] = std::max(est[a11], sqrt(sumsq(wc, 36)) + fabs((double)b->data[co]));
      bound[a11] = std::max(bound[a11], sumabs(wc, 36) + fabs((double)b->data[co]));
    }
    const int rc = set_act_exp(c, act_exp, a11, est[a11], bound[a11]);
    if (rc != IDC_OK) return rc;
  }
  {
    const HostTensor* w = find(c, "model_out.0.weight");
    const HostTensor* b = find(c, "model_out.0.bias");
    if (!check_dims(w, {2, 128, 1, 1}) || !check_dims(b, {2})) return fail(c, IDC_ERR_KEY, "missing/bad model_out.0.*");
    memcpy(H(c->wout), w->data.data(), 256 * sizeof(float));
    float* bo = (float*)H(c->bout);
    bo[0] = b->data[0]; bo[1] = b->data[1]; bo[2] = bo[3] = 0.f;
  }
  for (auto& op : c->ops) {
    float* bias = (float*)H(op.epi.bias);
    float* scale = (float*)H(op.epi.scale);
    float* shift = (float*)H(op.epi.shift);
    for (int i = 0; i < op.cout_pad; ++i) { bias[i] = 0.f; scale[i] = 1.f; shift[i] = 0.f; }
    const HostTensor* w[kMaxSrc] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    for (int s = 0; s < op.nsrc; ++s) {
      w[s] = find(c, op.wkey[s] + ".weight");
      const HostTensor* b = find(c, op.wkey[s] + ".bias");
      const int cin = op.src[s].cin, k = op.src_k[s];
      const bool ok = op.src_deconv[s] ? check_dims(w[s], {cin, op.cout, k, k}) : check_dims(w[s], {op.cout, cin, k, k});
      if (!ok || !check_dims(b, {op.cout})) return fail(c, IDC_ERR_KEY, "missing/bad %s.*", op.wkey[s].c_str());
      for (int i = 0; i < op.cout; ++i) bias[i] += b->data[i];
    }
    if (op.epi.has_bn) {
      const HostTensor* g = find(c, op.bnkey + ".weight");
      const HostTensor* b = find(c, op.bnkey + ".bias");
      const HostTensor* m = find(c, op.bnkey + ".running_mean");
      const HostTensor* v = find(c, op.bnkey + ".running_var");
      if (!check_dims(g, {op.cout}) || !check_dims(b, {op.cout}) || !check_dims(m, {op.cout}) ||
          !check_dims(v, {op.cout}))
        return fail(c, IDC_ERR_KEY, "missing/bad %s.*", op.bnkey.c_str());
      fold_bn(*g, *b, *m, *v, op.cout, scale, shift);
    }
    // weight value of (class, tap, ci, co)
    auto wval = [&](int cls, int t, int ci, int co) -> float {
      const Tap& tp = op.taps[cls][t];
      const HostTensor* ww = w[tp.src];
      const int cin = op.src[tp.src].cin, k = op.src_k[tp.src];
      if (op.src_deconv[tp.src])  // ConvTranspose2d / Caffe Deconvolution weight is [Cin][Cout][k][k]
        return ww->data[(((size_t)ci * op.cout + co) * k + tp.ky) * k + tp.kx];
      return ww->data[(((size_t)co * cin + ci) * k + tp.ky) * k + tp.kx];
    };
    if (op.out_buf >= 0 && c->bufs[op.out_buf].H > 0) {
      double& e_out = est[op.out_buf];
      double& b_out = bound[op.out_buf];
      for (int co = 0; co < op.cout; ++co) {
        double v = 0.0;
        if (op.epi.has_bn) {
          auto t = [&](const char* sfx) { return (double)find(c, op.bnkey + sfx)->data[co]; };
          const double var = t(".running_var"), mean = t(".running_mean");
          v = fabs(t(".weight")) * sqrt(var + mean * mean) / sqrt(var + (double)kBnEps) + fabs(t(".bias"));
        } else {
          double bsum = 0.0;
          for (int s = 0; s < op.nsrc; ++s) {
            const int cin = op.src[s].cin, kk = op.src_k[s] * op.src_k[s];
            const float* wd = w[s]->data.data();
            double n2 = 0.0;
            if (op.src_deconv[s])   // [cin][cout][k][k]
              for (int ci = 0; ci < cin; ++ci) n2 += sumsq(wd + ((size_t)ci * op.cout + co) * kk, kk);
            else
              n2 = sumsq(wd + (size_t)co * cin * kk, (size_t)cin * kk);
            v += sqrt(n2) * est[op.src[s].buf];
            bsum += (double)find(c, op.wkey[s] + ".bias")->data[co];
          }
          v += fabs(bsum);
          for (int cls = 0; cls < op.ncls; ++cls) {   // the taps of one output-parity class reach one output pixel
            double l1 = 0.0;
            for (int t = 0; t < op.ntaps; ++t) {
              const int s = op.taps[cls][t].src;
              double a = 0.0;
              for (int ci = 0; ci < op.src[s].cin; ++ci) a += fabs((double)wval(cls, t, ci, co));
              l1 += a * bound[op.src[s].buf];
            }
            b_out = std::max(b_out, l1 + fabs(bsum));
          }
        }
        e_out = std::max(e_out, v);
      }
      if (op.epi.has_bn) b_out = e_out;
      const int rc = set_act_exp(c, act_exp, op.out_buf, e_out, op.epi.has_bn ? -1.0 : b_out);
      if (rc != IDC_OK) return rc;
    }
    if (c->simt) {
      float* dst = (float*)H(op.w_simt);
      memset(dst, 0, sizeof(float) * (size_t)op.ncls * op.K * op.cout_pad);
      for (int cls = 0; cls < op.ncls; ++cls) {
        int k0 = 0;
        for (int t = 0; t < op.ntaps; ++t) {
          const int cin = op.src[op.taps[cls][t].src].cin;
          for (int ci = 0; ci < cin; ++ci)
            for (int co = 0; co < op.cout; ++co)
              dst[((size_t)cls * op.K + k0 + ci) * op.cout_pad + co] = wval(cls, t, ci, co);
          k0 += cin;
        }
      }
    } else {
      // K-major FP16 hi/lo rows, one row per (class, cout); per-output-channel power-of-two scale so
      // the lo term stays in FP16's normal range; the epilogue multiplies by 1/scale (exact).
      // Sources stored at different exponents share one accumulator at source 0's: source s's weights are
      // pre-multiplied by 2^(S_0 - S_s) (exact), so every product carries 2^(S_0 + e).
      const int s_in = c->bufs[op.src[0].buf].exp;
      const int s_out = (op.out_f32 || op.fuse_out_head) ? 0 : c->bufs[op.out_buf].exp;
      float srcmul[kMaxSrc];
      for (int s = 0; s < op.nsrc; ++s) srcmul[s] = ldexpf(1.f, s_in - c->bufs[op.src[s].buf].exp);
      auto wq = [&](int cls, int t, int ci, int co) { return wval(cls, t, ci, co) * srcmul[op.taps[cls][t].src]; };
      __half* hi = (__half*)H(op.w_hi);
      __half* lo = (__half*)H(op.w_lo);
      memset(hi, 0, sizeof(__half) * (size_t)op.ncls * op.K * op.cout_pad);
      memset(lo, 0, sizeof(__half) * (size_t)op.ncls * op.K * op.cout_pad);
      for (int co = 0; co < op.cout; ++co) {
        float mx = 0.f;
        for (int cls = 0; cls < op.ncls; ++cls)
          for (int t = 0; t < op.ntaps; ++t) {
            const int cin = op.src[op.taps[cls][t].src].cin;
            for (int ci = 0; ci < cin; ++ci) mx = fmaxf(mx, fabsf(wq(cls, t, ci, co)));
          }
        int e = 0;
        if (mx > 0.f) {
          frexpf(mx, &e);       // mx = f * 2^e, f in [0.5, 1)
          e = 9 - e;            // scaled max in [256, 512)
          e = std::max(-24, std::min(24, e));
        }
        const float sc = ldexpf(1.f, e);
        // acc = sum (a * 2^S_in)(w * 2^e); stored output = v * 2^S_out  (all exact powers of two)
        bias[co] = ldexpf(bias[co], e + s_in);
        scale[co] = ldexpf(scale[co], -(e + s_in) + s_out);
        shift[co] = ldexpf(shift[co], s_out);
        for (int cls = 0; cls < op.ncls; ++cls) {
          int k0 = 0;
          for (int t = 0; t < op.ntaps; ++t) {
            const int cin = op.src[op.taps[cls][t].src].cin;
            for (int ci = 0; ci < cin; ++ci) {
              const size_t idx = ((size_t)cls * op.cout_pad + co) * op.K + k0 + ci;
              split_f16(wq(cls, t, ci, co) * sc, hi[idx], lo[idx]);
            }
            k0 += cin;
          }
        }
      }
    }
  }
  if (c->glob) {
    for (int l = 0; l < 4; ++l) {
      const int cin = l == 0 ? 316 : 512;
      const std::string k = kGlobKeys[l];
      const HostTensor* w = find(c, k + ".weight");
      const HostTensor* b = find(c, k + ".bias");
      const HostTensor* g = find(c, k + ".bn.weight");
      const HostTensor* bb = find(c, k + ".bn.bias");
      const HostTensor* m = find(c, k + ".bn.running_mean");
      const HostTensor* v = find(c, k + ".bn.running_var");
      if (!check_dims(w, {512, cin}) || !check_dims(b, {512}) || !check_dims(g, {512}) || !check_dims(bb, {512}) ||
          !check_dims(m, {512}) || !check_dims(v, {512}))
        return fail(c, IDC_ERR_KEY, "missing/bad %s.* (global hints)", k.c_str());
      memcpy(H(c->gw[l]), w->data.data(), sizeof(float) * 512 * cin);
      memcpy(H(c->gb[l]), b->data.data(), sizeof(float) * 512);
      fold_bn(*g, *bb, *m, *v, 512, (float*)H(c->gscale[l]), (float*)H(c->gshift[l]));
    }
  }
  return IDC_OK;
}

int alloc_workspace(Ctx* c) {
  if (c->bufs.size() > kRangeInputBit) return fail(c, IDC_ERR_STATE, "%zu buffers: the range word has 31 bits", c->bufs.size());
  for (auto& b : c->bufs) {
    if (b.H == 0) continue;
    const size_t elems = (size_t)c->max_n * b.H * b.W * b.C;
    if (c->simt) {
      CUDA_TRY(c, cudaMalloc(b.p0.put(), elems * sizeof(float)));
    } else {
      CUDA_TRY(c, cudaMalloc(b.p0.put(), elems * sizeof(__half)));
      if (!c->fast) CUDA_TRY(c, cudaMalloc(b.p1.put(), elems * sizeof(__half)));
    }
  }
  if (c->dist) CUDA_TRY(c, cudaMalloc(c->logits.put(), sizeof(float) * (size_t)c->max_n * (c->H / 4) * (c->W / 4) * 576));
  if (c->caffe313) {
    CUDA_TRY(c, cudaMalloc(c->logits313.put(), sizeof(float) * (size_t)c->max_n * (c->H / 4) * (c->W / 4) * 320));
    CUDA_TRY(c, cudaMalloc(c->pts313.put(), sizeof(float) * 313 * 2));
  }
  for (auto& op : c->ops)
    if (op.out_f32) op.out_f32_ptr = (op.name == "pred313") ? c->logits313.get() : c->logits.get();
  if (c->glob) {
    CUDA_TRY(c, cudaMalloc(c->gvec.put(), sizeof(float) * (size_t)c->max_n * 512));
    CUDA_TRY(c, cudaMalloc(c->gtmp.put(), sizeof(float) * (size_t)2 * c->max_n * 512));
  }
  CUDA_TRY(c, cudaHostAlloc(c->h_err.put(), 64, cudaHostAllocMapped));
  memset(c->h_err.get(), 0, 64);
  CUDA_TRY(c, cudaHostGetDevicePointer(&c->d_err, c->h_err.get(), 0));
  c->d_range = reinterpret_cast<unsigned*>(c->d_err + 1);
  CUDA_TRY(c, cudaStreamCreateWithFlags(c->own_stream.put(), cudaStreamNonBlocking));
  return IDC_OK;
}

// Forwards are refused from here until every plan and the split-K workspace are in place: a failed (re-)plan leaves
// weights_ready false until a later plan succeeds.
int plan_engines(Ctx* c) {
  c->weights_ready = false;
  if (c->simt) { c->weights_ready = true; return IDC_OK; }
  c->splitk_ws_floats = 0; c->splitk_max_tiles = 0;
  for (auto& op : c->ops) {
    int rc = umma_plan_op(c, op);
    if (rc != IDC_OK) return rc;
  }
  c->splitk_ws.reset();
  c->splitk_counters.reset();
  if (c->splitk_ws_floats) {
    CUDA_TRY(c, cudaMalloc(c->splitk_ws.put(), c->splitk_ws_floats * sizeof(float)));
    CUDA_TRY(c, cudaMalloc(c->splitk_counters.put(), sizeof(int) * 2 * (size_t)c->splitk_max_tiles));
    CUDA_TRY(c, cudaMemset(c->splitk_counters.get(), 0, sizeof(int) * 2 * (size_t)c->splitk_max_tiles));
  }
  c->weights_ready = true;
  return IDC_OK;
}

// a code the device watchdog left in the mapped flag: clear it and fail with msg (which formats the code); then the
// buffers whose FP16 stores saturated since the last check: clear the word and fail with IDC_ERR_RANGE, naming them
int take_device_flags(Ctx* c, const char* msg) {
  volatile int* flag = c->h_err.get();
  const int werr = flag[0];
  if (werr) {
    flag[0] = 0;
    return fail(c, IDC_ERR_WATCHDOG, msg, werr);
  }
  const unsigned range = (unsigned)flag[1];
  if (!range) return IDC_OK;
  flag[1] = 0;
  std::string names;
  for (unsigned b = 0; b < 32; ++b) {
    if (!(range & (1u << b))) continue;
    if (!names.empty()) names += ", ";
    if (b == kRangeInputBit) names += "conv1_1 input";
    else if (b < c->bufs.size()) names += c->bufs[b].name + " (S = " + std::to_string(c->bufs[b].exp) + ")";
  }
  return fail(c, IDC_ERR_RANGE,
              "activation values reached 65504, FP16's largest value, at their storage exponent in: %s (values above it "
              "saturated; lower the exponent with act_exp.<buffer>)", names.c_str());
}

// idc_forward_host's copy/compute overlap (eager path, batches >= 8): the batch is cut into image chunks; conv1_1 of
// chunk k waits for the L, ab and mask copies of chunk k only (issued on HostPipeStreams::s_in), and the last op (c10_2
// + fused model_out) runs per chunk so that the D2H of ab chunk k (on HostPipeStreams::s_out) overlaps the compute of
// chunk k+1.  Everything in between runs on the whole batch.
struct HostPipe {
  static constexpr int kMaxChunks = 8;   // == the size of HostPipeStreams::ev_in / ev_out
  int nchunks = 0;
  int start[kMaxChunks + 1] = {};        // image ranges [start[k], start[k+1])
  float* ab_dst = nullptr;    // pinned host destination of out_ab: the caller's buffer or its twin in h_out
};

// One copy of an idc_forward_host call: the caller's buffer `user`, the device region `dev` and its page-locked twin
// `twin` (HostStaging).  A staged copy goes through the twin; the CPU moves the bytes between it and `user`.  The hint
// block is its own twin (user == twin): it is never staged.
struct HostCopy {
  char* user = nullptr;
  char* dev = nullptr;
  char* twin = nullptr;
  size_t bytes = 0;             // 0: the call has no such tensor (dev and twin are still its place)
  bool d2h = false, staged = false;
  char* host() const { return staged ? twin : user; }
};
// the copy list, in issue order: the inputs, then the outputs
enum { kCpHints, kCpL, kCpAb, kCpMask, kCpGlob, kCpOutAb, kCpRgb, kCpAbq, kCpDist, kNumCopies };

// idc_set_click: layout of the click answer block (device d_clickout, pinned host h_clickout)
constexpr int kClickInit = 8, kClickMaxIter = 100;                       // the defaults of LhnContext.ab_reccs
constexpr size_t kClickHdr = 32, kClickPmf = 544 * sizeof(float);
constexpr size_t kClickRes = (size_t)kClickInit * (3 * 32 + 2) * sizeof(double);
constexpr size_t kClickCopy = kClickHdr + kClickPmf + kClickRes;         // what travels back per click
constexpr size_t kClickBytes = kClickCopy + 529 * 2 * sizeof(float);     // + the default gamut grid (device only)

cudaError_t new_stream(Stream& s) { return cudaStreamCreateWithFlags(s.put(), cudaStreamNonBlocking); }
cudaError_t new_event(Event& e) { return cudaEventCreateWithFlags(e.put(), cudaEventDisableTiming); }

// After the class conv of a small-batch forward: the clicked pixel's pmf straight from its 529 logits (same per-row
// softmax routine as the full map, so the same bits), K-means on it (K from the click header), the block to pinned host
// memory.  Runs next to the full-map softmax on a branch of the dist head's side branch.
bool click_tail_on(Ctx* c, int n) { return c->click_mode && c->click && n <= 4; }

cudaError_t click_tail(Ctx* c, int n, cudaStream_t st) {
  if (!click_tail_on(c, n)) return cudaSuccess;
  char* out = c->click->d_clickout.get();
  int* hdr = reinterpret_cast<int*>(out);
  float* pmf = reinterpret_cast<float*>(out + kClickHdr);
  double* res = reinterpret_cast<double*>(out + kClickHdr + kClickPmf);
  const float* pts = reinterpret_cast<const float*>(out + kClickCopy);
  cudaError_t e = launch_click_pmf(c, c->click->d_click, n, hdr, pmf, st);
  if (e != cudaSuccess) return e;
  if ((e = launch_ab_reccs(pmf, 1, pts, 0, kClickMaxIter, kClickInit, res, st, hdr)) != cudaSuccess) return e;
  c->launch_count += 2;
  return cudaMemcpyAsync(c->click->h_clickout.get(), out, kClickCopy, cudaMemcpyDeviceToHost, st);
}

// persistent-grid cap (CTAs, even) that leaves kClickInit SMs to the side branch
int side_branch_cap(Ctx* c) { return ((c->num_sms - kClickInit) / 2) * 2; }

int run_forward(Ctx* c, int n, const float* L, const float* ab, const float* mask, float maskcent, const float* glob,
                float* out_ab, float* out_dist, uint8_t* out_rgb, cudaStream_t st, const HostPipe* hp = nullptr,
                double* out_abq = nullptr, const char* hints_dev = nullptr) {
  c->launch_count = 0;
  c->gadd_active = false;
  c->click_served = false;
  pdl_break(c);                        // whatever precedes this forward on `st` is not one of its kernels
  std::vector<Event>* ev = nullptr;
  auto mark = [&]() -> cudaError_t {
    if (!ev) return cudaSuccess;
    Event e;
    cudaError_t ce = cudaSuccess;
    if (!c->prof_pool.empty()) { e = std::move(c->prof_pool.back()); c->prof_pool.pop_back(); }
    else ce = cudaEventCreate(e.put());
    if (ce == cudaSuccess) ce = cudaEventRecord(e.get(), st);
    if (ce != cudaSuccess) return ce;
    ev->push_back(std::move(e));
    pdl_break(c);                      // per-op timing: kernels must not overlap their predecessors
    return cudaSuccess;
  };
  if (c->profiling) { c->prof_runs.emplace_back(); ev = &c->prof_runs.back(); }
  CUDA_TRY(c, mark());
  if (hp) CUDA_TRY(c, cudaStreamWaitEvent(st, c->pipe->ev_in[0].get(), 0));     // covers the glob vector too
  if (glob && c->glob) {
    CUDA_TRY(c, launch_global_mlp(c, n, glob, st));
    c->gadd_active = true;
  }
  const size_t HW = (size_t)c->H * c->W;
  const bool c11_umma = c->opt.conv1_1_umma && !c->simt && c->w11_umma.get();
  // hint mode: the ab / mask planes conv1_1 reads are rasterised here from the hint block (already on the device)
  if (hints_dev) CUDA_TRY(c, launch_hint_raster(c, n, c->H, c->W, hints_dev, const_cast<float*>(ab), const_cast<float*>(mask), st));
  if (hp) {
    for (int k = 0; k < hp->nchunks; ++k) {
      CUDA_TRY(c, cudaStreamWaitEvent(st, c->pipe->ev_in[k].get(), 0));
      pdl_break(c);
      if (c11_umma) CUDA_TRY(c, launch_conv1_1_umma(c, hp->start[k + 1] - hp->start[k], L, ab, mask, maskcent, st, hp->start[k]));
      else CUDA_TRY(c, launch_conv1_1(c, hp->start[k + 1] - hp->start[k], L, ab, mask, maskcent, st, hp->start[k]));
    }
  } else {
    if (c11_umma) CUDA_TRY(c, launch_conv1_1_umma(c, n, L, ab, mask, maskcent, st));
    else CUDA_TRY(c, launch_conv1_1(c, n, L, ab, mask, maskcent, st));
  }
  CUDA_TRY(c, mark());
  // Interactive batches: the dist head (class 1x1 conv + 529-way softmax) only depends on conv8_3, and decoder levels
  // 9-10 do not depend on it -> it runs on a side stream (a parallel branch of the click graph) on the ~20 SMs the
  // 128-CTA launches of the main chain leave idle, instead of sitting between c8_3 and up9 on the critical path.
  const bool side_dist = c->opt.side_dist && !c->simt && out_dist && n <= 4 && !hp && !ev;
  bool forked = false;
  for (size_t oi = 0; oi < c->ops.size(); ++oi) {
    ConvOp& op = c->ops[oi];
    if (side_dist && op.kind == OP_CLASS && op.name == "class") {
      if (!c->side) {
        auto g = std::make_unique<SideBranch>();
        CUDA_TRY(c, new_stream(g->s_side));
        CUDA_TRY(c, new_stream(g->s_click));
        for (Event* e : {&g->ev_fork, &g->ev_join, &g->ev_click[0], &g->ev_click[1]}) CUDA_TRY(c, new_event(*e));
        c->side = std::move(g);
      }
      const SideBranch& sb = *c->side;
      const cudaStream_t side = sb.s_side.get(), side_click = sb.s_click.get();
      const cudaEvent_t ev_click[2] = {sb.ev_click[0].get(), sb.ev_click[1].get()};
      cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
      CUDA_TRY(c, cudaStreamIsCapturing(st, &cap));
      const bool main_chain = c->chain;
      CUDA_TRY(c, cudaEventRecord(sb.ev_fork.get(), st));
      CUDA_TRY(c, cudaStreamWaitEvent(side, sb.ev_fork.get(), 0));
      pdl_break(c);                                        // first kernel of the branch follows an event wait
      CUDA_TRY(c, umma_run_op(c, op, n, nullptr, (float)c->opt.tanh_scale, side, 0, 16));
      const bool click = click_tail_on(c, n);
      if (click) {   // idc_set_click: clicked pixel's pmf + suggestions only need the logits -> a branch of the branch
        CUDA_TRY(c, cudaEventRecord(ev_click[0], side));
        CUDA_TRY(c, cudaStreamWaitEvent(side_click, ev_click[0], 0));
        CUDA_TRY(c, click_tail(c, n, side_click));
        CUDA_TRY(c, cudaEventRecord(ev_click[1], side_click));
        if (cap != cudaStreamCaptureStatusActive) pdl_break(c);      // live stream: the record sits between class and softmax
      }
      CUDA_TRY(c, launch_softmax529(c, n, out_dist, side));          // PDL-chained behind `class` on the side stream
      if (click) CUDA_TRY(c, cudaStreamWaitEvent(side, ev_click[1], 0));
      CUDA_TRY(c, cudaEventRecord(sb.ev_join.get(), side));
      // in a capture the event record is not a node: up9 keeps its programmatic edge to c8_3; on a live stream the
      // record sits between the two kernels, so the next launch is serialised normally
      c->chain = (cap == cudaStreamCaptureStatusActive) ? main_chain : false;
      forked = true;
      continue;
    }
    if (c->simt) {
      CUDA_TRY(c, simt_run_op(c, op, n, st));
    } else if (hp && op.fuse_out_head) {
      for (int k = 0; k < hp->nchunks; ++k) {
        const int i0 = hp->start[k], nk = hp->start[k + 1] - i0;
        CUDA_TRY(c, umma_run_op(c, op, nk, out_ab, (float)c->opt.tanh_scale, st, i0));
        CUDA_TRY(c, cudaEventRecord(c->pipe->ev_out[k].get(), st));
        pdl_break(c);
        CUDA_TRY(c, cudaStreamWaitEvent(c->pipe->s_out.get(), c->pipe->ev_out[k].get(), 0));
        CUDA_TRY(c, cudaMemcpyAsync(hp->ab_dst + (size_t)i0 * 2 * HW, out_ab + (size_t)i0 * 2 * HW,
                                    (size_t)nk * 2 * HW * sizeof(float), cudaMemcpyDeviceToHost, c->pipe->s_out.get()));
      }
    } else {
      // announced click: the suggestion kernel (8 CTAs of 1024 threads, a whole SM each) runs on the side branch next
      // to decoder levels 9-10; a full-width launch would queue behind it on 8 SMs and finish that much later.  Leaving 8
      // SMs free costs little: 512 tiles are 4 rounds on 132 and on 124 CTAs alike.
      const int cap = (forked && c->click_mode && c->click) ? side_branch_cap(c) : 0;
      CUDA_TRY(c, umma_run_op(c, op, n, op.fuse_out_head ? out_ab : nullptr, (float)c->opt.tanh_scale, st, 0, cap));
    }
    CUDA_TRY(c, mark());
  }
  const bool fused = !c->simt && !(c->flags & IDC_FLAG_KEEP_CONV10);
  if (!fused) CUDA_TRY(c, launch_out_head(c, n, out_ab, st));
  if (out_dist && !forked) {
    CUDA_TRY(c, launch_softmax529(c, n, out_dist, st));
    CUDA_TRY(c, click_tail(c, n, st));
    pdl_break(c);
  }
  if (out_rgb) {
    CUDA_TRY(c, launch_lab2rgb(c, n, c->H, c->W, L, 50.0f, out_ab, out_rgb, st, out_abq));
    c->launch_count++;
  }
  if (forked) {
    CUDA_TRY(c, cudaStreamWaitEvent(st, c->side->ev_join.get(), 0));   // join: whatever follows on `st` sees the distribution
    pdl_break(c);
  }
  CUDA_TRY(c, mark());
  pdl_break(c);
  c->last_n = n;
  return IDC_OK;
}

int check_forward_args(Ctx* c, int n, int h, int w, const void* L, const void* ab, const void* mask, const void* glob,
                       const void* out_ab, const void* out_dist, bool resident_l_ok = false, bool hints_ok = false) {
  if (!c->weights_ready) return fail(c, IDC_ERR_STATE, "idc_forward before idc_finalize_weights");
  if (n < 1 || n > c->max_n) return fail(c, IDC_ERR_ARG, "n=%d outside [1,%d]", n, c->max_n);
  if (h != c->H || w != c->W) return fail(c, IDC_ERR_ARG, "geometry %dx%d != ctx geometry %dx%d", h, w, c->H, c->W);
  const bool hint_mode = hints_ok && !ab && !mask;     // idc_set_hints list instead of planes
  if ((!L && !resident_l_ok) || ((!ab || !mask) && !hint_mode) || !out_ab)
    return fail(c, IDC_ERR_ARG, "null L/ab/mask/out_ab");
  if (out_dist && !c->dist) return fail(c, IDC_ERR_ARG, "out_dist requires IDC_FLAG_DIST");
  if (glob && !c->glob) return fail(c, IDC_ERR_ARG, "glob requires IDC_FLAG_GLOBAL_HINTS");
  return IDC_OK;
}

}  // namespace

// =============================================================================================
extern "C" {

const char* idc_version(void) { return "idc_b200 0.2 sm_90a (wgmma split-fp16 + fp32 simt engines)"; }

int idc_create(int device, int max_n, int h, int w, unsigned flags, idc_ctx** out) {
  if (!out) return IDC_ERR_ARG;
  *out = nullptr;
  if (max_n < 1 || h < 8 || w < 8 || (h % 8) || (w % 8)) return IDC_ERR_ARG;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return IDC_ERR_CUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return IDC_ERR_CUDA;
  if (prop.major != 9 || prop.minor != 0) return IDC_ERR_UNSUPPORTED;  // sm_90a cubins only; no fallback
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  std::unique_ptr<idc_ctx> c(new idc_ctx());
  c->dev = device; c->num_sms = prop.multiProcessorCount; c->max_n = max_n; c->H = h; c->W = w; c->flags = flags;
  c->simt = flags & IDC_FLAG_ENGINE_SIMT;
  c->fast = (flags & IDC_FLAG_FAST_FP16) && !c->simt;
  c->dist = flags & IDC_FLAG_DIST;
  c->glob = flags & IDC_FLAG_GLOBAL_HINTS;
  c->caffe313 = flags & IDC_FLAG_CAFFE313;
  build_plan(c.get());
  int rc = alloc_workspace(c.get());
  if (rc != IDC_OK) {
    fprintf(stderr, "idc_create: %s\n", c->err.c_str());
    return rc;
  }
  *out = c.release();
  return IDC_OK;
}

int idc_set_option(idc_ctx* c, const char* name, int value) {
  if (!c || !name) return IDC_ERR_ARG;
  if (!strncmp(name, "act_exp.", 8)) {     // storage exponent of one buffer: baked into the packed weights
    auto it = c->buf_index.find(name + 8);
    if (it == c->buf_index.end() || c->bufs[it->second].H == 0) return fail(c, IDC_ERR_KEY, "no activation '%s'", name + 8);
    if (value < kActExpMin || value > kActExpMax)
      return fail(c, IDC_ERR_ARG, "%s = %d outside [%d, %d]", name, value, kActExpMin, kActExpMax);
    if (c->weights_adopted)
      return fail(c, IDC_ERR_STATE, "%s must be set before the weights are packed (idc_finalize_weights)", name);
    c->act_exp_override[name + 8] = value;
    return IDC_OK;
  }
  struct { const char* n; int* v; } tab[] = {
      {"halo", &c->opt.halo}, {"pairs", &c->opt.pairs}, {"mt", &c->opt.mt},
      {"chunk_kb", &c->opt.chunk_kb}, {"split_k", &c->opt.split_k}, {"host_pipe", &c->opt.host_pipe},
      {"pdl", &c->opt.pdl}, {"tanh_scale", &c->opt.tanh_scale}, {"side_dist", &c->opt.side_dist},
      {"conv1_1_umma", &c->opt.conv1_1_umma}};
  for (auto& t : tab)
    if (!strcmp(t.n, name)) {
      *t.v = value;
      if (c->weights_adopted && strcmp(name, "host_pipe") && strcmp(name, "tanh_scale") && strcmp(name, "side_dist") && strcmp(name, "conv1_1_umma")) {      // plan-time option changed after planning: re-plan
        CUDA_TRY(c, cudaSetDevice(c->dev));
        CUDA_TRY(c, cudaDeviceSynchronize());
        int rc = plan_engines(c);
        if (rc != IDC_OK) return rc;
      }
      c->graph_exec.reset();
      return IDC_OK;
    }
  return fail(c, IDC_ERR_KEY, "unknown option '%s'", name);
}

int idc_load_tensor(idc_ctx* c, const char* key, const void* data, int dtype, int ndim, const int64_t* dims) {
  if (!c || !key || !data || ndim < 0 || ndim > 8 || (ndim && !dims)) return fail(c, IDC_ERR_ARG, "bad load_tensor args");
  HostTensor t;
  size_t count = 1;
  for (int i = 0; i < ndim; ++i) {
    if (dims[i] < 0) return fail(c, IDC_ERR_ARG, "negative dim");
    t.dims.push_back(dims[i]);
    count *= (size_t)dims[i];
  }
  t.data.resize(count);
  switch (dtype) {
    case IDC_F32: memcpy(t.data.data(), data, count * sizeof(float)); break;
    case IDC_F64: for (size_t i = 0; i < count; ++i) t.data[i] = (float)((const double*)data)[i]; break;
    case IDC_I64: for (size_t i = 0; i < count; ++i) t.data[i] = (float)((const int64_t*)data)[i]; break;
    default: return fail(c, IDC_ERR_ARG, "unknown dtype %d", dtype);
  }
  c->raw[key] = std::move(t);
  c->weights_ready = c->weights_adopted = false;
  return IDC_OK;
}

int idc_reserve_weights(idc_ctx* c) {
  if (!c) return IDC_ERR_ARG;
  CUDA_TRY(c, cudaSetDevice(c->dev));
  if (!c->arena.get()) {
    c->arena_bytes = layout_arena(c, nullptr);
    CUDA_TRY(c, cudaMalloc(c->arena.put(), c->arena_bytes));
    layout_arena(c, c->arena.get());
  }
  return IDC_OK;
}

int idc_finalize_weights(idc_ctx* c) {
  if (!c) return IDC_ERR_ARG;
  int rc = idc_reserve_weights(c);
  if (rc != IDC_OK) return rc;
  std::vector<char> host(c->arena_bytes, 0);
  rc = pack_weights(c, host.data());
  if (rc != IDC_OK) return rc;
  CUDA_TRY(c, cudaMemcpy(c->arena.get(), host.data(), c->arena_bytes, cudaMemcpyHostToDevice));
  return idc_adopt_weights(c);
}

int idc_adopt_weights(idc_ctx* c) {
  if (!c || !c->arena.get()) return fail(c, IDC_ERR_STATE, "no arena");
  CUDA_TRY(c, cudaSetDevice(c->dev));
  // the 313 bin centres are not part of the arena: a context that received it loads caffe.pts_in_hull itself
  if (c->caffe313) {
    const HostTensor* pts = find(c, "caffe.pts_in_hull");
    if (!check_dims(pts, {313, 2})) return fail(c, IDC_ERR_KEY, "missing/bad caffe.pts_in_hull [313,2]");
    CUDA_TRY(c, cudaMemcpy(c->pts313.get(), pts->data.data(), sizeof(float) * 626, cudaMemcpyHostToDevice));
  }
  // conv1_1 takes its weights as a kernel parameter: read them back from the (possibly received) arena
  CUDA_TRY(c, cudaMemcpy(c->h_w11.w, c->w11, sizeof(c->h_w11.w), cudaMemcpyDeviceToHost));
  CUDA_TRY(c, cudaMemcpy(c->h_w11.b, c->b11, sizeof(c->h_w11.b), cudaMemcpyDeviceToHost));
  std::vector<int> exps(c->bufs.size());
  CUDA_TRY(c, cudaMemcpy(exps.data(), c->act_exp, exps.size() * sizeof(int), cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < exps.size(); ++i) c->bufs[i].exp = exps[i];
  if (!c->simt) CUDA_TRY(c, conv1_1_umma_pack(c));      // tensor-core conv1_1: derived on the device, so ranks != 0 need nothing extra
  int rc = plan_engines(c);                             // sets weights_ready
  if (rc != IDC_OK) return rc;
  c->raw.clear();
  c->weights_adopted = true;
  c->graph_exec.reset();
  return IDC_OK;
}

int idc_weights_arena(idc_ctx* c, void** dev_ptr, size_t* bytes) {
  if (!c || !dev_ptr || !bytes) return IDC_ERR_ARG;
  if (!c->arena.get()) return fail(c, IDC_ERR_STATE, "arena not allocated");
  *dev_ptr = c->arena.get(); *bytes = c->arena_bytes;
  return IDC_OK;
}

int idc_forward(idc_ctx* c, int n, int h, int w, const float* L, const float* ab, const float* mask, float maskcent,
                const float* glob, float* out_ab, float* out_dist, uint8_t* out_rgb, void* stream) {
  if (!c) return IDC_ERR_ARG;
  int rc = check_forward_args(c, n, h, w, L, ab, mask, glob, out_ab, out_dist);
  if (rc != IDC_OK) return rc;
  CUDA_TRY(c, cudaSetDevice(c->dev));
  rc = take_device_flags(c, "device pipeline watchdog fired earlier (code %d)");   // left by an earlier (asynchronous) forward
  if (rc != IDC_OK) return rc;
  return run_forward(c, n, L, ab, mask, maskcent, glob, out_ab, out_dist, out_rgb, (cudaStream_t)stream);
}

static bool is_pinned(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost;
}

int idc_forward_host(idc_ctx* c, int n, int h, int w, const float* L, const float* ab, const float* mask,
                     float maskcent, const float* glob, float* out_ab, float* out_dist, uint8_t* out_rgb) {
  return idc_forward_host_q(c, n, h, w, L, ab, mask, maskcent, glob, out_ab, out_dist, out_rgb, nullptr);
}

// The copies of one idc_forward_host call (see HostStaging for the regions).  The inputs sit packed for n at the head
// of d_in; the outputs land in d_small on the click graph (`graph`), in d_out, d_rgb and AbqStaging otherwise.
static void host_copies(Ctx* c, int n, bool graph, const float* L, const float* ab, const float* mask, const float* glob,
                        float* out_ab, float* out_dist, uint8_t* out_rgb, double* out_abq, HostCopy* cp) {
  const HostStaging& sg = *c->stage;
  const size_t HW = (size_t)c->H * c->W, HW4 = (size_t)(c->H / 4) * (c->W / 4);
  auto set = [&](int k, const void* user, void* dev, void* twin, size_t bytes, bool d2h) {
    cp[k] = {(char*)user, (char*)dev, (char*)twin, user ? bytes : 0, d2h};
  };
  const size_t b_L = (size_t)n * HW * sizeof(float), b_ab = 2 * b_L, b_rgb = (size_t)n * 3 * HW, b_q = 2 * b_ab;
  char* d_in = (char*)sg.d_in.get(); char* h_in = (char*)sg.h_in.get();
  char* hints = (!ab && !mask) ? c->hints->h_hints.get() : nullptr;
  set(kCpHints, hints, hints ? c->hints->d_hints.get() : nullptr, hints, kHintBlockBytes, false);
  set(kCpL, L, d_in, h_in, b_L, false);
  set(kCpAb, ab, d_in + b_L, h_in + b_L, b_ab, false);
  set(kCpMask, mask, d_in + 3 * b_L, h_in + 3 * b_L, b_L, false);
  set(kCpGlob, glob, d_in + 4 * b_L, h_in + 4 * b_L, (size_t)n * 316 * sizeof(float), false);
  if (graph) {
    char* d = sg.d_small.get(); char* h = sg.h_small.get();
    set(kCpOutAb, out_ab, d, h, b_ab, true);
    set(kCpRgb, out_rgb, d + b_ab, h + b_ab, b_rgb, true);
    set(kCpAbq, out_abq, d + b_ab + b_rgb, h + b_ab + b_rgb, b_q, true);
  } else {
    set(kCpOutAb, out_ab, sg.d_out.get(), sg.h_out.get(), b_ab, true);
    set(kCpRgb, out_rgb, sg.d_rgb.get(), sg.h_rgb.get(), b_rgb, true);
    set(kCpAbq, out_abq, c->abq ? c->abq->d_abq.get() : nullptr, c->abq ? c->abq->h_abq.get() : nullptr, b_q, true);
  }
  const size_t dist_off = (size_t)c->max_n * 2 * HW;
  set(kCpDist, out_dist, sg.d_out.get() + dist_off, sg.h_out.get() + dist_off, (size_t)n * 529 * HW4 * sizeof(float), true);
}

// images [i0, i1) of a per-image copy
static HostCopy image_range(HostCopy e, int n, int i0, int i1) {
  const size_t per = e.bytes / n;
  e.user += i0 * per; e.dev += i0 * per; e.twin += i0 * per;
  e.bytes = (i1 - i0) * per;
  return e;
}

static void stage_inputs(const HostCopy* cp, int count) {
  for (int k = 0; k < count; ++k) if (cp[k].bytes && cp[k].staged && !cp[k].d2h) memcpy(cp[k].twin, cp[k].user, cp[k].bytes);
}

static void unstage_outputs(const HostCopy* cp, int count) {
  for (int k = 0; k < count; ++k) if (cp[k].bytes && cp[k].staged && cp[k].d2h) memcpy(cp[k].user, cp[k].twin, cp[k].bytes);
}

static cudaError_t copy_async(const HostCopy& e, size_t bytes, cudaStream_t st) {
  return e.d2h ? cudaMemcpyAsync(e.host(), e.dev, bytes, cudaMemcpyDeviceToHost, st)
               : cudaMemcpyAsync(e.dev, e.host(), bytes, cudaMemcpyHostToDevice, st);
}

// cp[0, count) as ONE copy when they follow each other both on the host and on the device, one copy each otherwise.
// All or nothing: caller buffers that merely touch may be separate allocations, which one copy cannot span; the click
// buffers and each twin are one block.
static cudaError_t issue_copies(const HostCopy* cp, int count, cudaStream_t st) {
  const HostCopy* a = nullptr;
  size_t bytes = 0;
  bool one = true;
  for (int k = 0; k < count; ++k) {
    if (!cp[k].bytes) continue;
    if (a) one = one && cp[k].host() == a->host() + bytes && cp[k].dev == a->dev + bytes;
    else a = &cp[k];
    bytes += cp[k].bytes;
  }
  if (!a || one) return a ? copy_async(*a, bytes, st) : cudaSuccess;
  for (int k = 0; k < count; ++k) {
    cudaError_t e = cp[k].bytes ? copy_async(cp[k], cp[k].bytes, st) : cudaSuccess;
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

static int run_host_forward(Ctx* c, int n, float maskcent, const HostCopy* cp, bool want_dist, cudaStream_t st,
                            const HostPipe* hp) {
  auto f = [&](int k) { return reinterpret_cast<float*>(cp[k].dev); };
  auto on = [&](int k) { return cp[k].bytes != 0; };
  return run_forward(c, n, f(kCpL), f(kCpAb), f(kCpMask), maskcent, on(kCpGlob) ? f(kCpGlob) : nullptr, f(kCpOutAb),
                     want_dist ? f(kCpDist) : nullptr, on(kCpRgb) ? reinterpret_cast<uint8_t*>(cp[kCpRgb].dev) : nullptr,
                     st, hp, on(kCpAbq) ? reinterpret_cast<double*>(cp[kCpAbq].dev) : nullptr,
                     on(kCpHints) ? cp[kCpHints].dev : nullptr);
}

// Small batches (the interactive click): ONE graph launch does everything -- the H2D of the inputs, the kernels
// (chained by programmatic dependent launch), the D2H of the results.
//   * page-locked caller buffers (idc_host_alloc; see LhnContext.click_buffers): the copy nodes read / write the
//     caller's memory directly -- no CPU copy at all.  Buffers laid out back to back ([L | ab | mask | glob],
//     [ab | rgb | abq]) travel as ONE copy each way.  The graph is keyed on the pointers and re-captured when they change.
//   * otherwise every copy is staged: the CPU copies through the twins, which are one copy node each way.
//   * hint mode: the list length lives in the fixed-size hint block, so editing the hints never re-captures the graph.
static int forward_host_graph(Ctx* c, int n, float maskcent, HostCopy* cp, bool want_dist) {
  cudaStream_t st = c->own_stream.get();
  const bool copy_dist = cp[kCpDist].bytes, want_rgb = cp[kCpRgb].bytes, want_glob = cp[kCpGlob].bytes;
  const bool want_q = cp[kCpAbq].bytes, hint_mode = cp[kCpHints].bytes, have_L = cp[kCpL].bytes;
  const uintptr_t flags = (uintptr_t)n | ((uintptr_t)want_dist << 8) | ((uintptr_t)want_rgb << 9) | ((uintptr_t)want_glob << 10) |
                          ((uintptr_t)want_q << 11) | ((uintptr_t)copy_dist << 12) | ((uintptr_t)c->click_mode << 13) |
                          ((uintptr_t)hint_mode << 14);
  const void* direct_key[8] = {(void*)(flags | (1u << 16)), cp[kCpL].user, cp[kCpAb].user, cp[kCpMask].user,
                               cp[kCpGlob].user, cp[kCpOutAb].user, cp[kCpRgb].user, cp[kCpAbq].user};
  // fast path: same pinned buffers as the captured graph -> replay without touching the driver's pointer tables
  const bool replay = c->graph_exec.get() && !copy_dist && memcmp(direct_key, c->graph_ptrs, sizeof(direct_key)) == 0 &&
                      c->graph_maskcent == maskcent;
  bool direct = replay || !copy_dist;
  for (int k = 0; k < kNumCopies && direct && !replay; ++k)
    direct = !cp[k].bytes || cp[k].user == cp[k].twin || is_pinned(cp[k].user);
  for (int k = 0; k < kNumCopies; ++k) cp[k].staged = !direct && cp[k].user != cp[k].twin;
  const void* staged_key[8] = {(void*)(flags | ((uintptr_t)have_L << 17)), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  const void** key = direct ? direct_key : staged_key;
  stage_inputs(cp, kCpOutAb);
  if (!replay && (!c->graph_exec.get() || memcmp(key, c->graph_ptrs, sizeof(staged_key)) != 0 || c->graph_maskcent != maskcent)) {
    c->graph_exec.reset();
    cudaGraph_t g = nullptr;
    CUDA_TRY(c, cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    const bool prof = c->profiling;
    c->profiling = false;            // event timing is meaningless inside a capture
    cudaError_t ce = issue_copies(cp, kCpOutAb, st);
    int rc = ce == cudaSuccess ? run_host_forward(c, n, maskcent, cp, want_dist, st, nullptr) : IDC_OK;
    if (rc == IDC_OK && ce == cudaSuccess) ce = issue_copies(cp + kCpOutAb, kCpDist - kCpOutAb, st);   // [ab | rgb | abq]
    if (rc == IDC_OK && ce == cudaSuccess) ce = issue_copies(cp + kCpDist, 1, st);
    c->profiling = prof;
    cudaError_t ce2 = cudaStreamEndCapture(st, &g);
    if (rc != IDC_OK) { if (g) cudaGraphDestroy(g); return rc; }
    if (ce != cudaSuccess) { if (g) cudaGraphDestroy(g); CUDA_TRY(c, ce); }
    CUDA_TRY(c, ce2);
    ce = cudaGraphInstantiate(c->graph_exec.put(), g, 0);
    cudaGraphDestroy(g);
    CUDA_TRY(c, ce);
    c->graph_captures++;
    memcpy(c->graph_ptrs, key, sizeof(staged_key));
    c->graph_maskcent = maskcent;
    c->graph_launches = c->launch_count;
  }
  if (c->dbg_graph_timing) CUDA_TRY(c, cudaEventRecord(c->dbg_ev[0].get(), st));
  CUDA_TRY(c, cudaGraphLaunch(c->graph_exec.get(), st));
  if (c->dbg_graph_timing) CUDA_TRY(c, cudaEventRecord(c->dbg_ev[1].get(), st));
  c->launch_count = c->graph_launches;
  c->last_n = n;
  CUDA_TRY(c, cudaStreamSynchronize(st));
  if (c->dbg_graph_timing) cudaEventElapsedTime(&c->dbg_graph_ms, c->dbg_ev[0].get(), c->dbg_ev[1].get());
  return IDC_OK;
}

// Every other call: eager copies on the context's stream, with the chunked overlap of HostPipe for batches >= 8.
// Caller memory is staged tensor by tensor, and each input is copied on its own, so the CPU stages the next input
// while the last one is in flight.
static int forward_host_eager(Ctx* c, int n, float maskcent, HostCopy* cp, bool want_dist) {
  for (int k = 0; k < kNumCopies; ++k) cp[k].staged = cp[k].bytes && cp[k].user != cp[k].twin && !is_pinned(cp[k].user);
  cudaStream_t st = c->own_stream.get();
  // large batches: chunked copy/compute overlap (see HostPipe); option host_pipe=0 turns it off for A/B runs
  const bool pipe_on = c->opt.host_pipe != 0;
  const bool fused_head = !c->simt && !(c->flags & IDC_FLAG_KEEP_CONV10);
  HostPipe hp;
  bool last_splits = false;
  for (auto& op : c->ops) if (op.fuse_out_head) last_splits = umma_op_uses_split_k(op);
  if (pipe_on && n >= 8 && fused_head && !last_splits && !c->profiling) {
    hp.nchunks = n >= 32 ? 4 : 2;   // measured: 8 chunks at n = 64 is 1.3 % slower end to end than 4
    for (int k = 0; k <= hp.nchunks; ++k) hp.start[k] = (int)((long long)n * k / hp.nchunks);
    hp.ab_dst = reinterpret_cast<float*>(cp[kCpOutAb].host());
    if (!c->pipe) {
      auto g = std::make_unique<HostPipeStreams>();
      CUDA_TRY(c, new_stream(g->s_in));
      CUDA_TRY(c, new_stream(g->s_out));
      for (int k = 0; k < HostPipe::kMaxChunks; ++k) {
        CUDA_TRY(c, new_event(g->ev_in[k]));
        CUDA_TRY(c, new_event(g->ev_out[k]));
      }
      c->pipe = std::move(g);
    }
  }
  auto put = [](const HostCopy& e, cudaStream_t s) { stage_inputs(&e, 1); return issue_copies(&e, 1, s); };
  if (hp.nchunks) {
    // the glob vector and the hint block go ahead of the first chunk, so ev_in[0] (which the MLP and the raster launch
    // wait for) covers them
    const cudaStream_t s_in = c->pipe->s_in.get();
    CUDA_TRY(c, put(cp[kCpGlob], s_in));
    CUDA_TRY(c, put(cp[kCpHints], s_in));
    for (int k = 0; k < hp.nchunks; ++k) {
      for (int j = kCpL; j <= kCpMask; ++j) CUDA_TRY(c, put(image_range(cp[j], n, hp.start[k], hp.start[k + 1]), s_in));
      CUDA_TRY(c, cudaEventRecord(c->pipe->ev_in[k].get(), s_in));
    }
  } else {
    for (int k = 0; k < kCpOutAb; ++k) CUDA_TRY(c, put(cp[k], st));
  }
  int rc = run_host_forward(c, n, maskcent, cp, want_dist, st, hp.nchunks ? &hp : nullptr);
  if (rc != IDC_OK) return rc;
  for (int k = hp.nchunks ? kCpRgb : kCpOutAb; k < kNumCopies; ++k)   // with HostPipe, run_forward brings ab back
    CUDA_TRY(c, issue_copies(cp + k, 1, st));
  CUDA_TRY(c, cudaStreamSynchronize(st));
  if (hp.nchunks) CUDA_TRY(c, cudaStreamSynchronize(c->pipe->s_out.get()));
  return IDC_OK;
}

static int ensure_host_staging(idc_ctx* c) {
  if (c->stage) return IDC_OK;
  const size_t HW = (size_t)c->H * c->W, HW4 = (size_t)(c->H / 4) * (c->W / 4);
  const int small_n = c->max_n < 4 ? c->max_n : 4;
  const size_t in_floats = (size_t)c->max_n * (4 * HW + 316);
  const size_t out_floats = (size_t)c->max_n * (2 * HW + (c->dist ? 529 * HW4 : 0));
  const size_t small_bytes = (size_t)small_n * (2 * HW * 4 + 3 * HW + 2 * HW * 8);
  auto g = std::make_unique<HostStaging>();
  CUDA_TRY(c, cudaMalloc(g->d_in.put(), in_floats * sizeof(float)));
  CUDA_TRY(c, cudaMalloc(g->d_out.put(), out_floats * sizeof(float)));
  CUDA_TRY(c, cudaMalloc(g->d_rgb.put(), (size_t)c->max_n * HW * 3));
  CUDA_TRY(c, cudaMalloc(g->d_small.put(), small_bytes));
  CUDA_TRY(c, cudaMallocHost(g->h_in.put(), in_floats * sizeof(float)));
  CUDA_TRY(c, cudaMallocHost(g->h_out.put(), out_floats * sizeof(float)));
  CUDA_TRY(c, cudaMallocHost(g->h_rgb.put(), (size_t)c->max_n * HW * 3));
  CUDA_TRY(c, cudaMallocHost(g->h_small.put(), small_bytes));
  c->stage = std::move(g);
  return IDC_OK;
}

int idc_set_image(idc_ctx* c, int n, int h, int w, const float* L) {
  if (!c) return IDC_ERR_ARG;
  if (n < 0 || n > c->max_n) return fail(c, IDC_ERR_ARG, "n=%d outside [0,%d]", n, c->max_n);
  if (n == 0 || !L) { c->image_n = 0; return IDC_OK; }
  if (h != c->H || w != c->W) return fail(c, IDC_ERR_ARG, "geometry %dx%d != ctx geometry %dx%d", h, w, c->H, c->W);
  CUDA_TRY(c, cudaSetDevice(c->dev));
  int rc = ensure_host_staging(c);
  if (rc != IDC_OK) return rc;
  c->image_n = 0;
  CUDA_TRY(c, cudaStreamSynchronize(c->own_stream.get()));
  // the L planes sit at the head of the input block for every batch size (small and large path alike)
  CUDA_TRY(c, cudaMemcpy(c->stage->d_in.get(), L, (size_t)n * c->H * c->W * sizeof(float), cudaMemcpyHostToDevice));
  c->image_n = n;
  return IDC_OK;
}

int idc_set_hints(idc_ctx* c, int count, const idc_hint* hints) {
  if (!c) return IDC_ERR_ARG;
  if (count < 0 || count > IDC_MAX_HINTS) return fail(c, IDC_ERR_ARG, "count=%d outside [0,%d]", count, IDC_MAX_HINTS);
  if (count && !hints) return fail(c, IDC_ERR_ARG, "null hint list");
  if (!c->hints) {
    CUDA_TRY(c, cudaSetDevice(c->dev));
    auto g = std::make_unique<HintBlock>();
    CUDA_TRY(c, cudaMalloc(g->d_hints.put(), kHintBlockBytes));
    CUDA_TRY(c, cudaMallocHost(g->h_hints.put(), kHintBlockBytes));
    memset(g->h_hints.get(), 0, kHintBlockBytes);
    c->hints = std::move(g);
  }
  // every idc_forward_host(_q) has synchronised before returning: no copy of the block is in flight
  char* block = c->hints->h_hints.get();
  *reinterpret_cast<int*>(block) = count;
  if (count) memcpy(block + kHintHdrBytes, hints, (size_t)count * sizeof(idc_hint));
  return IDC_OK;
}

int idc_forward_host_q(idc_ctx* c, int n, int h, int w, const float* L, const float* ab, const float* mask,
                       float maskcent, const float* glob, float* out_ab, float* out_dist, uint8_t* out_rgb,
                       double* out_abq) {
  if (!c) return IDC_ERR_ARG;
  // NULL L: idc_set_image; NULL ab and mask: idc_set_hints
  int rc = check_forward_args(c, n, h, w, L, ab, mask, glob, out_ab, out_dist, /*resident_l_ok=*/true, /*hints_ok=*/true);
  if (rc != IDC_OK) return rc;
  if (out_abq && !out_rgb) return fail(c, IDC_ERR_ARG, "out_abq (quantised ab) is derived from out_rgb: pass both");
  const bool hint_mode = !ab && !mask;
  if (hint_mode) {
    if (!c->hints) return fail(c, IDC_ERR_STATE, "ab and mask are NULL but idc_set_hints was never called");
    const char* block = c->hints->h_hints.get();
    const int count = *reinterpret_cast<const int*>(block);
    const idc_hint* hs = reinterpret_cast<const idc_hint*>(block + kHintHdrBytes);
    for (int i = 0; i < count; ++i)
      if (hs[i].img < 0 || hs[i].img >= n) return fail(c, IDC_ERR_ARG, "hint %d: img=%d outside [0,%d)", i, hs[i].img, n);
  }
  CUDA_TRY(c, cudaSetDevice(c->dev));
  rc = take_device_flags(c, "device pipeline watchdog fired earlier (code %d)");   // left over from an asynchronous idc_forward
  if (rc != IDC_OK) return rc;
  rc = ensure_host_staging(c);
  if (rc != IDC_OK) return rc;
  if (!L && c->image_n != n)
    return fail(c, IDC_ERR_STATE, "L_mc is NULL but no %d-image set is resident (idc_set_image)", n);
  const bool use_graph = !(c->flags & IDC_FLAG_NO_GRAPH) && n <= 4;
  if (!use_graph && out_abq && !c->abq) {
    const size_t bytes = (size_t)c->max_n * 2 * c->H * c->W * sizeof(double);
    auto g = std::make_unique<AbqStaging>();
    CUDA_TRY(c, cudaMalloc(g->d_abq.put(), bytes));
    CUDA_TRY(c, cudaMallocHost(g->h_abq.put(), bytes));
    c->abq = std::move(g);
  }
  HostCopy cp[kNumCopies];
  host_copies(c, n, use_graph, L, ab, mask, glob, out_ab, out_dist, out_rgb, out_abq, cp);
  const bool want_dist = out_dist || (c->dist_resident && c->dist);
  c->click_served = false;
  rc = use_graph ? forward_host_graph(c, n, maskcent, cp, want_dist) : forward_host_eager(c, n, maskcent, cp, want_dist);
  if (rc != IDC_OK) return rc;
  unstage_outputs(cp, kNumCopies);
  c->dist_valid_n = want_dist ? n : 0;
  c->click_served = use_graph && want_dist && c->click_mode && c->click;   // the side branch delivered the click's answer
  if (L) c->image_n = n;               // the planes just uploaded are the resident image now
  return take_device_flags(c, "device pipeline watchdog fired (code %d)");
}

void* idc_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (bytes == 0 || cudaHostAlloc(&p, bytes, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  return p;
}

int idc_host_free(void* p) {
  if (!p) return IDC_ERR_ARG;
  return cudaFreeHost(p) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_set_dist_resident(idc_ctx* c, int on) {
  if (!c) return IDC_ERR_ARG;
  if (on && !c->dist) return fail(c, IDC_ERR_ARG, "resident dist requires IDC_FLAG_DIST");
  c->dist_resident = on != 0;
  return IDC_OK;
}

// does the pinned click block hold the answer for this pixel?
static bool click_answers(idc_ctx* c, int img, int y4, int x4) {
  if (!c->click_served || !c->click) return false;
  const int* hdr = reinterpret_cast<const int*>(c->click->h_clickout.get());
  return hdr[7] == 1 && hdr[0] == img && hdr[1] == y4 && hdr[2] == x4;
}

int idc_set_click(idc_ctx* c, int img, int y4, int x4, int K) {
  if (!c) return IDC_ERR_ARG;
  if (!c->dist) return fail(c, IDC_ERR_ARG, "idc_set_click requires IDC_FLAG_DIST");
  if (K < 0 || K > 32) return fail(c, IDC_ERR_ARG, "idc_set_click: need 0 <= K <= 32");
  CUDA_TRY(c, cudaSetDevice(c->dev));
  if (!c->click) {
    auto g = std::make_unique<ClickBlock>();
    CUDA_TRY(c, cudaHostAlloc(g->h_click.put(), 64, cudaHostAllocMapped));
    memset(g->h_click.get(), 0, 64);
    g->h_click.get()[1] = -1;
    CUDA_TRY(c, cudaHostGetDevicePointer(&g->d_click, g->h_click.get(), 0));
    CUDA_TRY(c, cudaMalloc(g->d_clickout.put(), kClickBytes));
    CUDA_TRY(c, cudaMemset(g->d_clickout.get(), 0, kClickBytes));
    CUDA_TRY(c, cudaMallocHost(g->h_clickout.put(), kClickCopy));
    memset(g->h_clickout.get(), 0, kClickCopy);
    float pts[529 * 2];   // the PyTorch wrapper's gamut grid (data/colorize_image.py:283): bin i = (g[i % 23], g[i / 23])
    for (int i = 0; i < 529; ++i) { pts[2 * i] = -110.f + 10.f * (i % 23); pts[2 * i + 1] = -110.f + 10.f * (i / 23); }
    CUDA_TRY(c, cudaMemcpy(g->d_clickout.get() + kClickCopy, pts, sizeof(pts), cudaMemcpyHostToDevice));
    c->click = std::move(g);
  }
  volatile int* h = c->click->h_click.get();
  h[0] = img; h[1] = y4; h[2] = x4; h[3] = K; h[4] = h[4] + 1;
  c->click_mode = y4 >= 0;           // part of the graph key: switching the mode re-captures the click graph once
  c->click_served = false;
  return IDC_OK;
}

int idc_fetch_dist(idc_ctx* c, int img, int y4, int x4, float* out) {
  if (!c || !out) return IDC_ERR_ARG;
  if (img < 0 || img >= c->dist_valid_n || !c->stage)
    return fail(c, IDC_ERR_STATE, "no resident distribution for image %d (run idc_forward_host with resident mode on)", img);
  const int H4 = c->H / 4, W4 = c->W / 4;
  const size_t HW = (size_t)c->H * c->W, HW4 = (size_t)H4 * W4;
  const float* d = c->stage->d_out.get() + (size_t)c->max_n * 2 * HW + (size_t)img * 529 * HW4;
  CUDA_TRY(c, cudaSetDevice(c->dev));
  if (y4 < 0) {
    CUDA_TRY(c, cudaMemcpy(out, d, 529 * HW4 * sizeof(float), cudaMemcpyDeviceToHost));
    return IDC_OK;
  }
  if (y4 >= H4 || x4 < 0 || x4 >= W4) return fail(c, IDC_ERR_ARG, "pixel (%d,%d) outside the %dx%d grid", y4, x4, H4, W4);
  if (click_answers(c, img, y4, x4)) {       // idc_set_click: the forward already brought this pixel back
    memcpy(out, c->click->h_clickout.get() + kClickHdr, 529 * sizeof(float));
    return IDC_OK;
  }
  // one float per bin, bins are HW4 floats apart (NCHW)
  CUDA_TRY(c, cudaMemcpy2D(out, sizeof(float), d + (size_t)y4 * W4 + x4, HW4 * sizeof(float), sizeof(float), 529,
                           cudaMemcpyDeviceToHost));
  return IDC_OK;
}

// shared by idc_ab_reccs / idc_ab_reccs_pmf.  scratch (doubles): [kReccsMaxInit][3*32+2] results, then the 529x2
// gamut points as floats.
constexpr size_t kReccsScratchBytes = (size_t)kReccsMaxInit * kReccsRes * sizeof(double) + 529 * 2 * sizeof(float);

static bool reccs_args_ok(int K, int max_iter, int n_init) {
  return K >= 1 && K <= 32 && max_iter >= 1 && n_init >= 1 && n_init <= kReccsMaxInit;
}

// the restart reccs_best picks, as float32 outputs
static void reccs_pick(const double* res, int K, int n_init, float* centers_host, float* conf_host, int* iters_out) {
  const int stride = 3 * K + 2;
  const double* r = res + (size_t)reccs_best(res, K, n_init) * stride;
  for (int i = 0; i < 2 * K; ++i) centers_host[i] = (float)r[i];
  if (conf_host) for (int k = 0; k < K; ++k) conf_host[k] = (float)r[2 * K + k];
  if (iters_out) *iters_out = (int)r[3 * K];
}

static cudaError_t reccs_run(const float* pmf_dev, size_t bin_stride, double* scratch, int K, int max_iter, int n_init,
                             const float* pts_host, float* centers_host, float* conf_host, int* iters_out) {
  float pts[529 * 2];
  if (pts_host) {
    memcpy(pts, pts_host, sizeof(pts));
  } else {   // the PyTorch wrapper's gamut grid (data/colorize_image.py:283, quirk q3): bin i = (g[i % 23], g[i / 23])
    for (int i = 0; i < 529; ++i) { pts[2 * i] = -110.f + 10.f * (i % 23); pts[2 * i + 1] = -110.f + 10.f * (i / 23); }
  }
  float* pts_dev = reinterpret_cast<float*>(scratch + (size_t)kReccsMaxInit * kReccsRes);
  cudaError_t e = cudaMemcpy(pts_dev, pts, sizeof(pts), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return e;
  if ((e = launch_ab_reccs(pmf_dev, bin_stride, pts_dev, K, max_iter, n_init, scratch, 0)) != cudaSuccess) return e;
  const int stride = 3 * K + 2;
  double res[kReccsMaxInit * kReccsRes];
  if ((e = cudaMemcpy(res, scratch, (size_t)n_init * stride * sizeof(double), cudaMemcpyDeviceToHost)) != cudaSuccess) return e;
  reccs_pick(res, K, n_init, centers_host, conf_host, iters_out);
  return cudaSuccess;
}

int idc_ab_reccs(idc_ctx* c, int img, int y4, int x4, int K, int max_iter, int n_init, const float* pts_host,
                 float* centers_host, float* conf_host, int* iters_out) {
  if (!c || !centers_host) return IDC_ERR_ARG;
  if (!reccs_args_ok(K, max_iter, n_init))
    return fail(c, IDC_ERR_ARG, "idc_ab_reccs: need 1 <= K <= 32, max_iter >= 1, 1 <= n_init <= %d", kReccsMaxInit);
  if (img < 0 || img >= c->dist_valid_n || !c->stage)
    return fail(c, IDC_ERR_STATE, "no resident distribution for image %d (run idc_forward_host with resident mode on)", img);
  const int H4 = c->H / 4, W4 = c->W / 4;
  if (y4 < 0 || y4 >= H4 || x4 < 0 || x4 >= W4) return fail(c, IDC_ERR_ARG, "pixel (%d,%d) outside the %dx%d grid", y4, x4, H4, W4);
  const size_t HW = (size_t)c->H * c->W, HW4 = (size_t)H4 * W4;
  // idc_set_click with the same pixel and K, default restarts / iterations / gamut grid: the click graph already
  // clustered this pmf on its side branch and the results are in pinned host memory
  const char* clickout = c->click ? c->click->h_clickout.get() : nullptr;
  if (click_answers(c, img, y4, x4) && reinterpret_cast<const int*>(clickout)[3] == K && max_iter == kClickMaxIter &&
      n_init == kClickInit) {
    bool default_pts = pts_host == nullptr;
    if (!default_pts) {
      default_pts = true;
      for (int i = 0; i < 529 && default_pts; ++i)
        default_pts = pts_host[2 * i] == -110.f + 10.f * (i % 23) && pts_host[2 * i + 1] == -110.f + 10.f * (i / 23);
    }
    if (default_pts) {
      reccs_pick(reinterpret_cast<const double*>(clickout + kClickHdr + kClickPmf), K, n_init, centers_host, conf_host,
                 iters_out);
      return IDC_OK;
    }
  }
  const float* d = c->stage->d_out.get() + (size_t)c->max_n * 2 * HW + (size_t)img * 529 * HW4 + (size_t)y4 * W4 + x4;
  CUDA_TRY(c, cudaSetDevice(c->dev));
  if (!c->d_reccs.get()) CUDA_TRY(c, cudaMalloc(c->d_reccs.put(), kReccsScratchBytes));
  CUDA_TRY(c, reccs_run(d, HW4, c->d_reccs.get(), K, max_iter, n_init, pts_host, centers_host, conf_host, iters_out));
  return IDC_OK;
}

int idc_ab_reccs_pmf(int device, const float* pmf_host, int K, int max_iter, int n_init, const float* pts_host,
                     float* centers_host, float* conf_host, int* iters_out) {
  if (!pmf_host || !centers_host || !reccs_args_ok(K, max_iter, n_init)) return IDC_ERR_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  DevMem<char> buf;
  if (cudaMalloc(buf.put(), kReccsScratchBytes + 529 * sizeof(float)) != cudaSuccess) return IDC_ERR_CUDA;
  float* pmf_dev = reinterpret_cast<float*>(buf.get() + kReccsScratchBytes);
  cudaError_t e = cudaMemcpy(pmf_dev, pmf_host, 529 * sizeof(float), cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = reccs_run(pmf_dev, 1, reinterpret_cast<double*>(buf.get()), K, max_iter, n_init, pts_host, centers_host, conf_host,
                  iters_out);
  return e == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

// The heads a batched suggestion call reads: the entry point's name, the head it needs, and the grid its queries
// address (the pixels of a forward's image divided by `div`).
struct ReccsHead {
  const char* fn;
  const char* head;
  int div;
};
static const ReccsHead kReccsHead529 = {"idc_ab_reccs_batch", "the 529-bin head (IDC_FLAG_DIST)", 4};
static const ReccsHead kReccsHead313 = {"idc_caffe313_reccs_batch", "the Caffe 313-bin head (IDC_FLAG_CAFFE313)", 1};

// The host checks of a batched suggestion call for a context with / without `hd`'s head whose last forward carried
// n_img images of h x w; the message names the first bad query.
static int reccs_batch_check(const ReccsHead& hd, bool head, int n_img, int h, int w, int q, const int32_t* queries, int K,
                             int max_iter, int n_init, char* msg, size_t cap) {
  if (!head) return snprintf(msg, cap, "%s needs %s", hd.fn, hd.head), IDC_ERR_STATE;
  if (n_img < 1) return snprintf(msg, cap, "%s: no forward has run on this context", hd.fn), IDC_ERR_STATE;
  if (q < 1 || q > IDC_MAX_RECCS_QUERIES || !queries)
    return snprintf(msg, cap, "%s: need 1 <= q <= %d queries, got %d", hd.fn, IDC_MAX_RECCS_QUERIES, q), IDC_ERR_ARG;
  if (!reccs_args_ok(K, max_iter, n_init))
    return snprintf(msg, cap, "%s: need 1 <= K <= 32, max_iter >= 1, 1 <= n_init <= %d", hd.fn, kReccsMaxInit),
           IDC_ERR_ARG;
  const int GH = h / hd.div, GW = w / hd.div;
  for (int i = 0; i < q; ++i) {
    const int32_t* t = queries + 3 * (size_t)i;
    if (t[0] < 0 || t[0] >= n_img)
      return snprintf(msg, cap, "%s: query %d: image %d outside the last forward's [0, %d)", hd.fn, i, t[0], n_img),
             IDC_ERR_ARG;
    if (t[1] < 0 || t[1] >= GH || t[2] < 0 || t[2] >= GW)
      return snprintf(msg, cap, "%s: query %d: pixel (%d,%d) outside the %dx%d grid", hd.fn, i, t[1], t[2], GH, GW),
             IDC_ERR_ARG;
  }
  return IDC_OK;
}

static int caffe313_reccs_check(bool head, int n_img, int h, int w, int q, const int32_t* queries, float S, int K,
                                int max_iter, int n_init, char* msg, size_t cap) {
  const int rc = reccs_batch_check(kReccsHead313, head, n_img, h, w, q, queries, K, max_iter, n_init, msg, cap);
  if (rc == IDC_OK && !std::isfinite(S))
    return snprintf(msg, cap, "%s: S = %g is not finite", kReccsHead313.fn, (double)S), IDC_ERR_ARG;
  return rc;
}

// The context's batched-suggestion scratch, room for q queries.  Grows stream-ordered: neither the release nor the
// allocation waits for the device.
static cudaError_t reccs_batch_scratch(Ctx* c, int q, cudaStream_t st) {
  if (q <= c->reccs_batch_q) return cudaSuccess;
  if (c->d_reccs_batch.get()) {
    const cudaError_t e = cudaFreeAsync(c->d_reccs_batch.release(), st);
    if (e != cudaSuccess) return e;
  }
  c->reccs_batch_q = 0;
  const cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(c->d_reccs_batch.put()), reccs_batch_scratch_bytes(q), st);
  if (e == cudaSuccess) c->reccs_batch_q = q;
  return e;
}

int idc_ab_reccs_batch(idc_ctx* c, int q, const int32_t* queries_host, int K, int max_iter, int n_init,
                       const float* pts_host, float* centers_dev, float* conf_dev, int32_t* iters_dev, float* pmf_dev,
                       void* stream) {
  if (!c) return IDC_ERR_ARG;
  char msg[256];
  const int rc = reccs_batch_check(kReccsHead529, c->dist, c->last_n, c->H, c->W, q, queries_host, K, max_iter, n_init,
                                   msg, sizeof(msg));
  if (rc != IDC_OK) return fail(c, rc, "%s", msg);
  if (!centers_dev) return fail(c, IDC_ERR_ARG, "idc_ab_reccs_batch: NULL centers");
  const cudaStream_t st = (cudaStream_t)stream;
  CUDA_TRY(c, cudaSetDevice(c->dev));
  CUDA_TRY(c, reccs_batch_scratch(c, q, st));
  CUDA_TRY(c, launch_reccs_batch(c, q, queries_host, pts_host, K, max_iter, n_init, c->d_reccs_batch.get(), centers_dev,
                                 conf_dev, iters_dev, pmf_dev, st));
  return IDC_OK;
}

int idc_ab_reccs_batch_check(int has_head, int n_img, int h, int w, int q, const int32_t* queries, int K, int max_iter,
                             int n_init, char* msg, size_t msg_bytes) {
  char buf[256];
  const int rc = reccs_batch_check(kReccsHead529, has_head != 0, n_img, h, w, q, queries, K, max_iter, n_init, buf,
                                   sizeof(buf));
  if (rc != IDC_OK && msg && msg_bytes) snprintf(msg, msg_bytes, "%s", buf);
  return rc;
}

int idc_caffe313_reccs_batch(idc_ctx* c, int q, const int32_t* queries_host, float S, int K, int max_iter, int n_init,
                             float* centers_dev, float* conf_dev, int32_t* iters_dev, float* pmf_dev, void* stream) {
  if (!c) return IDC_ERR_ARG;
  char msg[256];
  const int rc = caffe313_reccs_check(c->caffe313, c->last_n, c->H, c->W, q, queries_host, S, K, max_iter, n_init, msg,
                                      sizeof(msg));
  if (rc != IDC_OK) return fail(c, rc, "%s", msg);
  if (!centers_dev) return fail(c, IDC_ERR_ARG, "idc_caffe313_reccs_batch: NULL centers");
  const cudaStream_t st = (cudaStream_t)stream;
  CUDA_TRY(c, cudaSetDevice(c->dev));
  CUDA_TRY(c, reccs_batch_scratch(c, q, st));
  CUDA_TRY(c, launch_caffe313_reccs_batch(c, q, queries_host, S, K, max_iter, n_init, c->d_reccs_batch.get(),
                                          centers_dev, conf_dev, iters_dev, pmf_dev, st));
  return IDC_OK;
}

int idc_caffe313_reccs_batch_check(int has_head, int n_img, int h, int w, int q, const int32_t* queries, float S, int K,
                                   int max_iter, int n_init, char* msg, size_t msg_bytes) {
  char buf[256];
  const int rc = caffe313_reccs_check(has_head != 0, n_img, h, w, q, queries, S, K, max_iter, n_init, buf, sizeof(buf));
  if (rc != IDC_OK && msg && msg_bytes) snprintf(msg, msg_bytes, "%s", buf);
  return rc;
}

int idc_caffe313_pred_ab(idc_ctx* c, int n, float T, float* out_ab, void* stream) {
  if (!c || !out_ab || n < 1 || n > c->max_n) return IDC_ERR_ARG;
  if (!c->caffe313) return fail(c, IDC_ERR_STATE, "ctx was not created with IDC_FLAG_CAFFE313");
  CUDA_TRY(c, cudaSetDevice(c->dev));
  CUDA_TRY(c, launch_decode313(c, n, T, out_ab, (cudaStream_t)stream));
  return IDC_OK;
}

int idc_caffe313_dist_pixel(idc_ctx* c, int img, int y, int x, float S, float* out313_host) {
  if (!c || !out313_host || img < 0 || img >= c->max_n || y < 0 || y >= c->H || x < 0 || x >= c->W) return IDC_ERR_ARG;
  if (!c->caffe313) return fail(c, IDC_ERR_STATE, "ctx was not created with IDC_FLAG_CAFFE313");
  CUDA_TRY(c, cudaSetDevice(c->dev));
  if (!c->d_dist313.get()) CUDA_TRY(c, cudaMalloc(c->d_dist313.put(), 320 * sizeof(float)));
  CUDA_TRY(c, launch_dist313_pixel(c, img, y, x, S, c->d_dist313.get(), 0));
  CUDA_TRY(c, cudaMemcpy(out313_host, c->d_dist313.get(), 313 * sizeof(float), cudaMemcpyDeviceToHost));
  return IDC_OK;
}

int idc_caffe313_dist_map(idc_ctx* c, int n, float S, float* out_dist, void* stream) {
  if (!c || !out_dist || n < 1 || n > c->max_n) return IDC_ERR_ARG;
  if (!c->caffe313) return fail(c, IDC_ERR_STATE, "ctx was not created with IDC_FLAG_CAFFE313");
  CUDA_TRY(c, cudaSetDevice(c->dev));
  CUDA_TRY(c, launch_dist313_map(c, n, S, out_dist, (cudaStream_t)stream));
  return IDC_OK;
}

int idc_negentropy(int device, int n, int bins, int hw, const float* dist, float* out, void* stream) {
  if (n < 1 || n > 65535 || bins < 1 || hw < 1 || !dist || !out) return IDC_ERR_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_negentropy(n, bins, hw, dist, out, (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_dist_negentropy(idc_ctx* c, int img, float* out_host) {
  if (!c || !out_host) return IDC_ERR_ARG;
  if (img < 0 || img >= c->dist_valid_n || !c->stage)
    return fail(c, IDC_ERR_STATE, "no resident distribution for image %d (run idc_forward_host with resident mode on)", img);
  const size_t HW = (size_t)c->H * c->W, HW4 = (size_t)(c->H / 4) * (c->W / 4);
  const float* d = c->stage->d_out.get() + (size_t)c->max_n * 2 * HW + (size_t)img * 529 * HW4;
  CUDA_TRY(c, cudaSetDevice(c->dev));
  if (!c->d_negent.get()) CUDA_TRY(c, cudaMalloc(c->d_negent.put(), HW4 * sizeof(float)));
  CUDA_TRY(c, launch_negentropy(1, 529, (int)HW4, d, c->d_negent.get(), 0));
  CUDA_TRY(c, cudaMemcpy(out_host, c->d_negent.get(), HW4 * sizeof(float), cudaMemcpyDeviceToHost));
  return IDC_OK;
}

int idc_lab2rgb_u8(int device, int n, int h, int w, const float* L, const float* ab, uint8_t* rgb, void* stream) {
  if (n < 1 || h < 1 || w < 1 || !L || !ab || !rgb) return IDC_ERR_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_lab2rgb(nullptr, n, h, w, L, 0.0f, ab, rgb, (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_global_stats(int device, int h, int w, const uint8_t* rgb, const float* pts313, float* out316, void* stream) {
  if (h < 4 || w < 4 || (h % 4) || (w % 4) || !rgb || !pts313 || !out316) return IDC_ERR_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_global_stats(h, w, rgb, pts313, out316, (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_rgb2lab_f64(int device, int n, int h, int w, const uint8_t* rgb, double* lab, void* stream) {
  if (n < 1 || h < 1 || w < 1 || !rgb || !lab) return IDC_ERR_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_rgb2lab(n, h, w, rgb, lab, (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_zoom_lab2rgb_u8(int device, int h_in, int w_in, const double* ab, int h, int w, const double* L_full,
                        uint8_t* rgb, void* stream) {
  if (!ab) return IDC_ERR_ARG;
  return idc_render_planes_u8(device, h_in, w_in, ab, 1, 0, nullptr, 0, IDC_RENDER_L_PLANE, L_full, h, w, rgb, stream);
}

int idc_render_planes_u8(int device, int h_in, int w_in, const double* ab, int ab_order, int ab_f32, const double* mask,
                         int mask_f32, int l_mode, const double* L, int h, int w, uint8_t* rgb, void* stream) {
  if (h_in < 1 || w_in < 1 || h < 1 || w < 1 || !rgb) return IDC_ERR_ARG;
  if ((ab_order != 0 && ab_order != 1) || (ab_f32 != 0 && ab_f32 != 1) || (mask_f32 != 0 && mask_f32 != 1)) return IDC_ERR_ARG;
  if (l_mode == IDC_RENDER_L_PLANE ? !L : (l_mode == IDC_RENDER_L_MASK || l_mode == IDC_RENDER_L_SUP) ? !mask : true)
    return IDC_ERR_ARG;
  if ((size_t)h * w > (size_t)0x7fffffff * 256) return IDC_ERR_ARG;      // grid.x limit at 256 threads per block
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_render_planes(ab, ab_order, ab_f32, mask, mask_f32, l_mode, L, h_in, w_in, h, w, rgb,
                              (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_resize_u8_linear(int device, int h_src, int w_src, const uint8_t* src, int h_dst, int w_dst, uint8_t* dst, void* stream) {
  if (h_src < 1 || w_src < 1 || h_dst < 1 || w_dst < 1 || !src || !dst) return IDC_ERR_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_resize_linear_u8(src, h_src, w_src, dst, h_dst, w_dst, (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_cubic_lab2rgb_u8(int device, int h_in, int w_in, const double* ab, int h, int w, const double* L, uint8_t* rgb,
                         void* stream) {
  if (h_in < 1 || w_in < 1 || h < 1 || w < 1 || !ab || !L || !rgb) return IDC_ERR_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_cubic_lab2rgb(ab, h_in, w_in, L, h, w, rgb, (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_gamut_ab(int device, double L, int gamut_size, int D, uint8_t* rgb, uint8_t* mask, void* stream) {
  if (gamut_size < 0 || gamut_size > 4096 || D < 1 || !rgb || !mask) return IDC_ERR_ARG;
  const int A = (2 * gamut_size + D - 1) / D + 1;        // len(np.arange(-g, g + D, D))
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_gamut(L, gamut_size, D, A, rgb, mask, (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

// the photo table of a batch: 1 <= n <= IDC_MAX_PHOTOS, every photo at least 1 x 1, in ascending non-overlapping order
// X and the photo sides are bounded so that the kernels' 32-bit pixel and byte indices within one image cannot overflow
static bool photos_ok(int n, const idc_photo* t, int X) {
  if (n < 1 || n > IDC_MAX_PHOTOS || !t || X < 8 || X > IDC_MAX_PHOTO_X || (X % 8)) return false;
  int64_t end = 0;
  for (int i = 0; i < n; ++i) {
    if (t[i].h < 1 || t[i].w < 1 || t[i].h > IDC_MAX_PHOTO_SIDE || t[i].w > IDC_MAX_PHOTO_SIDE || t[i].off < end)
      return false;
    end = t[i].off + (int64_t)t[i].h * t[i].w;
  }
  return end <= (int64_t)0x7fffffff * 256;              // grid.x limit of the render at 256 threads per block
}

int idc_photo_prep(int device, int n, const idc_photo* photos, const uint8_t* src, int X, float* L_mc, uint8_t* rgb,
                   void* stream) {
  if (!photos_ok(n, photos, X) || !src || !L_mc) return IDC_ERR_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_photo_prep(n, photos, src, X, L_mc, rgb, (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_photo_render(int device, int n, const idc_photo* photos, const uint8_t* src, int X, const double* lab,
                     uint8_t* out, void* stream) {
  if (!photos_ok(n, photos, X) || !src || !lab || !out) return IDC_ERR_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_photo_render(n, photos, src, X, lab, out, (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_hint_raster(int device, int n, int h, int w, int count, const void* block, float* ab, float* mask, void* stream) {
  if (n < 1 || n > 65535 || h < 1 || w < 1 || count < 0 || count > IDC_MAX_HINTS || !block || !ab || !mask)
    return IDC_ERR_ARG;
  if ((size_t)h * w > (size_t)0x7fffffff - 256) return IDC_ERR_ARG;   // the kernel's int pixel index + one CTA
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_hint_raster(nullptr, n, h, w, static_cast<const char*>(block), ab, mask, (cudaStream_t)stream) == cudaSuccess
             ? IDC_OK : IDC_ERR_CUDA;
}

int idc_hint_fill_mean(int device, int n_blocks, int levels, int X, const double* lab, void* blocks, size_t block_stride,
                       void* stream) {
  if (n_blocks < 1 || n_blocks > 65535 || levels < 1 || X < 1 || X > IDC_MAX_PHOTO_X || !lab || !blocks) return IDC_ERR_ARG;
  if (block_stride < kHintHdrBytes || block_stride % 4 || (uintptr_t)blocks % 4) return IDC_ERR_ARG;   // int32 fields
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_hint_fill_mean(n_blocks, levels, X, lab, static_cast<char*>(blocks), block_stride, (cudaStream_t)stream)
             == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_global_stats_batch(int device, int n, int h, int w, const uint8_t* rgb, const float* pts313, float* out,
                           void* stream) {
  if (n < 1 || n > 65535 || h < 4 || w < 4 || (h % 4) || (w % 4) || h > IDC_MAX_PHOTO_X || w > IDC_MAX_PHOTO_X) return IDC_ERR_ARG;
  if (!rgb || !pts313 || !out) return IDC_ERR_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_global_stats_batch(n, h, w, rgb, pts313, out, (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_rgb_sse(int device, int n, int h, int w, const uint8_t* a, const uint8_t* b, int64_t* sse, void* stream) {
  if (n < 1 || n > 65535 || h < 1 || w < 1 || !a || !b || !sse) return IDC_ERR_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return IDC_ERR_CUDA;
  return launch_rgb_sse(n, (size_t)h * w * 3, a, b, sse, (cudaStream_t)stream) == cudaSuccess ? IDC_OK : IDC_ERR_CUDA;
}

int idc_act_exponent(idc_ctx* c, const char* name, int* exp_out) {
  if (!c || !name || !exp_out) return IDC_ERR_ARG;
  auto it = c->buf_index.find(name);
  if (it == c->buf_index.end() || c->bufs[it->second].H == 0) return fail(c, IDC_ERR_KEY, "no activation '%s'", name);
  if (!c->weights_ready) return fail(c, IDC_ERR_STATE, "idc_act_exponent before idc_finalize_weights");
  *exp_out = c->bufs[it->second].exp;
  return IDC_OK;
}

int idc_num_acts(idc_ctx* c) {
  int k = 0;
  if (c) for (auto& b : c->bufs) k += b.H > 0;
  return k;
}
const char* idc_act_name(idc_ctx* c, int i) {
  if (c && i >= 0)
    for (auto& b : c->bufs)
      if (b.H > 0 && i-- == 0) return b.name.c_str();
  return nullptr;
}

int idc_act_absmax(idc_ctx* c, const char* name, int n, float* out_host) {
  if (!c || !name || !out_host || n < 1 || n > c->max_n) return fail(c, IDC_ERR_ARG, "bad idc_act_absmax args");
  auto it = c->buf_index.find(name);
  if (it == c->buf_index.end() || c->bufs[it->second].H == 0) return fail(c, IDC_ERR_KEY, "no activation '%s'", name);
  if (!c->weights_ready) return fail(c, IDC_ERR_STATE, "idc_act_absmax before idc_finalize_weights");
  const ActBuf& b = c->bufs[it->second];
  if (b.C % 8) return fail(c, IDC_ERR_UNSUPPORTED, "activation %s: %d channels, idc_act_absmax reads 8 at a time", name, b.C);
  CUDA_TRY(c, cudaSetDevice(c->dev));
  if (!c->d_absmax.get()) CUDA_TRY(c, cudaMalloc(c->d_absmax.put(), sizeof(unsigned)));
  CUDA_TRY(c, cudaDeviceSynchronize());   // the forward that wrote the buffer may be running on any stream
  CUDA_TRY(c, launch_act_absmax(c, b, n, c->d_absmax.get(), 0));
  unsigned bits = 0;
  CUDA_TRY(c, cudaMemcpy(&bits, c->d_absmax.get(), sizeof(bits), cudaMemcpyDeviceToHost));
  float v;
  memcpy(&v, &bits, sizeof(v));
  *out_host = v * ldexpf(1.f, -b.exp);    // stored units -> value, the multiply idc_get_activation applies per element
  return IDC_OK;
}

int idc_set_act_range(idc_ctx* c, const char* name, double max_abs) {
  if (!c || !name) return IDC_ERR_ARG;
  auto it = c->buf_index.find(name);
  if (it == c->buf_index.end() || c->bufs[it->second].H == 0) return fail(c, IDC_ERR_KEY, "no activation '%s'", name);
  if (!std::isfinite(max_abs) || !(max_abs > 0.0))
    return fail(c, IDC_ERR_ARG, "range of activation %s = %g: must be finite and > 0", name, max_abs);
  if (c->weights_adopted)
    return fail(c, IDC_ERR_STATE, "the range of %s must be set before the weights are packed (idc_finalize_weights)", name);
  c->act_range[name] = max_abs;
  return IDC_OK;
}

int idc_get_activation(idc_ctx* c, const char* name, float* out, size_t out_floats, int* ch, int* h, int* w) {
  if (!c || !name) return IDC_ERR_ARG;
  auto it = c->buf_index.find(name);
  if (it == c->buf_index.end() || c->bufs[it->second].H == 0) return fail(c, IDC_ERR_KEY, "no activation '%s'", name);
  const ActBuf& b = c->bufs[it->second];
  if (ch) *ch = b.C;
  if (h) *h = b.H;
  if (w) *w = b.W;
  if (!out) return IDC_OK;
  const int n = c->last_n > 0 ? c->last_n : 1;
  if (out_floats < (size_t)n * b.C * b.H * b.W) return fail(c, IDC_ERR_ARG, "output too small");
  CUDA_TRY(c, cudaSetDevice(c->dev));
  CUDA_TRY(c, launch_act_to_nchw(c, b, n, out, 0));
  CUDA_TRY(c, cudaDeviceSynchronize());
  return IDC_OK;
}

int idc_set_activation(idc_ctx* c, const char* name, int n, const float* in) {
  if (!c || !name || !in || n < 1 || n > c->max_n) return IDC_ERR_ARG;
  auto it = c->buf_index.find(name);
  if (it == c->buf_index.end() || c->bufs[it->second].H == 0) return fail(c, IDC_ERR_KEY, "no activation '%s'", name);
  CUDA_TRY(c, cudaSetDevice(c->dev));
  CUDA_TRY(c, launch_nchw_to_act(c, c->bufs[it->second], n, in, 0));
  CUDA_TRY(c, cudaDeviceSynchronize());
  c->last_n = n;
  return IDC_OK;
}

int idc_run_op(idc_ctx* c, const char* op_name, int n, void* stream) {
  if (!c || !op_name || n < 1 || n > c->max_n) return IDC_ERR_ARG;
  if (!c->weights_ready) return fail(c, IDC_ERR_STATE, "weights not finalized");
  CUDA_TRY(c, cudaSetDevice(c->dev));
  for (auto& op : c->ops)
    if (op.name == op_name) {
      if (op.fuse_out_head) return fail(c, IDC_ERR_ARG, "op %s has a fused head; use IDC_FLAG_KEEP_CONV10", op_name);
      c->gadd_active = false;
      if (c->simt) CUDA_TRY(c, simt_run_op(c, op, n, (cudaStream_t)stream));
      else CUDA_TRY(c, umma_run_op(c, op, n, nullptr, (float)c->opt.tanh_scale, (cudaStream_t)stream));
      c->last_n = n;
      return IDC_OK;
    }
  return fail(c, IDC_ERR_KEY, "no op '%s'", op_name);
}

int idc_set_profiling(idc_ctx* c, int enable) {
  if (!c) return IDC_ERR_ARG;
  c->profiling = enable != 0;
  return IDC_OK;
}

int idc_get_profile(idc_ctx* c, float* ms, int max_slots) {
  if (!c || !ms) return IDC_ERR_ARG;
  const int slots = (int)c->ops.size() + 2;
  if (max_slots < slots) return fail(c, IDC_ERR_ARG, "need %d slots", slots);
  CUDA_TRY(c, cudaSetDevice(c->dev));
  CUDA_TRY(c, cudaDeviceSynchronize());
  const int rc = take_device_flags(c, "device pipeline watchdog fired (code %d)");
  if (rc != IDC_OK) return rc;
  for (int i = 0; i < slots; ++i) ms[i] = 0.f;
  int runs = 0;
  for (auto& ev : c->prof_runs) {
    if ((int)ev.size() == slots + 1) {
      for (int i = 0; i < slots; ++i) {
        float t = 0.f;
        cudaEventElapsedTime(&t, ev[i].get(), ev[i + 1].get());
        ms[i] += t;
      }
      runs++;
    }
    for (Event& e : ev) c->prof_pool.push_back(std::move(e));
  }
  c->prof_runs.clear();
  if (runs) for (int i = 0; i < slots; ++i) ms[i] /= runs;
  return slots;
}

double idc_op_flops(idc_ctx* c, int i) {
  return (c && i >= 0 && i < (int)c->ops.size()) ? c->ops[i].flops_per_image : 0.0;
}

// experiments (tools/click_breakdown.py): device time of the click graph (copy nodes included), measured with two
// events around the graph launch.  enable = 1 / 0; returns the last span in *ms when non-null.
extern "C" int idc_debug_graph_timing(idc_ctx* c, int enable, float* ms) {
  if (!c) return IDC_ERR_ARG;
  CUDA_TRY(c, cudaSetDevice(c->dev));
  if (enable && !c->dbg_ev[0].get()) {
    Event ev[2];
    CUDA_TRY(c, cudaEventCreate(ev[0].put()));
    CUDA_TRY(c, cudaEventCreate(ev[1].put()));
    c->dbg_ev[0] = std::move(ev[0]);
    c->dbg_ev[1] = std::move(ev[1]);
  }
  c->dbg_graph_timing = enable != 0 && c->dbg_ev[0].get();
  if (ms) *ms = c->dbg_graph_ms;
  return IDC_OK;
}

int idc_num_ops(idc_ctx* c) { return c ? (int)c->ops.size() : 0; }
const char* idc_op_name(idc_ctx* c, int i) {
  return (c && i >= 0 && i < (int)c->ops.size()) ? c->ops[i].name.c_str() : nullptr;
}
int idc_last_launch_count(idc_ctx* c) { return c ? c->launch_count : 0; }
int idc_graph_captures(idc_ctx* c) { return c ? c->graph_captures : 0; }

double idc_flops_per_image(idc_ctx* c) {
  if (!c) return 0;
  double f = 2.0 * c->H * c->W * 64.0 * 36.0 + 2.0 * c->H * c->W * 2.0 * 128.0;  // model1.0 + model_out
  for (auto& op : c->ops) f += op.flops_per_image;
  return f;
}

const char* idc_last_error(idc_ctx* c) { return c ? c->err.c_str() : "null ctx"; }

int idc_destroy(idc_ctx* c) {
  if (!c) return IDC_ERR_ARG;
  cudaSetDevice(c->dev);
  cudaDeviceSynchronize();
  delete c;
  return IDC_OK;
}

}  // extern "C"
