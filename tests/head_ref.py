"""FP64 evaluations of the three heads of the Local Hints Network, each with a bound on how far the engine's FP32
evaluation of the same head may lie from it (test infrastructure; imports only oracle/ and tests/).

The heads are evaluated on the operands the engine's kernels consumed, read back after a forward
(LhnContext.get_activation: the wgmma engine's FP16 hi + lo planes carry ~22 bits, which FP32 holds exactly), so the
trunk's error stays out of the heads' bars.  Like tests/op_ref.py's (out, mag), every function returns the FP64 value
together with its bound; the bounds are formulas in 2^-24 (one FP32 rounding) times the magnitudes the kernels add.

  * regression head, model_out (1x1 128 -> 2) + scale * tanh (scale 110, or 100 for the Caffe-scaled models):
      - reg_from_conv10: on conv10_2 (out_head_kernel: SIMT engine, or IDC_FLAG_KEEP_CONV10);
      - reg_from_a10_1: c10_2 in FP64 from a10_1 (op_ref, exact mode) and then the head: the fused head of the wgmma
        engine's c10_2 epilogue consumes the FP32 accumulator, which is never stored.
    bound = scale * sech^2(max(|pre| - dpre, 0)) * dpre + 4 ulp32(|ab|) (tanhf <= 2 ulp, the x scale one rounding), with
      dpre = sum_c |w_out,c| * C10 * 2^-24 * mag10_c + C_HEAD * 2^-24 * (sum_c |w_out,c * v_c| + |b_out|).
  * distribution head, model_class (1x1 256 -> 529) + softmax(0.2 z) (softmax529_row): dist_head gives p64 and, per bin,
    the interval [lo, hi] of FP32 values the kernel may return.  In log space this is
      |ln p - ln p64| <= 0.2 (dz_k + max_j dz_j) + eps_k,  dz = C_CLS * 2^-24 * mag_z, mag_z = sum |w a| + |b|,
    eps_k = the roundings of softmax529_row: the x 0.2f (0.2f is 0.2 (1 + 1.5e-8)) and its rounding, the max
    subtraction, expf (<= 2 ulp), the 17-term lane sums and the 5-step butterfly (21 additions on every path), the
    reciprocal and the multiply.  The interval is built by carrying each step's relative bound and rounding the ends
    to the FP32 grid where the kernel rounds (to nearest, subnormals kept: float64 -> float32 is that rounding); a bin
    whose exp may fall below FLT_MIN also carries the error of the subtracted max, which the absolute rounding there
    does not cancel (test_head_ref_cpu feeds an FP32 restatement of the routine logits off by the budget).  So
    below FLT_MIN the rule becomes absolute: a bin whose interval rounds to 0 at both ends must be exactly 0 (p64
    clearly below 2^-150), one whose lower end rounds to 2^-149 or more must not be 0 (p64 clearly above 2^-149),
    and within the bound of either edge both outcomes are allowed.
    |sum p - 1| <= SUM_ULPS * 2^-24 + 529 * 2^-150: the sum, the reciprocal and the 529 products, each relative to
    the kernel's own exps; the FP64 exps cancel.
  * global-hints vector, dense_relu_bn_kernel x 4: glob_vector bounds the FP32 vector by each layer's own roundings
    (C_MLP of the dot product and the bias add, C_BN of the folded BatchNorm) carried to the output through the
    absolute Jacobian of the layers after it; glob_diff_bound is the bar of conv4_3(with the vector) -
    conv4_3(without it) against the vector.
  * peaked(sd, batch, target): model_class alone rescaled so that max |0.2 z| on a batch is `target` (e.g. 100), which
    sends many FP32 bins to 0 and into the subnormal range as a trained checkpoint's sharp pmfs do.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import caffe_spec, lhn_ref
from tests import op_ref

U = 2.0 ** -24                 # one FP32 rounding (round to nearest), relative
FLT_MIN = 2.0 ** -126

# --- accumulation constants, in units of 2^-24 * (the magnitude summed) ----------------------------------------------
# c10_2 on the wgmma engine: hi/lo operands (a 2^-22 weight split and the dropped lo*lo term), the tensor core's chunk
# sums (chunk_kb = 2) and 9 chunk adds, bias, LeakyReLU and the exact 2^-e scale.  Measured on an H100 80GB HBM3
# (700 W) on the stored conv10_2 of IDC_FLAG_KEEP_CONV10 (the same kernel and sums as the fused head's): 4.87 needed
# at most (rho = 0.3, 64^2, n = 3); 8 leaves 1.6x.
C10 = 8.0
# class (1x1, K = 256): the same kernel and operand split, chunk_kb = 1 and 4 chunk adds, so at most c10_2's constant.
# The pmfs cannot resolve it: on the same card the largest log-space deviation left over after softmax529_row's own
# roundings is 0.015 of a 16-unit logit term (0.24 units) on the peaked network, 0 on the others.  The SIMT engine sums
# the 256 products in one FP32 accumulator: 0.005 of 257 units (1.3) measured on the synthetic network; 16 leaves 12x
# (the worst case of a 256-term chain, 257 units, would make the bar 16x looser than TOL_DIST on the largest bins).
C_CLS = {"wgmma": 8.0, "simt": 16.0}
# the model_out dot product: the fused head chains 32 fmaf per lane and adds over the quad in 2 shuffle steps, the
# unfused out_head_kernel chains 16 and adds over 8 lanes in 3 steps; + the bias add.  35 covers both (analytic).
C_HEAD = 35.0
# softmax529_row's roundings, relative, on top of the logit and subtraction terms: expf 2 ulp = 4 units, 21 additions
# of positive terms, the reciprocal and the multiply
EXPF_UNITS = 4.0
SUM_ADDS = 21.0
SUM_ULPS = SUM_ADDS + 2.0 + 1.0           # the sum's 21 additions, 1 / sum, the products; +1 for second-order terms
# dense_relu_bn_kernel: a lane chains ceil(512 / 32) = 16 fmaf (10 for layer 0's 316 inputs), a 5-step butterfly, the
# bias add: 22 units (analytic).  The folded BatchNorm: scale and shift rounded to FP32 on the host, the multiply-add:
# 4 units of |scale * relu| + |beta| + |mean * scale|.
C_MLP = 22.0
C_BN = 4.0


def _d(x):
    return torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).double()


def ulp32(x):
    """The FP32 ulp of |x| (float64 tensor)."""
    a = np.abs(x.detach().cpu().numpy()).astype(np.float32)
    return torch.from_numpy(np.spacing(a).astype(np.float64))


def rn32(x):
    """float64 tensor -> the nearest FP32 value (round to nearest even, subnormals kept), as float64."""
    return x.double().float().double()


# ---------------------------------------------------------------------------------------------------------------------
# regression head
# ---------------------------------------------------------------------------------------------------------------------
def reg_head(sd, v, scale=110.0, dv=None):
    """model_out + scale * tanh on conv10_2 values v [n,128,H,W] (any float dtype), whose own error is at most dv
    (None: v is exactly what the head read).  -> (ab64 [n,2,H,W], bound), float64."""
    v = _d(v)
    w = _d(sd["model_out.0.weight"])[:, :, 0, 0]          # [2, 128]
    b = _d(sd["model_out.0.bias"])
    pre = torch.einsum("oc,nchw->nohw", w, v) + b[None, :, None, None]
    mag = torch.einsum("oc,nchw->nohw", w.abs(), v.abs()) + b.abs()[None, :, None, None]
    dpre = C_HEAD * U * mag
    if dv is not None:
        dpre = dpre + torch.einsum("oc,nchw->nohw", w.abs(), _d(dv))
    ab = scale * torch.tanh(pre)
    slope = 1.0 / torch.cosh((pre.abs() - dpre).clamp(min=0.0)) ** 2
    return ab, scale * slope * dpre + 4.0 * ulp32(ab)


def reg_from_conv10(sd, conv10_2, scale=110.0):
    """The unfused head (out_head_kernel) on its conv10_2 readback."""
    return reg_head(sd, conv10_2, scale)


def reg_from_a10_1(sd, a10_1, scale=110.0):
    """c10_2 (FP64, op_ref exact mode, LeakyReLU included) from the a10_1 readback, then the head: the fused head."""
    v, mag10 = op_ref.run_op("c10_2", sd, {"a10_1": _d(a10_1)})
    return reg_head(sd, v, scale, dv=C10 * U * mag10)


# ---------------------------------------------------------------------------------------------------------------------
# distribution head
# ---------------------------------------------------------------------------------------------------------------------
def class_logits(sd, conv8_3):
    """z = W conv8_3 + b and mag_z = |W| |conv8_3| + |b| in float64, [n,529,h,w] each."""
    a = _d(conv8_3)
    w, b = _d(sd["model_class.0.weight"]), _d(sd["model_class.0.bias"])
    return F.conv2d(a, w, b), F.conv2d(a.abs(), w.abs(), b.abs())


def dist_head(sd, conv8_3, engine="wgmma"):
    """softmax(0.2 z) in FP64 on the conv8_3 readback and the FP32 interval the kernel's pmf must lie in.
    -> dict p64, lo, hi ([n,529,h,w] float64; lo / hi are FP32 values), logbound (the log-space bound of a bin in
    the normal range), logit_term (its part 0.2 (dz_k + max_j dz_j)), sum_bound."""
    z, mag = class_logits(sd, conv8_3)
    dz = C_CLS[engine] * U * mag
    y = 0.2 * z
    m = y.amax(dim=1, keepdim=True)
    t = y - m
    # the kernel's y_j = RN(z~_j * 0.2f): 0.2 dz_j, 0.2f's own 1.5e-8 (a quarter unit) and the rounding.  It subtracts
    # its max, whose own error (up to max_j E_j) shifts every t_j alike.  Where the exps are rounded relatively (FP32's
    # normal range) that shift scales the bin and the sum by one factor and cancels in the ratio (the subnormal terms
    # of the sum are below 529 2^-126 of a sum >= 1).  An exp below FLT_MIN is rounded on an absolute grid, where the
    # shift moves it across rounding edges: a bin whose exp may land there is bounded with the shift in its argument
    # and in every term of the sum it is divided by.
    E = 0.2 * dz + 1.25 * U * y.abs()
    ex = EXPF_UNITS * U
    D = E + 1.000001 * U * t.abs()
    D_shift = D + E.amax(dim=1, keepdim=True)

    def interval(Dk):
        e_lo = rn32(torch.exp(t - Dk) * (1.0 - ex))
        e_hi = rn32(torch.exp(t + Dk) * (1.0 + ex))
        s_lo = rn32(e_lo.sum(dim=1, keepdim=True) * (1.0 - SUM_ADDS * U))
        s_hi = rn32(e_hi.sum(dim=1, keepdim=True) * (1.0 + SUM_ADDS * U))
        inv_lo, inv_hi = rn32(1.0 / s_hi), rn32(1.0 / s_lo)
        return rn32(e_lo * inv_lo), rn32(e_hi * inv_hi)

    lo, hi = interval(D)
    lo_s, hi_s = interval(D_shift)
    sub = torch.exp(t - D_shift) * (1.0 - ex) < FLT_MIN                # the bin's exp may be rounded below FLT_MIN
    lo, hi = torch.where(sub, lo_s, lo), torch.where(sub, hi_s, hi)
    p64 = torch.softmax(y, dim=1)
    logbound = E + E.amax(dim=1, keepdim=True) + U * (t.abs() + (p64 * t.abs()).sum(dim=1, keepdim=True)
                                                      + EXPF_UNITS * 2 + SUM_ADDS + 2)
    return {"p64": p64, "lo": lo, "hi": hi, "logbound": logbound, "logit_term": 0.2 * (dz + dz.amax(dim=1, keepdim=True)),
            "sum_bound": SUM_ULPS * U + 529 * 2.0 ** -150}


def dist_check(p, ref):
    """The kernel's pmf p [n,529,h,w] against dist_head's ref.  -> dict: frac (worst fraction of the interval's
    half-width on the side p lies, <= 1 passes), where (n, bin, y, x) of it, bad (bins outside [lo, hi]), sum_err,
    zero_must / zero_may / zero_got (bins that must be 0, may be 0, are 0), sub (bins in the subnormal range)."""
    p = _d(p)
    p64, lo, hi = ref["p64"], ref["lo"], ref["hi"]
    up = p >= p64
    width = torch.where(up, hi - p64, p64 - lo)
    dev = (p - p64).abs()
    frac = torch.where(dev == 0, torch.zeros_like(dev), dev / width.clamp(min=1e-320))
    frac = torch.where((p == 0) & (lo == 0), torch.zeros_like(frac), frac)          # a zero the interval allows
    i = int(torch.argmax(frac))
    where = np.unravel_index(i, tuple(frac.shape))
    bad = int(((p < lo) | (p > hi)).sum())
    return {"frac": float(frac.reshape(-1)[i]), "where": tuple(int(k) for k in where), "bad": bad,
            "sum_err": float((p.sum(dim=1) - 1.0).abs().max()),
            "zero_must": hi == 0, "zero_may": lo == 0, "zero_got": p == 0, "sub": (p > 0) & (p < FLT_MIN)}


# ---------------------------------------------------------------------------------------------------------------------
# global hints
# ---------------------------------------------------------------------------------------------------------------------
def glob_vector(gsd, glob316):
    """caffe_spec.global_hints_vector in FP64 and its FP32 bound, [n,512] each.

    Each layer l rounds its dot product and bias add (C_MLP units of |W||x| + |b|) and its folded BatchNorm (C_BN
    units); those local errors reach the output through the layers after l, to first order through their Jacobian
    J_l = d x_4 / d x_l = prod diag(scale * relu') W, so the bound is sum_l |J_l| (local error of layer l).  |J_l|, not
    the product of the |W|, is what keeps the bound near the errors' size: the |W| product grows ~25x per 512-input
    layer.  A unit whose pre-activation lies within the crude |W|-propagated bound of 0 counts as active."""
    x = _d(glob316)
    v = caffe_spec.global_hints_vector(gsd, x.numpy(), dtype=torch.float64)
    crude = torch.zeros_like(x)
    layers = []
    for l in range(4):
        t = lambda k: _d(gsd["glob.%d.%s" % (l, k)])
        w, b = t("weight"), t("bias")
        s = F.linear(x, w, b)
        es = C_MLP * U * (F.linear(x.abs(), w.abs()) + b.abs())
        ds = F.linear(crude, w.abs()) + es
        act = (s > -ds).double()
        r = F.relu(s)
        sc = t("bn.weight") / torch.sqrt(t("bn.running_var") + caffe_spec.BN_EPS)
        x = r * sc + (t("bn.bias") - t("bn.running_mean") * sc)
        ex = C_BN * U * ((r * sc).abs() + t("bn.bias").abs() + (t("bn.running_mean") * sc).abs())
        crude = sc.abs() * ds + ex
        layers.append((w, sc * act, ex + (sc * act).abs() * es))
    assert torch.allclose(x, v, rtol=0, atol=1e-12)
    d = torch.zeros_like(v)
    J = torch.eye(v.shape[1], dtype=torch.float64).expand(v.shape[0], -1, -1)
    for l in range(3, -1, -1):
        w, gain, local = layers[l]
        d = d + torch.einsum("nij,nj->ni", J.abs(), local)
        if l:
            J = torch.einsum("nij,nj,jk->nik", J, gain, w)
    return v, d


def bn_shift(sd, key="model4.6"):
    """The folded BatchNorm shift beta - mean * gamma / sqrt(var + eps) of a layer, float64 [C]."""
    g, b, m, v = (_d(sd[key + s]) for s in (".weight", ".bias", ".running_mean", ".running_var"))
    return b - m * g / torch.sqrt(v + lhn_ref.BN_EPS)


def c4_3_glob(sd, a4_2, vec):
    """conv4_3 with the global-hints vector added, FP64 from the a4_2 readback -> (out, mag)."""
    out, mag = op_ref.run_op("c4_3", sd, {"a4_2": _d(a4_2)})
    return out + _d(vec)[:, :, None, None], mag


def glob_diff_bound(sd, o_glob, o_plain, vec, dvec, S=None):
    """Bar of conv4_3(with the vector) - conv4_3(without it) against the FP64 vector vec (bound dvec), per element:
    the MLP bound, the FP32 shift + g (in value units: |shift + g| 2^-24), the two epilogue roundings (2^-24 |o|) and,
    on the wgmma engine (S = conv4_3's storage exponent), the two hi/lo storage roundings (2^-22 |o| + 2^-(25 + S)
    each)."""
    o1, o2 = _d(o_glob), _d(o_plain)
    g = _d(vec)[:, :, None, None]
    sh = bn_shift(sd)[None, :, None, None]
    bar = _d(dvec)[:, :, None, None] + U * (sh + g).abs() + U * (o1.abs() + o2.abs())
    if S is not None:
        bar = bar + 2.0 ** -22 * (o1.abs() + o2.abs()) + 2 * 2.0 ** (-25 - S)
    return bar


# ---------------------------------------------------------------------------------------------------------------------
# peaked class head
# ---------------------------------------------------------------------------------------------------------------------
def peaked(sd, batch, target=100.0, maskcent=0.5):
    """-> a copy of sd with model_class (weight and bias by one factor) scaled so that max |0.2 z| on `batch` =
    (L, ab, mask) is `target`; model_out is left as it is (calibrated.head_gain scales both heads)."""
    L, ab, mask = batch
    out = {k: (v if torch.is_tensor(v) else torch.from_numpy(np.ascontiguousarray(v))) for k, v in sd.items()}
    with torch.no_grad():
        _, inter = lhn_ref.lhn_forward(out, L, ab, mask, maskcent, ref_quirks=False, return_intermediates=True,
                                       dtype=torch.float64)
        z = lhn_ref._conv(out, "model_class.0", inter["conv8_3"])
    g = target / float((0.2 * z).abs().max())
    for k in ("model_class.0.weight", "model_class.0.bias"):
        out[k] = (out[k].double() * g).float()
    return out
