"""FP64 reference of every op of the Local Hints Network, one op at a time (test infrastructure; imports only oracle/ and
tests/).

Each op is evaluated in float64 from the input activations it is given, wired as oracle/lhn_ref.py wires the network:
3x3 convs (dilated in blocks 5 and 6, on the ::2-decimated input at the first conv of blocks 2-4), the 4x4 stride-2
transposed convs of the decoder plus their 3x3 shortcut, bias, ReLU / LeakyReLU(0.2) and eval-mode BatchNorm.  conv1_1
takes L, ab, mask and maskcent and applies the input pack cat(L/100, ab/110, mask - maskcent) itself.

Two operand modes:
  * "exact": the operands as given, in float64.  Chained, the ops reproduce lhn_forward(..., dtype=torch.float64).
  * "fp16": the operands IDC_FLAG_FAST_FP16 feeds the tensor core, held exactly in float64:
      - an input buffer b is fp16-RN(a * 2^S_b) (S_b = the context's act_exponent(b), FP16 subnormals kept);
      - a weight of source s is w * 2^(S_0 - S_s) (ops with several sources share source 0's accumulator scale), times
        the per-output-channel 2^e that puts the channel's largest such weight in [256, 512), rounded to fp16-RN
        (idc_finalize_weights; conv1_1: conv1_1_pack_kernel, without the clamp of e to [-24, 24]);
      - conv1_1's input is the correctly rounded FP32 L/100, ab/110 and mask - maskcent at the fixed 2^6 (kInExp);
      - the parameters are the FP32 values the engine holds.
    The products are summed in float64 and the epilogue is applied in float64, so what is left between the engine and
    this reference is the engine's accumulation, its FP32 epilogue and the final FP16 rounding of the stored value.

Every op returns (out, mag): out is the value before any storage rounding, mag bounds the size of the terms the engine
adds per element, in output units: |BN scale| * (sum |a*w| + |bias|) + |BN beta| + |BN mean * BN scale| (no BN: scale 1,
the last two 0).  An accumulation error of c units in the last place of FP32 is then at most c * 2^-24 * mag.
"""
import functools

import numpy as np
import torch
import torch.nn.functional as F

from oracle import lhn_ref

IN_EXP = 6          # kInExp: conv1_1's packed input is stored x 2^6
W_TOP = 9           # the largest scaled weight of an output channel is in [2^8, 2^9)
FP16_MAX = 65504.0

# op -> (output buffer, [(weight key, source buffer, kind, dilation)], activation, BatchNorm key).  kind: "conv" 3x3,
# "sub" 3x3 on the source's [:, :, ::2, ::2], "deconv" 4x4 stride-2 transposed conv.  Source 0 is the engine's source 0.
SPEC = {
    "c1_2": ("conv1_2", [("model1.2", "a1_1", "conv", 1)], "relu", "model1.4"),
    "c2_1": ("a2_1", [("model2.0", "conv1_2", "sub", 1)], "relu", None),
    "c2_2": ("conv2_2", [("model2.2", "a2_1", "conv", 1)], "relu", "model2.4"),
    "c3_1": ("a3_1", [("model3.0", "conv2_2", "sub", 1)], "relu", None),
    "c3_2": ("a3_2", [("model3.2", "a3_1", "conv", 1)], "relu", None),
    "c3_3": ("conv3_3", [("model3.4", "a3_2", "conv", 1)], "relu", "model3.6"),
    "c4_1": ("a4_1", [("model4.0", "conv3_3", "sub", 1)], "relu", None),
    "c4_2": ("a4_2", [("model4.2", "a4_1", "conv", 1)], "relu", None),
    "c4_3": ("conv4_3", [("model4.4", "a4_2", "conv", 1)], "relu", "model4.6"),
    "c5_1": ("a5_1", [("model5.0", "conv4_3", "conv", 2)], "relu", None),
    "c5_2": ("a5_2", [("model5.2", "a5_1", "conv", 2)], "relu", None),
    "c5_3": ("conv5_3", [("model5.4", "a5_2", "conv", 2)], "relu", "model5.6"),
    "c6_1": ("a6_1", [("model6.0", "conv5_3", "conv", 2)], "relu", None),
    "c6_2": ("a6_2", [("model6.2", "a6_1", "conv", 2)], "relu", None),
    "c6_3": ("conv6_3", [("model6.4", "a6_2", "conv", 2)], "relu", "model6.6"),
    "c7_1": ("a7_1", [("model7.0", "conv6_3", "conv", 1)], "relu", None),
    "c7_2": ("a7_2", [("model7.2", "a7_1", "conv", 1)], "relu", None),
    "c7_3": ("conv7_3", [("model7.4", "a7_2", "conv", 1)], "relu", "model7.6"),
    "up8": ("a8_1", [("model8up.0", "conv7_3", "deconv", 1), ("model3short8.0", "conv3_3", "conv", 1)], "relu", None),
    "c8_2": ("a8_2", [("model8.1", "a8_1", "conv", 1)], "relu", None),
    "c8_3": ("conv8_3", [("model8.3", "a8_2", "conv", 1)], "relu", "model8.5"),
    "up9": ("a9_1", [("model9up.0", "conv8_3", "deconv", 1), ("model2short9.0", "conv2_2", "conv", 1)], "relu", None),
    "c9_2": ("conv9_3", [("model9.1", "a9_1", "conv", 1)], "relu", "model9.3"),
    "up10": ("a10_1", [("model10up.0", "conv9_3", "deconv", 1), ("model1short10.0", "conv1_2", "conv", 1)], "relu",
             None),
    "c10_2": ("conv10_2", [("model10.1", "a10_1", "conv", 1)], "leaky", None),
}
MODES = ("exact", "fp16")


def f16(x):
    """float64 tensor -> fp16 round-to-nearest-even of every element, as float64 (subnormals kept; beyond 65504 the
    result is the unsaturated rounding, which callers check against FP16_MAX)."""
    x = x.double()
    u = ulp16(x)
    return torch.round(x / u) * u                   # x / ulp is exact; torch.round rounds half to even


def pow2(q):
    """Integer-valued tensor q -> 2^q in float64, built from the exponent bits: exact on every device (a library pow
    need not be; |q| <= 1022)."""
    return ((q.long() + 1023) << 52).view(torch.float64)


def ulp16(x):
    """The fp16 ulp of the binade of every element of x (2^-24 in the subnormal range), float64."""
    _, e = torch.frexp(x.double())                  # |x| = m * 2^e, m in [0.5, 1): the binade's exponent is e - 1
    return pow2(torch.clamp(e - 1, min=-14) - 10)


def _fp32(x):
    """float64 -> the nearest FP32 value, as float64."""
    return x.double().float().double()


def _param(sd, key, mode, device):
    v = sd[key]
    t = v if torch.is_tensor(v) else torch.from_numpy(np.ascontiguousarray(v))
    t = t.to(device)
    return _fp32(t) if mode == "fp16" else t.double()


def _chan_exp(mx):
    """[cout] largest |weight| -> the e with mx * 2^e in [256, 512) (e = 0 for an all-zero channel)."""
    _, ex = torch.frexp(mx)
    return torch.where(mx > 0, W_TOP - ex, torch.zeros_like(ex))


def _apply(kind, dil, a, w):
    if kind == "deconv":
        return F.conv_transpose2d(a, w, stride=2, padding=1)
    if kind == "sub":
        a = a[:, :, ::2, ::2]
    return F.conv2d(a, w, padding=dil * (w.shape[-1] // 2), dilation=dil)


def _epilogue(sd, t, mag, bias, act, bn, mode):
    """act(t + bias), then BatchNorm; and the magnitude bound in output units."""
    dev = t.device
    t = t + bias[None, :, None, None]
    mag = mag + bias.abs()[None, :, None, None]
    t = F.relu(t) if act == "relu" else F.leaky_relu(t, 0.2)
    if bn is None:
        return t, mag
    g, b, m, v = (_param(sd, bn + s, mode, dev) for s in (".weight", ".bias", ".running_mean", ".running_var"))
    out = F.batch_norm(t, m, v, g, b, False, 0.0, lhn_ref.BN_EPS)
    gs = (g / torch.sqrt(v + lhn_ref.BN_EPS))
    mag = gs.abs()[None, :, None, None] * mag + (b.abs() + (m * gs).abs())[None, :, None, None]
    return out, mag


def run_op(name, sd, acts, mode="exact", exps=None):
    """One op of SPEC on the input activations `acts` ({buffer: [n, C, H, W] tensor}, any float dtype, CPU or GPU).
    mode "fp16" needs exps = {buffer: storage exponent} for the op's sources.  -> (out, mag), float64."""
    assert mode in MODES
    out_buf, srcs, act, bn = SPEC[name]
    dev = acts[srcs[0][1]].device
    ws, xs = [], []
    for key, src, kind, dil in srcs:
        ws.append(_param(sd, key + ".weight", mode, dev))
        a = acts[src].double()
        if mode == "fp16":
            a = f16(_fp32(a) * 2.0 ** exps[src]) * 2.0 ** -exps[src]
        xs.append(a)
    if mode == "fp16":
        # one power-of-two scale per output channel over all sources, after source s is put at source 0's exponent
        mul = [2.0 ** (exps[srcs[0][1]] - exps[src]) for _, src, _, _ in srcs]
        co_dim = [1 if kind == "deconv" else 0 for _, _, kind, _ in srcs]
        mx = torch.stack([(w * m).abs().transpose(0, d).reshape(w.shape[d], -1).max(dim=1).values
                          for w, m, d in zip(ws, mul, co_dim)]).max(dim=0).values
        e = torch.clamp(_chan_exp(mx), -24, 24)
        for i, (w, m, d) in enumerate(zip(ws, mul, co_dim)):
            sc = pow2(e).reshape([-1 if j == d else 1 for j in range(4)]) * m
            ws[i] = f16(w * sc) / sc
    val = mag = 0.0
    for (key, src, kind, dil), a, w in zip(srcs, xs, ws):
        val = val + _apply(kind, dil, a, w)
        mag = mag + _apply(kind, dil, a.abs(), w.abs())
    bias = sum(_param(sd, key + ".bias", mode, dev) for key, *_ in srcs)
    return _epilogue(sd, val, mag, bias, act, bn, mode)


OPS = {name: functools.partial(run_op, name) for name in SPEC}


def conv1_1(sd, L, ab, mask, maskcent=0.0, mode="exact"):
    """The input pack cat(L/100, ab/110, mask - maskcent) and model1.0 + ReLU -> (a1_1, mag), float64.
    mode "fp16": the operands of conv1_1_umma_kernel<false>."""
    assert mode in MODES
    L, ab, mask = (torch.as_tensor(x) for x in (L, ab, mask))
    dev = L.device
    w = _param(sd, "model1.0.weight", mode, dev)
    if mode == "exact":
        x = torch.cat((L.double() / 100.0, ab.double() / 110.0, mask.double() - maskcent), dim=1)
    else:
        # the kernel's x / 100 and x / 110 are correctly rounded FP32 quotients (a float64 quotient rounded to FP32 is
        # one); mask - maskcent is one FP32 subtraction
        mc = float(np.float32(maskcent))
        x = torch.cat((_fp32(_fp32(L) / 100.0), _fp32(_fp32(ab) / 110.0), _fp32(_fp32(mask) - mc)), dim=1)
        x = f16(x * 2.0 ** IN_EXP) / 2.0 ** IN_EXP
        sc = pow2(_chan_exp(w.abs().reshape(64, -1).max(dim=1).values))[:, None, None, None]
        w = f16(w * sc) / sc
    val = F.conv2d(x, w, padding=1)
    mag = F.conv2d(x.abs(), w.abs(), padding=1)
    return _epilogue(sd, val, mag, _param(sd, "model1.0.bias", mode, dev), "relu", None, mode)


def chain(sd, L, ab, mask, maskcent=0.0):
    """conv1_1 and every op of SPEC in network order, each fed the previous outputs -> {buffer: tensor}, float64:
    the exact-mode ops chained, which is lhn_forward in float64."""
    acts = {"a1_1": conv1_1(sd, L, ab, mask, maskcent)[0]}
    for name, (out, *_) in SPEC.items():
        acts[out] = run_op(name, sd, acts)[0]
    return acts
