"""Trained-like variants of a state_dict, and the storage exponents the wgmma engine picks for them (test
infrastructure; imports only oracle/).

The synthetic weights of oracle/synth.py differ from a trained checkpoint in two ways that matter for the size of the
activations: the filters are zero-mean i.i.d. Gaussians, whose sums over many inputs cancel, and the BatchNorm running
statistics are random numbers unrelated to the activations.  These helpers remove both:

  * calibrate_bn(sd, batch): every BatchNorm's running_mean / running_var become the FP64 batch statistics of its
    input, in network order, as training leaves them (biased variance, so eval mode reproduces the batch-statistics
    forward exactly; kept as float64 tensors, which the engine and the FP32 oracle round to FP32 alike);
  * coherent(sd, rho): rho * std(W) is added to every trunk, decoder and shortcut filter, so neighbouring inputs add
    up instead of cancelling;
  * head_gain(sd, batch): model_out and model_class are rescaled so that the largest |pre-tanh| and the largest
    |0.2 * logit| on the batch are 1.5; otherwise tanh saturates at +-110 and hides ab errors;
  * act_estimates(sd): the magnitude estimate, the bound and the storage exponent S_b that idc_finalize_weights
    computes for every stored buffer (DESIGN §3), restated in numpy.
"""
import numpy as np
import torch

from oracle import lhn_ref, synth

# every filter of the trunk, the decoder and the shortcuts; not the input layer or the two heads
COHERENT_KEYS = [k for k, *_ in synth.CONV_LAYERS if k not in ("model1.0", "model_out.0", "model_class.0")]

# The plan of the engine: (output buffer, [(weight key, source buffer, transposed)], BatchNorm key or None), in plan
# order.  Source None is the packed conv1_1 input, magnitude 1.
_PLAN = [
    ("a1_1", [("model1.0", None, False)], None),
    ("conv1_2", [("model1.2", "a1_1", False)], "model1.4"),
    ("a2_1", [("model2.0", "conv1_2", False)], None),
    ("conv2_2", [("model2.2", "a2_1", False)], "model2.4"),
    ("a3_1", [("model3.0", "conv2_2", False)], None),
    ("a3_2", [("model3.2", "a3_1", False)], None),
    ("conv3_3", [("model3.4", "a3_2", False)], "model3.6"),
    ("a4_1", [("model4.0", "conv3_3", False)], None),
    ("a4_2", [("model4.2", "a4_1", False)], None),
    ("conv4_3", [("model4.4", "a4_2", False)], "model4.6"),
    ("a5_1", [("model5.0", "conv4_3", False)], None),
    ("a5_2", [("model5.2", "a5_1", False)], None),
    ("conv5_3", [("model5.4", "a5_2", False)], "model5.6"),
    ("a6_1", [("model6.0", "conv5_3", False)], None),
    ("a6_2", [("model6.2", "a6_1", False)], None),
    ("conv6_3", [("model6.4", "a6_2", False)], "model6.6"),
    ("a7_1", [("model7.0", "conv6_3", False)], None),
    ("a7_2", [("model7.2", "a7_1", False)], None),
    ("conv7_3", [("model7.4", "a7_2", False)], "model7.6"),
    ("a8_1", [("model8up.0", "conv7_3", True), ("model3short8.0", "conv3_3", False)], None),
    ("a8_2", [("model8.1", "a8_1", False)], None),
    ("conv8_3", [("model8.3", "a8_2", False)], "model8.5"),
    ("hyper", [("caffe.conv%d_pred" % l, "conv%d_3" % l, True) for l in (4, 5, 6, 7)]
     + [("caffe.conv3_pred", "conv3_3", False), ("caffe.conv8_pred", "conv8_3", False)], None),
    ("a9_1", [("model9up.0", "conv8_3", True), ("model2short9.0", "conv2_2", False)], None),
    ("conv9_3", [("model9.1", "a9_1", False)], "model9.3"),
    ("a10_1", [("model10up.0", "conv9_3", True), ("model1short10.0", "conv1_2", False)], None),
    ("conv10_2", [("model10.1", "a10_1", False)], None),
]
BN_KEYS = [k for k, _ in synth.BN_LAYERS]
BN_OUT = {bn: buf for buf, _, bn in _PLAN if bn}          # BN key -> the buffer it produces
ACT_EXP_REF = 7                                           # kActExpRef
BOUND_EXP_REF = 11                                        # kActExpBound
FP16_MAX = 65504.0


def _np64(v):
    """A tensor as the engine holds it (idc_load_tensor keeps FP32), in float64."""
    return (v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)).astype(np.float32).astype(np.float64)


def _as_torch(sd):
    return {k: (v if torch.is_tensor(v) else torch.from_numpy(np.ascontiguousarray(v))) for k, v in sd.items()}


def calibrate_bn(sd, batch, maskcent=0.5):
    """-> a copy of sd whose BatchNorm running statistics are the FP64 batch statistics of each BN's input on `batch`
    = (L, ab, mask), taken in network order (each BN's input already sees the calibrated BNs before it)."""
    L, ab, mask = batch
    stats = {}
    with torch.no_grad():
        lhn_ref.lhn_forward(sd, L, ab, mask, maskcent, ref_quirks=False, dtype=torch.float64, batch_stats=stats)
    out = _as_torch(sd)
    for key, (mean, var) in stats.items():
        out[key + ".running_mean"] = mean           # float64: the FP64 oracle sees the exact statistics
        out[key + ".running_var"] = var
    return out


def coherent(sd, rho):
    """-> a copy of sd with rho * std(W) added to every element of the trunk, decoder and shortcut filters."""
    out = _as_torch(sd)
    if rho == 0:
        return out
    for k in COHERENT_KEYS:
        w = out[k + ".weight"].double()
        out[k + ".weight"] = (w + rho * float(w.std())).float()
    return out


def head_gain(sd, batch, maskcent=0.5, target=1.5):
    """-> a copy of sd with model_out scaled so that max |pre-tanh| on `batch` is `target`, and model_class scaled so
    that max |0.2 * logit| is `target` (weight and bias by the same factor)."""
    L, ab, mask = batch
    out = _as_torch(sd)
    with torch.no_grad():
        _, inter = lhn_ref.lhn_forward(out, L, ab, mask, maskcent, ref_quirks=False, return_intermediates=True,
                                       dtype=torch.float64)
        pre = lhn_ref._conv(out, "model_out.0", inter["conv10_2"])
        logit = lhn_ref._conv(out, "model_class.0", inter["conv8_3"]) * 0.2
    for key, m in (("model_out.0", float(pre.abs().max())), ("model_class.0", float(logit.abs().max()))):
        g = target / m
        out[key + ".weight"] = (out[key + ".weight"].double() * g).float()
        out[key + ".bias"] = (out[key + ".bias"].double() * g).float()
    return out


def trained_like(sd, rho, batch, maskcent=0.5):
    """coherent(rho), then calibrate_bn and head_gain on `batch`: the network the calibrated tests run."""
    return head_gain(calibrate_bn(coherent(sd, rho), batch, maskcent), batch, maskcent)


def _ceil_log2(est):
    m, e = np.frexp(est)
    return int(e - 1) if m == 0.5 else int(e)


def exponent(est):
    """S_b = kActExpRef - ceil(log2 est_b) (kActExpRef for est 0)."""
    return ACT_EXP_REF if est <= 0 else ACT_EXP_REF - _ceil_log2(est)


def _class_l1(w, transposed):
    """[cout, classes]: sum of |w| over the inputs and the taps that reach an output pixel of each output-parity class.
    A 3x3 conv has one class (all 9 taps); a 4x4 stride-2 transposed conv has four, each a 2x2 sub-kernel
    (oy = 2 iy - 1 + ky: even rows take ky in {1, 3}, odd rows ky in {0, 2})."""
    a = np.abs(w)
    if not transposed:
        return a.sum(axis=(1, 2, 3))[:, None]                           # [cout, cin, k, k]
    taps = ((1, 3), (0, 2))
    return np.stack([a[:, :, taps[py]][:, :, :, taps[px]].sum(axis=(0, 2, 3))      # [cin, cout, 4, 4]
                     for py in (0, 1) for px in (0, 1)], axis=1)


def act_estimates(sd, caffe313=False, with_bound=True):
    """-> {buffer: (est, bound, S)} for every buffer the engine can store (conv10_2 as stored with keep_conv10; hyper
    with caffe313), computed as idc_finalize_weights computes them (DESIGN §3):
      * a BatchNorm output: est = bound = max_c |gamma_c| sqrt(var_c + mean_c^2) / sqrt(var_c + eps) + |beta_c|,
        S = 7 - ceil(log2 est);
      * any other conv output: est = max_c sum_s ||W_s[c]||_2 * est(s) + |sum_s bias_s[c]| (a typical size), and
        bound = the max over output channels c and output-parity classes of sum_s ||W_s[c, class]||_1 * bound(s) +
        |sum_s bias_s[c]| (a true bound while the BatchNorm outputs stay within their estimates);
        S = min(7 - ceil(log2 est), 11 - ceil(log2 bound)).
    The packed conv1_1 input counts as magnitude 1.  with_bound=False: S from est alone (the 2-norm rule, which
    trained-like networks exceed by far more than FP16's headroom)."""
    out = {}
    for buf, srcs, bn in _PLAN:
        if buf == "hyper" and not caffe313:
            continue
        if bn:
            g, b, m, v = (_np64(sd[bn + s]) for s in (".weight", ".bias", ".running_mean", ".running_var"))
            est = bound = float(np.max(np.abs(g) * np.sqrt(v + m * m) / np.sqrt(v + lhn_ref.BN_EPS) + np.abs(b)))
            s = exponent(est)
        else:
            l2, l1, bias = 0.0, 0.0, 0.0
            for key, src, tr in srcs:
                w = _np64(sd[key + ".weight"])
                n2 = np.sqrt((w ** 2).sum(axis=(0, 2, 3) if tr else (1, 2, 3)))
                l2 = l2 + n2 * (1.0 if src is None else out[src][0])
                l1 = l1 + _class_l1(w, tr) * (1.0 if src is None else out[src][1])
                bias = bias + _np64(sd[key + ".bias"])
            est = float(np.max(l2 + np.abs(bias)))
            bound = float(np.max(l1 + np.abs(bias)[:, None]))
            s = exponent(est)
            if with_bound:
                s = min(s, BOUND_EXP_REF - _ceil_log2(bound))
        out[buf] = (est, bound, s)
    return out


def stored_max(inter, est):
    """{buffer: max |a| * 2^S_b}: the largest value the FP16 hi plane of each buffer would hold."""
    return {b: float(inter[b].abs().max()) * 2.0 ** e[-1] for b, e in est.items() if b in inter}
