"""Calibrated storage exponents restated in numpy, and a network that needs them (test infrastructure; imports only
oracle/ and tests/calibrated.py).

With a measured range the wgmma engine stores buffer b with S_b = kActExpCal - ceil(log2 max_abs) (DESIGN §3); an
act_exp.<buffer> override wins over a range, and a buffer without a range keeps the weight-derived exponent of
tests/calibrated.act_estimates.
"""
import torch

from oracle import lhn_ref
from tests import calibrated

ACT_EXP_CAL = 10                    # kActExpCal
ACT_EXP_MIN, ACT_EXP_MAX = -24, 24  # kActExpMin, kActExpMax


def exponent_from_range(max_abs):
    """S = kActExpCal - ceil(log2 max_abs): the measured maximum is stored in (2^(kActExpCal-1), 2^kActExpCal]."""
    return ACT_EXP_CAL - calibrated._ceil_log2(max_abs)


def expected_exponents(sd, ranges=None, overrides=None, caffe313=False):
    """{buffer: S} for every buffer the engine can store: override, else measured range (> 0), else the estimate."""
    out = {}
    for b, (_, _, s) in calibrated.act_estimates(sd, caffe313=caffe313).items():
        if ranges and ranges.get(b, 0) > 0:
            s = exponent_from_range(ranges[b])
        if overrides and b in overrides:
            s = overrides[b]
        out[b] = s
    return out


STALE_BUFFER = "conv4_3"
STALE_SHIFT = 12


def stale_statistics(sd, batch=None, maskcent=0.5):
    """-> a copy of sd whose conv4_3 BatchNorm sees inputs 2^12 times larger than its running statistics say: the conv
    feeding it (model4.4, weight and bias) times 2^12, the statistics untouched, and the consumers of conv4_3 (model5.0,
    caffe.conv4_pred where present) times 2^-12, so conv4_3 is ~4000x its weight-derived estimate.
    conv4_3 is then no longer centred (4096 * scale * relu(x) + shift), which leaves every BatchNorm after it with
    statistics of a distribution it no longer sees and the heads with a gain fitted to another network.  With `batch`
    = (L, ab, mask) the rest of the network is brought back to a sane function, as training would leave it: the
    BatchNorms after model4.6 get the FP64 statistics of their inputs on the batch, in network order, and the heads
    are rescaled (calibrated.head_gain).  Only model4.6 stays stale."""
    out = dict(sd)
    for key in ("model4.4.weight", "model4.4.bias"):
        out[key] = torch.as_tensor(out[key]) * 2.0 ** STALE_SHIFT
    for key in ("model5.0.weight", "caffe.conv4_pred.weight"):
        if key in out:
            out[key] = torch.as_tensor(out[key]) * 2.0 ** -STALE_SHIFT
    if batch is None:
        return out
    later = calibrated.BN_KEYS[calibrated.BN_KEYS.index("model4.6") + 1:]
    for bn in later:
        # the BatchNorm's input statistics from its output y = (x - m) * g / sqrt(v + eps) + b, inverted per channel
        with torch.no_grad():
            _, inter = lhn_ref.lhn_forward(out, *batch, maskcent, ref_quirks=False, return_intermediates=True,
                                           dtype=torch.float64)
        y = inter[calibrated.BN_OUT[bn]]
        g, b, m, v = (torch.as_tensor(out[bn + k]).double() for k in (".weight", ".bias", ".running_mean", ".running_var"))
        k = torch.sqrt(v + lhn_ref.BN_EPS) / g
        out[bn + ".running_mean"] = (y.mean(dim=(0, 2, 3)) - b) * k + m
        out[bn + ".running_var"] = y.var(dim=(0, 2, 3), unbiased=False) * k * k
    return calibrated.head_gain(out, batch, maskcent)
