"""CPU: the FP64 heads of tests/head_ref.py and their bounds.  The heads equal the FP64 oracle's (lhn_forward in
float64: out_reg, dist64 and the glob_add path), every bound is >= 0 and grows with the magnitudes it covers, the peaked
network reaches FP32 underflow, and the pmf interval applies the subnormal rule at 2^-150, 2^-149 and FLT_MIN."""
import numpy as np
import pytest
import torch

from oracle import caffe_spec, lhn_ref, synth
from tests import head_ref, util


@pytest.fixture(scope="module")
def batch():
    return util.small_batch(2, 32, seed=41)


@pytest.fixture(scope="module")
def fp64(synth_sd, batch):
    with torch.no_grad():
        (reg, dist), inter = lhn_ref.lhn_forward(synth_sd, *batch, 0.5, dist=True, ref_quirks=False,
                                                 return_intermediates=True, dtype=torch.float64)
    return reg, dist, inter


def test_regression_head_is_the_oracle(synth_sd, fp64):
    reg, _, inter = fp64
    for scale in (110.0, 100.0):
        a, bound = head_ref.reg_from_a10_1(synth_sd, inter["a10_1"], scale)
        b, bound_c = head_ref.reg_from_conv10(synth_sd, inter["conv10_2"], scale)
        want = reg * (scale / 110.0)
        assert util.maxabs(a, want) <= 1e-12 * scale and util.maxabs(b, want) <= 1e-12 * scale
        assert bool((bound >= 0).all()) and bool((bound_c >= 0).all())
        assert bool((bound >= bound_c).all())          # the fused head's bound adds c10_2's own error


def test_distribution_head_is_the_oracle(synth_sd, fp64):
    _, dist, inter = fp64
    ref = head_ref.dist_head(synth_sd, inter["conv8_3"])
    assert util.maxabs(ref["p64"], dist) <= 1e-15
    assert bool((ref["lo"] <= ref["p64"]).all()) and bool((ref["p64"] <= ref["hi"]).all())
    assert bool((ref["logbound"] > 0).all()) and 0 < ref["sum_bound"] < 1e-5
    # the FP32 rounding of p64 itself lies inside the interval
    p32 = head_ref.rn32(ref["p64"])
    assert bool(((ref["lo"] <= p32) & (p32 <= ref["hi"])).all())
    simt = head_ref.dist_head(synth_sd, inter["conv8_3"], engine="simt")
    assert bool((simt["lo"] <= ref["lo"]).all()) and bool((simt["hi"] >= ref["hi"]).all())


def test_glob_path_is_the_oracle(synth_sd, batch):
    gsd = caffe_spec.synthetic_glob_state_dict()
    glob_ab, sat = synth.synthetic_glob(2, seed=3)
    glob = np.concatenate([glob_ab, sat], axis=1)
    vec, dvec = head_ref.glob_vector(gsd, glob)
    assert bool((dvec > 0).all())
    with torch.no_grad():
        _, inter = lhn_ref.lhn_forward(synth_sd, *batch, 0.5, glob_add=vec, ref_quirks=False,
                                       return_intermediates=True, dtype=torch.float64)
    out, mag = head_ref.c4_3_glob(synth_sd, inter["a4_2"], vec)
    assert util.maxabs(out, inter["conv4_3"]) <= 1e-12 * float(inter["conv4_3"].abs().max())
    assert bool((mag >= 0).all())
    plain = out - vec[:, :, None, None]
    bar = head_ref.glob_diff_bound(synth_sd, out, plain, vec, dvec, S=7)
    assert bool((bar > 0).all())


def test_bounds_grow_with_magnitude(synth_sd, fp64):
    """Doubling the operand doubles the magnitudes: the unsaturated bounds grow."""
    _, _, inter = fp64
    v = inter["conv10_2"]
    _, b1 = head_ref.reg_head(synth_sd, v * 1e-3)
    _, b2 = head_ref.reg_head(synth_sd, v * 2e-3)
    assert bool((b2 > b1).all())
    r1 = head_ref.dist_head(synth_sd, inter["conv8_3"] * 1e-2)
    r2 = head_ref.dist_head(synth_sd, inter["conv8_3"] * 2e-2)
    assert bool((r2["logbound"] > r1["logbound"]).all())
    gsd = caffe_spec.synthetic_glob_state_dict()
    glob = np.concatenate(synth.synthetic_glob(1, seed=4), axis=1)
    _, d1 = head_ref.glob_vector(gsd, glob * 0.5)
    _, d2 = head_ref.glob_vector(gsd, glob)
    assert float(d2.sum()) > float(d1.sum())


def test_peaked_network_reaches_underflow(synth_sd):
    b = util.small_batch(2, 64, seed=300)
    sd = head_ref.peaked(synth_sd, b, 100.0)
    for k in ("model_out.0.weight", "model_out.0.bias"):
        assert torch.equal(torch.as_tensor(sd[k]), torch.as_tensor(synth_sd[k])), k
    with torch.no_grad():
        _, inter = lhn_ref.lhn_forward(sd, *b, 0.5, ref_quirks=False, return_intermediates=True, dtype=torch.float64)
    z, _ = head_ref.class_logits(sd, inter["conv8_3"])
    assert abs(float((0.2 * z).abs().max()) - 100.0) < 1e-3
    ref = head_ref.dist_head(sd, inter["conv8_3"])
    n_zero, n_sub = int((ref["hi"] == 0).sum()), int(((ref["lo"] > 0) & (ref["hi"] < head_ref.FLT_MIN)).sum())
    print("peaked 64^2: %d bins must be 0, %d must be subnormal, of %d" % (n_zero, n_sub, ref["p64"].numel()))
    assert n_zero > 0 and n_sub > 0


def _one_bin(logit_gap):
    """A two-level pmf: bin 0 at z = 0 and the other 528 at z = -logit_gap / 0.2, on a 1x1 'conv8_3' through an
    identity class head -> dist_head's dict."""
    sd = {"model_class.0.weight": torch.zeros(529, 256, 1, 1, dtype=torch.float64),
          "model_class.0.bias": torch.full((529,), -logit_gap / 0.2, dtype=torch.float64)}
    sd["model_class.0.bias"][0] = 0.0
    return head_ref.dist_head(sd, torch.zeros(1, 256, 1, 1, dtype=torch.float64))


def test_subnormal_rule_at_the_edges():
    """p64 of the small bins = exp(-gap) / (1 + 528 exp(-gap)) ~ exp(-gap), put at 2^-150, 2^-149 and FLT_MIN and
    just either side: clearly below 2^-150 -> must be 0; at 2^-150 (the rounding tie, ties to even: 0) and within the
    bound of it -> may be 0; clearly above 2^-149 -> must not be 0; at FLT_MIN -> a normal FP32 value, exact bounds."""
    ln2 = np.log(2.0)
    for e, must_zero, may_zero in ((152, True, True), (150, False, True), (148.5, False, False),
                                   (126, False, False)):
        r = _one_bin(e * ln2)
        p, lo, hi = float(r["p64"][0, 1]), float(r["lo"][0, 1]), float(r["hi"][0, 1])
        assert abs(np.log2(p) + e) < 1e-6, (e, p)
        assert (hi == 0) == must_zero, (e, lo, hi)
        assert (lo == 0) == may_zero, (e, lo, hi)
    # p64 ~ FLT_MIN: both ends are normal FP32 values, within the log-space bound (and the final rounding) of p64
    r = _one_bin(126 * ln2 - 1e-3)
    p, lo, hi, lb = (float(r[k][0, 1]) for k in ("p64", "lo", "hi", "logbound"))
    assert head_ref.FLT_MIN <= lo < p < hi, (lo, p, hi)
    assert lo >= p * np.exp(-lb) * (1 - 2.0 ** -23) and hi <= p * np.exp(lb) * (1 + 2.0 ** -23), (lo, p, hi, lb)
    # a value below the smallest subnormal at the tie: RN(2^-150) = 0, RN(2^-150 (1 + 2^-20)) = 2^-149
    t = torch.tensor([2.0 ** -150, 2.0 ** -150 * (1 + 2.0 ** -20), 2.0 ** -149 * 1.49, 2.0 ** -149 * 1.51],
                     dtype=torch.float64)
    assert head_ref.rn32(t).tolist() == [0.0, 2.0 ** -149, 2.0 ** -149, 2.0 ** -148]


def _softmax529_row_fp32(z):
    """softmax529_row restated in float32 on logits z [P,529] (float64): y = z * 0.2f, the max, t = y - max, exp
    correctly rounded (within expf's 2 ulp), 17-term lane sums then the 5-step butterfly, 1 / sum, the products."""
    y = (z.astype(np.float32) * np.float32(0.2)).astype(np.float32)
    t = (y - y.max(axis=1, keepdims=True)).astype(np.float32)
    e = np.exp(t.astype(np.float64)).astype(np.float32)
    pad = np.zeros((z.shape[0], 17 * 32), np.float32)
    pad[:, :529] = e
    lanes = np.zeros((z.shape[0], 32), np.float32)
    for j in range(17):
        lanes = (lanes + pad[:, 32 * j:32 * j + 32]).astype(np.float32)
    for o in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[:, np.arange(32) ^ o]).astype(np.float32)
    inv = (np.float32(1.0) / lanes[:, :1]).astype(np.float32)
    return (e * inv).astype(np.float32)


@pytest.mark.parametrize("net", ["synthetic", "rho0.3"])
def test_interval_holds_fp32_softmax_with_logit_errors(synth_sd, net):
    """An FP32 softmax529_row fed FP32 logits off by the full C_CLS budget lies in dist_head's interval, bin for bin,
    including the zero and subnormal bins of a peaked head: the largest logit moved by +-dz alone (an error of the
    max, common to every t_j, which the subnormal rounding does not cancel) and every logit moved by +-dz at random."""
    from tests import calibrated, gpu_cases
    b = util.small_batch(2, 64, seed=300)
    base = synth_sd if net == "synthetic" else calibrated.trained_like(synth_sd, 0.3, gpu_cases.calibration_batch())
    sd = head_ref.peaked(base, b, 100.0)
    with torch.no_grad():
        _, inter = lhn_ref.lhn_forward(sd, *b, 0.5, ref_quirks=False, return_intermediates=True)
    a = inter["conv8_3"].double()
    ref = head_ref.dist_head(sd, a)
    z, mag = head_ref.class_logits(sd, a)
    z = z.numpy()
    # the logit error budget, less the rounding of the perturbed logit to FP32 that the emulation adds on top
    dz = (head_ref.C_CLS["wgmma"] * head_ref.U * mag).numpy()
    dz = dz - head_ref.U * (np.abs(z) + dz)
    flat = lambda x: x.transpose(0, 2, 3, 1).reshape(-1, 529)
    lo, hi = flat(ref["lo"].numpy()), flat(ref["hi"].numpy())
    top = np.argmax(z, axis=1)[:, None]
    rs = np.random.RandomState(1)
    shifts = [np.where(np.arange(529)[None, :, None, None] == top, s * dz, 0.0) for s in (1, -1)]
    shifts.append(rs.choice([-1.0, 1.0], z.shape) * dz)
    for k, dlt in enumerate(shifts):
        p = _softmax529_row_fp32(flat(z + dlt)).astype(np.float64)
        bad = int(((p < lo) | (p > hi)).sum())
        assert bad == 0, (net, k, bad)
    assert int((ref["hi"] == 0).sum()) > 0 and int(((ref["lo"] > 0) & (ref["hi"] < head_ref.FLT_MIN)).sum()) > 0
