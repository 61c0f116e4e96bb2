"""CPU: the trained-like networks of tests/calibrated.py are what they claim to be, and the storage exponents the
engine picks for them (restated in act_estimates) keep every buffer inside FP16's range."""
import numpy as np
import pytest
import torch

from oracle import lhn_ref, synth
from tests import calibrated

RHOS = [0.0, 0.15, 0.3, 0.6, 1.0]

# DESIGN §3's table: the exponents of the synthetic weights (tools/act_range_table.py)
SYNTH_EXPONENTS = {
    "a1_1": 6, "conv1_2": 6, "a2_1": 5, "conv2_2": 6, "a3_1": 4, "a3_2": -2, "conv3_3": 6, "a4_1": 4, "a4_2": -3,
    "conv4_3": 5, "a5_1": 3, "a5_2": -3, "conv5_3": 6, "a6_1": 3, "a6_2": -3, "conv6_3": 6, "a7_1": 3, "a7_2": -3,
    "conv7_3": 6, "a8_1": 3, "a8_2": -3, "conv8_3": 6, "a9_1": 4, "conv9_3": 6, "a10_1": 4, "conv10_2": -1,
}


@pytest.fixture(scope="module")
def sd0():
    return synth.torch_state_dict(1234)


@pytest.fixture(scope="module")
def cal():
    return synth.synthetic_batch(4, 64, seed=0)


@pytest.fixture(scope="module")
def nets(sd0, cal):
    return {rho: calibrated.trained_like(sd0, rho, cal) for rho in RHOS}


def _inter64(sd, batch, maskcent=0.5):
    with torch.no_grad():
        _, inter = lhn_ref.lhn_forward(sd, *batch, maskcent, ref_quirks=False, return_intermediates=True,
                                       dtype=torch.float64)
    return inter


@pytest.mark.parametrize("rho", [0.0, 0.3])
def test_calibrated_bn_normalises_the_calibration_batch(sd0, cal, rho):
    """Eval-mode BatchNorm with the calibrated statistics: x_hat = (out - beta) / gamma has per-channel mean 0 and
    variance var / (var + eps) on the calibration batch (FP64), for every BatchNorm."""
    sd = calibrated.calibrate_bn(calibrated.coherent(sd0, rho), cal)
    inter = _inter64(sd, cal)
    for bn in calibrated.BN_KEYS:
        out = inter[calibrated.BN_OUT[bn]]
        g, b, v = (sd[bn + s].double() for s in (".weight", ".bias", ".running_var"))
        xh = (out - b[None, :, None, None]) / g[None, :, None, None]
        mean, var = xh.mean(dim=(0, 2, 3)), xh.var(dim=(0, 2, 3), unbiased=False)
        assert float(mean.abs().max()) < 1e-6, (bn, float(mean.abs().max()))
        assert float((var - v / (v + lhn_ref.BN_EPS)).abs().max()) < 1e-6, bn
        assert float(var.max()) > 0.99, bn


def test_coherent_zero_is_the_identity(sd0):
    out = calibrated.coherent(sd0, 0)
    assert set(out) == set(sd0)
    for k, v in sd0.items():
        assert torch.equal(out[k], v), k


def test_coherent_adds_rho_std(sd0):
    out = calibrated.coherent(sd0, 0.5)
    for k in calibrated.COHERENT_KEYS:
        w0, w1 = sd0[k + ".weight"].double(), out[k + ".weight"].double()
        assert float((w1 - w0 - 0.5 * float(w0.std())).abs().max()) < 1e-6 * float(w0.abs().max()), k
    for k in ("model1.0", "model_out.0", "model_class.0"):
        assert torch.equal(out[k + ".weight"], sd0[k + ".weight"])


def test_head_gain_keeps_tanh_unsaturated(nets, cal):
    for rho, sd in nets.items():
        with torch.no_grad():
            _, inter = lhn_ref.lhn_forward(sd, *cal, 0.5, ref_quirks=False, return_intermediates=True,
                                           dtype=torch.float64)
            pre = lhn_ref._conv(sd, "model_out.0", inter["conv10_2"])
            logit = lhn_ref._conv(sd, "model_class.0", inter["conv8_3"]) * 0.2
        assert abs(float(pre.abs().max()) - 1.5) < 1e-5, rho
        assert abs(float(logit.abs().max()) - 1.5) < 1e-5, rho


def test_synthetic_exponents(sd0):
    est = calibrated.act_estimates(sd0)
    assert {b: e[2] for b, e in est.items()} == SYNTH_EXPONENTS
    csd = dict(sd0)
    from oracle import caffe_spec
    csd.update({k: torch.from_numpy(v) for k, v in caffe_spec.synthetic_caffe313_state_dict().items()})
    assert "hyper" in calibrated.act_estimates(csd, caffe313=True)


def test_bound_holds_with_measured_inputs(nets, cal):
    """The 1-norm bound of every conv without a BatchNorm, taken per output-parity class, evaluated with the sources'
    measured max |a| instead of their estimates, is >= the measured max |a| of the output (FP64): the bound is true,
    and the tap selection of the transposed convs' classes is right.  Checked per output channel."""
    for rho in (0.0, 1.0):
        sd = nets[rho]
        inter = _inter64(sd, cal)
        for buf, srcs, bn in calibrated._PLAN:
            if bn or buf == "hyper":
                continue
            acc, bias = 0.0, 0.0
            for key, src, tr in srcs:
                w = calibrated._np64(sd[key + ".weight"])
                m = 1.0 if src is None else float(inter[src].abs().max())
                acc = acc + calibrated._class_l1(w, tr) * m
                bias = bias + calibrated._np64(sd[key + ".bias"])
            bound = (acc + np.abs(bias)[:, None]).max(axis=1)
            got = inter[buf].abs().amax(dim=(0, 2, 3)).numpy()
            assert np.all(got <= bound * (1 + 1e-12)), (rho, buf, float(np.max(got / bound)))
            assert float(np.max(got / bound)) > 0.1 or rho == 0.0, (rho, buf)   # and within 10x on coherent filters


@pytest.mark.parametrize("rho", [0.6, 1.0])
def test_two_norm_estimate_saturates(nets, cal, rho):
    """Guard: these networks are aimed at the limit.  With the exponent chosen from the 2-norm estimate alone, the
    largest stored value of at least one buffer exceeds 65504 (the trained-like filters add up coherently, which the
    2-norm of a filter does not see)."""
    inter = _inter64(nets[rho], cal)
    sm = calibrated.stored_max(inter, calibrated.act_estimates(nets[rho], with_bound=False))
    assert max(sm.values()) > calibrated.FP16_MAX, sm


@pytest.mark.parametrize("rho", RHOS)
def test_exponents_keep_headroom(nets, cal, rho):
    """With the bound, every buffer's largest stored value stays 8x below 65504, on the calibration batch and on a
    batch the network was not calibrated on."""
    est = calibrated.act_estimates(nets[rho])
    for batch in (cal, synth.synthetic_batch(3, 64, seed=1300, max_hints=4)):
        sm = calibrated.stored_max(_inter64(nets[rho], batch), est)
        assert max(sm.values()) < calibrated.FP16_MAX / 8, (rho, max(sm, key=sm.get), max(sm.values()))
