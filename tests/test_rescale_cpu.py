"""CPU: the power-of-two rescaled twins of tests/rescale.py compute the same network.  Checked in float64 through the
oracle: the twin's outputs equal the original's and every intermediate is exactly 2^k times the original's, to 1e-12
relative.  The GPU tests (test_gpu_act_range.py) rely on this to demand bit-identical engine outputs."""
import numpy as np
import pytest
import torch

from oracle import caffe_spec, lhn_ref, synth
from tests import rescale, util

TOL = 1e-12
F64 = torch.float64


@pytest.fixture(scope="module")
def full_sd(synth_sd):
    """The synthetic network plus the global-hints MLP and the Caffe 313-bin head."""
    sd = dict(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in caffe_spec.synthetic_glob_state_dict().items()})
    sd.update({k: torch.from_numpy(v) for k, v in
               caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=util.golden("pts_in_hull.npy")).items()})
    return sd


@pytest.fixture(scope="module")
def batch():
    L, ab, m = synth.synthetic_batch(2, 32, seed=41, max_hints=4)
    glob_ab, sat = synth.synthetic_glob(2, seed=5)
    return L, ab, m, np.concatenate([glob_ab, sat], axis=1).astype(np.float32)


def _forward(sd, batch, glob):
    L, ab, m, g316 = batch
    with torch.no_grad():
        gvec = caffe_spec.global_hints_vector(sd, g316, dtype=F64) if glob else None
        (reg, dist), inter = lhn_ref.lhn_forward(sd, L, ab, m, 0.5, dist=True, glob_add=gvec, ref_quirks=False,
                                                  return_intermediates=True, dtype=F64)
        pred, dist_s, logits, hyper = caffe_spec.caffe313_head(sd, inter, return_logits=True, dtype=F64)
    inter.update({"out_reg": reg, "dist64": dist, "pred_ab": pred, "dist_ab_S": dist_s, "logits313": logits,
                  "hyper": hyper})
    return inter


def _rel(a, b):
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-300))


def _check_twin(ref, twin, gains):
    assert set(ref) == set(twin)
    checked = 0
    for name, r in ref.items():
        k = gains.get(name, 0)           # names outside the family (the pre-BN ReLU outputs, the heads) keep gain 1
        err = _rel(twin[name], r * 2.0 ** k)
        assert err <= TOL, (name, k, err)
        checked += name in rescale.BUFFERS
    assert checked == len(rescale.BUFFERS)


@pytest.mark.parametrize("glob", [False, True], ids=["plain", "glob"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_gains_every_buffer(full_sd, batch, seed, glob):
    """k in [-12, 12] on every buffer at once, the distribution head, the Caffe head and (glob) the global hints."""
    gains = rescale.random_gains(seed, -12, 12)
    assert len(set(gains.values())) > 5
    _check_twin(_forward(full_sd, batch, glob), _forward(rescale.rescale(full_sd, gains), batch, glob), gains)


@pytest.mark.parametrize("buf", rescale.BUFFERS)
def test_one_buffer(full_sd, batch, buf):
    """k = +9 on one buffer: that buffer (only) scales, with the global hints on so conv4_3's rule includes the MLP."""
    gains = {buf: 9}
    ref = _forward(full_sd, batch, True)
    twin = _forward(rescale.rescale(full_sd, gains), batch, True)
    _check_twin(ref, twin, gains)
    assert _rel(twin[buf], ref[buf]) > 100.0          # the buffer really moved


def test_rescale_is_exact_and_leaves_the_input_alone(full_sd):
    """Scaled tensors are exactly 2^k times the originals in their own dtype; the input dict is not modified; BN running
    statistics never change."""
    before = {k: (v.clone() if torch.is_tensor(v) else np.copy(v)) for k, v in full_sd.items()}
    twin = rescale.rescale(full_sd, {"conv4_3": 7, "a8_1": -3, "conv10_2": 5})
    for k, v in full_sd.items():
        assert torch.equal(torch.as_tensor(v), torch.as_tensor(before[k])), k
    assert torch.equal(twin["model4.6.weight"], full_sd["model4.6.weight"] * 128.0)
    assert twin["model4.6.weight"].dtype == torch.float32
    assert torch.equal(twin["glob.3.bn.bias"], full_sd["glob.3.bn.bias"] * 128.0)
    assert torch.equal(twin["model5.0.weight"], full_sd["model5.0.weight"] / 128.0)
    assert torch.equal(twin["model5.0.bias"], full_sd["model5.0.bias"])
    assert torch.equal(twin["caffe.conv4_pred.weight"], full_sd["caffe.conv4_pred.weight"] / 128.0)
    for p in ("model8up.0", "model3short8.0"):
        assert torch.equal(twin[p + ".bias"], full_sd[p + ".bias"] / 8.0)
    assert torch.equal(twin["model8.1.weight"], full_sd["model8.1.weight"] * 8.0)
    assert torch.equal(twin["model_out.0.weight"], full_sd["model_out.0.weight"] / 32.0)
    assert torch.equal(twin["model_out.0.bias"], full_sd["model_out.0.bias"])
    for k in full_sd:
        if "running_" in k:
            assert twin[k] is full_sd[k]
    with pytest.raises(KeyError):
        rescale.rescale(full_sd, {"a5_3": 1})
    with pytest.raises(ValueError):
        rescale.rescale(full_sd, {"a5_1": 0.5})
