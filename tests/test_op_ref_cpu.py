"""CPU: the per-op FP64 reference of tests/op_ref.py.  Chained, its exact-mode ops are the FP64 oracle; its fp16 operand
rounding is torch's float -> half conversion; and its fp16 mode commutes with the power-of-two twins of
tests/rescale.py exactly, as the engine's storage exponents do."""
import numpy as np
import pytest
import torch

from oracle import lhn_ref, synth
from tests import calibrated, op_ref, rescale, util


@pytest.fixture(scope="module")
def batch():
    return util.small_batch(2, 32, seed=41)


@pytest.fixture(scope="module")
def rho03(synth_sd):
    return calibrated.trained_like(synth_sd, 0.3, synth.synthetic_batch(2, 32, seed=5))


def test_spec_matches_op_io():
    assert list(op_ref.SPEC) == list(util.OP_IO)
    for name, (out, srcs, _, _) in op_ref.SPEC.items():
        assert ([s for _, s, _, _ in srcs], out) == tuple(util.OP_IO[name]), name


@pytest.mark.parametrize("net", ["synthetic", "rho0.3"])
def test_chain_is_the_fp64_oracle(synth_sd, rho03, batch, net):
    """conv1_1 and the 25 ops, each fed the previous ones' outputs, reproduce every buffer of the FP64 oracle."""
    sd = synth_sd if net == "synthetic" else rho03
    with torch.no_grad():
        _, inter = lhn_ref.lhn_forward(sd, *batch, 0.5, ref_quirks=False, return_intermediates=True,
                                       dtype=torch.float64)
        got = op_ref.chain(sd, *batch, 0.5)
    assert set(got) == set(util.OP_IO[k][1] for k in util.OP_IO) | {"a1_1"}
    for b, v in got.items():
        err = util.maxabs(v, inter[b])
        assert err <= 1e-12 * max(1.0, float(inter[b].abs().max())), (b, err)


def _f16_cases():
    """Values across FP16's whole range: random normals and subnormals, every kind of tie, and values next to them."""
    rng = np.random.RandomState(7)
    r = (rng.uniform(1, 2, 4000) * 2.0 ** rng.randint(-26, 16, 4000) * rng.choice([-1, 1], 4000)).astype(np.float32)
    grid = np.float16(rng.uniform(-65504, 65504, 2000)).astype(np.float64)
    sub = np.arange(-1100, 1100) * 2.0 ** -24                       # the subnormals, zero and the first normals
    ties = np.concatenate([grid, sub]) + np.concatenate([op_ref.ulp16(torch.from_numpy(grid)).numpy(),
                                                         np.full(sub.size, 2.0 ** -24)]) / 2
    ties = ties[np.abs(ties) < 65504]
    nudged = np.concatenate([np.nextafter(ties.astype(np.float32), np.float32(np.inf)),
                             np.nextafter(ties.astype(np.float32), np.float32(-np.inf))]).astype(np.float64)
    return np.concatenate([r, grid, sub, ties, nudged, [0.0, -0.0, 65504.0, -65504.0, 2.0 ** -25, 3 * 2.0 ** -26]])


def test_f16_is_torch_half_rounding():
    """op_ref.f16 is round-to-nearest-even into FP16, subnormals included: it equals torch's float -> half conversion
    on every case, and fixes every FP16 value."""
    x = torch.from_numpy(_f16_cases())
    assert torch.equal(x.float().double(), x)                        # every case is an FP32 value
    want = x.float().half().double()
    got = op_ref.f16(x)
    bad = (got != want).nonzero().flatten()
    assert bad.numel() == 0, [(float(x[i]), float(got[i]), float(want[i])) for i in bad[:5]]
    assert torch.equal(op_ref.f16(want), want)
    # ties really are exercised: some round down, some up, and subnormals occur
    assert (want.abs() < 2.0 ** -14).sum() > 1000 and (want != x).sum() > 1000


def _inter(sd, batch):
    with torch.no_grad():
        return lhn_ref.lhn_forward(sd, *batch, 0.5, ref_quirks=False, return_intermediates=True)[1]


def test_fp16_mode_rounds_and_stays_close(synth_sd, batch):
    """The fp16 operands differ from the exact ones, and the result stays within FP16 operand error of the exact op."""
    inter = _inter(synth_sd, batch)
    exps = {b: e[2] for b, e in calibrated.act_estimates(synth_sd).items()}
    for name in ("c1_2", "c2_1", "c5_1", "up9", "c10_2"):
        ins, out = util.OP_IO[name]
        acts = {b: inter[b] for b in ins}
        ex, mag = op_ref.OPS[name](synth_sd, acts)
        fp, mag16 = op_ref.OPS[name](synth_sd, acts, mode="fp16", exps=exps)
        d = float((fp - ex).abs().max())
        assert 0 < d <= 2 ** -10 * float(mag.max()), (name, d)
        assert float((mag16 - mag).abs().max()) <= 2 ** -10 * float(mag.max()), name
    ex = op_ref.conv1_1(synth_sd, *batch, 0.5)[0]
    fp = op_ref.conv1_1(synth_sd, *batch, 0.5, mode="fp16")[0]
    assert 0 < float((fp - ex).abs().max()) <= 2 ** -10 * float(ex.abs().max())


def test_fp16_mode_scales_exactly_on_a_twin(synth_sd, batch):
    """A power-of-two twin (every buffer x 2^k_b, tests/rescale.py) moves every storage exponent by -k_b, so the fp16
    operands are the same numbers times powers of two: every op's output and magnitude scale by exactly 2^k_out."""
    gains = rescale.random_gains(11, -6, 6, buffers=rescale.STORED + ["conv10_2"])
    twin = rescale.rescale(synth_sd, gains)
    exps = {b: e[2] for b, e in calibrated.act_estimates(synth_sd).items()}
    exps2 = {b: e[2] for b, e in calibrated.act_estimates(twin).items()}
    assert all(exps2[b] == exps[b] - gains[b] for b in gains)
    inter = _inter(synth_sd, batch)
    for name in util.OP_IO:
        ins, out = util.OP_IO[name]
        v, m = op_ref.OPS[name](synth_sd, {b: inter[b] for b in ins}, mode="fp16", exps=exps)
        v2, m2 = op_ref.OPS[name](twin, {b: inter[b] * 2.0 ** gains[b] for b in ins}, mode="fp16", exps=exps2)
        assert torch.equal(v2, v * 2.0 ** gains[out]) and torch.equal(m2, m * 2.0 ** gains[out]), name
    v, m = op_ref.conv1_1(synth_sd, *batch, 0.5, mode="fp16")
    v2, m2 = op_ref.conv1_1(twin, *batch, 0.5, mode="fp16")
    assert torch.equal(v2, v * 2.0 ** gains["a1_1"]) and torch.equal(m2, m * 2.0 ** gains["a1_1"])
