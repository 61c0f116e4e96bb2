"""CPU: the oracle (oracle/lhn_ref.py) against the UNMODIFIED reference network run live (tests/live_ref.py), in FP64
and in FP32, on live inputs; and the sampled colour suggestions' tie rule against the reference wrapper.

test_oracle.py pins lhn_ref to one stored 64² vector of the reference.  Here the reference's own SIGGRAPHGenerator runs
beside it on every case: 8², 64², 72 x 88 and 256², maskcent 0 and 0.5, the synthetic network and a trained-like one
(rho = 0.3, tests/calibrated.py), both outputs of the distribution model and the regression-only model.  The reference
must be importable (a checkout, or what `__graft_entry__.build()` staged): without it these tests fail, they do not
skip."""
import numpy as np
import pytest
import torch

from oracle import lhn_ref, synth
from tests import calibrated, live_ref

GEOMS = [(8, 8), (64, 64), (72, 88), (256, 256)]
NETS = ["synthetic", 0.3]
# Worst cases measured over all 16 cases of each precision: 0 in the regression map and 0 in the distribution, in FP64
# and in FP32 -- the oracle calls the same torch functions, in the same order, as the reference's modules.  The bars
# are rounding noise only (ab is O(110), the pmf O(1)): a misread of the reference is orders of magnitude larger.
BAR = {torch.float64: {"reg": 1e-10, "dist": 1e-15}, torch.float32: {"reg": 1e-4, "dist": 1e-7}}


def _f32(sd):
    """The weights as the reference module holds them: its parameters and buffers are float32, so load_state_dict
    rounds the calibrated network's float64 BatchNorm statistics.  The oracle gets the same rounded values."""
    return {k: (v.float() if torch.is_floating_point(v) else v) for k, v in sd.items()}


@pytest.fixture(scope="module")
def nets(synth_sd):
    cal = synth.synthetic_batch(4, 64, seed=0)
    return {"synthetic": _f32(synth_sd), 0.3: _f32(calibrated.trained_like(synth_sd, 0.3, cal))}


def _inputs(H, W, seed):
    """One image: L_mc [1,H,W], ab [2,H,W], mask [1,H,W] float32, with hints (cropped from a larger grid for 8²)."""
    X = max(H, W, 32)
    L, ab, m = synth.synthetic_batch(1, X, seed=seed, max_hints=6)
    return tuple(np.ascontiguousarray(a[0, :, :H, :W]) for a in (L, ab, m))


def _worst(name, dtype, rows):
    reg = max(r[0] for r in rows)
    dist = max(r[1] for r in rows)
    print("%s %s: worst max|d reg| = %.3e, worst max|d dist| = %.3e over %d cases"
          % (name, str(dtype).replace("torch.", ""), reg, dist, len(rows)))
    return reg, dist


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
def test_oracle_equals_live_reference_network(nets, dtype):
    rows = []
    for net in NETS:
        sd = nets[net]
        ref_dist, ref_reg = live_ref.reference_net(sd, True, dtype), live_ref.reference_net(sd, False, dtype)
        for gi, (H, W) in enumerate(GEOMS):
            L, ab, m = _inputs(H, W, 40 + gi)
            for mc in (0.0, 0.5):
                quirk, up = live_ref.net_forward(ref_dist, dtype, L, ab, m, mc)
                plain = live_ref.net_forward(ref_reg, dtype, L, ab, m, mc)
                with torch.no_grad():
                    reg_q, dist64 = lhn_ref.lhn_forward(sd, L[None], ab[None], m[None], mc, dist=True, dtype=dtype)
                    reg = lhn_ref.lhn_forward(sd, L[None], ab[None], m[None], mc, ref_quirks=False, dtype=dtype)
                dist_up = lhn_ref.upsample4(dist64)[0].double().numpy()
                assert up.shape == dist_up.shape == (529, H, W)
                # the distribution model returns the regression map x 110 twice (models/pytorch/model.py); the oracle
                # with ref_quirks returns it the same way
                e_q = float(np.abs(quirk - reg_q[0].double().numpy()).max()) / 110.0
                e_r = float(np.abs(plain - reg[0].double().numpy()).max())
                e_d = float(np.abs(up - dist_up).max())
                case = (net, H, W, mc)
                assert e_q <= BAR[dtype]["reg"] and e_r <= BAR[dtype]["reg"], (case, e_q, e_r)
                assert e_d <= BAR[dtype]["dist"], (case, e_d)
                # the two reference models share the trunk and the regression head
                assert np.abs(quirk / 110.0 - plain).max() <= BAR[dtype]["reg"] + 1e-9 * np.abs(plain).max(), case
                rows.append((max(e_q, e_r), e_d))
    _worst("lhn_ref vs reference", dtype, rows)


def test_sampled_reccs_tie_rule_matches_reference():
    """get_ab_reccs(method='sampled') maps a uniform sample to a bin with np.digitize(u, cdf), so a sample equal to a
    CDF value belongs to the NEXT bin, and zero bins repeat a CDF value.  Random uniforms never land on a CDF value;
    here the draws are replaced, on both sides alike, by ones that include every CDF value, and the port's sample set,
    centres and confidences must equal the reference's bit for bit."""
    from interactive_deep_colorization_b200 import colorize_image as PCI
    CI = live_ref.reference_wrapper()
    X, h, w, N = 8, 5, 2, 4000
    rs = np.random.RandomState(7)
    pmf = rs.randint(0, 9, 529).astype(np.float32)
    pmf[rs.rand(529) < 0.5] = 0                        # runs of zero bins: repeated CDF values
    pmf /= pmf.sum()
    dist = np.zeros((529, X, X), np.float32)
    dist[:, h, w] = pmf
    with live_ref.precision(torch.float32):
        ref = CI.ColorizeImageTorchDist(Xd=X)
    ref.dist_ab, ref.dist_ab_set = dist, True
    port = PCI.ColorizeImageB200Dist(Xd=X)
    port.dist_ab, port.dist_ab_set = dist, True
    cdf = np.cumsum(pmf)
    cdf = cdf / cdf[-1]
    edges = np.unique(cdf[cdf < 1]).astype(np.float64)
    real_uniform = np.random.uniform

    def uniform(low=0.0, high=1.0, size=None):
        u = real_uniform(low, high, size)             # consumes the global state exactly as the real draw does
        u[:edges.size] = edges
        return u

    got = {}
    for name, cm in (("port", port), ("ref", ref)):
        np.random.seed(11)
        np.random.uniform = uniform
        try:
            kw = {"method": "sampled"} if cm is port else {}
            with live_ref.precision(torch.float32), live_ref.one_thread():
                got[name] = cm.get_ab_reccs(h, w, K=5, N=N, return_conf=True, **kw)
        finally:
            np.random.uniform = real_uniform
    u = np.random.RandomState(11).uniform(0, 1, N)
    u[:edges.size] = edges
    assert (np.digitize(u, cdf) != np.searchsorted(cdf, u, side="left")).sum() >= edges.size   # the ties matter
    for a, b in zip(got["port"], got["ref"]):
        assert np.array_equal(a, b), (a, b)
