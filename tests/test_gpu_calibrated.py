"""GPU: both engines on trained-like networks (tests/calibrated.py): BatchNorm statistics calibrated on data, filters
with a non-zero mean (rho * std(W) added), heads rescaled so tanh does not saturate.  Their activations are far larger
than the 2-norm magnitude estimate of the weights predicts (DESIGN §3), which is where the wgmma engine's FP16 storage
would saturate.  The wgmma engine must match the FP32 oracle there; the SIMT engine is the control.  A store that
does saturate must make the forward fail (IDC_ERR_RANGE) and name the buffer.

rho = 0 (calibrated BatchNorm on zero-mean filters) is ill-conditioned: the FP32 oracle is 1.1e-3 from the FP64
evaluation in ab, and the SIMT engine (FP32 as well, another summation order) 2.6e-3 from the FP32 oracle.  Every bar is
therefore max(bar, 4 x |FP32 oracle - FP64 oracle|); on the coherent networks that term stays below the plain bars.

A stored buffer of a whole forward carries the errors of every op before it: it is held to 5x the per-op bar of
tests/test_gpu_umma_ops.py (measured on an H100: up to 2.5x the per-op bar, in the dilated block 5, with the 2-norm
exponents and with the bounded ones alike); the per-op bar itself holds in the isolation pass."""
import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import _lib
from oracle import caffe_spec, lhn_ref, synth
from tests import calibrated, rescale, util

pytestmark = pytest.mark.gpu
TOL_AB = 1e-3        # BASELINE.json north_star: ab within 1e-3 max-abs of the reference
TOL_DIST = 1e-5
OP_BAR = 2e-5        # tests/test_gpu_umma_ops.py: per-op bar relative to max(1, |out|max)
CHAIN_BAR = 5 * OP_BAR   # a buffer of a whole forward, relative to max(1, |a|max)
COND = 4             # bars are at least COND x |FP32 oracle - FP64 oracle| (the network's own FP32 conditioning)
RHOS = [0.0, 0.15, 0.3, 0.6, 1.0]
ENGINES = ["wgmma", "simt"]


@pytest.fixture(scope="module")
def cal():
    return synth.synthetic_batch(4, 64, seed=0)


@pytest.fixture(scope="module")
def nets(synth_sd, cal):
    out = {"synthetic": synth_sd}
    out.update({rho: calibrated.trained_like(synth_sd, rho, cal) for rho in RHOS})
    return out


@pytest.fixture(scope="module")
def batch64():
    return util.small_batch(3, 64, seed=1300)


def _oracle(sd, batch, maskcent=0.5):
    """FP32 oracle (reg, dist, intermediates) and the conditioning of each output: COND x |FP32 - FP64|."""
    with torch.no_grad():
        (reg, dist), inter = lhn_ref.lhn_forward(sd, *batch, maskcent, dist=True, ref_quirks=False,
                                                 return_intermediates=True)
        (reg64, dist64), inter64 = lhn_ref.lhn_forward(sd, *batch, maskcent, dist=True, ref_quirks=False,
                                                       return_intermediates=True, dtype=torch.float64)
    cond = {"ab": COND * util.maxabs(reg, reg64), "dist": COND * util.maxabs(dist, dist64)}
    cond.update({b: COND * util.maxabs(inter[b], inter64[b]) for b in rescale.STORED + ["conv10_2"]})
    return reg, dist, inter, cond


@pytest.fixture(scope="module")
def oracles(nets, batch64):
    return {k: _oracle(sd, batch64) for k, sd in nets.items()}


def _with_caffe(sd):
    out = dict(sd)
    out.update({k: torch.from_numpy(v) for k, v in
                caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=util.golden("pts_in_hull.npy")).items()})
    return out


@pytest.mark.parametrize("net", ["synthetic", 0.0, 0.3, 1.0])
def test_exponents_match_host_estimate(nets, net):
    """idc_act_exponent equals tests/calibrated.act_estimates for every buffer (conv10_2 stored, Caffe hyper-column
    included): the engine's estimate and bound are the ones DESIGN §3 states."""
    sd = _with_caffe(nets[net])
    want = calibrated.act_estimates(sd, caffe313=True)
    ctx = util.make_ctx(sd, 64, 64, max_n=1, keep_conv10=True, caffe313=True)
    got = {b: ctx.act_exponent(b) for b in want}
    ctx.close()
    assert got == {b: e[2] for b, e in want.items()}, {b: (got[b], want[b]) for b in want if got[b] != want[b][2]}


def _check_forward(ctx, batch, ref, what, buffers=rescale.STORED, keep10=False):
    reg, dist, inter, cond = ref
    r = ctx.forward_host(*batch, 0.5, want_dist=True)
    e_ab, e_d = util.maxabs(r["ab"], reg), util.maxabs(r["dist"], dist)
    errs = {}
    for b in buffers + (["conv10_2"] if keep10 else []):
        got = ctx.get_activation(b, batch[0].shape[0]).cpu()
        scale = float(inter[b].abs().max())
        errs[b] = (util.maxabs(got, inter[b]), max(CHAIN_BAR * max(1.0, scale), cond[b]), scale)
    worst = max(errs, key=lambda b: errs[b][0] / errs[b][1])
    print("%s: ab %.2e (bar %.1e)  dist %.2e  worst buffer %s: %.2e of bar %.2e (|a|max %.3g)"
          % (what, e_ab, max(TOL_AB, cond["ab"]), e_d, worst, *errs[worst]))
    if not ctx.flags & _lib.FLAG_ENGINE_SIMT:
        # the storage exponents keep every buffer inside FP16's range: its largest value, stored, is below 65504
        stored = {b: float(inter[b].abs().max()) * 2.0 ** ctx.act_exponent(b) for b in errs}
        over = {b: v for b, v in stored.items() if v > calibrated.FP16_MAX}
        assert not over, (what, "stored above 65504", over)
    assert e_ab <= max(TOL_AB, cond["ab"]), (what, e_ab)
    assert e_d <= max(TOL_DIST, cond["dist"]), (what, e_d)
    bad = {b: v for b, v in errs.items() if v[0] > v[1]}
    assert not bad, (what, bad)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("rho", RHOS)
def test_trained_like_64(nets, oracles, batch64, rho, engine):
    """64², n = 3, the default plan (fused head, dist head on): ab, dist and every stored buffer against the FP32
    oracle; then the unfused plan, which also stores conv10_2."""
    for keep10 in (False, True):
        ctx = util.make_ctx(nets[rho], 64, 64, max_n=3, dist=True, engine=engine, keep_conv10=keep10)
        _check_forward(ctx, batch64, oracles[rho], "rho=%g %s keep_conv10=%d" % (rho, engine, keep10), keep10=keep10)
        ctx.close()


@pytest.mark.parametrize("engine", ENGINES)
def test_trained_like_ragged(nets, engine):
    """rho = 0.3 at 72 x 88, n = 2: ragged tiles on every level."""
    batch = tuple(np.ascontiguousarray(a[:, :, :72, :88]) for a in util.small_batch(2, 88, seed=77))
    ctx = util.make_ctx(nets[0.3], 72, 88, max_n=2, dist=True, engine=engine)
    _check_forward(ctx, batch, _oracle(nets[0.3], batch), "rho=0.3 72x88 %s" % engine)
    ctx.close()


@pytest.mark.parametrize("engine", ENGINES)
def test_trained_like_click_graph_256(nets, engine):
    """rho = 0.3 through the 256² click graph (n = 1, dist head resident, announced click): ab and the clicked
    pixel's pmf against the FP32 oracle."""
    L, ab, m = synth.synthetic_batch(1, 256, seed=31, max_hints=6)
    reg, dist, _, cond = _oracle(nets[0.3], (L, ab, m))
    ctx = util.make_ctx(nets[0.3], 256, 256, max_n=1, dist=True, engine=engine)
    ctx.set_dist_resident(True)
    ctx.set_click(0, 20, 41, 5)
    r = ctx.forward_host(L, ab, m, 0.5)
    pmf = ctx.fetch_dist(0, 20, 41)
    e_ab, e_p = util.maxabs(r["ab"], reg), util.maxabs(pmf, dist[0, :, 20, 41])
    print("rho=0.3 256² click %s: ab %.2e  pmf %.2e" % (engine, e_ab, e_p))
    assert e_ab <= max(TOL_AB, cond["ab"]) and e_p <= max(TOL_DIST, cond["dist"]), (e_ab, e_p)
    ctx.close()


@pytest.mark.parametrize("opt,val", [("halo", 3), ("mt", 2), ("split_k", 1)])
def test_trained_like_plan_variants(nets, oracles, batch64, opt, val):
    """rho = 0.3 with the halo-tile A operand on every eligible op, two M-tiles per CTA, split-K off."""
    ctx = util.make_ctx(nets[0.3], 64, 64, max_n=3, dist=True, options={opt: val})
    _check_forward(ctx, batch64, oracles[0.3], "rho=0.3 %s=%d" % (opt, val))
    ctx.close()


# the ops that produce the largest stored values on these networks: the second conv of each encoder block (two
# coherent convs with no BatchNorm between them) under the 2-norm estimate, and the decoder's up-sampling ops
ISOLATED = ["c3_1", "c3_2", "c4_2", "c5_2", "c6_2", "c7_2", "up8", "c8_2", "up9", "up10", "c10_2"]


@pytest.mark.parametrize("rho", [0.3, 1.0])
def test_trained_like_isolated_ops(nets, oracles, rho):
    """Per-op isolation: the FP32 oracle's activations are injected as each op's inputs, ONE op runs, its output is
    compared with the oracle's, so a failure names the layer."""
    reg, dist, inter, cond = oracles[rho]
    ctx = util.make_ctx(nets[rho], 64, 64, max_n=3, keep_conv10=True, use_graph=False)
    bad = {}
    for op in ISOLATED:
        ins, out = util.OP_IO[op]
        for nm in ins:
            ctx.set_activation(nm, inter[nm].cuda().contiguous())
        ctx.run_op(op, 3)
        torch.cuda.synchronize()
        err = util.maxabs(ctx.get_activation(out, 3), inter[out])
        scale = float(inter[out].abs().max())
        print("rho=%g op %-6s max|err| %.3e (|out|max %.3g)" % (rho, op, err, scale))
        if err >= OP_BAR * max(1.0, scale):
            bad[op] = (err, scale)
    ctx.close()
    assert not bad, bad


def _override_that_saturates(inter, buf):
    """The smallest exponent at which buf's largest value stores above 2 x 65504."""
    return int(np.floor(np.log2(2 * calibrated.FP16_MAX / float(inter[buf].abs().max())))) + 1


@pytest.mark.parametrize("fast", [False, True])
def test_saturation_is_reported(synth_sd, oracles, batch64, fast):
    """act_exp.a3_2 high enough that a3_2 stores above 65504: the forward fails with IDC_ERR_RANGE naming a3_2 and no
    other buffer (the wgmma epilogue, FAST_FP16 included); three steps lower the same forward passes."""
    _, _, inter, _ = oracles["synthetic"]
    s_bad = _override_that_saturates(inter, "a3_2")
    for s, fails in ((s_bad, True), (s_bad - 3, False)):
        ctx = util.make_ctx(synth_sd, 64, 64, max_n=3, fast_fp16=fast, options={"act_exp.a3_2": s})
        if fails:
            with pytest.raises(_lib.IdcError, match="a3_2") as ei:
                ctx.forward_host(*batch64, 0.5)
            assert ei.value.code == _lib.ERR_RANGE
            assert "conv1_2" not in str(ei.value) and "a4_1" not in str(ei.value)
        else:
            r = ctx.forward_host(*batch64, 0.5)
            if not fast:
                assert util.maxabs(r["ab"], oracles["synthetic"][0]) <= TOL_AB
        ctx.close()


def test_saturation_reported_on_every_path(synth_sd, oracles, batch64):
    """The asynchronous idc_forward reports at the next call on the context; the large-batch host path (n = 8, copy
    overlap) and conv1_1_umma_kernel's output (a1_1) and input pack report too; a report clears the word, so the next
    forward that stays in range passes."""
    _, _, inter, _ = oracles["synthetic"]
    L, ab, m = (util.dev(a) for a in batch64)
    ctx = util.make_ctx(synth_sd, 64, 64, max_n=3, options={"act_exp.a8_2": _override_that_saturates(inter, "a8_2")})
    ctx.forward_device(L, ab, m, 0.5)                # asynchronous: nothing to report yet
    torch.cuda.synchronize()
    with pytest.raises(_lib.IdcError, match="a8_2") as ei:
        ctx.forward_device(L, ab, m, 0.5)
    assert ei.value.code == _lib.ERR_RANGE
    ctx.close()
    big = tuple(np.ascontiguousarray(np.concatenate([a] * 3)[:8]) for a in batch64)
    ctx = util.make_ctx(synth_sd, 64, 64, max_n=8, options={"act_exp.a1_1": _override_that_saturates(inter, "a1_1")})
    with pytest.raises(_lib.IdcError, match="a1_1") as ei:
        ctx.forward_host(*big, 0.5)
    assert ei.value.code == _lib.ERR_RANGE
    ctx.close()
    ctx = util.make_ctx(synth_sd, 64, 64, max_n=3)
    L_big = np.ascontiguousarray(batch64[0] * np.float32(1e6))        # L / 100 * 2^6 far above 65504
    with pytest.raises(_lib.IdcError, match="conv1_1 input") as ei:
        ctx.forward_host(L_big, batch64[1], batch64[2], 0.5)
    assert ei.value.code == _lib.ERR_RANGE
    ctx.forward_host(*batch64, 0.5)
    ctx.close()
