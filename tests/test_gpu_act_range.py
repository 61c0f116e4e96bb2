"""GPU: the engines do not depend on the absolute size of the activations.

Every check loads a power-of-two rescaled twin of the network (tests/rescale.py: buffer b stores 2^k times the
original's values, the function is unchanged) next to the original and compares.  The SIMT engine scales every multiply
and add exactly, so it is bit-identical across the family.  The wgmma engine stores buffer b as FP16 hi/lo of
value * 2^S_b with S_b chosen from the weights (DESIGN §3); the choice shifts by exactly -k on the twin, so the stored
FP16 bits, and every output, are the same.  A fixed exponent would clamp large activations at FP16's 65504 without
an error: the k = +10 test is that case."""
import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import _lib
from oracle import caffe_spec, synth
from tests import rescale, util

pytestmark = pytest.mark.gpu
TOL_AB = 1e-3        # BASELINE.json north_star: ab within 1e-3 max-abs of the reference
FUSED = rescale.STORED + ["conv10_2"]      # the buffers of the default (fused-head) plan, conv10_2 kept in registers


def _exps(ctx):
    return {b: ctx.act_exponent(b) for b in rescale.STORED}


def _same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and np.array_equal(a, b), (what, int((a != b).sum()), util.maxabs(a, b))


def _fwd(ctx, batch, **kw):
    L, ab, m = batch
    return ctx.forward_host(L, ab, m, 0.5, **kw)


def _check_exps(exp0, exp1, gains):
    for b in rescale.STORED:
        assert exp1[b] == exp0[b] - gains.get(b, 0), (b, exp0[b], exp1[b], gains.get(b, 0))


@pytest.fixture(scope="module")
def batch64():
    return util.small_batch(3, 64, seed=1300)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_simt_random_gains_bit_identical(synth_sd, batch64, seed):
    """Control: k in [-12, 12] on every buffer; the FP32 engine's ab, dist and rgb are bit-identical."""
    b = tuple(a[:2] for a in batch64)
    gains = rescale.random_gains(seed, -12, 12, FUSED)
    ref = util.make_ctx(synth_sd, 64, 64, max_n=2, dist=True, engine="simt")
    twin = util.make_ctx(rescale.rescale(synth_sd, gains), 64, 64, max_n=2, dist=True, engine="simt")
    r0, r1 = _fwd(ref, b, want_dist=True, want_rgb=True), _fwd(twin, b, want_dist=True, want_rgb=True)
    for k in ("ab", "dist", "rgb"):
        _same(r1[k], r0[k], k)
    ref.close(); twin.close()


@pytest.fixture(scope="module")
def one_buffer_ctxs(synth_sd, batch64):
    """Original and twin contexts (64², n = 3, dist head); the twin context is reloaded for each twin."""
    ref = util.make_ctx(synth_sd, 64, 64, max_n=3, dist=True)
    twin = util.make_ctx(synth_sd, 64, 64, max_n=3, dist=True)
    out0 = _fwd(ref, batch64, want_dist=True)
    yield ref, twin, {k: np.copy(v) for k, v in out0.items() if v is not None}, _exps(ref)
    ref.close(); twin.close()


@pytest.mark.parametrize("buf", FUSED)
def test_wgmma_one_buffer(one_buffer_ctxs, synth_sd, batch64, buf):
    """k = -8 and +8 on one buffer: output bit-identical, the buffer's exponent shifted by exactly -k (the others
    unchanged), ab within TOL_AB of the FP32 oracle on the twin."""
    ref, twin, out0, exp0 = one_buffer_ctxs
    for k in (-8, 8):
        gains = {buf: k}
        sd = rescale.rescale(synth_sd, gains)
        twin.load_state_dict(sd)
        _check_exps(exp0, _exps(twin), gains)
        r = _fwd(twin, batch64, want_dist=True)
        _same(r["ab"], out0["ab"], (buf, k, "ab"))
        _same(r["dist"], out0["dist"], (buf, k, "dist"))
        err = util.maxabs(r["ab"], util.oracle_forward(sd, *batch64, 0.5))
        assert err <= TOL_AB, (buf, k, err)


_VARIANTS = [("mt", 2, -1), ("halo", 3, 1), ("pairs", 2, 0), ("split_k", 1, -1), ("conv1_1_umma", 0, 1)]


def test_wgmma_random_gains_plan_variants(synth_sd, batch64):
    """k in [-5, 5] on every buffer at once, one seeded draw per plan variant: ab and dist bit-identical."""
    b = tuple(a[:2] for a in batch64)
    ref = util.make_ctx(synth_sd, 64, 64, max_n=2, dist=True)
    twin = util.make_ctx(synth_sd, 64, 64, max_n=2, dist=True)
    exp0 = _exps(ref)
    for i, (opt, val, default) in enumerate([("default", None, None)] + _VARIANTS):
        gains = rescale.random_gains(100 + i, -5, 5, FUSED)
        twin.load_state_dict(rescale.rescale(synth_sd, gains))
        _check_exps(exp0, _exps(twin), gains)
        if val is not None:
            ref.set_option(opt, val); twin.set_option(opt, val)
        r0, r1 = _fwd(ref, b, want_dist=True, want_rgb=True), _fwd(twin, b, want_dist=True, want_rgb=True)
        for k in ("ab", "dist", "rgb"):
            _same(r1[k], r0[k], (opt, k))
        if val is not None:
            ref.set_option(opt, default); twin.set_option(opt, default)
    ref.close(); twin.close()


def test_wgmma_random_gains_ragged(synth_sd):
    """72 x 88, n = 2 (ragged tiles on every level), with the unfused head so conv10_2 is a stored buffer too."""
    batch = tuple(np.ascontiguousarray(a[:, :, :72, :88]) for a in util.small_batch(2, 88, seed=77))
    gains = rescale.random_gains(7, -5, 5, FUSED)
    sd = rescale.rescale(synth_sd, gains)
    for kw in (dict(), dict(keep_conv10=True)):
        ref = util.make_ctx(synth_sd, 72, 88, max_n=2, dist=True, **kw)
        twin = util.make_ctx(sd, 72, 88, max_n=2, dist=True, **kw)
        _check_exps(_exps(ref), _exps(twin), gains)
        if kw:
            assert twin.act_exponent("conv10_2") == ref.act_exponent("conv10_2") - gains["conv10_2"]
        r0, r1 = _fwd(ref, batch, want_dist=True), _fwd(twin, batch, want_dist=True)
        _same(r1["ab"], r0["ab"], (kw, "ab"))
        _same(r1["dist"], r0["dist"], (kw, "dist"))
        ref.close(); twin.close()


def test_wgmma_random_gains_click_graph_256(synth_sd):
    """256², n = 1 through the click graph with the dist head resident and an announced click: ab, rgb, the clicked
    pixel's pmf and its colour suggestions bit-identical."""
    L, ab, m = synth.synthetic_batch(1, 256, seed=31, max_hints=6)
    gains = rescale.random_gains(11, -5, 5, FUSED)
    ctxs = [util.make_ctx(sd, 256, 256, max_n=1, dist=True) for sd in (synth_sd, rescale.rescale(synth_sd, gains))]
    outs = []
    for ctx in ctxs:
        ctx.set_dist_resident(True)
        ctx.set_click(0, 20, 41, 5)
        r = ctx.forward_host(L, ab, m, 0.5, want_rgb=True)
        outs.append((np.copy(r["ab"]), np.copy(r["rgb"]), ctx.fetch_dist(0, 20, 41), ctx.ab_reccs(0, 20, 41, K=5)))
    (a0, g0, p0, c0), (a1, g1, p1, c1) = outs
    _same(a1, a0, "ab"); _same(g1, g0, "rgb"); _same(p1, p0, "pmf")
    _same(c1[0], c0[0], "centres"); _same(c1[1], c0[1], "mass")
    assert c1[2] == c0[2]
    for ctx in ctxs:
        ctx.close()


def test_wgmma_random_gains_global_hints(synth_sd, batch64):
    """Global hints: conv4_3's gain scales the MLP's last BatchNorm, so the added vector scales with it."""
    gsd = caffe_spec.synthetic_glob_state_dict()
    sd = dict(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in gsd.items()})
    glob_ab, sat = synth.synthetic_glob(2, seed=3)
    glob = np.ascontiguousarray(np.concatenate([glob_ab, sat], axis=1).astype(np.float32))
    b = tuple(a[:2] for a in batch64)
    gains = rescale.random_gains(21, -5, 5, FUSED)
    gains["conv4_3"] = 5
    ref = util.make_ctx(sd, 64, 64, max_n=2, global_hints=True)
    twin = util.make_ctx(rescale.rescale(sd, gains), 64, 64, max_n=2, global_hints=True)
    _check_exps(_exps(ref), _exps(twin), gains)
    r0, r1 = _fwd(ref, b, glob=glob), _fwd(twin, b, glob=glob)
    _same(r1["ab"], r0["ab"], "ab")
    gvec = caffe_spec.global_hints_vector(gsd, glob)
    assert util.maxabs(r0["ab"], util.oracle_forward(synth_sd, *b, 0.5, glob_add=gvec)) <= TOL_AB
    ref.close(); twin.close()


def test_wgmma_random_gains_caffe313(synth_sd, batch64):
    """Caffe 313-bin head: hyper (2^k times the original's, exactly), pred_ab and the dist_ab_S map bit-identical."""
    csd = caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=util.golden("pts_in_hull.npy"))
    sd = dict(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in csd.items()})
    gains = rescale.random_gains(31, -5, 5, rescale.BUFFERS)
    ctxs = [util.make_ctx(s, 64, 64, max_n=2, caffe313=True) for s in (sd, rescale.rescale(sd, gains))]
    assert ctxs[1].act_exponent("hyper") == ctxs[0].act_exponent("hyper") - gains["hyper"]
    L, ab, m = (util.dev(a[:2]) for a in batch64)
    outs = []
    for ctx in ctxs:
        r = ctx.forward_device(L, ab, m, 0.5)
        pred = ctx.caffe313_pred_ab(2)
        dmap = ctx.caffe313_dist_map(2)
        torch.cuda.synchronize()
        outs.append((r["ab"].cpu().numpy(), ctx.get_activation("hyper", 2).cpu().numpy(), pred.cpu().numpy(),
                     dmap.cpu().numpy()))
    (a0, h0, p0, d0), (a1, h1, p1, d1) = outs
    _same(a1, a0, "ab")
    _same(h1, h0 * np.float32(2.0 ** gains["hyper"]), "hyper")
    _same(p1, p0, "pred_ab")
    _same(d1, d0, "dist_ab_S")
    for ctx in ctxs:
        ctx.close()


def test_wgmma_large_activations(synth_sd, batch64):
    """k = +10 on every buffer: activations ~1000x the synthetic ones (conv2_2 reaches ~7700, far above the 1023 a
    fixed 2^6 storage scale can hold).  ab within TOL_AB of the FP32 oracle on the twin, and bit-identical to the
    original network."""
    gains = {b: 10 for b in FUSED}
    sd = rescale.rescale(synth_sd, gains)
    ref = util.make_ctx(synth_sd, 64, 64, max_n=3, dist=True, keep_conv10=True)
    twin = util.make_ctx(sd, 64, 64, max_n=3, dist=True, keep_conv10=True)
    _check_exps(_exps(ref), _exps(twin), gains)
    r0, r1 = _fwd(ref, batch64, want_dist=True), _fwd(twin, batch64, want_dist=True)
    (reg, dist), inter = util.oracle_forward(sd, *batch64, 0.5, dist=True, intermediates=True)
    big = max(float(inter[b].abs().max()) for b in rescale.STORED)
    assert big > 2000.0, big
    err = util.maxabs(r1["ab"], reg)
    print("k = +10 on every buffer: largest activation %.0f, max|d ab| vs the FP32 oracle %.3e" % (big, err))
    assert err <= TOL_AB, err
    assert util.maxabs(r1["dist"], dist) < 1e-5
    _same(r1["ab"], r0["ab"], "ab")
    for b in ("a1_1", "conv2_2", "conv4_3", "a8_1", "conv10_2"):
        got = twin.get_activation(b, 3).cpu()
        assert util.maxabs(got, inter[b]) <= 2e-4 * 1024, b          # the 2e-4 layer bar of the original, scaled
    ref.close(); twin.close()


def test_exponent_out_of_range_is_refused(synth_sd):
    """A twin whose exponent falls outside the supported range makes load_state_dict raise, naming the buffer; so does
    an out-of-range or late act_exp override."""
    ctx = util.make_ctx(synth_sd, 64, 64, max_n=1)
    s = ctx.act_exponent("conv4_3")
    with pytest.raises(_lib.IdcError, match="conv4_3"):
        ctx.load_state_dict(rescale.rescale(synth_sd, {"conv4_3": s + 30}))
    with pytest.raises(_lib.IdcError):
        _fwd(ctx, util.small_batch(1, 64))                 # no forward from a context whose weights were refused
    with pytest.raises(_lib.IdcError, match="a8_1"):
        ctx.load_state_dict(rescale.rescale(synth_sd, {"a8_1": -40}))
    ctx.load_state_dict(synth_sd)
    with pytest.raises(_lib.IdcError):
        ctx.set_option("act_exp.conv4_3", 3)              # the weights are packed: too late
    with pytest.raises(_lib.IdcError):
        ctx.set_option("act_exp.nosuchbuffer", 3)
    ctx.close()
    from interactive_deep_colorization_b200.engine import LhnContext
    c2 = LhnContext(device=0, max_n=1, H=64, W=64)
    with pytest.raises(_lib.IdcError):
        c2.set_option("act_exp.conv4_3", 99)
    c2.close()


def test_act_exp_override(synth_sd, batch64):
    """act_exp.<buffer> replaces the chosen exponent (two steps up on every buffer; small values then keep more of
    their lo plane, so the output moves by summation-level noise only)."""
    ref = util.make_ctx(synth_sd, 64, 64, max_n=3, dist=True)
    exp0 = _exps(ref)
    ctx = util.make_ctx(synth_sd, 64, 64, max_n=3, dist=True,
                        options={"act_exp." + b: e + 2 for b, e in exp0.items()})
    assert _exps(ctx) == {b: e + 2 for b, e in exp0.items()}
    r0, r1 = _fwd(ref, batch64, want_dist=True), _fwd(ctx, batch64, want_dist=True)
    assert util.maxabs(r1["ab"], r0["ab"]) < 1e-4
    assert util.maxabs(r1["dist"], r0["dist"]) < 1e-6
    ref.close(); ctx.close()


def test_set_get_activation_round_trip_large_values(synth_sd):
    """set_activation -> get_activation keeps ~22 significant bits for values up to 1e5 on a buffer whose exponent the
    weights moved down (a fixed 2^6 scale clamps them at 1023)."""
    ctx = util.make_ctx(rescale.rescale(synth_sd, {"a8_1": 10}), 64, 64, max_n=2)
    s = ctx.act_exponent("a8_1")
    assert s <= -4, s
    c, h, w = ctx.activation_shape("a8_1")
    g = torch.Generator().manual_seed(5)
    mag = 10.0 ** (torch.rand((2, c, h, w), generator=g) * 5.0)                 # 1 .. 1e5
    x = (mag * torch.sign(torch.rand((2, c, h, w), generator=g) - 0.5)).float()
    ctx.set_activation("a8_1", x.cuda().contiguous())
    y = ctx.get_activation("a8_1", 2).cpu()
    err = (y.double() - x.double()).abs()
    bound = x.double().abs() * 2.0 ** -20 + 2.0 ** (-24 - s)
    assert float(x.abs().max()) > 9e4
    assert bool((err <= bound).all()), float((err / bound).max())
    ctx.close()
