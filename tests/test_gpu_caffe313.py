"""GPU: the Caffe-spec 313-bin head (row a14) at the launchers' 256^2 and at ragged geometries, against an FP64
evaluation of oracle/caffe_spec.caffe313_head.

The head ops run in isolation: the FP32 oracle trunk's conv3_3 ... conv8_3 are injected with set_activation, read back
(the wgmma engine stores activations as FP16 hi + lo, ~22 bits), and the FP64 head is evaluated on exactly the tensors the
kernels saw, so the trunk's error stays out of the head's bars.  Then hyper (6 sources, 34 taps, 4 output-parity classes,
K = 12 800) and pred313 (313 of 320 columns, a ragged last n-tile) run, and the four head kernels read their logits:
decode313 (annealed mean), dist313_map / dist313_pixel (dist_ab_S) and negentropy.  The geometries reach the branches
64 x 64 never takes: a short last map CTA (W/4 % 8 != 0), an odd number of hyper rows, a decode grid that is not a whole
number of 8-cell blocks, non-square images, a batch below the context's max_n, and image offsets in the logits."""
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from interactive_deep_colorization_b200 import colorize_image as CI
from interactive_deep_colorization_b200 import prepost
from oracle import caffe_spec, color_ref, synth
from tests import caffe313_ref, util

pytestmark = pytest.mark.gpu
TOL_AB = 1e-3        # BASELINE.json north_star: ab within 1e-3 max-abs of the reference
TOL_MAP = 1e-5       # dist_ab_S against FP64, and |sum - 1|
TOL_ENT = 5e-5       # negentropy: both sides sum the bins in the same order; only logf and numpy's log differ
# End to end, the engine's trunk differs from the FP32 oracle trunk by FP32 summation-order noise (hyper 1.1e-5 apart
# on the wgmma engine at 256^2), and the head turns hyper noise into ~100x as much pred_ab error (T = 2.6 times the ab
# spread of the bins), so the chained pred_ab of the wgmma engine is 1.1e-3 from the FP64 head on the oracle trunk
# (H100, 256^2) while the head alone is within 2e-4.  The chained bar is the one test_caffe_named_wrappers holds the
# same head to; the head alone keeps the 1e-3 north star.
TOL_CHAIN = 2e-3
TRUNK = ("conv3_3", "conv4_3", "conv5_3", "conv6_3", "conv7_3", "conv8_3")

# (H, W, n, max_n): the product plan; H/4 = W/4 = 2 (one short map CTA, a 1 x 1 hyper grid, 2 of 8 decode warps busy);
# W/4 = 22 (map CTAs of 8 + 8 + 6 cells) with H/8 = 9 hyper rows; non-square both ways (W/4 = 50 and 10); a batch below
# max_n (image offsets n * H/4 in the logits); 512^2
GEOMS = [(256, 256, 1, 1), (8, 8, 1, 1), (72, 88, 2, 2), (40, 200, 1, 1), (200, 40, 1, 1), (128, 64, 3, 4),
         (512, 512, 1, 1)]


def _gid(g):
    return "%dx%d_n%d_max%d" % g


def _inputs(H, W, n, seed):
    """Random L and a few 7 x 7 hints per image, cropped from a square synthetic batch."""
    X = max(H, W, 32)
    L, ab, m = synth.synthetic_batch(n, X, seed=seed, max_hints=4)
    crop = lambda a: np.ascontiguousarray(a[:, :, :H, :W])
    return crop(L), crop(ab), crop(m)


@pytest.fixture(scope="module")
def weights(synth_sd):
    pts = util.golden("pts_in_hull.npy")
    csd = caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=pts)
    sd = dict(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in csd.items()})
    return sd, csd


_CASES = {}


def _case(synth_sd, geom):
    """Inputs and FP32 oracle trunk of one geometry (maskcent 0.5), built once per module."""
    if geom not in _CASES:
        H, W, n, _ = geom
        L, ab, m = _inputs(H, W, n, seed=H + 7 * W + n)
        _, inter = util.oracle_forward(synth_sd, L, ab, m, 0.5, intermediates=True)
        _CASES[geom] = {"L": L, "ab": ab, "m": m, "inter": {k: inter[k] for k in TRUNK}, "spec": {}}
    return _CASES[geom]


def _spec(csd, trunk):
    """FP64 and FP32 evaluations of the spec head on the same trunk tensors."""
    with torch.no_grad():
        pred64, dist64, logits64, hyper64 = caffe_spec.caffe313_head(csd, trunk, return_logits=True, dtype=torch.float64)
        pred32, _ = caffe_spec.caffe313_head(csd, trunk)
    return {"pred64": pred64.numpy(), "dist64": dist64.numpy(), "logits64": logits64.numpy(),
            "hyper64": hyper64.numpy(), "pred32": pred32.numpy()}


def _spec_from_hyper(csd, hyper):
    """pred_313 and the decode in FP64 on the hyper-column the engine produced and pred313 read (its own readback), with
    the closed-form x4 up-sample of tests/caffe313_ref.py: checks pred313 + decode313 / dist313 without hyper's error."""
    w = torch.as_tensor(np.asarray(csd["caffe.pred_313.weight"]), dtype=torch.float64)
    b = torch.as_tensor(np.asarray(csd["caffe.pred_313.bias"]), dtype=torch.float64)
    with torch.no_grad():
        logits = F.conv2d(torch.as_tensor(hyper, dtype=torch.float64), w, b).numpy()
    return {"pred": caffe313_ref.pred_ab(logits, csd["caffe.pts_in_hull"]), "dist": caffe313_ref.dist_ab_S(logits)}


def _pixels(H, W, seed):
    """Pixels checked bit for bit against the single-pixel lookup: all of them on the smallest grids; otherwise the last
    two cell rows and columns (where the x4 up-sample reads the zero padding past the last cell), the corners and 256
    seeded pixels."""
    if H * W <= 1024:
        return [(y, x) for y in range(H) for x in range(W)]
    px = {(y, x) for y in range(H - 8, H) for x in range(W)} | {(y, x) for y in range(H) for x in range(W - 8, W)}
    px |= {(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1)}
    rs = np.random.RandomState(seed)
    px |= set(zip(rs.randint(0, H, 256).tolist(), rs.randint(0, W, 256).tolist()))
    return sorted(px)


def _worst(d, logits64):
    n_, c_, y_, x_ = np.unravel_index(int(np.argmax(d)), d.shape)
    top2 = np.sort(logits64[n_, :, y_ // 4, x_ // 4])[-2:]
    return (n_, c_, y_, x_), float(top2[1] - top2[0])


def _entropy_err(got, want):
    """NaN at the same pixels (a bin that underflowed to exactly 0: 0 * log 0), then max-abs over the others."""
    assert np.array_equal(np.isnan(got), np.isnan(want)), (np.isnan(got).sum(), np.isnan(want).sum())
    ok = ~np.isnan(want)
    return util.maxabs(got[ok], want[ok])


def _run_isolated(ctx, case, csd, engine):
    """Inject the trunk, run hyper + pred313, read everything the head produces.  -> (outputs, spec on the readback)."""
    n = case["L"].shape[0]
    for nm in TRUNK:
        ctx.set_activation(nm, case["inter"][nm].cuda().contiguous())
    seen = {nm: ctx.get_activation(nm, n).cpu() for nm in TRUNK}
    if engine not in case["spec"]:
        case["spec"][engine] = (seen, _spec(csd, seen))
    seen0, spec = case["spec"][engine]
    for nm in TRUNK:                                   # the storage format does not depend on the plan options
        assert torch.equal(seen[nm], seen0[nm]), nm
    ctx.run_op("hyper", n)
    ctx.run_op("pred313", n)
    torch.cuda.synchronize()
    dmap = ctx.caffe313_dist_map(n)
    out = {"hyper": ctx.get_activation("hyper", n).cpu().numpy(), "pred": ctx.caffe313_pred_ab(n).cpu().numpy(),
           "map": dmap.cpu().numpy(), "neg": prepost.negentropy_gpu(dmap).cpu().numpy()}
    return out, spec


def _check_head(ctx, out, spec, csd, engine, tag):
    """The bars of the head against FP64; prints the numbers.  -> the errors.

    Two stages.  hyper against FP64 on the injected trunk, with test_single_op's per-op bar; then pred313 + the decode
    kernels against FP64 on the engine's own hyper.  The chained pred_ab (FP64 from the trunk) is held to the same bar on
    the wgmma engine.  The SIMT engine sums hyper's K = 12 800 products in one FP32 accumulator, so its hyper is ~8x
    further from FP64 than wgmma's (measured on an H100: 1.7e-5 vs 2.5e-6 at 256^2), and the T = 2.6 softmax turns that
    into a chained pred_ab error of 9.9e-4 at 256^2 and 1.4e-3 at 512^2; for it the chained number is printed, and both
    stages it is made of keep their bars."""
    H, W = ctx.H, ctx.W
    n = out["pred"].shape[0]
    hy, hy64 = out["hyper"], spec["hyper64"]
    assert hy.shape == hy64.shape == (n, 384, H // 4, W // 4)
    hy_err, hy_scale = util.maxabs(hy, hy64), float(np.abs(hy64).max())
    own = _spec_from_hyper(csd, hy)
    d = out["map"]
    assert d.shape == spec["dist64"].shape == (n, 313, H, W) and d.dtype == np.float32
    map_err, map_own = util.maxabs(d, spec["dist64"]), util.maxabs(d, own["dist"])
    map_sum = float(np.abs(d.sum(1, dtype=np.float64) - 1.0).max())
    pd = np.abs(out["pred"].astype(np.float64) - spec["pred64"])
    pred_err, pred_err32 = float(pd.max()), util.maxabs(out["pred"], spec["pred32"])
    pred_own = util.maxabs(out["pred"], own["pred"])
    ref32_vs_64 = util.maxabs(spec["pred32"], spec["pred64"])
    bar = max(1e-3, 2.0 * ref32_vs_64)
    (wn, wc, wy, wx), gap = _worst(pd, spec["logits64"])
    print("%s: hyper vs FP64 %.3e (|out|max %.2f); map vs FP64 %.3e (on its own hyper %.3e), max|sum-1| %.3e; pred_ab vs "
          "FP64 %.3e (on its own hyper %.3e), vs FP32 oracle %.3e (FP32 oracle vs FP64 %.3e), worst pixel (n=%d, c=%d, "
          "y=%d, x=%d) top-2 logit gap %.3f" % (tag, hy_err, hy_scale, map_err, map_own, map_sum, pred_err, pred_own,
                                                pred_err32, ref32_vs_64, wn, wc, wy, wx, gap))
    assert hy_err < 2e-5 * max(1.0, hy_scale), (tag, hy_err, hy_scale)
    assert map_err < TOL_MAP and map_own < TOL_MAP and map_sum < TOL_MAP, (tag, map_err, map_own, map_sum)
    assert pred_own <= bar, (tag, pred_own, ref32_vs_64)
    if engine == "wgmma":
        assert pred_err <= bar, (tag, pred_err, ref32_vs_64)
    for i in range(n):
        err = _entropy_err(out["neg"][i], caffe313_ref.negentropy(d[i]))
        assert err <= TOL_ENT, (tag, i, err)
    return hy_err, map_err, pred_err


def _check_pixels(ctx, dmap, tag):
    """Every image's corners and, on the last image, _pixels(): dist313_pixel_kernel == dist313_map_kernel, bit for bit."""
    n, _, H, W = dmap.shape
    todo = [(n - 1, y, x) for (y, x) in _pixels(H, W, seed=H * W)]
    todo += [(i, y, x) for i in range(n - 1) for (y, x) in ((0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1))]
    for (i, y, x) in todo:
        px = ctx.caffe313_dist_pixel(i, y, x)
        assert np.array_equal(px.view(np.uint32), dmap[i, :, y, x].view(np.uint32)), (tag, i, y, x)
    print("%s: %d map pixels equal the single-pixel lookup bit for bit" % (tag, len(todo)))


@pytest.mark.parametrize("engine", ["simt", "wgmma"])
@pytest.mark.parametrize("geom", GEOMS, ids=_gid)
def test_head_ops_against_fp64(weights, synth_sd, geom, engine):
    sd, csd = weights
    H, W, n, max_n = geom
    t0 = time.time()
    case = _case(synth_sd, geom)
    ctx = util.make_ctx(sd, H, W, max_n=max_n, engine=engine, caffe313=True, use_graph=False)
    try:
        out, spec = _run_isolated(ctx, case, csd, engine)
        tag = "%s %s" % (_gid(geom), engine)
        _check_head(ctx, out, spec, csd, engine, tag)
        _check_pixels(ctx, out["map"], tag)
    finally:
        ctx.close()
    print("%s: %.1f s" % (tag, time.time() - t0))


# wgmma plan options on the head ops.  At 256^2, batch 1 the hyper launch is 4 classes x 8 tiles x 3 n-tiles = 96 tiles:
# more than half an H100's 132 SMs, so the automatic plan does not split K there; (72, 88, 2, 2) (48 tiles, split 2) and
# (8, 8, 1, 1) (12 tiles, split 4) are the geometries where split_k = 1 changes the plan.
VARIANTS = {"mt1": {"mt": 1}, "mt2": {"mt": 2}, "pairs0": {"pairs": 0}, "pairs2": {"pairs": 2}, "halo0": {"halo": 0},
            "halo3": {"halo": 3}, "split_k1": {"split_k": 1}}
# same arithmetic in the same order, only other tiles, clusters or operand loads: bit-identical
SCHEDULING_ONLY = ("mt1", "mt2", "pairs0", "pairs2", "halo0", "halo3")


@pytest.mark.parametrize("geom", [(256, 256, 1, 1), (72, 88, 2, 2), (8, 8, 1, 1)], ids=_gid)
def test_head_ops_under_plan_options(weights, synth_sd, geom):
    sd, csd = weights
    H, W, n, max_n = geom
    case = _case(synth_sd, geom)
    names = ["auto"] + (list(VARIANTS) if geom[0] == 256 else ["split_k1"])
    outs = {}
    for name in names:
        ctx = util.make_ctx(sd, H, W, max_n=max_n, engine="wgmma", caffe313=True, use_graph=False,
                            options=VARIANTS.get(name, {}))
        try:
            outs[name], spec = _run_isolated(ctx, case, csd, "wgmma")
            _check_head(ctx, outs[name], spec, csd, "wgmma", "%s wgmma %s" % (_gid(geom), name))
        finally:
            ctx.close()
    for name in names[1:]:
        same = all(np.array_equal(outs[name][k], outs["auto"][k]) for k in ("hyper", "pred", "map"))
        print("%s %s: %s the automatic plan" % (_gid(geom), name, "bit-identical to" if same else "differs from"))
        if name in SCHEDULING_ONLY or geom == (256, 256, 1, 1):      # split_k = 1 is the automatic plan there
            assert same, name
        else:                                                        # a split K sums in another order
            assert not same, name


@pytest.mark.parametrize("engine", ["simt", "wgmma"])
def test_forward_device_256(weights, synth_sd, engine):
    """Trunk + head as a user of the Caffe backend gets them, against the FP64 head on the FP32 oracle trunk.  hyper
    keeps test_gpu_forward.test_caffe313_head's bar, and pred_ab on the engine's own hyper its 1e-3; the chained pred_ab
    is held to TOL_CHAIN on the wgmma engine and printed for the SIMT engine (2.5e-3 on an H100: its trunk and hyper sum
    in single FP32 accumulators, see _check_head)."""
    sd, csd = weights
    geom = (256, 256, 1, 1)
    case = _case(synth_sd, geom)
    if "oracle" not in case["spec"]:
        case["spec"]["oracle"] = (None, _spec(csd, case["inter"]))
    spec = case["spec"]["oracle"][1]
    with torch.no_grad():
        _, _, _, hyper32 = caffe_spec.caffe313_head(csd, case["inter"], return_logits=True)
    assert float(np.abs(spec["pred64"]).max()) > 5.0
    ctx = util.make_ctx(sd, 256, 256, max_n=1, engine=engine, caffe313=True)
    try:
        ctx.forward_device(util.dev(case["L"]), util.dev(case["ab"]), util.dev(case["m"]), 0.5)
        torch.cuda.synchronize()
        hyper = ctx.get_activation("hyper", 1).cpu().numpy()
        pred = ctx.caffe313_pred_ab(1).cpu().numpy()
        dmap = ctx.caffe313_dist_map(1).cpu().numpy()
    finally:
        ctx.close()
    hy_err = util.maxabs(hyper, hyper32)
    pd = np.abs(pred.astype(np.float64) - spec["pred64"])
    err64, err32, ref32_vs_64 = float(pd.max()), util.maxabs(pred, spec["pred32"]), util.maxabs(spec["pred32"], spec["pred64"])
    err_own = util.maxabs(pred, _spec_from_hyper(csd, hyper)["pred"])
    (wn, wc, wy, wx), gap = _worst(pd, spec["logits64"])
    map_err = util.maxabs(dmap, spec["dist64"])
    print("forward_device 256 %s: hyper vs FP32 oracle %.3e; map vs FP64 %.3e; pred_ab vs FP64 %.3e (on its own hyper "
          "%.3e), vs FP32 oracle %.3e (FP32 oracle vs FP64 %.3e), worst pixel (c=%d, y=%d, x=%d) top-2 logit gap %.3f"
          % (engine, hy_err, map_err, err64, err_own, err32, ref32_vs_64, wc, wy, wx, gap))
    assert hy_err < 3e-4, hy_err
    assert err_own <= max(1e-3, 2.0 * ref32_vs_64), (err_own, ref32_vs_64)
    if engine == "wgmma":
        assert err64 <= TOL_CHAIN, err64
    assert map_err < TOL_MAP, map_err


def _mortar_case():
    g = util.golden("lhn_256.npz")
    ab, m = np.zeros((2, 256, 256)), np.zeros((1, 256, 256))
    pts = [((135, 160), 3, (23, -69)), ((100, 160), 3, (0, 0)), ((252, 3), 2, (-40, 60)), ((5, 250), 3, (70, 10))]
    for loc, p, val in pts:
        CI.put_point(ab, m, loc, p, val)
    return g["img_rgb"], ab, m, pts


def _caffe313_sd(synth_sd, csd):
    sd = util.caffe_scaled(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in csd.items() if k != "caffe.pts_in_hull"})     # prep_net adds its own
    return sd


def test_caffe_dist_wrapper_256(weights, synth_sd):
    """ColorizeImageB200CaffeDist(Xd=256), as the launcher's b200-caffe backend builds it, on the mortar image."""
    _, csd = weights
    img, ab, m, _ = _mortar_case()
    cd = CI.ColorizeImageB200CaffeDist(Xd=256)
    cd.prep_net(0, state_dict=_caffe313_sd(synth_sd, csd), S=.2)
    cd.set_image(img)
    rgb = cd.net_forward(ab, m)
    assert rgb.shape == (256, 256, 3) and rgb.dtype == np.uint8
    L = cd.img_l_mc.astype(np.float32)[None]
    _, inter = util.oracle_forward(synth_sd, L, ab[None].astype(np.float32), m[None].astype(np.float32), 0.0,
                                   intermediates=True)
    spec = _spec(csd, {k: inter[k] for k in TRUNK})
    own = _spec_from_hyper(csd, cd._ctx.get_activation("hyper", 1).cpu().numpy())
    err64, ref32_vs_64 = util.maxabs(cd.output_ab_raw, spec["pred64"][0]), util.maxabs(spec["pred32"], spec["pred64"])
    err_own = util.maxabs(cd.output_ab_raw, own["pred"][0])
    print("ColorizeImageB200CaffeDist 256: output_ab_raw vs FP64 %.3e (on its own hyper %.3e; FP32 oracle vs FP64 %.3e)"
          % (err64, err_own, ref32_vs_64))
    assert err64 <= TOL_CHAIN and err_own <= max(1e-3, 2.0 * ref32_vs_64), (err64, err_own, ref32_vs_64)
    assert np.array_equal(rgb, color_ref.lab2rgb_transpose(cd.img_l, cd.output_ab_raw.astype(np.float64)))
    d = np.asarray(cd.dist_ab)
    dev_map = cd._ctx.caffe313_dist_map(1)[0].cpu().numpy()
    assert d.shape == (313, 256, 256) and np.array_equal(d.view(np.uint32), dev_map.view(np.uint32))
    assert util.maxabs(d, spec["dist64"][0]) < TOL_MAP
    for (y, x) in ((0, 0), (0, 255), (255, 0), (255, 255)):
        assert np.array_equal(np.asarray(cd.dist_ab[:, y, x]).view(np.uint32), d[:, y, x].view(np.uint32)), (y, x)
    cd.compute_entropy()
    assert cd.dist_entropy.shape == (256, 256) and cd.dist_entropy.dtype == np.float32
    err = _entropy_err(cd.dist_entropy, caffe313_ref.negentropy(d))
    print("ColorizeImageB200CaffeDist 256: compute_entropy vs numpy %.3e" % err)
    assert err <= TOL_ENT
    for (y, x) in ((135, 160), (255, 255), (0, 0)):
        rec, conf = cd.get_ab_reccs(y, x, K=9, return_conf=True)
        assert rec.shape == (9, 2) and conf.shape == (9,), (y, x)
        assert abs(conf.sum() - 1.0) < 1e-4 and np.all(conf >= 0) and np.all(np.diff(conf) <= 1e-9), (y, x, conf)
        assert np.all(np.abs(rec) <= 110.0), (y, x)


def test_caffe_wrapper_256(synth_sd):
    """ColorizeImageB200Caffe(Xd=256): the regression output is the oracle's, scaled from tanh x 110 to tanh x 100."""
    img, ab, m, _ = _mortar_case()
    cc = CI.ColorizeImageB200Caffe(Xd=256)
    cc.prep_net(0, state_dict=util.caffe_scaled(synth_sd))
    cc.set_image(img)
    rgb = cc.net_forward(ab, m)
    L = cc.img_l_mc.astype(np.float32)[None]
    ref = util.oracle_forward(synth_sd, L, ab[None].astype(np.float32), m[None].astype(np.float32), 0.0)[0] * (100.0 / 110.0)
    err = util.maxabs(cc.output_ab_raw, ref)
    print("ColorizeImageB200Caffe 256: output_ab_raw vs oracle x 100/110 %.3e" % err)
    assert err <= TOL_AB
    assert np.array_equal(rgb, color_ref.lab2rgb_transpose(cc.img_l, cc.output_ab_raw.astype(np.float64)))


def test_caffe_hint_list_equals_dense_256(weights, synth_sd):
    """The hint-list click (hints rasterised on the device) gives the dense click's bits, on both Caffe classes."""
    _, csd = weights
    img, ab, m, pts = _mortar_case()
    rects = CI.hints_from_points(pts, 256)
    for make, sd in ((lambda: CI.ColorizeImageB200CaffeDist(Xd=256), _caffe313_sd(synth_sd, csd)),
                     (lambda: CI.ColorizeImageB200Caffe(Xd=256), util.caffe_scaled(synth_sd))):
        dense, hinted = make(), make()
        for w in (dense, hinted):
            w.prep_net(0, state_dict=sd)
            w.set_image(img)
        r1 = dense.net_forward(ab, m)
        r2 = hinted.net_forward_hints(rects)
        name = type(dense).__name__
        assert np.array_equal(r1, r2), name
        assert np.array_equal(dense.output_ab_raw, hinted.output_ab_raw), name
        if isinstance(dense, CI.ColorizeImageB200CaffeDist):
            assert np.array_equal(np.asarray(dense.dist_ab), np.asarray(hinted.dist_ab))
