"""GPU: the wrappers and photo batches against the UNMODIFIED reference wrapper, run live on the CPU in FP32 and FP64
(tests/live_ref.py).

Sessions as the notebook and the GUI drive them: `load_image` of seeded synthetic photos written as PNG (including one
with a side above Xfullres_max, which the reference zooms to the cap with an order-1 zoom of uint8), then a sequence of
put_point edits with a net_forward after each.  After every forward the port is compared with the reference's own
numbers, not with a restatement of them:

  * raw ab within TOL_AB of the FP32 reference (the north star) and of the FP64 reference;
  * get_img_forward differs by at most 1, and only where the float64 renders of the two raw ab maps -- both computed
    by the reference's own lab2rgb_transpose -- fall on different sides of an integer, or lie within 1e-9 of one;
    get_img_fullres equals the reference's own zoom and render of the port's output_ab (except within 1e-9 of an
    edge), and differs from the reference's result only where those renders differ;
  * the quantised output_ab within 2 ulps of the channel scale where the RGB is equal;
  * the getters that depend only on the inputs equal the reference except within 1e-9 of a truncation edge;
  * get_result_PSNR equal bit for bit to the reference's formula on the port's RGB, and within the bound the differing
    values allow of the reference's own PSNR;
  * the distribution wrapper's return value (x 110 twice), dist_ab and its views, compute_entropy and both
    get_ab_reccs methods; the launcher's share_trunk + hint_click pairing over a 20-click run;
  * PhotoColorizer.colorize and reveal_sweep against one reference session per photo.

The reference runs on the CPU; FP64 sessions are a subset, so that the file's CPU work stays near three minutes."""
import time

import cv2
import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import colorize_image as CI
from interactive_deep_colorization_b200 import photos
from oracle import synth
from tests import calibrated, live_ref, util

pytestmark = pytest.mark.gpu
TOL_AB = 1e-3
# DESIGN §11: on coherent (trained-like) networks the wgmma engine's chunked tensor-core sums miss TOL_AB on some
# images, where the exact-FP32 SIMT engine does not.  Measured here on an H100 80GB HBM3 (700 W), rho = 0.3: 4.8e-3 on
# the 2000 x 37 photo at Xd 256, 1.1e-3 on the 256² photo at Xd 64.  Every other case is held to TOL_AB.
TOL_AB_WGMMA_COHERENT = 6e-3
TOL_DIST = 1e-5
AB_ULPS = 2                      # rgb2lab on the device vs float64 numpy, in ulps of 500 (a) and 200 (b)
ENTROPY_SLACK = 5e-5             # logf against numpy's log (DESIGN §2)
PHOTOS = {"389x530": (389, 530), "256": (256, 256), "8": (8, 8), "1x300": (1, 300), "300x1": (300, 1),
          "2000x37": (2000, 37), "10007x12": (10007, 12)}
F32, F64 = torch.float32, torch.float64
_T0 = [None]


def _photo(H, W, seed):
    """A seeded synthetic photo: a cubic up-sample of coarse noise plus fine noise."""
    rs = np.random.RandomState(seed)
    coarse = rs.randint(0, 256, (max(H // 48, 2), max(W // 48, 2), 3)).astype(np.uint8)
    img = cv2.resize(coarse, (W, H), interpolation=cv2.INTER_CUBIC).astype(np.int16)
    img += rs.randint(-12, 13, (H, W, 3)).astype(np.int16)
    return np.clip(img, 0, 255).astype(np.uint8)


@pytest.fixture(scope="module")
def paths(tmp_path_factory):
    _T0[0] = time.perf_counter()
    d = tmp_path_factory.mktemp("live_ref_photos")
    out = {}
    for i, (name, (H, W)) in enumerate(PHOTOS.items()):
        out[name] = str(d / (name + ".png"))
        assert cv2.imwrite(out[name], _photo(H, W, 60 + i)[:, :, ::-1])
    yield out
    print("\ntest_gpu_live_reference: %.1f s in this module" % (time.perf_counter() - _T0[0]))


@pytest.fixture(scope="module")
def nets(synth_sd):
    """The weights as the reference module holds them (float32; the calibrated network's float64 BatchNorm statistics
    are rounded by its load_state_dict), given to both sides."""
    f32 = lambda sd: {k: (v.float() if torch.is_floating_point(v) else v) for k, v in sd.items()}
    cal = synth.synthetic_batch(4, 64, seed=0)
    return {"synthetic": f32(synth_sd), 0.3: f32(calibrated.trained_like(synth_sd, 0.3, cal))}


def edits(X, n=None):
    """The put_point edits of a session, (loc, p, val) each; None = a forward with no hints."""
    rs = np.random.RandomState(X)
    five = [(tuple(rs.randint(4, X - 4, 2)), p, tuple(rs.uniform(-80, 80, 2))) for p in (0, 1, 3, 1, 3)]
    out = [None, ((X // 2, X // 3), 0, (37.0, -21.0))] + five + [
        ((X - 2, X - 1), 3, (-40.0, 55.0)),              # clipped by the bottom-right edge
        ((1, X // 2), 3, (60.0, 10.0)),                  # rows -2:5: numpy wraps the start, the slice is empty
        ((X // 2 + 1, X // 3 + 2), 3, (-15.0, -60.0)),   # overlaps the 1 x 1 point
    ]
    return out[:n]


def click_run(X, n=20, seed=5):
    """BASELINE config 5: n clicks of put_point, p in 0 ... 3."""
    rs = np.random.RandomState(seed)
    return [(tuple(rs.randint(0, X, 2)), int(rs.randint(0, 4)), tuple(rs.uniform(-90, 90, 2))) for _ in range(n)]


# ---------------------------------------------------------------------------------------------------------------
# comparison rules
# ---------------------------------------------------------------------------------------------------------------
def _floor255(r):
    return np.floor(r[0]).astype(np.int64)


def straddle(got, want, r_got, r_want, what, max_diff=1):
    """uint8 `got` vs `want`: every difference is at most max_diff (None: unbounded), and where they differ the float64
    renders behind them (r_*, as (255 * clip(lab2rgb), 255 * lab2rgb)) truncate to different integers, or one of them
    lies within 1e-9 of an integer (the device's pow / cbrt may round that one the other way).  -> fraction of values
    that differ."""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    d = got.astype(np.int64) - want.astype(np.int64)
    if max_diff is not None:
        assert np.abs(d).max(initial=0) <= max_diff, (what, int(np.abs(d).max()))
    diff = d != 0
    explained = (_floor255(r_got) != _floor255(r_want)) | util.render_edges(r_got[0], unclipped=r_got[1]) | \
        util.render_edges(r_want[0], unclipped=r_want[1])
    bad = np.argwhere(diff & ~explained)
    assert len(bad) == 0, (what, len(bad), [(tuple(i), r_got[0][tuple(i)], r_want[0][tuple(i)]) for i in bad[:4]])
    return float(diff.mean())


def ref_render_of(ref, fn, **swap):
    """The reference's own render `fn` (a getter name) with some of its attributes temporarily replaced by the port's
    values -> [(clipped, unclipped)] of its lab2rgb_transpose calls."""
    cm = ref.cm
    old = {k: getattr(cm, k) for k in swap}
    try:
        for k, v in swap.items():
            setattr(cm, k, v)
        return ref.render(fn)[1]
    finally:
        for k, v in old.items():
            setattr(cm, k, v)


def check_inputs(port, ref, what, fullres=True):
    """The getters that depend only on the inputs: equal to the reference except within 1e-9 of a truncation edge.
    -> number of values excluded as edges."""
    names = ["get_img_gray", "get_input_img", "get_img_mask", "get_sup_img"]
    if fullres:
        names += ["get_img_gray_fullres", "get_input_img_fullres", "get_img_mask_fullres", "get_sup_fullres"]
    n_edge = 0
    for name in names:
        want, seen = ref.render(name)
        got = getattr(port, name)()
        assert got.shape == want.shape and got.dtype == np.uint8, (what, name, got.shape, want.shape)
        edge = util.render_edges(seen[-1][0], unclipped=seen[-1][1])
        bad = np.argwhere((got != want) & ~edge)
        assert len(bad) == 0, (what, name, len(bad), bad[:4].tolist())
        n_edge += int(edge.sum())
    return n_edge


def sse_bound(port_rgb, ref, ref_rgb):
    """(ΔSSE of the port's RGB against the reference's, the bound Σ(2|e| + 1) over the differing values, e the
    reference's error there), both with the reference's own get_result_PSNR."""
    _, se_port = ref.call("get_result_PSNR", port_rgb, return_SE_map=True)
    _, se_ref = ref.call("get_result_PSNR", ref_rgb, return_SE_map=True)
    diff = port_rgb != ref_rgb
    e = ref.cm.img_rgb.astype(np.float64) - ref_rgb
    return float(se_port.sum() - se_ref.sum()), float((2 * np.abs(e[diff]) + 1).sum())


def check_psnr(port, ref, ref_rgb, what):
    """get_result_PSNR() and get_result_PSNR(result, return_SE_map=True) -> ΔPSNR against the reference's own."""
    rgb = port.get_img_forward()
    assert port.get_result_PSNR() == ref.call("get_result_PSNR", rgb), what
    p1, se1 = port.get_result_PSNR(ref_rgb, return_SE_map=True)
    p2, se2 = ref.call("get_result_PSNR", ref_rgb, return_SE_map=True)
    assert p1 == p2 and np.array_equal(se1, se2), what
    dsse, bound = sse_bound(rgb, ref, ref_rgb)
    assert abs(dsse) <= bound, (what, dsse, bound)
    return port.get_result_PSNR() - ref.call("get_result_PSNR", ref_rgb)


def tol_ab(net, engine):
    return TOL_AB_WGMMA_COHERENT if (net != "synthetic" and engine == "wgmma") else TOL_AB


def port_render(ref, L_mc, raw):
    """The float64 render of raw ab the port's uint8 result truncates: the reference's own lab2rgb_transpose, on the
    FP32 L_mc the network reads plus 50 (DESIGN §2: the forward's fused render reads that L, not the float64 img_l)."""
    L = np.asarray(L_mc, np.float32).astype(np.float64) + 50.0
    return live_ref.capture_renders(ref.CI, lambda: ref.CI.lab2rgb_transpose(L, raw))[1][0]


def check_forward(port, refs, what, fullres=True, tol=TOL_AB):
    """Every check of one net_forward of the colour wrapper.  refs: [(name, RefSession, its net_forward return)],
    the FP32 reference first.  Prints one line."""
    raw = port.output_ab_raw.astype(np.float64)
    ref32 = refs[0][1]
    raws = {name: r.raw_ab() for name, r, _ in refs}
    dist = {name: float(np.abs(raw - a).max()) for name, a in raws.items()}
    line = ["%s:" % what] + ["|ab - %s| %.2e" % kv for kv in dist.items()]
    if "fp64" in raws:
        line.append("|fp32 - fp64| %.2e" % float(np.abs(raws["fp32"] - raws["fp64"]).max()))
    for name, d in dist.items():
        assert d <= tol, (what, name, d)
    # uint8 forward: the port's raw ab through the reference's own render, against each reference's render
    r_port = port_render(ref32, port.img_l_mc, raw)
    for name, r, (ret, seen) in refs:
        f = straddle(port.get_img_forward(), ret, r_port, seen[0], (what, name, "rgb"))
        line.append("rgb!=%s %.1e" % (name, f))
    ref_rgb = refs[0][2][0]
    # quantised output_ab where the RGB is equal
    same = np.all(port.output_rgb == ref_rgb, axis=-1)
    u = np.abs(np.asarray(port.output_ab, np.float64) - ref32.cm.output_ab) / np.spacing(np.array([500.0, 200.0]))[:, None, None]
    assert u[:, same].max(initial=0) <= AB_ULPS, (what, float(u[:, same].max()))
    # full-resolution result: the port's quantised ab zoomed by the reference's own statements
    if fullres:
        full_ref = ref32.render("get_img_fullres")
        # a 1-LSB difference at the network size moves the quantised ab by up to ~1, and the zoom carries that into
        # a larger full-resolution difference: there the port must equal the reference's own zoom and render of the
        # port's output_ab, and differ from the reference's result only where those two renders differ
        r_full = ref_render_of(ref32, "get_img_fullres", output_ab=np.asarray(port.output_ab, np.float64))[0]
        got = port.get_img_fullres()
        straddle(got, _floor255(r_full).astype(np.uint8), r_full, r_full, (what, "fullres vs its own render"))
        f = straddle(got, full_ref[0], r_full, full_ref[1][0], (what, "fullres"), max_diff=None)
        line.append("fullres!=fp32 %.1e" % f)
    line.append("edges %d" % check_inputs(port, ref32, what, fullres))
    line.append("dPSNR %+.2e" % check_psnr(port, ref32, ref_rgb, what))
    print("  ".join(line))


# ---------------------------------------------------------------------------------------------------------------
# colour wrapper sessions
# ---------------------------------------------------------------------------------------------------------------
# (photo, Xd, maskcent, network, engine, FP64 reference too, hints as a device hint list, edits)
SESSIONS = [
    ("389x530", 256, True, "synthetic", "wgmma", True, False, None),
    ("389x530", 256, False, 0.3, "simt", False, True, None),
    ("256", 64, False, "synthetic", "wgmma", True, True, None),
    ("8", 64, True, 0.3, "wgmma", True, False, None),
    ("1x300", 64, False, "synthetic", "simt", True, False, None),
    ("300x1", 64, True, 0.3, "wgmma", False, True, None),
    ("2000x37", 256, True, 0.3, "wgmma", False, False, None),
    ("10007x12", 64, False, "synthetic", "wgmma", True, False, None),
    ("256", 256, True, 0.3, "simt", True, False, 4),
    ("389x530", 512, True, "synthetic", "wgmma", False, False, 3),
]


def _sid(s):
    return "%s-X%d-%s-%s-%s%s%s" % (s[0], s[1], "mc" if s[2] else "nomc", "synth" if s[3] == "synthetic" else "rho0.3",
                                   s[4], "-fp64" if s[5] else "", "-hints" if s[6] else "")


@pytest.mark.parametrize("sess", SESSIONS, ids=[_sid(s) for s in SESSIONS])
def test_colour_session_against_reference(paths, nets, sess):
    photo, X, mc, net, engine, fp64, as_hints, n_edits = sess
    sd = nets[net]
    refs = [("fp32", live_ref.RefSession(sd, X, mc, dtype=F32))]
    if fp64:
        refs.append(("fp64", live_ref.RefSession(sd, X, mc, dtype=F64)))
    port = CI.ColorizeImageB200(Xd=X, maskcent=mc, engine=engine)
    port.prep_net(state_dict=sd)
    port.load_image(paths[photo])
    for _, r in refs:
        r.call("load_image", paths[photo])
    ref32 = refs[0][1].cm
    assert np.array_equal(port.img_rgb, ref32.img_rgb)
    assert np.shape(port.img_l_fullres) == ref32.img_l_fullres.shape, (np.shape(port.img_l_fullres), ref32.img_l_fullres.shape)
    ab, mask = np.zeros((2, X, X)), np.zeros((1, X, X))
    points = []
    for k, e in enumerate(edits(X, n_edits)):
        if e is not None:
            CI.put_point(ab, mask, *e)
            points.append(e)
        if as_hints:
            port.net_forward_hints(CI.hints_from_points(points, X))
            assert np.array_equal(port.input_ab, ab) and np.array_equal(port.input_mask, mask)
        else:
            port.net_forward(ab.copy(), mask.copy())
        outs = [(name, r, r.render("net_forward", ab.copy(), mask.copy())) for name, r in refs]
        check_forward(port, outs, "%s edit %d" % (_sid(sess), k), tol=tol_ab(net, engine))


# ---------------------------------------------------------------------------------------------------------------
# distribution wrapper
# ---------------------------------------------------------------------------------------------------------------
def weighted_inertia(pmf, pts, centres):
    d = ((pts[:, None, :] - centres[None, :, :]) ** 2).sum(-1).min(1)
    return float((pmf * d).sum())


def check_dist(port, ret, refs, rs, what, whole=False):
    """One net_forward of the distribution wrapper against the references ([(name, RefSession, return value)],
    FP32 first).  -> (pixels whose sampled reccs drew identical samples, pixels compared)."""
    X = port.Xd
    for name, r, rret in refs:
        d = float(np.abs(ret - rret).max())
        assert d <= 110 * TOL_AB, (what, name, "x110 return", d)            # the x110 is applied twice on both sides
        assert float(np.abs(port.output_ab_raw.astype(np.float64) - r.raw_ab()).max()) <= TOL_AB, (what, name)
    assert np.array_equal(ret, port.output_ab_raw * 110.0), what
    pix = [tuple(p) for p in rs.randint(0, X, (24, 2))]
    grid = np.asarray(port.dist_ab)
    for name, r, _ in refs:
        ref_d = r.cm.dist_ab
        for h, w in pix:
            assert np.abs(port.dist_ab[:, h, w] - ref_d[:, h, w]).max() <= TOL_DIST, (what, name, h, w)
            assert np.abs(port.dist_ab_full[:, h, w] - r.cm.dist_ab_full[:, h, w]).max() <= TOL_DIST, (what, name)
        assert np.abs(grid[:, ::4, ::4] - ref_d[:, ::4, ::4]).max() <= TOL_DIST, (what, name)
        if whole:
            assert np.abs(grid - ref_d).max() <= TOL_DIST, (what, name)
    for h, w in pix[:4]:
        col = np.asarray(port.dist_ab[:, h, w], np.float64)
        assert np.array_equal(port.dist_ab_full[:, h, w], col)
        assert np.array_equal(port.dist_ab_grid[:, :, h, w], col.reshape(23, 23))
    if whole:
        assert np.array_equal(np.asarray(port.dist_ab_full), grid.astype(np.float64))
        assert np.array_equal(np.asarray(port.dist_ab_grid), grid.astype(np.float64).reshape(23, 23, X, X))
    # compute_entropy: NaN where a bin is 0, elsewhere within the first-order bound of the bins' differences
    ref32 = refs[0][1]
    port.compute_entropy()
    with np.errstate(divide="ignore", invalid="ignore"):
        ref32.call("compute_entropy")
    e_p, e_r = port.dist_entropy[::4, ::4], ref32.cm.dist_entropy[::4, ::4]
    d_p, d_r = grid[:, ::4, ::4].astype(np.float64), ref32.cm.dist_ab[:, ::4, ::4].astype(np.float64)
    one_zero = (d_p == 0).any(0) != (d_r == 0).any(0)
    assert np.array_equal(np.isnan(e_p)[~one_zero], np.isnan(e_r)[~one_zero]), what
    ok = ~np.isnan(e_r) & ~np.isnan(e_p)
    with np.errstate(divide="ignore"):
        bound = (np.abs(d_p - d_r) * (np.abs(np.log(d_r)) + 1)).sum(0) + ENTROPY_SLACK
    assert (np.abs(e_p - e_r) <= bound)[ok].all(), (what, float(np.abs(e_p - e_r)[ok].max()))
    # get_ab_reccs(method='sampled') after the same seed on both sides
    same = 0
    N = 2000
    for k, (h, w) in enumerate(pix[:6]):
        s = 100 + k
        got = []
        for cm, kw in ((port, {"method": "sampled"}), (ref32.cm, {})):
            np.random.seed(s)
            with live_ref.precision(F32), live_ref.one_thread():
                got.append(cm.get_ab_reccs(h, w, K=5, N=N, return_conf=True, **kw))
        u = np.random.RandomState(s).uniform(0, 1, N)
        cdf_p, cdf_r = np.cumsum(np.asarray(port.dist_ab[:, h, w])), np.cumsum(ref32.cm.dist_ab[:, h, w])
        cdf_p, cdf_r = cdf_p / cdf_p[-1], cdf_r / cdf_r[-1]
        if np.array_equal(np.digitize(u, cdf_p), np.digitize(u, cdf_r)):
            same += 1
            assert np.array_equal(got[0][0], got[1][0]) and np.array_equal(got[0][1], got[1][1]), (what, h, w)
    # method='gpu': the weighted k-means limit is at least as tight as the reference's sampled answer
    pts = ref32.cm.pts_in_hull.astype(np.float64)
    for k, (h, w) in enumerate(pix[6:9]):
        pmf = ref32.cm.dist_ab[:, h, w].astype(np.float64)
        np.random.seed(200 + k)
        with live_ref.precision(F32):
            c_ref = ref32.cm.get_ab_reccs(h, w, K=5)
        c_gpu = port.get_ab_reccs(h, w, K=5)
        assert weighted_inertia(pmf, pts, c_gpu) <= 1.01 * weighted_inertia(pmf, pts, c_ref), (what, h, w)
    return same, 6, int(one_zero.sum())


DIST_SESSIONS = [
    ("389x530", 256, True, "synthetic", "wgmma", True),
    ("256", 64, False, 0.3, "simt", True),
    ("8", 64, True, 0.3, "wgmma", False),
]


@pytest.mark.parametrize("sess", DIST_SESSIONS, ids=[_sid(s + (False,)) for s in DIST_SESSIONS])
def test_dist_session_against_reference(paths, nets, sess):
    photo, X, mc, net, engine, fp64 = sess
    sd = nets[net]
    refs = [("fp32", live_ref.RefSession(sd, X, mc, dist=True, dtype=F32))]
    if fp64:
        refs.append(("fp64", live_ref.RefSession(sd, X, mc, dist=True, dtype=F64)))
    port = CI.ColorizeImageB200Dist(Xd=X, maskcent=mc, engine=engine)
    port.prep_net(state_dict=sd)
    port.load_image(paths[photo])
    for _, r in refs:
        r.call("load_image", paths[photo])
    ab, mask = np.zeros((2, X, X)), np.zeros((1, X, X))
    rs = np.random.RandomState(X)
    same = total = 0
    for k, e in enumerate(edits(X, 4)):
        if e is not None:
            CI.put_point(ab, mask, *e)
        ret = port.net_forward(ab.copy(), mask.copy())
        outs = [(name, r, r.call("net_forward", ab.copy(), mask.copy())) for name, r in refs]
        s, n, one_zero = check_dist(port, ret, outs, rs, "%s edit %d" % (sess, k), whole=(X == 64))
        same, total = same + s, total + n
        print("%s edit %d: sampled reccs with identical samples %d of %d, pixels with one-sided zero bins %d"
              % (sess, k, s, n, one_zero))
    assert same * 2 > total, (same, total)


def test_launcher_pairing_over_a_click_run(paths, nets):
    """launcher.build_models with share_trunk, the GUI's hint_click before each click, against the reference pair
    (ColorizeImageTorch + ColorizeImageTorchDist, each with its own forward) over the 20-click run."""
    X, sd = 256, nets["synthetic"]
    ref_c = live_ref.RefSession(sd, X, True, dtype=F32)
    ref_d = live_ref.RefSession(sd, X, True, dist=True, dtype=F32)
    colour = CI.ColorizeImageB200(Xd=X, maskcent=True)
    colour.prep_net(state_dict=sd, dist=True)
    dist = CI.ColorizeImageB200Dist(Xd=X, maskcent=True)
    dist.share_trunk(colour)
    for m in (colour, dist):
        m.load_image(paths["389x530"])
    for r in (ref_c, ref_d):
        r.call("load_image", paths["389x530"])
    ab, mask = np.zeros((2, X, X)), np.zeros((1, X, X))
    pts = ref_d.cm.pts_in_hull.astype(np.float64)
    worst, ratio = 0.0, 0.0
    for k, (loc, p, val) in enumerate(click_run(X)):
        CI.put_point(ab, mask, loc, p, val)
        h, w = loc
        dist.hint_click(h, w, K=9)
        ret = dist.net_forward(ab.copy(), mask.copy())                  # predict_color, then the suggestions
        rret = ref_d.call("net_forward", ab.copy(), mask.copy())
        assert float(np.abs(ret - rret).max()) <= 110 * TOL_AB, k
        col = np.asarray(dist.dist_ab[:, h, w], np.float64)
        assert np.abs(col - ref_d.cm.dist_ab[:, h, w]).max() <= TOL_DIST, k
        np.random.seed(k)
        with live_ref.precision(F32):
            c_ref = ref_d.cm.get_ab_reccs(h, w, K=9)
        c_gpu = dist.get_ab_reccs(h, w, K=9)
        pmf = ref_d.cm.dist_ab[:, h, w].astype(np.float64)
        # K = 9 on the synthetic network's nearly flat pmfs has many local optima, and the device's restarts do not
        # always reach as good a one as the reference's sampled k-means: up to 6.5 % worse on an H100 (click 15;
        # DESIGN §11).  K = 5 is held to 1 % in the dist sessions.
        ratio = max(ratio, weighted_inertia(pmf, pts, c_gpu) / weighted_inertia(pmf, pts, c_ref))
        assert ratio <= 1.10, (k, ratio)
        colour.net_forward(ab.copy(), mask.copy())                      # compute_result
        out = [("fp32", ref_c, ref_c.render("net_forward", ab.copy(), mask.copy()))]
        worst = max(worst, util.maxabs(colour.output_ab_raw, dist.output_ab_raw))
        check_forward(colour, out, "pairing click %d" % k, fullres=(k % 5 == 4))
    print("pairing: worst weighted-inertia ratio of the K = 9 suggestions to the reference's %.4f" % ratio)
    assert worst == 0.0                              # one forward per click serves both models


# ---------------------------------------------------------------------------------------------------------------
# photo batches
# ---------------------------------------------------------------------------------------------------------------
BATCH_PHOTOS = ["389x530", "256", "8", "1x300", "300x1", "2000x37"]     # 10007 x 12 is refused by photo batches


def _batch_check(rgb, ab, psnr, ref, rret, what, tol):
    """A batch result (network-size rgb, raw ab, psnr) against a reference session after its net_forward."""
    d = float(np.abs(ab.astype(np.float64) - ref.raw_ab()).max())
    assert d <= tol, (what, d)
    r_port = port_render(ref, ref.cm.img_l - 50.0, ab.astype(np.float64))
    f = straddle(rgb, rret[0], r_port, rret[1][0], (what, "rgb"))
    assert psnr == ref.call("get_result_PSNR", rgb), what
    dsse, bound = sse_bound(rgb, ref, rret[0])
    assert abs(dsse) <= bound, (what, dsse, bound)
    return d, f, psnr - ref.call("get_result_PSNR")


def test_photo_batches_against_reference(paths, nets):
    X, sd = 64, nets[0.3]
    files = [paths[p] for p in BATCH_PHOTOS]
    pc = photos.PhotoColorizer(sd, Xd=X, batch=4, maskcent=True)      # passes of 4 and 2 photos
    res = list(pc.colorize(files, psnr=True))
    zeros = (np.zeros((2, X, X)), np.zeros((1, X, X)))
    for i, f in enumerate(files):
        ref = live_ref.RefSession(sd, X, True, dtype=F32)
        ref.call("load_image", f)
        rret = ref.render("net_forward", *zeros)
        d, fr, dp = _batch_check(res[i].rgb, res[i].ab, res[i].psnr, ref, rret, ("colorize", BATCH_PHOTOS[i]),
                                  tol_ab(0.3, "wgmma"))
        # full resolution: the port's RGB re-derived to output_ab by the reference's own statements, then zoomed
        ref.cm.output_rgb, keep = res[i].rgb, ref.cm.output_rgb
        ref.call("_set_out_ab_")
        r_full = ref.render("get_img_fullres")[1][0]
        ref.cm.output_rgb = keep
        ref.call("_set_out_ab_")
        full_ref = ref.render("get_img_fullres")
        straddle(res[i].fullres, _floor255(r_full).astype(np.uint8), r_full, r_full, ("colorize fullres own", BATCH_PHOTOS[i]))
        ff = straddle(res[i].fullres, full_ref[0], r_full, full_ref[1][0], ("colorize fullres", BATCH_PHOTOS[i]),
                      max_diff=None)
        print("colorize %s: |ab - fp32| %.2e  rgb!=fp32 %.1e  fullres!=fp32 %.1e  dPSNR %+.2e"
              % (BATCH_PHOTOS[i], d, fr, ff, dp))
    levels, seed = (0, 1, 5, 50), 4
    pc16 = photos.PhotoColorizer(sd, Xd=X, batch=16, maskcent=True)   # four photos per pass, then two
    sweep = list(pc16.reveal_sweep(files, levels=levels, seed=seed))
    for i, f in enumerate(files):
        ref = live_ref.RefSession(sd, X, True, dtype=F32)
        ref.call("load_image", f)
        pts = photos.reveal_points(X, max(levels), seed, i)
        assert np.array_equal(sweep[i].points, pts)
        for j, m in enumerate(levels):
            ab, mask = np.zeros((2, X, X)), np.zeros((1, X, X))
            for y0, x0, P in pts[:m]:                   # put_point's slice assignment, P x P from the corner
                ab[:, y0:y0 + P, x0:x0 + P] = ref.cm.img_ab[:, y0:y0 + P, x0:x0 + P].mean(axis=(1, 2))[:, None, None]
                mask[:, y0:y0 + P, x0:x0 + P] = 1
            rret = ref.render("net_forward", ab, mask)
            d, fr, dp = _batch_check(sweep[i].rgb[j], sweep[i].ab[j], sweep[i].psnr[j], ref, rret,
                                     ("reveal", BATCH_PHOTOS[i], m), tol_ab(0.3, "wgmma"))
            print("reveal %s level %d: |ab - fp32| %.2e  rgb!=fp32 %.1e  dPSNR %+.2e" % (BATCH_PHOTOS[i], m, d, fr, dp))
    pc.close()
    pc16.close()
