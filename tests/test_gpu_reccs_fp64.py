"""GPU: the colour-suggestion k-means (ab_reccs_kernel and the kernels around it, csrc/idc_heads.cu) against its FP64
statement, oracle/reccs_ref.weighted_kmeans_pmf, fed exactly the pmf the kernel used, on every path that runs it:
idc_ab_reccs_pmf on crafted pmfs, idc_ab_reccs on the resident distribution of the wgmma and SIMT engines, the announced
click, idc_ab_reccs_batch and idc_caffe313_reccs_batch with out_pmf, and the wrappers' get_ab_reccs(method='gpu').

Both sides compute in FP64 and round each other's decisions alike unless a decision is within rounding of a tie.  The
oracle traces the relative margin of every decision (seeding arg-max, Lloyd arg-min over all points, mass order, restart
pick).  A query whose seeding, mass-order and pick margins all exceed 1e-12 must give the oracle's picked restart, with
every float32 centre and mass within 1 ulp of float32(oracle), and its Lloyd iteration count -- one iteration apart at
most where a Lloyd label sits within rounding of a tie.  A query below the margin is checked only on weighted inertia
(within 1e-9 relative of the oracle's picked restart with its centres rounded to float32) and counted; only symmetric
crafted pmfs may have such queries.  The peaked network makes Lloyd ties: subnormal-weight bins pull a centre ~1e-10 off
its grid bin, perpendicular to the line to a bin 10 away, whose squared distances to it and to another grid centre then
both round to 100.0.  Most such labels belong to inert points (weight 0, or below 2^-60 of their clusters' mass:
reccs_ref's "lloyd_inert"), which move no centre or mass, only the step at which the assignment counts as stable; every
query with a Lloyd tie is still held to 1 ulp.  Each case prints the queries compared, the exclusions, the Lloyd ties (and how many of
them cost an iteration) and the worst centre / mass error in ulps."""
import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import prepost
from interactive_deep_colorization_b200.engine import LhnContext
from oracle import caffe_spec, reccs_ref as R, synth
from tests import calibrated, gpu_cases, head_ref, util

pytestmark = pytest.mark.gpu
GRID = R.torch_gamut_points()
PTS313 = prepost.pts_in_hull()
MARGIN = 1e-12


CENTRE_FLOOR = 2.0 ** -16   # ab units: a centre coordinate that cancels to ~0 (the uniform pmf's mean) is measured in
                            # ulps of 2^-16 (1.8e-12), still ~100x the FP64 sums' own rounding of a mean of |ab| <= 110


def _ulps(got, ref, floor=0.0):
    """|got - float32(ref)| in float32 ulps of float32(max(|ref|, floor))"""
    r = np.asarray(ref, np.float64).astype(np.float32)
    d = np.abs(np.asarray(got, np.float32).astype(np.float64) - r.astype(np.float64))
    return float((d / np.spacing(np.maximum(np.abs(r), np.float32(floor))).astype(np.float64)).max(initial=0.0))


class Tally:
    def __init__(self, name):
        self.name, self.n, self.excluded, self.uc, self.um = name, 0, 0, 0.0, 0.0
        self.lloyd_ties = self.inert_only = self.longer = 0

    def check(self, pmf, pts, K, max_iter, n_init, c, m, it, tag="", tie_ok=False):
        """One query: the kernel's (centres [K,2], mass [K], iterations) against the oracle on the same pmf.

        The seeding, mass-order and restart-pick decisions must be above the margin, unless tie_ok (a symmetric crafted
        pmf).  Then the centres and mass are within 1 ulp of the oracle's picked restart, and the iteration count is
        the oracle's -- or, where a Lloyd label sits within rounding of a tie, at most one off: on the peaked network
        those labels belong to points of weight 0 or far below their clusters' mass, which move no centre or mass and
        only decide when the assignment counts as stable.  A tie_ok query below the margin is checked on weighted
        inertia against the oracle's float32-rounded centres, to 1e-9 relative."""
        co, mo, io, mg = R.weighted_kmeans_pmf(pmf, pts, K, max_iter, n_init, trace=True)
        self.n += 1
        c, m = np.asarray(c, np.float32), np.asarray(m, np.float32)
        assert c.shape == (K, 2) and m.shape == (K,)
        uc, um = _ulps(c, co, CENTRE_FLOOR), _ulps(m, mo)
        if min(mg["seed"], mg["order"], mg["pick"]) > MARGIN:
            self.uc, self.um = max(self.uc, uc), max(self.um, um)
            lloyd_tie = min(mg["lloyd"], mg["lloyd_inert"]) <= MARGIN
            self.lloyd_ties += lloyd_tie
            self.inert_only += lloyd_tie and mg["lloyd"] > MARGIN
            self.longer += it != io
            assert uc <= 1 and um <= 1 and (it == io or (lloyd_tie and abs(int(it) - io) == 1)), \
                (self.name, tag, K, max_iter, n_init, it, io, uc, um, mg)
        else:
            assert tie_ok, ("below the margin", self.name, tag, K, max_iter, n_init, mg)
            self.excluded += 1
            e, eo = R.weighted_inertia(pmf, pts, c), R.weighted_inertia(pmf, pts, co.astype(np.float32))
            assert abs(e - eo) <= 1e-9 * eo, (self.name, tag, K, e, eo, mg)
        return mg

    def report(self):
        print("%s: %d queries compared, %d below the %g margin (symmetric pmfs); %d with a Lloyd label within rounding "
              "of a tie (%d of them on inert points only), %d of those one Lloyd iteration apart; worst centre %.2f ulp, "
              "worst mass %.2f ulp" % (self.name, self.n, self.excluded, MARGIN, self.lloyd_ties, self.inert_only,
                                       self.longer, self.uc, self.um))
        assert self.n > 0


# ---------------------------------------------------------------------------------------------------------------------
# idc_ab_reccs_pmf on crafted pmfs
# ---------------------------------------------------------------------------------------------------------------------
def _support(idx, w):
    p = np.zeros(529, np.float32)
    p[idx] = w
    return p


def _sm(seed, s=2.0):
    """softmax of seeded Gaussian logits of spread s"""
    z = np.random.RandomState(seed).randn(529) * s
    e = np.exp(z - z.max())
    return (e / e.sum()).astype(np.float32)


def _two_equal_top():
    p = _sm(11)
    top = np.argsort(p)
    p[top[-2]] = p[top[-1]]
    return p


def _dup_table():
    """the grid with bins 0..19 moved onto bins 200..219 (weighted duplicates), under a pmf that weighs them"""
    pts = GRID.copy()
    pts[:20] = GRID[200:220]
    return pts


# name -> (pmf, pts or None, [(K, max_iter, n_init)], the K at which the pmf's symmetry makes ties).  The small supports have dyadic weights, so every
# centre stays exactly on its bin and each tie they make (seeds repeated at bin 0, empty clusters) is exact.
KS = (1, 2, 3, 5, 9, 17, 32)
CRAFTED = {
    "support1": (_support([300], [1.0]), None, [(K, 100, n) for K in KS for n in (8, 16)], ()),
    "support2": (_support([40, 412], [0.75, 0.25]), None, [(K, 100, n) for K in KS for n in (8, 16)], ()),
    "support3_bin528": (_support([17, 250, 528], [0.5625, 0.28125, 0.15625]), None,
                        [(K, 100, n) for K in KS for n in (8, 16)], ()),
    # four bins of one weight: at K >= 4 equal single-bin masses, ordered by the stable sort (cluster index); at K = 2
    # two clusters of two bins each tie on mass
    "support4_equal": (_support([40, 100, 412, 470], [0.25] * 4), None, [(K, 100, n) for K in KS for n in (1, 8, 16)],
                       (2,)),
    "support5": (_support([3, 120, 261, 333, 515], [0.3125, 0.25, 0.1875, 0.15625, 0.09375]), None,
                 [(K, 100, n) for K in KS for n in (1, 8, 16)], ()),
    "softmax": (_sm(1), None, [(K, 100, n) for K in KS for n in (1, 8, 16)], ()),
    # the flat 1e-6 floor of the blobs makes clusters of equal mass at K = 32
    "blobs": (R.synthetic_pmf("blobs", 0).astype(np.float32), None, [(K, 100, 8) for K in KS], (32,)),
    "max_iter": (_sm(2), None, [(K, mi, 8) for K in (5, 9, 32) for mi in (1, 2, 3)], ()),
    "scale_1e-30": ((_sm(3, 3.0) * 1e-30).astype(np.float32), None, [(K, 100, 8) for K in (2, 5, 9, 32)], ()),
    "scale_1e30": ((_sm(4, 3.0) * 1e30).astype(np.float32), None, [(K, 100, 8) for K in (2, 5, 9, 32)], ()),
    "ab_swapped_grid": (_sm(5), GRID[:, ::-1].copy(), [(K, 100, 8) for K in (3, 9, 32)], ()),
    "duplicate_points": (_sm(6), _dup_table(), [(K, 100, 8) for K in (3, 9, 32)], ()),
    "two_equal_top": (_two_equal_top(), None, [(K, 100, n) for K in (1, 2, 5, 9) for n in (2, 8)], ()),
    "uniform": (np.full(529, 1.0 / 529, np.float32), None, [(K, 100, 8) for K in (1, 2, 5, 9)], (2, 5, 9)),
}


@pytest.mark.parametrize("name", list(CRAFTED))
def test_crafted_pmfs(name):
    pmf, pts, runs, tie_ks = CRAFTED[name]
    pp = GRID if pts is None else pts
    t = Tally("ab_reccs_pmf " + name)
    nz = int(np.count_nonzero(pmf))
    for K, max_iter, n_init in runs:
        c, m, it = prepost.ab_reccs_pmf_gpu(pmf, K=K, max_iter=max_iter, n_init=n_init, pts=pts)
        t.check(pmf, pp, K, max_iter, n_init, c, m, it, tie_ok=K in tie_ks)
        if name == "max_iter":
            assert it == max_iter                      # every one of these runs stops on the cap
        if K > nz:                                     # more clusters than non-zero bins: the rest are empty
            assert np.all(m[nz:] == 0) and np.array_equal(m[:nz], np.sort(pmf[pmf > 0])[::-1])
    t.report()


def test_caffe_padded_pmf_single_call():
    """get_ab_reccs of the Caffe wrapper feeds 313 bins zero-padded to 529 with (0, 0) rows; the oracle on the unpadded
    313 bins is the answer."""
    t = Tally("ab_reccs_pmf caffe313 padded")
    for seed in range(4):
        z = np.random.RandomState(20 + seed).randn(313) * (1.0 + 2 * seed)
        p313 = np.exp(z - z.max())
        p313 = (p313 / p313.sum()).astype(np.float32)
        p, q = np.zeros(529, np.float32), np.zeros((529, 2), np.float32)
        p[:313], q[:313] = p313, PTS313
        for K in (1, 5, 9, 32):
            c, m, it = prepost.ab_reccs_pmf_gpu(p, K=K, pts=q)
            t.check(p313, PTS313, K, 100, 8, c, m, it)
    t.report()


# ---------------------------------------------------------------------------------------------------------------------
# network pmfs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nets(synth_sd):
    rho = calibrated.trained_like(synth_sd, 0.3, gpu_cases.calibration_batch())
    return {"synth": synth_sd, "peak": head_ref.peaked(rho, util.small_batch(2, 64, seed=300), 100.0)}


def _resident(sd, X, n, engine="wgmma", seed=3):
    ctx = LhnContext(device=0, max_n=n, H=X, W=X, dist=True, engine=engine)
    ctx.load_state_dict(sd)
    ctx.set_dist_resident(True)
    L, ab, m = synth.synthetic_batch(n, X, seed=seed, max_hints=6)
    ctx.forward_host(L, ab, m, 0.5)
    return ctx, (L, ab, m)


def _pixels(ctx, n, G, count, seed):
    """(img, y4, x4): every image's corners, up to a third of the sample at pixels with a zero bin, then seeded ones"""
    q = []
    for i in range(n):
        q += [(i, 0, 0), (i, 0, G - 1), (i, G - 1, 0), (i, G - 1, G - 1)]
    rs = np.random.RandomState(seed)
    zero = []
    for i in range(n):
        d = ctx.fetch_dist(i)
        ys, xs = np.nonzero((d == 0).any(0))
        zero += [(i, int(y), int(x)) for y, x in zip(ys, xs)]
    if zero:
        q += [zero[j] for j in rs.choice(len(zero), min(len(zero), count // 3), replace=False)]
    while len(q) < count:
        q.append((int(rs.randint(n)), int(rs.randint(G)), int(rs.randint(G))))
    return q, len(zero)


@pytest.mark.parametrize("engine", ["wgmma", "simt"])
@pytest.mark.parametrize("net", ["synth", "peak"])
def test_resident_single_pixel(nets, engine, net):
    X, n = 64, 2
    ctx, _ = _resident(nets[net], X, n, engine)
    q, nzero = _pixels(ctx, n, X // 4, 40, 1)
    t = Tally("ab_reccs %s %s (%d pixels with a zero bin)" % (engine, net, nzero))
    if net == "peak":
        assert nzero > 0
    for j, (img, y4, x4) in enumerate(q):
        K = (9, 5, 1, 32, 17)[j % 5]
        c, m, it = ctx.ab_reccs(img, y4, x4, K=K)
        t.check(ctx.fetch_dist(img, y4, x4), GRID, K, 100, 8, c, m, it, (img, y4, x4))
    ctx.close()
    t.report()


@pytest.mark.parametrize("net", ["synth", "peak"])
def test_announced_click(nets, net):
    """set_click + forward_host: the click graph's side branch clusters the clicked pixel with K from the click header;
    ab_reccs / fetch_dist for that pixel are answered from the block it brought back."""
    X = 128
    ctx = LhnContext(device=0, max_n=1, H=X, W=X, dist=True)
    ctx.load_state_dict(nets[net])
    ctx.set_dist_resident(True)
    L, ab, m = synth.synthetic_batch(1, X, seed=12, max_hints=5)
    t = Tally("click %s" % net)
    G = X // 4
    for y4, x4, K in ((0, 0, 9), (G - 1, G - 1, 32), (0, G - 1, 1), (G - 1, 0, 5), (10, 20, 17), (31, 7, 2)):
        ctx.set_click(0, y4, x4, K)
        ctx.forward_host(L, ab, m, 0.5)
        c, f, it = ctx.ab_reccs(0, y4, x4, K=K)
        t.check(ctx.fetch_dist(0, y4, x4), GRID, K, 100, 8, c, f, it, (y4, x4))
    ctx.close()
    t.report()


def _batch(ctx, q, K, max_iter=100, n_init=8, caffe=False):
    out_pmf = torch.full((len(q), 529), -1.0, dtype=torch.float32, device="cuda")
    if caffe:
        c, f, it = ctx.caffe313_reccs_batch(q, K=K, S=0.2, max_iter=max_iter, n_init=n_init, out_pmf=out_pmf)
    else:
        c, f, it = ctx.ab_reccs_batch(q, K=K, max_iter=max_iter, n_init=n_init, out_pmf=out_pmf)
    torch.cuda.synchronize()
    return c.cpu().numpy(), f.cpu().numpy(), it.cpu().numpy(), out_pmf.cpu().numpy()


@pytest.mark.parametrize("net", ["synth", "peak"])
def test_batch_many_queries(nets, net):
    """Every pixel of three 128^2 images in order: 3072 queries, two query launches (2048 + 1024), queries crossing
    images; the oracle on ~200 of them: both sides of each image and launch boundary, corners, zero-bin pixels."""
    X, n = 128, 3
    ctx, _ = _resident(nets[net], X, n, seed=7)
    G = X // 4
    q = np.array([(i, y, x) for i in range(n) for y in range(G) for x in range(G)], np.int32)
    assert len(q) > 2048
    c, f, it, pmf = _batch(ctx, q, 9)
    sample, _ = _pixels(ctx, n, G, 120, 2)
    idx = [int(i * G * G + y * G + x) for i, y, x in sample]
    idx += [G * G - 1, G * G, 2 * G * G - 1, 2 * G * G, 2047, 2048, len(q) - 1]
    rs = np.random.RandomState(3)
    idx += list(rs.randint(0, len(q), 60))
    t = Tally("ab_reccs_batch %s, %d queries" % (net, len(q)))
    for i in sorted(set(idx)):
        t.check(pmf[i], GRID, 9, 100, 8, c[i], f[i], it[i], tuple(q[i]))
    ctx.close()
    t.report()


def test_batch_parameters(nets):
    """K x n_init x max_iter on the peaked network's pmfs (zero bins), queries crossing images, with out_pmf."""
    X, n = 64, 2
    ctx, _ = _resident(nets["peak"], X, n, seed=9)
    q, nzero = _pixels(ctx, n, X // 4, 4 * n + 12, 4)    # 4 n corners, then 4 sampled pixels with a zero bin
    assert nzero >= 4
    q = np.array(q[:4] + q[4 * n:4 * n + 4], np.int32)     # image 0's corners and the zero-bin pixels (both images)
    assert len(set(map(tuple, q.tolist()))) == 8
    t = Tally("ab_reccs_batch peak K x n_init x max_iter")
    for K in (1, 2, 5, 9, 17, 32):
        for n_init in (1, 8, 16):
            for max_iter in (2, 100):
                c, f, it, pmf = _batch(ctx, q, K, max_iter, n_init)
                for i in range(len(q)):
                    t.check(pmf[i], GRID, K, max_iter, n_init, c[i], f[i], it[i], tuple(q[i]))
    ctx.close()
    t.report()


@pytest.fixture(scope="module")
def csd(synth_sd):
    sd = util.caffe_scaled(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=PTS313).items()})
    return sd


@pytest.mark.parametrize("H,W", [(256, 256), (72, 88)])
def test_caffe313_batch(csd, H, W):
    n = 2
    ctx = util.make_ctx(csd, H, W, max_n=n, caffe313=True)
    L, ab, m = synth.synthetic_batch(n, max(H, W), seed=5, max_hints=4)
    crop = lambda a: util.dev(a[:, :, :H, :W])
    ctx.forward_device(crop(L), crop(ab), crop(m), 0.0)
    torch.cuda.synchronize()
    rs = np.random.RandomState(6)
    q = []
    for i in range(n):
        q += [(i, 0, 0), (i, 0, W - 1), (i, H - 1, 0), (i, H - 1, W - 1)]
    q += list(zip(rs.randint(0, n, 40), rs.randint(0, H, 40), rs.randint(0, W, 40)))
    q = np.array(q, np.int32)
    t = Tally("caffe313_reccs_batch %dx%d" % (H, W))
    for K in (1, 5, 9, 32):
        c, f, it, pmf = _batch(ctx, q, K, caffe=True)
        assert not pmf[:, 313:].any()
        for i in range(len(q)) if K == 9 else range(0, len(q), 4):
            t.check(pmf[i, :313], PTS313, K, 100, 8, c[i], f[i], it[i], tuple(q[i]))
    ctx.close()
    t.report()


def test_wrappers_get_ab_reccs(synth_sd, csd):
    from interactive_deep_colorization_b200 import colorize_image as CI
    g = util.golden("lhn_256.npz")
    a5, m5 = synth.synthetic_hints(256, 5, 0)
    pix = [(0, 0), (255, 255), (0, 255), (255, 0), (128, 128), (37, 201), (190, 64), (77, 77)]
    cd = CI.ColorizeImageB200Dist(Xd=256, maskcent=True)
    cd.prep_net(state_dict=synth_sd)
    cd.set_image(g["img_rgb"])
    cd.net_forward(a5, m5)
    t = Tally("ColorizeImageB200Dist.get_ab_reccs")
    for h, w in pix:
        for K in (5, 9):
            c, f = cd.get_ab_reccs(h, w, K=K, return_conf=True)
            # the iteration count is not returned: the single-pixel call on the same forward gives it
            it = cd._dist_ctx.ab_reccs(0, h // 4, w // 4, K=K, pts=cd.pts_in_hull)[2]
            t.check(np.asarray(cd.dist_ab[:, h, w], np.float32), cd.pts_in_hull, K, 100, 8, c.astype(np.float32),
                    f.astype(np.float32), it, (h, w))
    t.report()
    dm = CI.ColorizeImageB200CaffeDist(Xd=256)
    dm.prep_net(state_dict=csd)
    dm.set_image(g["img_rgb"])
    dm.net_forward(a5, m5)
    t = Tally("ColorizeImageB200CaffeDist.get_ab_reccs")
    for h, w in pix:
        for K in (5, 9):
            c, f = dm.get_ab_reccs(h, w, K=K, return_conf=True)
            p313 = np.asarray(dm.dist_ab[:, h, w], np.float32)
            p, qq = np.zeros(529, np.float32), np.zeros((529, 2), np.float32)
            p[:313], qq[:313] = p313, dm.pts_in_hull
            it = prepost.ab_reccs_pmf_gpu(p, K=K, pts=qq)[2]
            t.check(p313, dm.pts_in_hull, K, 100, 8, c.astype(np.float32), f.astype(np.float32), it, (h, w))
    t.report()
