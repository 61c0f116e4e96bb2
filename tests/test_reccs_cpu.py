"""Row f2 oracle checks (CPU): the deterministic weighted-k-means restatement vs the reference's
sample-and-cluster procedure (data/colorize_image.py:322-354), which is stochastic -> statistical parity."""
import numpy as np
import pytest

from oracle import reccs_ref as R
from tests import util

P = R.torch_gamut_points()


def _match(a, b):
    """greedy nearest matching distance between two centre sets"""
    b = list(map(tuple, b))
    worst = 0.0
    for c in a:
        d = [np.hypot(c[0] - q[0], c[1] - q[1]) for q in b]
        j = int(np.argmin(d))
        worst = max(worst, d[j])
        b.pop(j)
    return worst


def test_gamut_table_matches_reference_grid():
    assert P.shape == (529, 2) and tuple(P[1]) == (-100.0, -110.0) and tuple(P[23]) == (-110.0, -100.0)   # quirk q3


@pytest.mark.parametrize("kind,seed", [("blobs", 0), ("softmax", 1), ("softmax", 2), ("uniform", 0)])
def test_weighted_limit_is_at_least_as_good_as_sampling(kind, seed):
    pmf = R.synthetic_pmf(kind, seed)
    c, mass, iters = R.weighted_kmeans_pmf(pmf, P, 5)
    cs, confs, _ = R.sampled_reccs(pmf, P, 5, 25000, seed)
    assert abs(mass.sum() - 1) < 1e-12 and np.all(np.diff(mass) <= 1e-15)
    # objective of the population problem the reference approximates by sampling
    assert R.weighted_inertia(pmf, P, c) <= 1.01 * R.weighted_inertia(pmf, P, cs)


def test_well_separated_modes_agree_with_sampling():
    pmf = np.full(529, 1e-9)
    idx, w = [30, 262, 500], [0.55, 0.3, 0.15]
    for i, wi in zip(idx, w):
        pmf[i] = wi
    c, mass, _ = R.weighted_kmeans_pmf(pmf, P, 3)
    cs, confs, _ = R.sampled_reccs(pmf, P, 3, 25000, 0)
    assert _match(c, cs) < 0.5 and np.allclose(mass, confs, atol=0.01)
    assert np.allclose(c, P[idx], atol=1e-3) and np.allclose(mass, w, atol=1e-6)


def test_deterministic_and_restart_monotone():
    pmf = R.synthetic_pmf("softmax", 3)
    a = R.weighted_kmeans_pmf(pmf, P, 7, n_init=8)
    b = R.weighted_kmeans_pmf(pmf, P, 7, n_init=8)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    e1 = R.weighted_inertia(pmf, P, R.weighted_kmeans_pmf(pmf, P, 7, n_init=1)[0])
    assert R.weighted_inertia(pmf, P, a[0]) <= e1 + 1e-12


def test_against_reference_run_in_golden():
    """tests/golden/lhn_dist_256.npz holds get_ab_reccs(128,128,K=9) of the reference itself (seeded)."""
    gd = util.golden("lhn_dist_256.npz")
    pmf = gd["dist_rows"][:, 4, 4]                      # dist[:, 128, 128] = 64-grid (32,32) = rows[::8] index 4
    ref = gd["reccs_128_128_K9"]
    c, mass, _ = R.weighted_kmeans_pmf(pmf, P, 9)
    assert R.weighted_inertia(pmf, P, c) <= 1.01 * R.weighted_inertia(pmf, P, ref)


def _support(idx, w):
    p = np.zeros(529)
    p[idx] = w
    return p


def test_trace_leaves_the_answer_unchanged():
    for kind, seed in (("softmax", 1), ("blobs", 0), ("uniform", 0)):
        pmf = R.synthetic_pmf(kind, seed)
        for K, n_init, max_iter in ((5, 8, 100), (9, 16, 3)):
            a = R.weighted_kmeans_pmf(pmf, P, K, max_iter, n_init)
            b = R.weighted_kmeans_pmf(pmf, P, K, max_iter, n_init, trace=True)
            assert len(a) == 3 and len(b) == 4
            assert all(np.array_equal(x, y) for x, y in zip(a, b[:3]))
            assert b[3]["min"] == min(b[3][k] for k in ("seed", "lloyd", "order", "pick"))
            assert b[3]["lloyd_inert"] >= 0


def test_margins_on_hand_built_cases():
    # five points on the a axis, weights 0.6 at 0 and 0.4 at 40.  Seeding: the first seed's rank gap (0.6 - 0.4) / 0.6
    # = 1/3; the second seed is the 0.4 bin (score 0.4 * 40^2) against zero scores -> margin 1
    line = np.array([[0, 0], [10, 0], [20, 0], [30, 0], [40, 0]], np.float64)
    pmf = np.array([0.6, 0, 0, 0, 0.4])
    c, mass, it, m = R.weighted_kmeans_pmf(pmf, line, 2, n_init=1, trace=True)
    assert np.array_equal(c, [[0, 0], [40, 0]]) and np.allclose(mass, [0.6, 0.4]) and it == 1
    assert m["seed"] == pytest.approx(1 / 3) and m["order"] == pytest.approx(1 / 3) and m["restart"] == 0
    # Lloyd: the weighted points sit on their centres (margin 1).  Of the zero-weight points, the one at 20 is
    # equidistant from both centres -- an exact tie (integer distances), so no margin; the closest decision left is the
    # point at 10 (or 30): d = 100 against 900 -> 8/9.  Zero-weight labels are traced apart and stay out of "min"
    assert m["lloyd"] == 1.0 and m["lloyd_inert"] == pytest.approx(8 / 9) and m["min"] == pytest.approx(1 / 3)
    # the same point 1e-7 off the tie: a genuine near-tie, margin ((20 + e)^2 - (20 - e)^2) / (20 + e)^2 -- of a
    # zero-weight point, then of a weighted one
    off = line.copy()
    off[2, 0] += 1e-7
    m2 = R.weighted_kmeans_pmf(pmf, off, 2, n_init=1, trace=True)[3]
    near = 80e-7 / (20 + 1e-7) ** 2
    assert m2["lloyd_inert"] == pytest.approx(near, rel=1e-6) and m2["lloyd"] == 1.0
    m2 = R.weighted_kmeans_pmf(np.array([0.6, 0, 1e-3, 0, 0.4]), off, 2, n_init=1, trace=True)[3]
    assert m2["lloyd"] < 1e-7 and m2["min"] == min(m2["lloyd"], m2["pick"])       # the 1e-3 moves centre 0 a little
    # two restarts at inertia 0 tie at any scale (margin 1 against the 1e-300 floor of the threshold); with weight at
    # 10 as well, restart 1 (seeded from the 0.4 bin) converges to the same clusters: a tie on a positive inertia,
    # margin 1e-9 to the threshold.  Restart 0 wins both
    m3 = R.weighted_kmeans_pmf(pmf, line, 2, n_init=2, trace=True)[3]
    assert m3["pick"] == 1.0 and m3["restart"] == 0
    m3 = R.weighted_kmeans_pmf(np.array([0.5, 0.1, 0, 0, 0.4]), line, 2, n_init=2, trace=True)[3]
    assert m3["pick"] == pytest.approx(1e-9) and m3["restart"] == 0
    # seeding: two bins at -20 and +20 with equal pmf values tie exactly (lowest index wins in any rounding) ...
    pair = np.array([[0, 0], [20, 0], [-20, 0]], np.float64)
    m4 = R.weighted_kmeans_pmf(np.array([0.5, 0.25, 0.25]), pair, 2, n_init=1, trace=True)[3]
    assert m4["seed"] == pytest.approx(0.5)                         # only the first seed's rank gap is left
    # ... and 1e-13 apart they are a near-tie below the 1e-12 bar
    m5 = R.weighted_kmeans_pmf(np.array([0.5, 0.25, 0.25 * (1 + 1e-13)]), pair, 2, n_init=1, trace=True)[3]
    assert 0 < m5["seed"] < 1e-12 and m5["min"] == m5["seed"]
    # equal non-zero masses of clusters holding more than one bin: a tie the stable order cannot make exact
    quad = np.array([[0, 0], [10, 0], [100, 0], [110, 0]], np.float64)
    m6 = R.weighted_kmeans_pmf(np.array([0.3, 0.2, 0.2, 0.3]), quad, 2, n_init=1, trace=True)[3]
    assert m6["order"] == 0.0


def test_more_clusters_than_support_keep_empty_centres():
    """K above the number of non-zero bins: the seeds after the support repeat at bin 0 (every score is 0: the
    arg-max takes the lowest index), those clusters stay empty with mass 0 and keep their centre, and the stable mass
    order puts them after the support in cluster order.  Restarts seeded from zero-weight bins (n_init above the
    support) tie on inertia 0 with restart 0, which wins."""
    idx, w = [300, 40, 412], [0.5, 0.3125, 0.1875]      # dyadic: every centre stays exactly on its bin
    pmf = _support(idx, w)
    for K in (3, 4, 9, 32):
        for n_init in (1, 8, 16):
            c, mass, it, m = R.weighted_kmeans_pmf(pmf, P, K, n_init=n_init, trace=True)
            assert np.array_equal(c[:3], P[idx]) and np.array_equal(mass[:3], w)
            assert np.all(mass[3:] == 0) and np.all(c[3:] == P[0]) and it == 1
            assert m["restart"] == 0 and m["min"] > 1e-6, m
    # a restart seeded from a zero-weight bin keeps that seed as an empty cluster of its own
    c, mass, _ = R._one_restart(pmf, P, 5, 100, 7)
    z = np.lexsort((np.arange(529), -pmf))[7]
    assert pmf[z] == 0 and np.array_equal(c[3], P[z]) and np.array_equal(c[4], P[0]) and np.all(mass[3:] == 0)


def test_equal_single_bin_masses_keep_cluster_order():
    pmf = _support([500, 20], [0.5, 0.5])
    c, mass, _, m = R.weighted_kmeans_pmf(pmf, P, 2, trace=True)
    # the first seed is the lower index among equal weights (bin 20): its cluster 0 comes first in the stable order
    assert np.array_equal(c, P[[20, 500]]) and np.array_equal(mass, [0.5, 0.5]) and np.isinf(m["order"])


def test_caffe_padded_table_equals_the_313_bin_table():
    """What the Caffe distribution wrapper and idc_caffe313_reccs_batch feed the kernel: 529 slots, the 313 bin centres
    then 216 rows of (0, 0) with zero weight -- (0, 0) is also a real bin.  The oracle gives the same answer on the
    padded pair as on the 313 bins: centres, mass, iterations, and the margins."""
    pts = util.golden("pts_in_hull.npy").astype(np.float64)
    assert np.sum(np.all(pts == 0, 1)) == 1
    rs = np.random.RandomState(3)
    p313 = []
    for s in (1.0, 3.0, 8.0):
        z = rs.randn(313) * s
        e = np.exp(z - z.max())
        p313.append((e / e.sum()).astype(np.float32))
    p313.append(np.where(np.arange(313) % 50 == 0, 0.2, 0.0).astype(np.float32))     # 7 bins, K above the support
    pad_pts = np.zeros((529, 2))
    pad_pts[:313] = pts
    for p in p313:
        pad = np.zeros(529, np.float32)
        pad[:313] = p
        for K, n_init, max_iter in ((1, 8, 100), (5, 8, 100), (9, 16, 100), (32, 8, 100), (9, 8, 2)):
            a = R.weighted_kmeans_pmf(p, pts, K, max_iter, n_init, trace=True)
            b = R.weighted_kmeans_pmf(pad, pad_pts, K, max_iter, n_init, trace=True)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2], (K, n_init)
            assert a[3]["restart"] == b[3]["restart"]
