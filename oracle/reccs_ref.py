"""ORACLE (test infrastructure only -- never imported by the product path).

Colour suggestions at one pixel, SURVEY row f2.

* `sampled_reccs`  -- restatement of the reference procedure, /root/reference/data/colorize_image.py:322-354:
  cumulative sum of the pixel's pmf -> N uniform draws -> bin lookup (np.digitize) -> sklearn KMeans(K) on the
  drawn gamut points -> centres ordered by cluster occupancy.  Stochastic (np.random + KMeans init).
* `weighted_kmeans_pmf` -- the deterministic N -> infinity limit of it that the CUDA kernel
  (csrc/idc_heads.cu: ab_reccs_kernel) implements: weighted k-means over the gamut points with the pmf as
  weights; greedy farthest-point seeding (heaviest bin first, then argmax w * d^2, lowest index on ties),
  FP64 Lloyd iterations until the assignment is stable; best of n_init restarts.  Every sum is correctly rounded
  (math.fsum), so the statement has one answer whatever the bin order, and zero-weight padding leaves it alone.

Parity: the kernel is checked against `weighted_kmeans_pmf` on every path that runs it, to 1 float32 ulp of the
centres and mass with equal Lloyd iterations wherever the traced decision margins (trace=True) exceed 1e-12
(tests/test_gpu_reccs_fp64.py); `weighted_kmeans_pmf` is checked
against `sampled_reccs` statistically (tests/test_reccs_cpu.py).  The reference holds no vectors for this
function (its output is random), so parity with the reference itself is statistical only.
"""
import math

import numpy as np


def torch_gamut_points():
    """Bin -> ab table of the PyTorch wrapper (reference data/colorize_image.py:283; quirk q3)."""
    g = np.arange(-110, 120, 10)
    return np.array(np.meshgrid(g, g)).reshape((2, 529)).T.astype(np.float64)


def weighted_kmeans_pmf(pmf, pts, K, max_iter=100, n_init=8, trace=False):
    """Best (lowest weighted inertia) of n_init restarts; restart v seeds from the bin of weight-rank v.
    Restarts within 1e-9 relative of the best count as ties -> lowest v.

    trace=True appends a dict of margins: the smallest relative margin of each kind of decision the run took, over
    every restart -- "seed" (each seeding arg-max, the weight ranks of the first seed included: winner against
    runner-up), "lloyd" (each Lloyd arg-min over the points that can move a centre) -- and, of the picked restart,
    "order" (adjacent masses of the stable mass sort) and "lloyd_inert" (each Lloyd arg-min over the inert points); "pick"
    (each restart's inertia against the 1e-9 tie threshold, relative to the best inertia); "min" of seed, lloyd, order
    and pick, and "restart", the index picked.  A point is inert when its weight is 0, or below INERT = 2^-60 of the
    mass of both clusters its arg-min hesitates between: its label moves a centre by at most 2^-60 of the distance to
    the point and a mass by 2^-60 relative, far below an FP64 ulp.  It decides whether the assignment counts as stable,
    so a flipped inert label costs one Lloyd iteration: the other side stops one iteration later, on the same centres
    (exactly for zero weight).  "lloyd_inert" stays out of "min"; inert labels of the other restarts change nothing the
    answer depends on.  A decision whose candidates are computed exactly in any rounding (equal pmf values, coinciding
    centres, squared distances that are exact in FP64, zero scores and zero masses) has no margin (inf): every
    implementation resolves it the same way.  A margin below ~1e-12 means another correct FP64 implementation (FMA
    contraction, another summation order) may take the other branch."""
    runs = [_one_restart(pmf, pts, K, max_iter, v, trace) for v in range(n_init)]
    e = np.array([weighted_inertia(pmf, pts, r[0]) for r in runs])
    thr = e.min() * (1.0 + 1e-9) + 1e-300
    pick = int(np.nonzero(e <= thr)[0][0])
    if not trace:
        return runs[pick]
    m = {"seed": min(r[3]["seed"] for r in runs), "lloyd": min(r[3]["lloyd"] for r in runs),
         "order": runs[pick][3]["order"], "lloyd_inert": runs[pick][3]["lloyd_inert"],
         "pick": float(np.min(np.abs(e - thr)) / max(e.min(), 1e-300)), "restart": pick}
    m["min"] = min(m["seed"], m["lloyd"], m["order"], m["pick"])
    return runs[pick][:3] + (m,)


def _fsum(a):
    """correctly rounded sum: no summation order, so zero-weight entries (padding) cannot change it.  A deliberate
    departure from numpy's pairwise sums (which the statement used before): the answer moves in its last bits only"""
    return math.fsum(np.asarray(a, np.float64).ravel().tolist())


def _gap(hi, lo):
    """relative margin between a winning value hi and a losing value lo <= hi (inf when both are 0)"""
    return np.inf if hi == lo == 0 else (hi - lo) / abs(hi)


def _sq_exact(p, c):
    """Is the FP64 (px - cx)^2 + (py - cy)^2 the exact value, so that any rounding order or FMA gives it too?"""
    from fractions import Fraction as F
    d = float((p[0] - c[0]) ** 2 + (p[1] - c[1]) ** 2)
    return F(d) == (F(float(p[0])) - F(float(c[0]))) ** 2 + (F(float(p[1])) - F(float(c[1]))) ** 2


def _seed_margin(s, pmf, w, P, cen, top):
    """Margin of one seeding arg-max over scores s = w * mind (winner top).  Exact ties: equal zero scores; or tied
    scores from exactly computed distances to the nearest centre with either the same pmf value or every weight and
    product exact (the pmf's sum, w = pmf / sum and w * mind all exact in FP64)."""
    from fractions import Fraction as F
    tied = np.nonzero(s == s[top])[0]
    if s[top] > 0 and tied.size > 1:
        near = [int(np.argmin(((cen - P[i]) ** 2).sum(1))) for i in tied]
        d = [float(((cen[k] - P[i]) ** 2).sum()) for i, k in zip(tied, near)]
        if not all(_sq_exact(P[i], cen[k]) for i, k in zip(tied, near)):
            return 0.0
        same = np.all(pmf[tied] == pmf[top]) and np.all(np.asarray(d) == d[0])
        if not same:
            tot = _fsum(pmf)
            if F(tot) != sum(F(float(x)) for x in pmf if x != 0) or not all(
                    F(float(w[i])) == F(float(pmf[i])) / F(tot) and F(float(s[i])) == F(float(w[i])) * F(di)
                    for i, di in zip(tied, d)):
                return 0.0
    rest = np.delete(s, tied)
    return _gap(s[top], rest.max()) if rest.size else np.inf


def _lloyd_margins(d, P, c):
    """Margin of the arg-min of every row of d [points, K].  A tie is exact when the tied centres coincide or every
    tied distance is exact in FP64."""
    out = np.full(d.shape[0], np.inf)
    if d.shape[1] == 1:
        return out
    s = np.sort(d, 1)
    with np.errstate(invalid="ignore", divide="ignore"):
        g = (s[:, 1] - s[:, 0]) / s[:, 1]
    out[s[:, 1] != s[:, 0]] = g[s[:, 1] != s[:, 0]]
    for i in np.nonzero(s[:, 1] == s[:, 0])[0]:
        tied = np.nonzero(d[i] == s[i, 0])[0]
        if not (all(np.array_equal(c[k], c[tied[0]]) for k in tied) or all(_sq_exact(P[i], c[k]) for k in tied)):
            out[i] = 0.0
            continue
        rest = np.delete(d[i], tied)
        if rest.size:
            out[i] = _gap(rest.min(), s[i, 0])
    return out


INERT = 2.0 ** -60     # a point of weight below INERT x the mass of both clusters it hesitates between is inert


def _one_restart(pmf, pts, K, max_iter, v, trace=False):
    raw = np.asarray(pmf, np.float64)
    w = raw / _fsum(raw)
    P = np.asarray(pts, np.float64)
    c = np.empty((K, 2))
    rank = np.lexsort((np.arange(w.size), -w))             # weight rank, lowest index first among equals
    c[0] = P[rank[v]]
    seed = np.inf
    for r in range(v + 1 if trace else 0):                 # the first seed: v + 1 arg-max rounds, winners taken out
        a, b = rank[r], rank[r + 1] if r + 1 < w.size else None
        if b is not None and raw[a] != raw[b]:
            seed = min(seed, _gap(w[a], w[b]))
    mind = ((P - c[0]) ** 2).sum(1)
    for j in range(1, K):
        s = w * mind
        top = int(np.argmax(s))
        if trace:
            seed = min(seed, _seed_margin(s, raw, w, P, c[:j], top))
        c[j] = P[top]
        mind = np.minimum(mind, ((P - c[j]) ** 2).sum(1))
    labels = np.full(P.shape[0], -1)
    iters = 0
    lloyd = lloyd_inert = np.inf
    while iters < max_iter:
        d = ((P[:, None, :] - c[None, :, :]) ** 2).sum(2)
        new = np.argmin(d, 1)
        if trace:
            g = _lloyd_margins(d, P, c)
            mk = np.bincount(new, weights=w, minlength=K)
            two = np.argsort(d, 1, kind="stable")[:, :2] if K > 1 else np.zeros((w.size, 2), int)
            inert = (w == 0) | (w <= INERT * np.minimum(mk[two[:, 0]], mk[two[:, 1]]))
            lloyd = min(lloyd, float(g[~inert].min(initial=np.inf)))
            lloyd_inert = min(lloyd_inert, float(g[inert].min(initial=np.inf)))
        if np.array_equal(new, labels):
            break
        labels = new
        for k in range(K):
            sel = labels == k
            m = _fsum(w[sel])
            if m > 0:
                c[k] = (_fsum(w[sel] * P[sel, 0]) / m, _fsum(w[sel] * P[sel, 1]) / m)
        iters += 1
    mass = np.array([_fsum(w[labels == k]) for k in range(K)])
    order = np.argsort(-mass, kind="stable")
    if not trace:
        return c[order], mass[order], iters
    ms = mass[order]
    om = np.inf
    for a, b in zip(order[:-1], order[1:]):
        if mass[a] == mass[b] and mass[a] > 0:
            # the same single non-zero pmf value in both clusters: equal in every rounding, the stable order decides
            na, nb = raw[(labels == a) & (raw != 0)], raw[(labels == b) & (raw != 0)]
            if not (na.size == nb.size == 1 and na[0] == nb[0]):
                om = 0.0
        else:
            om = min(om, _gap(mass[a], mass[b]))
    return c[order], ms, iters, {"seed": seed, "lloyd": lloyd, "lloyd_inert": lloyd_inert, "order": om}


def sampled_reccs(pmf, pts, K=5, N=25000, seed=0):
    from sklearn.cluster import KMeans
    rng = np.random.RandomState(seed)
    cmf = np.cumsum(np.asarray(pmf, np.float64))
    cmf = cmf / cmf[-1]
    inds = np.digitize(rng.uniform(0, 1.0, N), bins=cmf)
    samples = np.asarray(pts)[inds, :]
    km = KMeans(n_clusters=K, n_init=10, random_state=seed).fit(samples)
    cnt = np.histogram(km.labels_, np.arange(0, K + 1))[0]
    order = np.argsort(cnt)[::-1]
    return km.cluster_centers_[order, :], cnt[order] / float(N), float(km.inertia_) / N


def weighted_inertia(pmf, pts, centers):
    w = np.asarray(pmf, np.float64)
    w = w / _fsum(w)
    d = ((np.asarray(pts, np.float64)[:, None, :] - np.asarray(centers, np.float64)[None]) ** 2).sum(2)
    return _fsum(w * d.min(1))


def synthetic_pmf(kind, seed=0):
    """Test pmfs over the 529 bins."""
    rng = np.random.RandomState(seed)
    P = torch_gamut_points()
    if kind == "uniform":
        return np.full(529, 1.0 / 529)
    if kind == "blobs":       # 3 Gaussian blobs of unequal mass + a small floor
        mu = np.array([[-60.0, 40.0], [50.0, 50.0], [20.0, -70.0]])
        a = np.array([0.6, 0.3, 0.1])
        p = sum(ai * np.exp(-((P - m) ** 2).sum(1) / (2 * 12.0 ** 2)) for ai, m in zip(a, mu))
        return p / p.sum() + 1e-6
    if kind == "softmax":     # what the dist head produces: softmax of random logits
        z = rng.randn(529) * 2.0
        e = np.exp(z - z.max())
        return e / e.sum()
    if kind == "peaked":      # nearly one-hot
        p = np.full(529, 1e-7)
        p[rng.randint(529)] = 1.0
        return p / p.sum()
    raise ValueError(kind)
