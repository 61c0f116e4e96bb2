"""Float64 numpy statement of the Levin baseline (DESIGN.md §4b), the oracle of idc_levin_weights / idc_levin_solve:
the weight rule (vectorised, each operation in the order the kernel rounds it), the reachability rule (a breadth-first
search over non-zero weights from the hinted pixels) and a direct sparse solve on the pixels that reach a hint, with 0
on the rest; the solver's right-hand side and true relative residual rounded as the kernel rounds them, and the layout
of its workspace."""
import collections
import math

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as sla

# neighbour k: (dy, dx), the 3 x 3 window in row-major order without its centre (the plane order of idc_levin_weights)
OFFSETS = ((-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 1), (1, -1), (1, 0), (1, 1))
LN001 = np.log(0.01)
VAR_SCALE = 0.6
SIGMA_FLOOR = 2e-6


def _shift(a, dy, dx):
    """a[y + dy, x + dx] where that lies inside, else 0; and the mask of where it does."""
    h, w = a.shape
    out = np.zeros_like(a)
    inside = np.zeros(a.shape, bool)
    ys, yd = slice(max(dy, 0), h + min(dy, 0)), slice(max(-dy, 0), h + min(-dy, 0))
    xs, xd = slice(max(dx, 0), w + min(dx, 0)), slice(max(-dx, 0), w + min(-dx, 0))
    out[yd, xd] = a[ys, xs]
    inside[yd, xd] = True
    return out, inside


def sigma(L):
    """The per-pixel s of the weight rule for one L plane [h,w] float64 -> (s, Y, neighbours [8,h,w], inside [8,h,w])."""
    Y = np.asarray(L, np.float64) / 100.0
    nb, inside = zip(*(_shift(Y, dy, dx) for dy, dx in OFFSETS))
    nb, inside = np.stack(nb), np.stack(inside)
    total, cnt = Y.copy(), np.ones_like(Y)
    for k in range(8):                                   # sequential sums, p first, as the kernel adds them
        total = np.where(inside[k], total + nb[k], total)
        cnt = np.where(inside[k], cnt + 1.0, cnt)
    mean = total / cnt
    dev = (Y - mean) * (Y - mean)
    m = np.full_like(Y, np.inf)
    for k in range(8):
        e = nb[k] - mean
        dev = np.where(inside[k], dev + e * e, dev)
        d = nb[k] - Y
        m = np.where(inside[k], np.minimum(m, d * d), m)
    s = VAR_SCALE * (dev / cnt)
    s = np.maximum(s, -m / LN001)
    s = np.maximum(s, SIGMA_FLOOR)
    return s, Y, nb, inside


def weights(L, normalise=True):
    """L [h,w] float64 (channel 0 of the photo's Lab) -> w [8,h,w] float64: w[k, y, x] = the weight of neighbour k of
    (y, x), 0 outside the image.  normalise=False: the un-normalised exp(-d^2 / s)."""
    s, Y, nb, inside = sigma(L)
    e = np.zeros_like(nb)
    with np.errstate(under="ignore"):
        for k in range(8):
            d = nb[k] - Y
            e[k] = np.where(inside[k], np.exp(-(d * d) / s), 0.0)
    if not normalise:
        return e
    tot = np.zeros_like(Y)
    for k in range(8):
        tot = tot + e[k]
    return e / tot


def _edges(w):
    """w [8,h,w] -> (rows, cols, vals): pixel p -> neighbour q with w_pq != 0, flattened row-major."""
    _, h, wd = w.shape
    idx = np.arange(h * wd).reshape(h, wd)
    rows, cols, vals = [], [], []
    for k, (dy, dx) in enumerate(OFFSETS):
        q, inside = _shift(idx, dy, dx)
        sel = inside & (w[k] != 0)
        rows.append(idx[sel])
        cols.append(q[sel])
        vals.append(w[k][sel])
    return np.concatenate(rows), np.concatenate(cols), np.concatenate(vals)


def reaching(w, hinted):
    """Free pixels from which a path of non-zero weights leads to a hinted pixel -> bool [h,w].  A breadth-first search
    backwards from the hints: p joins when w_pq != 0 for a q already found."""
    _, h, wd = w.shape
    rows, cols, _ = _edges(w)
    hinted = hinted.reshape(-1)
    into = collections.defaultdict(list)                 # q -> the pixels p with w_pq != 0
    for p, q in zip(rows.tolist(), cols.tolist()):
        into[q].append(p)
    seen = hinted.copy()
    queue = collections.deque(np.flatnonzero(hinted).tolist())
    while queue:
        q = queue.popleft()
        for p in into[q]:
            if not seen[p]:
                seen[p] = True
                queue.append(p)
    return (seen & ~hinted).reshape(h, wd)


def solve(w, ab_hint, mask):
    """w [8,h,w]; ab_hint [2,h,w] and mask [h,w] (hinted: mask > 0) -> u [2,h,w] float64: the hints on hinted pixels,
    spsolve of u_p - sum_q w_pq u_q = 0 on the free pixels that reach a hint (the hinted u_q moved to the right), 0 on
    every other pixel."""
    _, h, wd = w.shape
    hinted = np.asarray(mask).reshape(h, wd) > 0
    ab_hint = np.asarray(ab_hint, np.float64).reshape(2, h * wd)
    u = np.zeros((2, h * wd))
    u[:, hinted.reshape(-1)] = ab_hint[:, hinted.reshape(-1)]
    R = reaching(w, hinted).reshape(-1)
    if not R.any():
        return u.reshape(2, h, wd)
    rows, cols, vals = _edges(w)
    W = sp.csr_matrix((vals, (rows, cols)), shape=(h * wd, h * wd))
    ridx = np.flatnonzero(R)
    A = sp.identity(len(ridx), format="csc") - W[ridx][:, ridx].tocsc()
    Wrh = W[ridx][:, np.flatnonzero(hinted.reshape(-1))]
    for c in range(2):
        b = Wrh @ ab_hint[c, hinted.reshape(-1)]
        u[c, ridx] = sla.spsolve(A, b)
    return u.reshape(2, h, wd)


def rhs(w, ab_hint, mask):
    """b [2,h,w] float64 of the system reduced to the free pixels: b_p = sum over hinted neighbours q of w_pq c_q on
    free p, 0 on hinted p.  Summed over k in neighbour order with each product and sum rounded on its own, from the
    float32 hint, as levin_rhs in idc_levin.cu does, so it is the solver's b bit for bit."""
    _, h, wd = w.shape
    hinted = np.asarray(mask).reshape(h, wd) > 0
    c = np.asarray(ab_hint, np.float32).reshape(2, h, wd).astype(np.float64)
    b = np.zeros((2, h, wd))
    for k, (dy, dx) in enumerate(OFFSETS):
        hq, inside = _shift(hinted, dy, dx)
        for ch in range(2):
            cq, _ = _shift(c[ch], dy, dx)
            b[ch] = np.where(inside & hq, b[ch] + w[k] * cq, b[ch])
    b[:, hinted] = 0.0
    return b


def _apply(w, x, hinted):
    """(A x)_p = x_p - sum_q w_pq x_q on free p (0 on hinted p), with x taken as 0 on hinted pixels: levin_apply's
    order and roundings."""
    x = np.where(hinted, 0.0, x)
    acc = np.zeros_like(x)
    for k, (dy, dx) in enumerate(OFFSETS):
        xq, inside = _shift(x, dy, dx)
        acc = np.where(inside, acc + w[k] * xq, acc)
    return np.where(hinted, 0.0, x - acc)


def residual(w, ab_hint, mask, u):
    """The true relative residual ||b - A u||_2 / ||b||_2 of each channel -> float64 [2]; u [2,h,w], its hinted entries
    ignored; 0 for a channel whose b is 0.  Each element b_p - (A u)_p is rounded as the solver's true-residual check
    rounds it, and the squares are summed exactly (math.fsum), so only the order of the solver's final sum differs."""
    _, h, wd = w.shape
    hinted = np.asarray(mask).reshape(h, wd) > 0
    b = rhs(w, ab_hint, mask)
    out = np.zeros(2)
    for ch in range(2):
        r = b[ch] - _apply(w, np.asarray(u[ch], np.float64), hinted)
        nb = math.fsum((b[ch] * b[ch]).ravel())
        if nb > 0:
            out[ch] = math.sqrt(math.fsum((r * r).ravel())) / math.sqrt(nb)
    return out


# The solver workspace's vectors per image and channel, in levin_solve_kernel's order (idc_levin.cu)
WS_VECS = ("u", "r", "rhat", "p", "v", "t")


def workspace(ws, h, w, image, channel, vec="u"):
    """One FP64 vector [h,w] of idc_levin_solve's workspace (a host copy, any dtype: it is viewed as float64): by
    default the solution u.  The layout is levin_solve_kernel's (idc_levin.cu): vector v of channel c of image i
    starts at double ((i * 2 + c) * 6 + v) * h * w, v in WS_VECS order; r holds s in place during an iteration."""
    d = np.ascontiguousarray(ws).reshape(-1).view(np.float64)
    o = ((image * 2 + channel) * len(WS_VECS) + WS_VECS.index(vec)) * h * w
    return d[o:o + h * w].reshape(h, w)


def matrix_rows(w, hinted):
    """The full system's matrix (hinted rows: u_p = c_p) as a scipy CSR matrix, for row-sum checks."""
    _, h, wd = w.shape
    rows, cols, vals = _edges(w)
    free = ~hinted.reshape(-1)
    keep = free[rows]
    W = sp.csr_matrix((vals[keep], (rows[keep], cols[keep])), shape=(h * wd, h * wd))
    return sp.identity(h * wd, format="csr") - W
