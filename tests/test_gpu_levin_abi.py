"""GPU: idc_levin_weights and idc_levin_solve across the whole C ABI against the float64 statements of
tests/levin_ref.py: non-square, thin and tiny images, the largest network size, sparse and dense hints, known answers
that every branch of the solver's stopping logic must give bit for bit, and batches that need a second wave of CTAs.

Every solved channel is held to the same contract: relres is the TRUE relative residual of the u the solver leaves in
its workspace (levin_ref.residual, rounded as the kernel rounds each element), out_ab is float32(u) on free pixels and
the hint on hinted ones bit for bit, and a converged u is within TOL_AB of spsolve."""
import math

import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import _lib, photos
from oracle import color_ref
from tests import levin_ref
from tests.test_gpu_levin import TOL_AB, _edges_photo, _st, _weights
from tests.test_gpu_reveal import _paint, _photo

pytestmark = pytest.mark.gpu
TOL = photos.LEVIN_TOL
DBL_MIN = np.finfo(np.float64).tiny
# thin (every pixel has a clipped window), tiny, hw < 512 (threads without a pixel in every reduction), odd and
# non-square with hw not a multiple of 256 or 512, and the largest network size
SHAPES = [(2, 37), (37, 2), (2, 2), (8, 8), (24, 40), (33, 517), (512, 512)]
REPORT = {}


def _lab(rgb):
    """float64 Lab [3,h,w] of a uint8 RGB photo (the host statement of rgb2lab)."""
    return np.ascontiguousarray(color_ref.rgb2lab(rgb).transpose(2, 0, 1))


def _labs(h, w):
    """Two of test_gpu_reveal's seeded photos and the hard-edge image, at h x w."""
    return [_lab(_photo(h, w, 40 + i)) for i in range(2)] + [_lab(_edges_photo(h, w))]


def _launch(wts, ab, mask, levels, tol=TOL, max_iter=photos.LEVIN_MAX_ITER):
    """idc_levin_solve on device weights [P,8,h,w] and host planes ab [n,2,h,w], mask [n,h,w], into outputs and a
    workspace that start as garbage -> (out_ab float32 [n,2,h,w], iters [n,2], relres [n,2], workspace bytes)."""
    lib = _lib.load()
    n, _, h, w = ab.shape
    d_ab, d_mask = (torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in (ab, mask))
    out = torch.full((n, 2, h, w), float("nan"), device="cuda")
    iters = torch.full((n, 2), -7, dtype=torch.int32, device="cuda")
    relres = torch.full((n, 2), float("nan"), dtype=torch.float64, device="cuda")
    nbytes = lib.idc_levin_workspace_bytes(n, h, w)
    ws = torch.full((nbytes // 8,), float("nan"), dtype=torch.float64, device="cuda")
    assert lib.idc_levin_solve(0, n, levels, h, w, wts.data_ptr(), d_ab.data_ptr(), d_mask.data_ptr(), tol, max_iter,
                               out.data_ptr(), iters.data_ptr(), relres.data_ptr(), ws.data_ptr(), nbytes, _st()) == 0
    return out.cpu().numpy(), iters.cpu().numpy(), relres.cpu().numpy(), ws.cpu().numpy().view(np.uint8)


def _u(ws, j, h, w):
    return np.stack([levin_ref.workspace(ws, h, w, j, c) for c in range(2)])


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _check_contract(w, ab, mask, got, relres, ws, j, tol=TOL):
    """out_ab and relres of image j against its workspace u -> the relative relres mismatch (0 where both are 0)."""
    h, wd = mask.shape
    hinted = mask > 0
    u = _u(ws, j, h, wd)
    assert (u[:, hinted] == 0).all(), j                          # only free pixels are ever written
    assert np.array_equal(_bits(got), _bits(np.where(hinted, ab, u.astype(np.float32)))), j
    res = levin_ref.residual(w, ab, mask, u)
    for c in range(2):
        assert abs(relres[c] - res[c]) <= max(1e-6 * res[c], 4 * np.spacing(tol)), (j, c, relres[c], res[c])
    return max(abs(relres[c] - res[c]) / res[c] if res[c] else 0.0 for c in range(2))


def _check_solve(w, ab, mask, got, relres, ws, j):
    """A converged image: the contract, relres <= tol and spsolve within TOL_AB -> (max |d ab|, relres mismatch)."""
    assert (relres <= TOL).all(), (j, relres)
    mis = _check_contract(w, ab, mask, got, relres, ws, j)
    err = float(np.abs(got - levin_ref.solve(w, ab, mask)).max())
    assert err <= TOL_AB, (j, err)
    return err, mis


@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%d" % s for s in SHAPES])
def test_weights_on_every_shape(shape):
    labs = _labs(*shape)
    got = _weights(labs).cpu().numpy()
    flips = 0
    for i, lab in enumerate(labs):
        want = levin_ref.weights(lab[0])
        e = levin_ref.weights(lab[0], normalise=False)
        inside = levin_ref.sigma(lab[0])[3]
        under = e < 2 * DBL_MIN                     # subnormal or about to be: exp and e / tot may round it either way
        bad = ~under & ~(np.abs(got[i] - want) <= 1e-13 * np.abs(want))
        assert not bad.any(), (i, np.argwhere(bad)[:5].tolist())
        # where exp underflows, both sides are below 2 DBL_MIN / 0.01 (the closest neighbour keeps e >= 0.01)
        assert (np.abs(got[i][under]) < 200 * DBL_MIN).all() and (got[i][~inside] == 0).all()
        flips += int((under & ((got[i] == 0) != (want == 0))).sum())
        # d^2 <= 2 dev and s >= 0.6 dev / cnt keep every exponent >= -30: no weight inside the image underflows
        assert (got[i][inside] >= math.exp(-30) / 8 * (1 - 1e-12)).all(), i
    REPORT.setdefault("zero-pattern flips", {})[shape] = flips
    print("levin weights %dx%d: %d zero-pattern differences, all where exp underflows" % (shape + (flips,)))


def _masks(h, w, seed):
    """Single-pixel points: 1, 5, 50 and a quarter of the pixels (a prefix of one permutation, at least one pixel
    left free), and about 90 % of the pixels hinted."""
    rs = np.random.RandomState(seed)
    hw = h * w
    order = rs.permutation(hw)
    out = []
    for m in (1, 5, 50, hw // 4):
        k = np.zeros(hw, np.float32)
        k[order[:max(1, min(m, hw - 1))]] = 1
        out.append(k)
    k = (rs.rand(hw) < 0.9).astype(np.float32)
    k[order[0]], k[order[-1]] = 1, 0
    return [m.reshape(h, w) for m in out + [k]]


@pytest.mark.parametrize("shape", SHAPES[:-1], ids=["%dx%d" % s for s in SHAPES[:-1]])
def test_solve_on_every_shape(shape):
    """Three photos x five masks in one launch (levels = 5); the hint planes carry the photo's colour on every pixel,
    so a free pixel's colour must not leak in."""
    h, w = shape
    labs = _labs(h, w)
    masks = _masks(h, w, 1000 * h + w)
    ab = np.stack([np.float32(lab[1:]) for lab in labs for _ in masks])
    mask = np.stack([m for _ in labs for m in masks])
    wts = _weights(labs)
    w_host = wts.cpu().numpy()
    got, iters, relres, ws = _launch(wts, ab, mask, len(masks))
    stats = [_check_solve(w_host[j // len(masks)], ab[j], mask[j], got[j], relres[j], ws, j) for j in range(len(ab))]
    REPORT.setdefault("solve", {})[shape] = (max(s[0] for s in stats), max(s[1] for s in stats), int(iters.max()))
    print("levin solve %dx%d: max |d ab| = %.3g, max relres mismatch = %.3g, iterations max %d"
          % ((h, w) + REPORT["solve"][shape]))


def test_solve_512_with_500_points():
    X = 512
    lab = _lab(_photo(X, X, 47))
    ab, mask, _ = _paint(lab, photos.reveal_points(X, 500, 11, 0))
    wts = _weights([lab])
    got, iters, relres, ws = _launch(wts, ab[None], mask, 1)
    err, mis = _check_solve(wts.cpu().numpy()[0], ab, mask[0], got[0], relres[0], ws, 0)
    REPORT.setdefault("solve", {})[(X, X)] = (err, mis, int(iters.max()))
    print("levin solve 512x512, 500 points: max |d ab| = %.3g, relres mismatch = %.3g, iterations %s"
          % (err, mis, iters[0].tolist()))


@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%d" % s for s in SHAPES])
def test_isolated_free_pixels_take_one_exact_step(shape):
    """Every pixel hinted but (3i, 3j): A = I on the free set, so the first step is exact (s = t = 0, omega = 0) and
    u = b bit for bit."""
    h, w = shape
    labs = _labs(h, w)
    mask = np.ones((h, w), np.float32)
    mask[::3, ::3] = 0
    ab = np.stack([np.float32(lab[1:]) for lab in labs])
    wts = _weights(labs)
    w_host = wts.cpu().numpy()
    got, iters, relres, ws = _launch(wts, ab, np.stack([mask] * len(labs)), 1)
    assert (iters == 1).all() and (relres == 0).all(), (iters.tolist(), relres.tolist())
    for j in range(len(labs)):
        b = levin_ref.rhs(w_host[j], ab[j], mask)
        assert np.array_equal(_bits(got[j]), _bits(np.where(mask > 0, ab[j], b.astype(np.float32)))), j
        assert np.array_equal(_u(ws, j, h, w), b), j


def _stochastic_weights(h, w, seed):
    """Hand-built rows: random positive weights on the in-image neighbours summing to 1, except that the 2 x 2 block
    at (5, 5) points only inside itself (a closed set), (4, 5) points only into that block and (9, 9) has no weight at
    all: those six pixels reach no hint.  No other pixel points at them, so every pixel that reaches a hint has only
    neighbours whose u is c."""
    rs = np.random.RandomState(seed)
    inside = levin_ref.sigma(np.zeros((h, w)))[3]
    wt = np.where(inside, rs.rand(8, h, w) + 0.05, 0.0)
    k = {o: i for i, o in enumerate(levin_ref.OFFSETS)}
    block = {(5, 5), (5, 6), (6, 5), (6, 6)}
    dark = block | {(4, 5), (9, 9)}
    for y in range(h):
        for x in range(w):
            for (dy, dx), i in k.items():
                q = (y + dy, x + dx)
                if (y, x) in block | {(4, 5)} and q not in block or (y, x) not in dark and q in dark:
                    wt[i, y, x] = 0.0
    wt[:, 9, 9] = 0.0
    tot = wt.sum(0)
    return wt / np.where(tot > 0, tot, 1.0), sorted(dark)


def test_one_colour_everywhere_it_reaches():
    """Every hint a (c_a, c_b): u = c on each pixel that reaches a hint and 0 elsewhere.  ||u - c|| <= ||A_RR^-1||_2
    tol ||b||, A_RR the system on the reaching pixels; out_ab is float32(u)."""
    h, w = 24, 40                                                # 960 pixels: warp 15 holds pixels in every sum
    wt, dark = _stochastic_weights(h, w, 3)
    rs = np.random.RandomState(4)
    colour = np.array([23.5, -61.25], np.float32)
    masks, abs_ = [], []
    for frac in (0.0, 0.01, 0.3):
        m = (rs.rand(h, w) < frac).astype(np.float32)
        m[12, 20] = 1
        for y, x in dark:
            m[y, x] = 0
        masks.append(m)
        ab = (rs.rand(2, h, w) * 200 - 100).astype(np.float32)    # free pixels carry other colours: not hints
        ab[:, m > 0] = colour[:, None]
        abs_.append(ab)
    ab, mask = np.stack(abs_), np.stack(masks)
    got, iters, relres, ws = _launch(torch.from_numpy(wt[None]).cuda(), ab, mask, len(masks))
    for j in range(len(masks)):
        hinted = mask[j] > 0
        reach = levin_ref.reaching(wt, hinted)
        assert all(not reach[p] for p in dark) and reach.sum() == h * w - hinted.sum() - len(dark)
        _check_solve(wt, ab[j], mask[j], got[j], relres[j], ws, j)
        ridx = np.flatnonzero(reach.ravel())
        A = levin_ref.matrix_rows(wt, hinted).toarray()[np.ix_(ridx, ridx)]
        inv_norm = np.linalg.norm(np.linalg.inv(A), 2)
        b = levin_ref.rhs(wt, ab[j], mask[j])
        for c in range(2):
            bound = inv_norm * TOL * np.linalg.norm(b[c]) + np.spacing(abs(colour[c]))
            assert np.abs(got[j, c][reach] - colour[c]).max() <= bound, (j, c)
            assert (got[j, c][~reach & ~hinted] == 0).all() and (got[j, c][hinted] == colour[c]).all()


def _symmetry_case(shape, seed):
    h, w = shape
    lab = _lab(_photo(h, w, seed))
    wts = _weights([lab])
    assert wts[wts > 0].min().item() > 1e-15                    # no subnormal product: doubling commutes with rounding
    return lab, wts


@pytest.mark.parametrize("shape", [(24, 40), (64, 64)])
def test_channels_swap_and_scale_bit_for_bit(shape):
    """The two channels run the same FP64 operations in lockstep: swapping the a and b planes swaps every result, and
    b = 2 a gives out_b = 2 out_a with the same iterations and relres, bit for bit."""
    h, w = shape
    lab, wts = _symmetry_case(shape, 50)
    A, B = np.float32(lab[1]), np.float32(lab[2])
    ab, mask = [], []
    for m in _masks(h, w, 7)[1:4]:
        for planes in ((A, B), (B, A), (A, 2 * A)):
            ab.append(np.stack(planes))
            mask.append(m)
    ab, mask = np.stack(ab), np.stack(mask)
    got, iters, relres, ws = _launch(wts, ab, mask, len(ab))
    for j in range(0, len(ab), 3):
        assert np.array_equal(_bits(got[j + 1]), _bits(got[j][::-1]))
        assert iters[j + 1].tolist() == iters[j][::-1].tolist() and relres[j + 1].tolist() == relres[j][::-1].tolist()
        assert np.array_equal(_bits(got[j + 2, 1]), _bits(2 * got[j + 2, 0]))
        assert iters[j + 2, 0] == iters[j + 2, 1] and relres[j + 2, 0] == relres[j + 2, 1]
        # and channel a of (A, 2A) is channel a of (A, B): the other channel's hints do not touch it
        assert np.array_equal(_bits(got[j + 2, 0]), _bits(got[j, 0])) and iters[j + 2, 0] == iters[j, 0]
    assert (relres <= TOL).all()


def test_zero_channel_stops_at_once_and_leaves_the_other_alone():
    """All a hints 0 (b = 0 in that channel, colours on free pixels that are not hints): iters 0, relres 0, exact zeros;
    the other channel equals a launch in which both channels carry its hints, bit for bit, workspace u included."""
    h, w = 33, 40
    lab, wts = _symmetry_case((h, w), 51)
    m = _masks(h, w, 8)[2]
    B = np.float32(lab[2])
    Z = np.where(m > 0, 0, np.float32(lab[1])).astype(np.float32)
    ab = np.stack([np.stack(p) for p in ((Z, B), (B, B), (B, Z))])
    got, iters, relres, ws = _launch(wts, ab, np.stack([m] * 3), 3)
    assert iters[0, 0] == 0 and relres[0, 0] == 0 and (got[0, 0] == 0).all() and (_u(ws, 0, h, w)[0] == 0).all()
    assert iters[2, 1] == 0 and relres[2, 1] == 0 and (got[2, 1] == 0).all()
    assert iters[1, 0] > 0
    for j, c in ((0, 1), (2, 0)):
        assert np.array_equal(_bits(got[j, c]), _bits(got[1, c])) and iters[j, c] == iters[1, c]
        assert relres[j, c] == relres[1, c] and np.array_equal(_u(ws, j, h, w)[c], _u(ws, 1, h, w)[c])


def test_singular_system_breaks_down_restarts_and_stops_at_max_iter():
    """Free pixels (1, 1) and (1, 2) of a 4 x 4 image point at each other with weight 1 and at the hint above with 0.5:
    A = [[1, -1], [-1, 1]].  Channel a's hints give b = (1, 1), a null vector of A, so (rhat, v) = (b, A b) = 0 at
    every attempt and there is no solution: break down, restart from u = 0 with p = v = 0, until max_iter; relres 1.
    Channel b's give b = (1, -1), an eigenvector: one exact step to u = (0.5, -0.5)."""
    h = w = 4
    k = {o: i for i, o in enumerate(levin_ref.OFFSETS)}
    wt = np.zeros((8, h, w))
    wt[k[(0, 1)], 1, 1] = wt[k[(0, -1)], 1, 2] = 1.0
    wt[k[(-1, 0)], 1, 1] = wt[k[(-1, 0)], 1, 2] = 0.5
    mask = np.ones((h, w), np.float32)
    mask[1, 1] = mask[1, 2] = 0
    ab = np.full((2, h, w), 7.0, np.float32)
    ab[:, 0, 1] = (2, 2)
    ab[:, 0, 2] = (2, -2)
    max_iter = 37
    got, iters, relres, ws = _launch(torch.from_numpy(wt[None]).cuda(), ab[None], mask[None], 1, max_iter=max_iter)
    assert iters[0].tolist() == [max_iter, 1] and relres[0].tolist() == [1.0, 0.0]
    _check_contract(wt, ab, mask, got[0], relres[0], ws, 0)
    free = mask == 0
    assert got[0, 0][free].tolist() == [0.0, 0.0] and got[0, 1][free].tolist() == [0.5, -0.5]
    # the state channel a stops in is the state every attempt starts from: r = rhat = p = b, v = A p = 0, u = 0
    vec = {name: levin_ref.workspace(ws, h, w, 0, 0, name)[free].tolist() for name in levin_ref.WS_VECS}
    assert vec == {"u": [0.0, 0.0], "r": [1.0, 1.0], "rhat": [1.0, 1.0], "p": [1.0, 1.0], "v": [0.0, 0.0],
                   "t": [1.0, 1.0]}, vec


def _hard_case():
    """A 64 x 64 photo with 5 points: hundreds of iterations."""
    lab = _lab(_photo(64, 64, 52))
    ab, mask, _ = _paint(lab, photos.reveal_points(64, 5, 12, 0))
    return _weights([lab]), ab, mask


@pytest.mark.parametrize("max_iter", [1, 7, 50])
def test_max_iter_stops_with_the_true_residual(max_iter):
    wts, ab, mask = _hard_case()
    got, iters, relres, ws = _launch(wts, ab[None], mask, 1, max_iter=max_iter)
    assert (iters == max_iter).all() and (relres > TOL).all(), (iters.tolist(), relres.tolist())
    _check_contract(wts.cpu().numpy()[0], ab, mask[0], got[0], relres[0], ws, 0)


def test_very_tight_tol_reports_the_true_residual():
    """tol 1e-14 is at FP64's floor for this system: whatever the outcome, relres is the true residual, and a channel
    either reached tol or spent max_iter."""
    wts, ab, mask = _hard_case()
    tol = 1e-14
    got, iters, relres, ws = _launch(wts, ab[None], mask, 1, tol=tol)
    w_host = wts.cpu().numpy()[0]
    mis = _check_contract(w_host, ab, mask[0], got[0], relres[0], ws, 0, tol=tol)
    assert ((relres[0] <= tol) | (iters[0] == photos.LEVIN_MAX_ITER)).all()
    # a restart replaces rhat = b with the true residual of the moment
    b = levin_ref.rhs(w_host, ab, mask[0])
    restarted = [not np.array_equal(levin_ref.workspace(ws, 64, 64, 0, c, "rhat"), b[c]) for c in range(2)]
    REPORT["tight tol"] = (iters[0].tolist(), relres[0].tolist(), restarted, mis)
    print("levin tol 1e-14 at 64x64: iterations %s, relres %s, restarted %s, relres mismatch %.3g"
          % REPORT["tight tol"])


def test_batch_of_300_with_7_levels_equals_solo_launches():
    """n = 300 images of 16 x 24, levels = 7: 43 photos, the last with 6 levels, and more CTAs than an H100 has SMs.
    The levels mix 0, 1 and many hints.  Each image equals a launch of it alone with its photo's weights, bit for bit,
    workspace u included."""
    h, w, levels, n = 16, 24, 7, 300
    counts = (0, 1, 2, 5, 20, 96, 300)
    labs = [_lab(_photo(h, w, 100 + p)) for p in range(-(-n // levels))]
    ab, mask = [], []
    for j in range(n):
        order = np.random.RandomState(j // levels).permutation(h * w)
        m = np.zeros(h * w, np.float32)
        m[order[:counts[j % levels]]] = 1
        mask.append(m.reshape(h, w))
        ab.append(np.float32(labs[j // levels][1:]))
    ab, mask = np.stack(ab), np.stack(mask)
    wts = _weights(labs)
    w_host = wts.cpu().numpy()
    got, iters, relres, ws = _launch(wts, ab, mask, levels)
    for j in range(n):
        p = j // levels
        one = _launch(wts[p:p + 1], ab[j:j + 1], mask[j:j + 1], 1)
        assert np.array_equal(_bits(got[j]), _bits(one[0][0])), j
        assert iters[j].tolist() == one[1][0].tolist() and relres[j].tolist() == one[2][0].tolist(), j
        assert np.array_equal(_u(ws, j, h, w), _u(one[3], 0, h, w)), j
        if counts[j % levels] == 0:
            assert iters[j].tolist() == [0, 0] and relres[j].tolist() == [0.0, 0.0] and (got[j] == 0).all()
        else:
            _check_solve(w_host[p], ab[j], mask[j], got[j], relres[j], ws, j)
