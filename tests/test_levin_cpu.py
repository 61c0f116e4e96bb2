"""CPU: the Levin baseline of reveal sweeps -- its float64 oracle (tests/levin_ref.py: the weight rule, its floors, the
reachability rule and the degenerate cases, the solver's right-hand side, true residual and workspace layout), the
argument checks of idc_levin_solve (idc_levin_check and the device
entry points, IDC_ERR_ARG before any device call), the method's argument checks and the command line."""
import ctypes
import os

import numpy as np
import pytest
import scipy.sparse as sp

import ideepcolor_b200 as cli
from interactive_deep_colorization_b200 import _lib, photos
from tests import levin_ref
from tests.test_reveal_cpu import FakeColorizer, _img


def _smooth(h, w, seed):
    rs = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w]
    return 30 + 40 * np.sin(x / 7.0) * np.cos(y / 11.0) + rs.rand(h, w) * 5


def _edges(h, w):
    """Flat regions and hard edges: four constant blocks, one of them with a ramp."""
    L = np.full((h, w), 20.0)
    L[:, w // 2:] = 80.0
    L[h // 2:, :w // 3] = 50.0
    L[:h // 3, w // 2:] += np.linspace(0, 5, w - w // 2)
    return L


@pytest.mark.parametrize("L", [_smooth(24, 31, 0), _edges(20, 26), np.full((9, 7), 42.0)])
def test_free_rows_sum_to_one(L):
    w = levin_ref.weights(L)
    assert np.allclose(w.sum(0), 1.0, rtol=0, atol=1e-14)
    hinted = np.zeros(L.shape, bool)
    hinted[3, 4] = True
    A = levin_ref.matrix_rows(w, hinted)
    rows = np.asarray(A.sum(1)).ravel()
    assert np.abs(rows[~hinted.ravel()]).max() <= 1e-14                 # u_p - sum w_pq u_q: the rows sum to 0
    assert rows[hinted.ravel()].tolist() == [1.0]
    # outside the image: weight 0
    assert (w[0, 0, :] == 0).all() and (w[0, :, 0] == 0).all() and (w[7, -1, :] == 0).all() and (w[7, :, -1] == 0).all()


def test_floors_engage_on_a_flat_patch_and_at_a_hard_edge():
    # flat: var = 0 and m = 0, so s is the 2e-6 floor and every weight is equal
    s, *_ = levin_ref.sigma(np.full((6, 6), 37.0))
    assert (s == levin_ref.SIGMA_FLOOR).all()
    w = levin_ref.weights(np.full((6, 6), 37.0))
    assert np.allclose(w[:, 2, 2], 1 / 8.0, rtol=0, atol=1e-15)
    assert np.allclose(w[[4, 6, 7], 0, 0], 1 / 3.0, rtol=0, atol=1e-15)
    # a pixel alone on its side of a hard edge: the closest neighbour is across the edge, 0.6 var would let its weight
    # underflow, and the -m / ln 0.01 floor decides s
    L = np.full((5, 5), 10.0)
    L[2, 2] = 90.0
    s, Y, nb, inside = levin_ref.sigma(L)
    m = (0.8) ** 2
    assert s[2, 2] == pytest.approx(-m / np.log(0.01), rel=1e-12)
    assert s[2, 2] > 0.6 * np.var(np.r_[np.full(8, 0.1), 0.9])
    e = levin_ref.weights(L, normalise=False)
    assert e[:, 2, 2].min() == pytest.approx(0.01, rel=1e-12)


@pytest.mark.parametrize("L", [_smooth(24, 31, 1), _edges(20, 26), np.random.RandomState(5).rand(16, 16) * 100])
def test_closest_neighbour_keeps_one_hundredth(L):
    e = levin_ref.weights(L, normalise=False)
    _, Y, nb, inside = levin_ref.sigma(L)
    d2 = np.where(inside, (nb - Y) ** 2, np.inf)
    closest = np.argmin(d2, axis=0)
    kept = np.take_along_axis(e, closest[None], 0)[0]
    assert (kept >= 0.01 * (1 - 1e-12)).all()
    assert (e.max(0) <= 1.0).all()


@pytest.mark.parametrize("L", [_smooth(17, 23, 2), _edges(20, 26)])
def test_one_hint_gives_its_colour_everywhere(L):
    w = levin_ref.weights(L)
    mask = np.zeros(L.shape, np.float32)
    mask[5, 7] = 1
    ab = np.zeros((2,) + L.shape, np.float32)
    ab[:, 5, 7] = (23.5, -61.25)
    u = levin_ref.solve(w, ab, mask)
    reach = levin_ref.reaching(w, mask > 0)
    assert reach.sum() == L.size - 1                     # every weight here is non-zero: everything reaches the hint
    # relative to the hint colour: a direct solve of ~500 unknowns leaves a few ulps
    assert np.abs(u[0] - 23.5).max() <= 1e-12 * 23.5 and np.abs(u[1] + 61.25).max() <= 1e-12 * 61.25


def test_hard_edge_keeps_each_side_near_its_hint():
    L = np.full((24, 24), 15.0)
    L[:, 12:] = 85.0
    L += np.random.RandomState(3).rand(24, 24) * 0.5
    w = levin_ref.weights(L)
    mask = np.zeros(L.shape, np.float32)
    ab = np.zeros((2,) + L.shape, np.float32)
    mask[12, 3], ab[:, 12, 3] = 1, (40, 10)
    mask[12, 20], ab[:, 12, 20] = 1, (-30, -50)
    u = levin_ref.solve(w, ab, mask)
    # within 5% of the distance between the two hint colours (70 in a, 60 in b) of its own side's hint everywhere
    assert np.abs(u[0, :, :12] - 40).max() < 3.0 and np.abs(u[1, :, :12] - 10).max() < 3.0
    assert np.abs(u[0, :, 12:] + 30).max() < 3.0 and np.abs(u[1, :, 12:] + 50).max() < 3.0


def _closed_pair_weights():
    """A 4 x 4 image whose weights are set by hand: pixels (0, 0) and (0, 1) point only at each other (a closed,
    hint-free pair); every other pixel points at its row neighbours; (3, 3) is hinted."""
    w = np.zeros((8, 4, 4))
    k = {o: i for i, o in enumerate(levin_ref.OFFSETS)}
    w[k[(0, 1)], 0, 0] = 1.0
    w[k[(0, -1)], 0, 1] = 1.0
    for y in range(4):
        for x in range(4):
            if y == 0 and x < 2:
                continue
            nbs = [o for o in ((0, -1), (0, 1), (1, 0), (-1, 0)) if 0 <= y + o[0] < 4 and 0 <= x + o[1] < 4
                   and not (y + o[0] == 0 and x + o[1] < 2)]
            for o in nbs:
                w[k[o], y, x] = 1.0 / len(nbs)
    return w


def test_closed_hint_free_pair_is_zero():
    w = _closed_pair_weights()
    mask = np.zeros((4, 4), np.float32)
    mask[3, 3] = 1
    ab = np.zeros((2, 4, 4), np.float32)
    ab[:, 3, 3] = (12.0, -7.0)
    reach = levin_ref.reaching(w, mask > 0)
    assert not reach[0, 0] and not reach[0, 1] and reach.sum() == 13
    u = levin_ref.solve(w, ab, mask)
    assert (u[:, 0, :2] == 0).all()
    assert np.abs(u[0][reach] - 12).max() <= 1e-12 and np.abs(u[1][reach] + 7).max() <= 1e-12


def test_level_zero_is_zero():
    w = levin_ref.weights(_smooth(10, 12, 4))
    u = levin_ref.solve(w, np.full((2, 10, 12), 9.0, np.float32), np.zeros((10, 12), np.float32))
    assert (u == 0).all()


def _hints(L, frac, seed):
    """A mask of about frac of the pixels and hint planes with a colour on EVERY pixel (free ones too: not hints)."""
    rs = np.random.RandomState(seed)
    mask = (rs.rand(*L.shape) < frac).astype(np.float32)
    ab = (rs.rand(2, *L.shape) * 200 - 100).astype(np.float32)
    return ab, mask


@pytest.mark.parametrize("L", [_smooth(17, 23, 5), _edges(20, 26), _smooth(2, 9, 6)])
def test_rhs_is_the_hinted_columns_summed_in_neighbour_order(L):
    w = levin_ref.weights(L)
    ab, mask = _hints(L, 0.3, 7)
    hinted = mask > 0
    b = levin_ref.rhs(w, ab, mask)
    assert (b[:, hinted] == 0).all()
    # bit for bit: a scalar loop over k in neighbour order, each product and sum rounded on its own
    h, wd = L.shape
    for y in range(h):
        for x in range(wd):
            if hinted[y, x]:
                continue
            for c in range(2):
                acc = 0.0
                for k, (dy, dx) in enumerate(levin_ref.OFFSETS):
                    yy, xx = y + dy, x + dx
                    if 0 <= yy < h and 0 <= xx < wd and hinted[yy, xx]:
                        acc = acc + float(w[k, y, x]) * float(ab[c, yy, xx])
                assert b[c, y, x] == acc, (c, y, x)
    # and W_fh c_h of the sparse matrix solve() builds, to rounding
    rows, cols, vals = levin_ref._edges(w)
    W = sp.csr_matrix((vals, (rows, cols)), shape=(L.size, L.size))
    for c in range(2):
        want = W[:, hinted.ravel()] @ ab[c].ravel()[hinted.ravel()].astype(np.float64)
        want[hinted.ravel()] = 0
        assert np.abs(b[c].ravel() - want).max() <= 1e-13 * max(np.abs(want).max(), 1)


def test_residual_is_the_true_relative_residual():
    L = _smooth(19, 21, 8)
    w = levin_ref.weights(L)
    ab, mask = _hints(L, 0.05, 9)
    hinted = mask > 0
    b = levin_ref.rhs(w, ab, mask)
    # u = 0: r = b exactly
    assert levin_ref.residual(w, ab, mask, np.zeros((2,) + L.shape)).tolist() == [1.0, 1.0]
    # the direct solve: a residual at rounding level
    u = levin_ref.solve(w, ab, mask)
    assert (levin_ref.residual(w, ab, mask, u) <= 1e-13).all()
    # a perturbed u: against the sparse matrix of matrix_rows, to rounding; the hinted entries of u do not count
    rs = np.random.RandomState(10)
    v = u + rs.randn(*u.shape) * 1e-3
    v[:, hinted] = 1e30
    A = levin_ref.matrix_rows(w, hinted)
    free = ~hinted.ravel()
    got = levin_ref.residual(w, ab, mask, v)
    for c in range(2):
        x = np.where(hinted, 0.0, v[c]).ravel()
        r = (b[c].ravel() - A @ x)[free]
        want = np.linalg.norm(r) / np.linalg.norm(b[c])
        assert abs(got[c] - want) <= 1e-12 * want
    # a channel whose b is 0 (every hint 0 in a): 0
    ab0 = ab.copy()
    ab0[0][hinted] = 0
    assert levin_ref.residual(w, ab0, mask, v)[0] == 0.0


def test_workspace_reads_each_vector_at_its_offset():
    n, h, w, V = 3, 4, 5, len(levin_ref.WS_VECS)
    hw = h * w
    # a synthetic buffer: the double at ((i * 2 + c) * 6 + v) * hw + p holds i * 1e4 + c * 1e3 + v * 1e2 + p
    ws = np.zeros(n * 2 * V * hw)
    for i in range(n):
        for c in range(2):
            for v in range(V):
                o = ((i * 2 + c) * V + v) * hw
                ws[o:o + hw] = i * 1e4 + c * 1e3 + v * 1e2 + np.arange(hw)
    raw = ws.view(np.uint8)                       # a byte copy, as a device workspace comes back
    for i in range(n):
        for c in range(2):
            for v, name in enumerate(levin_ref.WS_VECS):
                want = (i * 1e4 + c * 1e3 + v * 1e2 + np.arange(hw)).reshape(h, w)
                assert np.array_equal(levin_ref.workspace(raw, h, w, i, c, name), want), (i, c, name)
            assert np.array_equal(levin_ref.workspace(ws, h, w, i, c), levin_ref.workspace(raw, h, w, i, c, "u"))
    assert _lib.load().idc_levin_workspace_bytes(n, h, w) == ws.nbytes     # the C ABI sizes exactly this layout


def test_levin_abi_argument_checks():
    lib = _lib.load()
    P = ctypes.c_void_p(64)          # never dereferenced: the checks run on the host
    n, h, w = 6, 64, 48
    need = lib.idc_levin_workspace_bytes(n, h, w)
    assert need == n * 2 * 6 * h * w * 8
    for bad in ((0, h, w), (65536, h, w), (n, 1, w), (n, h, 1), (n, _lib.MAX_PHOTO_X + 1, w)):
        assert lib.idc_levin_workspace_bytes(*bad) == 0
    good = [n, 3, h, w, P, P, P, 1e-10, 100, P, P, P, P, need]
    msg = ctypes.create_string_buffer(256)
    assert lib.idc_levin_check(*good, msg, 256) == 0
    bad = {0: [0, 65536], 1: [0, n + 1, -1], 2: [1, 0, _lib.MAX_PHOTO_X + 1], 3: [1, 0, _lib.MAX_PHOTO_X + 1],
           4: [None], 5: [None], 6: [None], 7: [0.0, -1e-3, 1.0, float("nan"), float("inf")],
           8: [0, -5, _lib.LEVIN_MAX_ITER + 1], 9: [None], 10: [None], 11: [None], 12: [None, ctypes.c_void_p(68)],
           13: [need - 1, 0]}
    for i, values in bad.items():
        for v in values:
            args = list(good)
            args[i] = v
            assert lib.idc_levin_check(*args, msg, 256) == _lib.ERR_ARG, (i, v)
            assert msg.value, (i, v)
            # the device entry point runs the same checks first, so nothing here reaches a device call
            assert lib.idc_levin_solve(0, *args[:13], args[13], None) == _lib.ERR_ARG, (i, v)
    assert lib.idc_levin_check(*good, None, 0) == 0
    for args in ((0, 0, h, w, P, P, None), (0, n, 1, w, P, P, None), (0, n, h, w, None, P, None),
                 (0, n, h, w, P, None, None)):
        assert lib.idc_levin_weights(*args) == _lib.ERR_ARG, args
    for args in ((0, 0, h, w, P, P, P, None), (0, n, 0, w, P, P, P, None), (0, n, h, w, None, P, P, None),
                 (0, n, h, w, P, None, P, None), (0, n, h, w, P, P, None, None)):
        assert lib.idc_lab2rgb_u8_mc(*args) == _lib.ERR_ARG, args


class FakeLevinDevice(object):
    def __init__(self):
        self.log = []

    def submit_reveal(self, imgs, points, levels, levin=None):
        self.log.append((levels, levin))
        return imgs, points, levels

    def collect_reveal(self, token):
        imgs, points, levels = token
        return [photos.RevealResult(np.zeros(len(levels)), None, None, p) for p in points]

    def discard(self, token):
        pass

    def close(self):
        pass


class FakeLevinColorizer(FakeColorizer):
    def _make_backend(self, state_dict):
        return FakeLevinDevice()


def test_method_arguments():
    pc = FakeLevinColorizer(None, Xd=64, batch=6)
    list(pc.reveal_sweep([_img(0), _img(1)], levels=(0, 5), seed=2))
    list(pc.reveal_sweep([_img(0), _img(1)], levels=(0, 5), seed=2, method="levin"))
    list(pc.reveal_sweep([_img(0)], levels=(3,), method="levin", levin_tol=1e-6, levin_max_iter=50))
    assert pc._backend.log[0] == ((0, 5), None)
    assert pc._backend.log[1] == ((0, 5), (photos.LEVIN_TOL, photos.LEVIN_MAX_ITER, [0, 1]))
    assert pc._backend.log[2] == ((3,), (1e-6, 50, [0]))
    n = len(pc._backend.log)
    for kw in ({"method": "Levin"}, {"method": None}, {"method": "levin", "levin_tol": 0},
               {"method": "levin", "levin_tol": 1.0}, {"method": "levin", "levin_tol": float("nan")},
               {"method": "levin", "levin_max_iter": 0}, {"method": "levin", "levin_max_iter": 2.5},
               {"method": "levin", "levin_max_iter": True}):
        with pytest.raises(ValueError):
            pc.reveal_sweep([_img(0)], levels=(0, 1), **kw)
    assert len(pc._backend.log) == n


def test_cli_reveal_levin_parsing():
    base = ["--color_model", "m.pth", "--image_dir", "d", "--out", "o"]
    assert cli.parse_args(base + ["--reveal_sweep", "0,5", "--reveal_levin"]).reveal_levin
    assert not cli.parse_args(base + ["--reveal_sweep", "0,5"]).reveal_levin
    with pytest.raises(SystemExit):
        cli.parse_args(base + ["--reveal_levin"])                                 # needs --reveal_sweep


def test_cli_reveal_levin_csv(tmp_path, monkeypatch, capsys):
    import cv2
    import torch
    d = tmp_path / "photos"
    d.mkdir()
    for i, name in enumerate(("b.png", "a.png", "c.jpg")):
        cv2.imwrite(str(d / name), _img(10 * (i + 1)))
    torch.save({}, str(tmp_path / "m.pth"))
    seen = []

    class Fake(FakeColorizer):
        def reveal_sweep(self, paths, levels, seed, method="network"):
            seen.append(method)
            off = 100.0 if method == "levin" else 0.0
            return iter(photos.RevealResult(np.array([off + i + 10.0 * j for j in range(len(levels))]), None, None,
                                            None) for i in range(len(paths)))

    monkeypatch.setattr(photos, "PhotoColorizer", Fake)
    out = tmp_path / "out"
    rc = cli.main(["--color_model", str(tmp_path / "m.pth"), "--image_dir", str(d), "--out", str(out),
                   "--reveal_sweep", "0,5,20", "--batch", "6", "--load_size", "64", "--reveal_levin"])
    assert rc == 0
    assert sorted(seen) == ["levin", "network"]
    assert sorted(os.listdir(str(out))) == ["reveal_psnr.csv", "reveal_psnr_levin.csv"]
    net = (out / "reveal_psnr.csv").read_text().splitlines()
    lev = (out / "reveal_psnr_levin.csv").read_text().splitlines()
    assert net[0] == lev[0] == "image,0,5,20"
    assert [l.split(",")[0] for l in lev[1:]] == ["a.png", "b.png", "c.jpg", "mean"]
    assert [float(v) for v in net[1].split(",")[1:]] == [0.0, 10.0, 20.0]
    assert [float(v) for v in lev[1].split(",")[1:]] == [100.0, 110.0, 120.0]
    assert [float(v) for v in lev[-1].split(",")[1:]] == [101.0, 111.0, 121.0]
    # without the flag the network's CSV is the same file, and no baseline is run
    seen.clear()
    out2 = tmp_path / "out2"
    cli.main(["--color_model", str(tmp_path / "m.pth"), "--image_dir", str(d), "--out", str(out2),
              "--reveal_sweep", "0,5,20", "--batch", "6", "--load_size", "64"])
    assert seen == ["network"] and os.listdir(str(out2)) == ["reveal_psnr.csv"]
    assert (out2 / "reveal_psnr.csv").read_text() == (out / "reveal_psnr.csv").read_text()
