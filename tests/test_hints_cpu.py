"""CPU: hint lists (idc_set_hints semantics) and the gamut map oracle.

* the numpy raster oracle equals cv2.rectangle painting (the GUI's PointEdit.updateInput) on random edits;
* hints_from_points equals put_point, numpy slice semantics included (negative starts wrap to an empty slice);
* the launcher's list builder equals get_input() + rgb2lab of a Qt-free fake GUI, within one float32 ulp;
* converting each hint colour on its own vs inside a 256x256 image differs by at most one float32 ulp, over all 2^24
  uint8 colours;
* oracle/gamut_ref.py equals the reference's abGrid.update_gamut (tests/golden/gamut_ref.npz)."""
import os

import numpy as np
import pytest

from interactive_deep_colorization_b200 import color
from interactive_deep_colorization_b200 import colorize_image as CI
from interactive_deep_colorization_b200 import launcher
from oracle import gamut_ref, hints_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _random_rects(rs, n, X, n_img=1):
    out = np.zeros(n, CI.HINT_LIST_DTYPE)
    for i in range(n):
        y0, x0 = rs.randint(-6, X + 6, 2)
        h, w = rs.randint(-2, 12, 2)                   # negative extents: empty rectangles
        ab = (0.0, 0.0) if rs.rand() < 0.15 else tuple(rs.uniform(-110, 110, 2))   # zero-colour hints carry mask 1
        out[i] = (rs.randint(n_img), y0, x0, y0 + h, x0 + w) + ab
    return out


def test_raster_oracle_matches_cv2_rectangle():
    import cv2
    rs = np.random.RandomState(0)
    X = 48
    for trial in range(40):
        rects = _random_rects(rs, rs.randint(0, 30), X)
        if trial == 0:                                 # every border crossed, full cover, overlaps
            rects = np.array([(0, -5, -5, 3, 3, 1, 2), (0, X - 3, X - 3, X + 9, X + 9, 3, 4), (0, -1, 10, X, 12, 5, 6),
                              (0, 0, 0, X - 1, X - 1, 0, 0), (0, 20, 20, 21, 21, 7, 8)], CI.HINT_LIST_DTYPE)
        ab, mask = hints_ref.raster(rects, 1, X, X, dtype=np.float64)
        im_a, im_b = np.zeros((X, X)), np.zeros((X, X))
        m = np.zeros((X, X), np.uint8)
        for r in rects:
            if r["y1"] < r["y0"] or r["x1"] < r["x0"]:
                continue                               # cv2 would reorder the corners; an inverted hint is empty
            tl, br = (int(r["x0"]), int(r["y0"])), (int(r["x1"]), int(r["y1"]))
            cv2.rectangle(im_a, tl, br, float(r["a"]), -1)
            cv2.rectangle(im_b, tl, br, float(r["b"]), -1)
            cv2.rectangle(m, tl, br, 255, -1)
        assert np.array_equal(ab[0, 0], im_a) and np.array_equal(ab[0, 1], im_b)
        assert np.array_equal(mask[0, 0], (m > 0).astype(np.float64))
        # the product's host raster (lazy wrapper planes) is the same function of the list
        pab, pmask = CI.raster_hints(rects, X)
        assert np.array_equal(pab, ab[0]) and np.array_equal(pmask, mask[0])


def test_hints_from_points_matches_put_point():
    rs = np.random.RandomState(1)
    X = 40
    for trial in range(60):
        pts = []
        for _ in range(rs.randint(1, 12)):
            loc = rs.randint(-8, X + 8, 2)
            pts.append((loc, int(rs.randint(0, 6)), rs.uniform(-100, 100, 2)))
        if trial == 0:                                 # wrapped negative starts: put_point paints nothing there
            pts = [((1, 20), 3, (10., 20.)), ((20, 2), 4, (30., 40.)), ((-5, -5), 1, (5., 5.)), ((X - 1, X - 1), 2, (1., 1.))]
        ab, mask = np.zeros((2, X, X)), np.zeros((1, X, X))
        for loc, p, val in pts:
            CI.put_point(ab, mask, loc, p, val)
        rects = CI.hints_from_points(pts, X)
        rab, rmask = hints_ref.raster(rects, 1, X, X, dtype=np.float64)
        assert np.array_equal(rab[0], ab) and np.array_equal(rmask[0], mask), trial


class _Pt(object):
    def __init__(self, x, y):
        self._x, self._y = x, y

    def x(self):
        return self._x

    def y(self):
        return self._y


class _Color(object):
    def __init__(self, rgb):
        self.rgb = rgb

    def red(self):
        return self.rgb[0]

    def green(self):
        return self.rgb[1]

    def blue(self):
        return self.rgb[2]


class FakePointEdit(object):
    """Qt-free stand-in for ui/ui_control.py PointEdit: the test's own window -> load_size mapping."""

    def __init__(self, pnt, rgb, width, win_size=512, load_size=256, img_size=(480, 360)):
        self.pnt, self.color, self.width = _Pt(*pnt), _Color(rgb), width
        self.load_size, self.img_w, self.img_h = load_size, img_size[0], img_size[1]
        self.scale = float(max(img_size)) / load_size
        self.dw, self.dh = (win_size - img_size[0]) // 2, (win_size - img_size[1]) // 2

    def scale_point(self, in_x, in_y, w):
        return (int((in_x - self.dw) / float(self.img_w) * self.load_size) + w,
                int((in_y - self.dh) / float(self.img_h) * self.load_size) + w)

    def paint(self, im, mask):
        import cv2
        w = int(self.width / self.scale)
        tl = self.scale_point(self.pnt.x(), self.pnt.y(), -w)
        br = self.scale_point(self.pnt.x(), self.pnt.y(), w)
        cv2.rectangle(mask, tl, br, 255, -1)
        cv2.rectangle(im, tl, br, tuple(int(v) for v in self.color.rgb), -1)


class FakeUIControl(object):
    def __init__(self, edits, load_size=256):
        self.userEdits, self.load_size = edits, load_size

    def get_input(self):
        im = np.zeros((self.load_size, self.load_size, 3), np.uint8)
        mask = np.zeros((self.load_size, self.load_size, 1), np.uint8)
        for ue in self.userEdits:
            ue.paint(im, mask)
        return im, mask


def fake_edits(rs, n):
    return [FakePointEdit((int(rs.randint(0, 512)), int(rs.randint(0, 512))), tuple(int(v) for v in rs.randint(0, 256, 3)),
                          int(rs.randint(1, 12))) for _ in range(n)]


def dense_gui_planes(ui):
    """compute_result's statements (ui/gui_draw.py:273-277)."""
    im, mask = ui.get_input()
    return color.rgb2lab(im).transpose((2, 0, 1))[1:3], (mask > 0.0).transpose((2, 0, 1))


def _ulps32(a, b):
    a32, b32 = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a32.astype(np.float64) - b32.astype(np.float64)) / np.spacing(np.maximum(np.abs(a32), np.abs(b32)))


def test_gui_hint_list_matches_dense_get_input():
    rs = np.random.RandomState(2)
    for trial in range(25):
        ui = FakeUIControl(fake_edits(rs, rs.randint(0, 25)))
        rects = launcher.gui_hint_list(ui)
        ab_d, mask_d = dense_gui_planes(ui)
        ab_h, mask_h = CI.raster_hints(rects, 256)
        assert np.array_equal(mask_h > 0, mask_d), trial
        assert np.all(_ulps32(ab_h, ab_d) <= 1), trial


def test_per_colour_conversion_within_one_float32_ulp_of_dense():
    """All 2^24 uint8 colours: converted the way the hook does (one rgb2lab batch of <= 64 distinct colours) vs inside
    a 256x256 painted image (the dense GUI path).  Every difference is <= 1 float32 ulp in a or b."""
    g, b = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    n_diff = 0
    for r0 in range(0, 256, 16):
        rgb = np.empty((16, 256, 256, 3), np.uint8)
        rgb[..., 0] = np.arange(r0, r0 + 16, dtype=np.uint8)[:, None, None]
        rgb[..., 1], rgb[..., 2] = g, b
        dense = np.stack([color.rgb2lab(im) for im in rgb])                     # 256x256 images, as get_input paints
        batched = color.rgb2lab(rgb.reshape(-1, 64, 3)).reshape(dense.shape)   # [1, 64, 3] batches, stacked
        u = np.maximum(_ulps32(batched[..., 1], dense[..., 1]), _ulps32(batched[..., 2], dense[..., 2]))
        assert u.max() <= 1
        n_diff += int(np.count_nonzero(u))
    print("colours whose float32 ab differs by one ulp between the two layouts: %d" % n_diff)


def _golden_gamut():
    g = np.load(os.path.join(ROOT, "tests", "golden", "gamut_ref.npz"))
    shape = tuple(g["mask_shape"])
    mask = np.unpackbits(g["mask"], axis=-1)[..., :shape[-1]].astype(bool)
    return g, mask


def test_gamut_oracle_matches_reference_golden():
    g, mask = _golden_gamut()
    for i, L in enumerate(g["L"]):
        rgb, m = gamut_ref.update_gamut(float(L), int(g["gamut_size"]), int(g["D"]))
        assert np.array_equal(m, mask[i]), L
        assert np.array_equal(rgb, g["masked_rgb"][i]), L


@pytest.mark.parametrize("D", [1, 2, 3])
def test_gamut_oracle_grid_matches_arange(D):
    a, b = gamut_ref.grid(110, D)
    A = len(np.arange(-110, 110 + D, D))
    assert a.shape == (A, A) and np.all(a[:, 0] == np.arange(-110, 110 + D, D)) and np.all(b[0] == a[:, 0])
