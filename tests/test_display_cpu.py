"""CPU: the cubic resize rule the GUI's display step restates (tests/cubic_ref.py, what cubic_lab2rgb_kernel follows)
against the installed cv2.resize(INTER_CUBIC) on float64 ab planes, bit for bit."""
import cv2
import numpy as np
import pytest

from tests import cubic_ref

# (h_in, w_in, H, W): up-scales, down-scales, the exact 2x, 1-pixel outputs and inputs, odd and prime sizes
GEOMETRIES = [(256, 256, 512, 512), (256, 256, 384, 600), (256, 256, 200, 256), (256, 256, 700, 700),
              (256, 256, 513, 511), (256, 256, 128, 128), (256, 256, 100, 80), (256, 256, 1, 1), (256, 256, 1, 300),
              (256, 256, 91, 1), (64, 96, 37, 1), (64, 64, 128, 128), (1, 1, 5, 7), (1, 256, 3, 512), (97, 89, 251, 257),
              (13, 17, 1031, 1033), (1009, 1013, 23, 29)]


def gui_window(h, w, win=512):
    """(win_h, win_w) the GUI shows an h x w photo at (ui/gui_draw.py read_image): the long side scaled to `win`, both
    sides rounded to a multiple of 4."""
    r = win / float(max(h, w))
    return int(round(r * h / 4.0) * 4), int(round(r * w / 4.0) * 4)


# the display sizes of a square photo, 3456 x 5184, 4000 x 6000 (both orientations), 4:3, 16:9 and 507 x 600, at the
# default 512-pixel window, from the 256 x 256 network output
GUI_GEOMETRIES = sorted({(256, 256) + gui_window(h, w) for (h, w) in ((512, 512), (3456, 5184), (5184, 3456),
                                                                      (4000, 6000), (3000, 4000), (1080, 1920),
                                                                      (507, 600))})


def random_geometries(n, seed=0):
    """A seeded sweep of (h_in, w_in, H, W) with every side in 1 ... 1100."""
    rs = np.random.RandomState(seed)
    return [tuple(int(v) for v in rs.randint(1, 1101, 4)) for _ in range(n)]


def _cv2_display(ab, H, W):
    """The GUI's statement (ui/gui_draw.py:281): ab [2,h,w] -> [H,W,2]."""
    out = cv2.resize(ab.transpose((1, 2, 0)), (W, H), interpolation=cv2.INTER_CUBIC)
    return out.reshape(H, W, 2)


def test_gui_window_sizes():
    assert gui_window(3456, 5184) == (340, 512) and gui_window(5184, 3456) == (512, 340)
    assert gui_window(3000, 4000) == (384, 512) and gui_window(1080, 1920) == (288, 512)
    assert (256, 256, 512, 512) in GUI_GEOMETRIES and len(GUI_GEOMETRIES) == 6


@pytest.mark.parametrize("h_in,w_in,H,W", GEOMETRIES + GUI_GEOMETRIES)
def test_cubic_resize_equals_cv2(h_in, w_in, H, W):
    ab = np.random.RandomState(h_in * 31 + W).uniform(-110, 110, (2, h_in, w_in))
    got = cubic_ref.resize(ab.transpose((1, 2, 0)), W, H)
    assert got.shape == (H, W, 2) and np.array_equal(got, _cv2_display(ab, H, W))


def test_cubic_resize_random_sweep_equals_cv2():
    rs = np.random.RandomState(1)
    for (h_in, w_in, H, W) in random_geometries(40):
        ab = rs.uniform(-110, 110, (2, h_in, w_in))
        got = cubic_ref.resize(ab.transpose((1, 2, 0)), W, H)
        assert np.array_equal(got, _cv2_display(ab, H, W)), (h_in, w_in, H, W)


def test_cubic_weights_equal_cv2_on_one_hot_rows():
    """Each output of a one-hot row is one tap's weight (or the sum of the clamped taps): the float32 weights
    themselves, isolated from the sums."""
    for (n_in, n_out) in ((256, 512), (256, 600), (256, 200), (7, 1033), (1013, 29)):
        idx, w = cubic_ref.taps(n_in, n_out)
        for j in sorted({0, 1, n_in // 2, n_in - 2, n_in - 1}):
            row = np.zeros((1, n_in))
            row[0, j] = 1.0
            got = cv2.resize(row, (n_out, 1), interpolation=cv2.INTER_CUBIC)[0]
            want = np.where(idx == j, w.astype(np.float64), 0.0).sum(axis=0)
            assert np.array_equal(got, want), (n_in, n_out, j)

