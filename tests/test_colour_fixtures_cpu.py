"""CPU: the fixtures of tests/test_gpu_colour_exhaustive.py hold what that file relies on, without a device: the
all-colour layout, the chunked oracle, the Lab grid, the linear-RGB knee points and the host cell rule of
the global statistics."""
import numpy as np
import pytest

from oracle import color_ref
from tests import test_gpu_colour_exhaustive as X


@pytest.fixture(scope="module")
def colours():
    return X.all_colours()


def test_all_colour_layout(colours):
    rgb = colours
    assert rgb.shape == (64, 512, 512, 3) and rgb.dtype == np.uint8
    idx = (rgb[..., 0].astype(np.int64) << 16) | (rgb[..., 1].astype(np.int64) << 8) | rgb[..., 2]
    assert np.array_equal(idx.reshape(-1), np.arange(1 << 24))          # every colour exactly once, in order
    assert tuple(rgb[1, 2, 3]) == (4, 4, 3)                              # i = 1 << 18 | 2 << 9 | 3


def test_chunked_oracle_equals_unchunked(colours):
    rgb = colours
    part = rgb[14:18]                                                    # straddles a chunk boundary
    got = X.oracle_rgb2lab(part)
    assert np.array_equal(got[:2], X.oracle_rgb2lab(rgb[:16])[14:])     # same image, other chunk position
    whole = color_ref.rgb2lab(part)
    assert np.array_equal(got, whole) or X.lab_ulps(got, whole).max() <= 1
    flat = color_ref.rgb2lab(part.reshape(-1, 3)).reshape(part.shape)
    assert X.lab_ulps(got, flat).max() <= 1


def test_lab_ulps_scale():
    ref = np.array([[50.0, 0.0, 0.0]])
    assert X.lab_ulps(ref, ref).max() == 0
    got = ref + np.spacing(X.LAB_SCALE) * np.array([3, -2, 1])
    assert np.array_equal(X.lab_ulps(got, ref)[0], [3, 2, 1])


def test_grid():
    L, ab = X.grid_L(), X.grid_ab()
    assert L[0] == 0 and L[-1] == 100 and np.all(np.diff(L) > 0)
    for v in (1e-6, 7.9999, 8.001, 99.999, 8.0, 50.0):
        assert v in L
    knee = 116.0 * X.FINV_KNEE - 16.0
    assert knee in L and abs(knee - 8.0000056) < 1e-12
    assert (knee + 16.0) / 116.0 == pytest.approx(X.FINV_KNEE, abs=1e-15)
    assert ab[0] == -128 and ab[-1] == 127.5 and len(ab) == 512
    img = X.grid_image(8.0)
    assert img.shape == (3, 512, 512) and img[1, 5, 9] == ab[5] and img[2, 5, 9] == ab[9]
    # the grid crosses the fz < 0 clamp (fz = fy - b / 200) at every L, and the ab planes are exact in float32
    fz = (img[0] + 16) / 116 - img[2] / 200
    assert (fz < 0).any() and (fz > 0).any()
    assert np.array_equal(img[1:].astype(np.float32), img[1:])


def test_knee_points_land_at_the_gamma_knee():
    pts = X.knee_lab()
    lin = color_ref.lab2linear(pts)
    t = np.spacing(X.GAMMA_KNEE)
    off = (lin - X.GAMMA_KNEE) / t
    at = np.abs(off) <= X.KNEE_SIDE_ULPS
    assert at.any(-1).all()                                              # every point has a channel in the window
    for ch in range(3):
        o = off[at[:, ch], ch]
        assert (o < 0).sum() >= 10 and (o > 0).sum() >= 10, (ch, (o < 0).sum(), (o > 0).sum())
    # these points are where srgb_gamma's branch is decided; the two branches meet within 1e-5 of each other in
    # 255 units there (10.3147...), so either branch truncates to 10
    for c in lin[at]:
        assert int(255 * 12.92 * c) == int(255 * (1.055 * c ** (1 / 2.4) - 0.055)) == 10


def test_stats_host_rule_matches_the_oracle_histogram():
    """stats_cells_host on oracle Lab reproduces caffe_spec.global_stats' histogram up to cells within 1e-3 of a bin
    boundary (the oracle pools with numpy's mean, not the sequential sum)."""
    from oracle import caffe_spec
    rs = np.random.RandomState(2)
    img = rs.randint(0, 256, (64, 96, 3)).astype(np.uint8)
    lab = color_ref.rgb2lab(img).transpose(2, 0, 1)[None]
    bins = X.stats_cells_host(lab)[0]
    hist = np.bincount(bins, minlength=313) / bins.size
    ref = caffe_spec.global_stats(img, X.PTS)
    assert np.abs(hist - ref[:313]).sum() * bins.size / 2 <= 2
