"""GPU: the full-resolution renders (render_planes_kernel, idc_render_planes_u8) -- get_img_fullres,
get_img_gray_fullres, get_input_img_fullres, get_img_mask_fullres and get_sup_fullres of the wrapper classes (reference
data/colorize_image.py:119-158) -- against scipy.ndimage.zoom + oracle/color_ref, and against ColorizeImageBase's own
statements on the same object."""
import cv2
import numpy as np
import pytest
from scipy.ndimage import zoom

from interactive_deep_colorization_b200 import _lib, color, prepost
from interactive_deep_colorization_b200 import colorize_image as CI
from oracle import color_ref
from tests import util, zoom_ref
from tests.test_gpu_configs import _caffe_scaled, _glob_sd

pytestmark = pytest.mark.gpu
PLANE, MASK, SUP = _lib.RENDER_L_PLANE, _lib.RENDER_L_MASK, _lib.RENDER_L_SUP
GETTERS = ("get_img_fullres", "get_img_gray_fullres", "get_input_img_fullres", "get_img_mask_fullres",
           "get_sup_fullres")
# two output sizes past 256 whose float64 ratio 255/(n-1) rounds up (the last row / column reads cval)
OVER = [n for n in range(400, 800) if zoom_ref.overshoot(256, n)[-1]][:2]


def _rgb255(lab2rgb, L, ab):
    """255 * clip(lab2rgb, 0, 1) of L [1,H,W] and ab [2,H,W]: a render before its truncating cast."""
    return np.clip(lab2rgb(np.concatenate((L, ab), axis=0).transpose((1, 2, 0))), 0, 1) * 255


def _close(got, want, what):
    """The bar get_img_fullres meets: every value within 1 LSB, fewer than 1e-3 of them off."""
    assert got.shape == want.shape and got.dtype == np.uint8, (what, got.shape, want.shape)
    d = np.abs(got.astype(int) - want.astype(int))
    assert d.max() <= 1 and (d > 0).mean() < 1e-3, (what, int(d.max()), float((d > 0).mean()))


def _planes(h_in, w_in, H, W, dtype, seed):
    rs = np.random.RandomState(seed)
    ab = rs.uniform(-80, 80, (2, h_in, w_in)).astype(dtype)
    mask = (rs.rand(1, h_in, w_in) < 0.3).astype(dtype)
    mask[0, rs.rand(h_in, w_in) < 0.1] = 0.37          # fractional values exercise the L arithmetic
    L = rs.uniform(0, 100, (1, H, W))
    return ab, mask, L


@pytest.mark.parametrize("h_in,w_in,H,W", [(256, 256, 256, 256), (256, 256, 507, 600), (256, 256, 100, 80),
                                           (64, 64, 75, 91), (256, 256, 1, 300), (64, 64, 91, 1),
                                           (256, 256, 45, 53), (256, 256, OVER[0], OVER[1]), (256, 256, 768, 1280)])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_render_planes_kernel_against_scipy(h_in, w_in, H, W, dtype):
    ab, mask, L = _planes(h_in, w_in, H, W, dtype, seed=H * 7 + W)
    f = (1, H / h_in, W / w_in)
    zeros = np.zeros((2, H, W))
    gray = prepost.render_planes_gpu(H, W, L=L)
    _close(gray, color_ref.lab2rgb_transpose(L, zeros), "gray")
    # get_img_fullres: scipy's order-1 zoom of the (output) ab with the full-resolution L, exact off truncation edges
    full = prepost.fullres_rgb_gpu(ab, L)
    rgb255 = _rgb255(color_ref.lab2rgb, L, zoom(ab, f, order=1))
    util.assert_render_exact(full, rgb255.astype(np.uint8), rgb255, ("fullres", H, W, dtype.__name__))
    for order in (0, 1):
        z_ab = zoom(ab, f, order=order)
        assert z_ab.dtype == dtype and z_ab.shape == (2, H, W)
        inp = prepost.render_planes_gpu(H, W, ab=ab, ab_order=order, L=L)
        _close(inp, color_ref.lab2rgb_transpose(L, z_ab), ("input", order))
        sup = prepost.render_planes_gpu(H, W, ab=ab, ab_order=order, mask=mask, l_mode=SUP)
        _close(sup, color_ref.lab2rgb_transpose(50 * zoom(mask, f, order=0), z_ab), ("sup", order))
    m = prepost.render_planes_gpu(H, W, mask=mask, l_mode=MASK)
    _close(m, color_ref.lab2rgb_transpose(100. * (1 - zoom(mask, f, order=0)), zeros), "mask")
    # overshoot rows / columns carry the cval sample, ab = 0 and m = 0: the mask render's white (L = 100 gives
    # (255, 254, 255): G = 254.9988 truncates), the supervision render's black, the input render's grey
    oy, ox = zoom_ref.overshoot(h_in, H), zoom_ref.overshoot(w_in, W)
    white = color_ref.lab2rgb_transpose(np.full((1, 1, 1), 100.), np.zeros((2, 1, 1)))[0, 0]
    assert list(white) == [255, 254, 255]
    inp = prepost.render_planes_gpu(H, W, ab=ab, ab_order=1, L=L)
    sup = prepost.render_planes_gpu(H, W, ab=ab, ab_order=0, mask=mask, l_mode=SUP)
    for sel in ((oy, slice(None)), (slice(None), ox)):
        assert np.all(m[sel] == white) and np.all(sup[sel] == 0)
        assert np.array_equal(inp[sel], gray[sel]) and np.array_equal(full[sel], gray[sel])
    if (H, W) in ((45, 53), tuple(OVER), (768, 1280)):
        assert oy.sum() == 1 and ox.sum() == 1


def test_binary_mask_render_is_exact():
    """L in {0, 100} with ab = 0: L = 0 is exactly black; at L = 100 R and B clip to 255 and G = 254.9988 sits far from
    the truncation edge, so the device equals the host bit for bit."""
    rs = np.random.RandomState(3)
    for dtype in (np.float64, np.float32):
        mask = (rs.rand(1, 256, 256) < 0.4).astype(dtype)
        for (H, W) in ((507, 600), (45, 53), (1080, 1920)):
            got = prepost.render_planes_gpu(H, W, mask=mask, l_mode=MASK)
            want = color_ref.lab2rgb_transpose(100. * (1 - zoom(mask, (1, H / 256., W / 256.), order=0)),
                                               np.zeros((2, H, W)))
            assert np.array_equal(got, want), (dtype, H, W)


def test_render_planes_error_codes():
    import torch
    lib = _lib.load()
    d = torch.zeros(64, dtype=torch.float64, device="cuda")
    rgb = torch.empty((8, 8, 3), dtype=torch.uint8, device="cuda")
    p = d.data_ptr()
    assert lib.idc_render_planes_u8(0, 4, 4, p, 1, 0, None, 0, MASK, p, 8, 8, rgb.data_ptr(), None) == -1
    assert lib.idc_render_planes_u8(0, 4, 4, p, 2, 0, p, 0, PLANE, p, 8, 8, rgb.data_ptr(), None) == -1
    assert lib.idc_render_planes_u8(0, 4, 4, p, 1, 0, p, 0, PLANE, p, 8, 8, rgb.data_ptr(), None) == 0
    torch.cuda.synchronize()


# ----- the wrapper getters -----
def _photo(H, W, seed):
    """A smooth seeded synthetic photo (a cubic up-sample of coarse noise)."""
    coarse = np.random.RandomState(seed).randint(0, 256, (max(H // 64, 2), max(W // 64, 2), 3)).astype(np.uint8)
    return cv2.resize(coarse, (W, H), interpolation=cv2.INTER_CUBIC)


def _load(cm, tmp_path, H, W, seed=0):
    path = str(tmp_path / ("photo_%d_%d.png" % (H, W)))
    cv2.imwrite(path, np.ascontiguousarray(_photo(H, W, seed)[:, :, ::-1]))
    cm.load_image(path)


POINTS = [([135, 160], 3, [23, -69]), ([100, 60], 5, [-40, 15.5]), ([250, 3], 2, [60, 60]), ([0, 255], 4, [-10, -80])]


def _wrapper(kind, synth_sd, tmp_path):
    """A wrapper of `kind` with the seeded synthetic weights and a 507 x 600 photo loaded."""
    if kind == "torch":
        cm = CI.ColorizeImageB200(Xd=256)
        cm.prep_net(state_dict=synth_sd)
    elif kind == "caffe":
        cm = CI.ColorizeImageB200Caffe(Xd=256)
        cm.prep_net(0, state_dict=_caffe_scaled(synth_sd))
    else:
        cm = CI.ColorizeImageB200GlobDist(Xd=256)
        cm.prep_net(state_dict=_glob_sd(synth_sd)[0])
    _load(cm, tmp_path, 507, 600, seed=1)
    return cm


def _fullres_rgb255(cm):
    """get_img_fullres's host statement before its truncating cast (ColorizeImageBase.get_img_fullres)."""
    return _rgb255(color.lab2rgb, np.asarray(cm.img_l_fullres), cm._to_fullres(cm.output_ab, cm.output_ab, 1))


def _check_getters(cm, what):
    """The device renders first (the host statements below copy the full-resolution L to the host)."""
    dev = {g: getattr(cm, g)() for g in GETTERS}
    assert cm.img_l_fullres._host is None and cm.img_lab_fullres._host is None, what    # L never left the device
    for g in GETTERS:
        host = getattr(CI.ColorizeImageBase, g)(cm)
        if g == "get_img_mask_fullres":
            assert np.array_equal(dev[g], host), (what, g)
        elif g == "get_img_fullres":
            util.assert_render_exact(dev[g], host, _fullres_rgb255(cm), (what, g))
        else:
            _close(dev[g], host, (what, g))


@pytest.mark.parametrize("kind", ["torch", "caffe", "globdist"])
def test_wrapper_getters_match_the_host_statements(kind, synth_sd, tmp_path):
    from interactive_deep_colorization_b200.prepost import DeviceLab
    ab, m = np.zeros((2, 256, 256)), np.zeros((1, 256, 256))
    for (loc, p, val) in POINTS:
        CI.put_point(ab, m, loc, p, val)
    cm = _wrapper(kind, synth_sd, tmp_path)
    assert isinstance(cm.img_l_fullres, DeviceLab)
    cm.net_forward(ab, m)
    _check_getters(cm, (kind, "dense"))
    cm = _wrapper(kind, synth_sd, tmp_path)
    cm.net_forward_hints(CI.hints_from_points(POINTS, 256))
    assert "_input_ab" not in cm.__dict__                               # the planes are rasterised when first read
    _check_getters(cm, (kind, "hints"))
    assert np.array_equal(cm.input_ab, ab) and np.array_equal(cm.input_mask, m)
    cm = _wrapper(kind, synth_sd, tmp_path)
    cm.net_forward(ab.astype(np.float32), m.astype(np.float32))         # float32 planes: scipy / numpy give float32
    _check_getters(cm, (kind, "float32"))


def test_input_render_of_an_18_megapixel_photo(synth_sd, tmp_path):
    """256^2 hints -> 3456 x 5184 (the size of the reference's bird_gray.jpg), the GUI's save_result call."""
    cm = CI.ColorizeImageB200(Xd=256)
    cm.prep_net(state_dict=synth_sd)
    _load(cm, tmp_path, 3456, 5184, seed=2)
    ab, m = np.zeros((2, 256, 256)), np.zeros((1, 256, 256))
    for (loc, p, val) in POINTS:
        CI.put_point(ab, m, loc, p, val)
    cm.net_forward(ab, m)
    got = cm.get_input_img_fullres()
    assert cm.img_l_fullres._host is None
    _close(got, CI.ColorizeImageBase.get_input_img_fullres(cm), "18 MP input render")


def test_fullres_render_of_a_24_megapixel_photo(synth_sd, tmp_path):
    """256^2 -> 4000 x 6000: the float64 ratio 255 / (n - 1) rounds up on both axes, so scipy's last row and last
    column read cval (ab = 0) and get_img_fullres shows them grey, like the reference."""
    cm = CI.ColorizeImageB200(Xd=256)
    cm.prep_net(state_dict=synth_sd)
    _load(cm, tmp_path, 4000, 6000, seed=3)
    ab, m = np.zeros((2, 256, 256)), np.zeros((1, 256, 256))
    for (loc, p, val) in POINTS:
        CI.put_point(ab, m, loc, p, val)
    cm.net_forward(ab, m)
    got = cm.get_img_fullres()
    gray = cm.get_img_gray_fullres()
    assert cm.img_l_fullres._host is None
    oy, ox = zoom_ref.overshoot(256, 4000), zoom_ref.overshoot(256, 6000)
    assert oy.sum() == 1 and oy[-1] and ox.sum() == 1 and ox[-1]
    assert np.array_equal(got[-1], gray[-1]) and np.array_equal(got[:, -1], gray[:, -1])
    assert np.any(got[:-1, :-1] != gray[:-1, :-1])                      # the hints do colour the inside
    util.assert_render_exact(got, CI.ColorizeImageBase.get_img_fullres(cm), _fullres_rgb255(cm), "24 MP fullres render")
