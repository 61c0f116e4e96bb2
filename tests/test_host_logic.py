"""CPU: host-side mirror of the reference wrapper (no GPU work)."""
import numpy as np

from interactive_deep_colorization_b200 import colorize_image as CI
from interactive_deep_colorization_b200.model import SIGGRAPHGeneratorB200
from oracle import color_ref, synth
from tests import util


def test_preconditions_return_minus_one(capsys):
    cm = CI.ColorizeImageB200(Xd=64)
    ab, m = np.zeros((2, 64, 64)), np.zeros((1, 64, 64))
    assert cm.net_forward(ab, m) == -1                  # reference :85-87
    assert "image" in capsys.readouterr().out
    cm.set_image(np.zeros((64, 64, 3), np.uint8))
    assert cm.net_forward(ab, m) == -1                  # reference :88-90
    assert "net" in capsys.readouterr().out


def test_image_prep_matches_reference_golden():
    g = util.golden("lhn_256.npz")
    cm = CI.ColorizeImageB200(Xd=256)
    cm.set_image(g["img_rgb"])
    assert np.max(np.abs(cm.img_l_mc - g["img_l_mc"])) < 1e-9
    assert cm.img_l.shape == (1, 256, 256) and cm.img_ab.shape == (2, 256, 256)
    assert cm.get_img_gray().shape == (256, 256, 3)
    # quantised output_ab path (reference :196-198)
    cm.output_rgb = g["mc0_kat_rgb"][None]            # the stored pixels as a 1 x K image (the conversion is per pixel)
    cm._set_out_ab_()
    assert np.max(np.abs(cm.output_ab[:, 0] - g["mc0_kat_output_ab"])) < 1e-4
    # full-res rendering: img_rgb_fullres == img_rgb here, so zoom factor is 1 (any full-size output will do)
    cm.output_rgb = g["img_rgb"]
    cm._set_out_ab_()
    assert np.array_equal(cm.get_img_fullres(), color_ref.lab2rgb_transpose(cm.img_l, cm.output_ab))


def test_put_point_and_hint_normalisation():
    ab, m = np.zeros((2, 256, 256)), np.zeros((1, 256, 256))
    CI.put_point(ab, m, [135, 160], 3, [23, -69])
    assert m.sum() == 49 and ab[0, 135, 160] == 23 and ab[1, 132, 163] == -69 and ab[0, 131, 160] == 0
    cm = CI.ColorizeImageB200(Xd=256, maskcent=True)
    assert cm.mask_cent == .5 and cm.mask_mult == 1. and cm.l_mean == 50.
    cm.img_l_set = cm.net_set = True
    assert CI.ColorizeImageBase.net_forward(cm, ab, m) == 0
    assert np.array_equal(cm.input_ab_mc, ab) and np.array_equal(cm.input_mask_mult, m)


def test_state_dict_keys_match_synthetic_reference_keys():
    sd = synth.synthetic_state_dict()
    net = SIGGRAPHGeneratorB200(dist=True)
    own = net.state_dict()
    assert set(own.keys()) == set(sd.keys())
    for k, v in sd.items():
        assert tuple(own[k].shape) == tuple(v.shape), k


def test_lazy_upsampled_dist():
    d64 = np.random.RandomState(0).rand(529, 4, 4).astype(np.float32)
    lazy = CI._LazyUpsampledDist(d64)
    full = np.repeat(np.repeat(d64, 4, 1), 4, 2)
    assert lazy.shape == (529, 16, 16)
    assert np.array_equal(lazy[:, 7, 9], full[:, 7, 9])
    assert np.array_equal(np.asarray(lazy), full)


def test_reccs_are_sorted_by_mass():
    cd = CI.ColorizeImageB200Dist(Xd=16)
    pmf = np.zeros(529, np.float32)
    pmf[[10, 300, 500]] = [0.6, 0.3, 0.1]
    cd.dist_ab = CI._LazyUpsampledDist(np.tile(pmf[:, None, None], (1, 4, 4)))
    cd.dist_ab_set = True
    np.random.seed(0)
    centers, conf = cd.get_ab_reccs(5, 5, K=3, N=5000, return_conf=True, method='sampled')
    assert np.allclose(centers[0], cd.pts_in_hull[10]) and np.allclose(centers[2], cd.pts_in_hull[500])
    assert conf[0] > conf[1] > conf[2] and abs(conf.sum() - 1) < 1e-9


def test_headless_cli_hint_parsing():
    import ideepcolor_b200 as cli
    a = cli.parse_args(["--color_model", "w.pth", "--suggest", "9", "--pytorch_maskcent"])
    assert a.load_size == 256 and a.suggest == 9 and a.pytorch_maskcent and a.gpu == 0
    assert cli.hint_ab({"ab": [23, -69]}) == [23.0, -69.0]
    white = cli.hint_ab({"rgb": [255, 255, 255]})
    assert abs(white[0]) < 0.01 and abs(white[1]) < 0.01
    red = cli.hint_ab({"rgb": [255, 0, 0]})
    assert abs(red[0] - 80.09) < 0.05 and abs(red[1] - 67.20) < 0.05      # sRGB red in CIELAB (D65)


def test_launcher_argument_surface_and_click_hook():
    """Row f4: the launcher keeps ideepcolor.py's argument names (:13-46) and re-enables the per-click predict_color()
    the reference commented out (ui/gui_draw.py:134,142) by wrapping update_ui -- checked on a stand-in class."""
    from interactive_deep_colorization_b200 import launcher
    a = launcher.parse_args(["--image_file", "x.jpg", "--dist_model", "w.pth", "--load_size", "128", "--win_size", "514"])
    assert a.backend == "b200" and a.color_model == "w.pth" and a.load_size == 128 and a.gpu == 0 and not a.pytorch_maskcent

    class FakeDraw(object):
        def __init__(self):
            self.calls, self.flag = 0, False

        def update_ui(self, move_point=True):
            return self.flag                      # is_predict: True on a new / erased point

        def predict_color(self):
            self.calls += 1
    launcher.enable_per_click_suggestions(FakeDraw)
    launcher.enable_per_click_suggestions(FakeDraw)          # idempotent
    d = FakeDraw()
    assert d.update_ui(move_point=False) is False and d.calls == 0
    d.flag = True
    assert d.update_ui() is True and d.calls == 1
    import pytest
    with pytest.raises(SystemExit):
        launcher.build_models(launcher.parse_args(["--backend", "nope"]))


class _FakeCtx(object):
    """Stands in for LhnContext in the wrapper-logic tests: 'forward' is a cheap deterministic function of the staged
    image and hints, so the tests can tell a re-used result from a recomputed one without a GPU."""

    def __init__(self, X):
        self.H = self.W = X
        self.device = 0
        self._wrapper_click, self._wrapper_staged_l, self._wrapper_last, self._wrapper_shared = None, [], None, False
        self.calls, self.image_uploads, self.L = 0, 0, None
        self._dist_resident = False

    def click_buffers(self, n=1, glob=False):
        X = self.H
        return {"L_mc": np.zeros((n, 1, X, X), np.float32), "ab": np.zeros((n, 2, X, X), np.float32),
                "mask": np.zeros((n, 1, X, X), np.float32), "glob": np.zeros((n, 316), np.float32) if glob else None,
                "out_ab": np.zeros((n, 2, X, X), np.float32), "out_rgb": np.zeros((n, X, X, 3), np.uint8),
                "out_abq": np.zeros((n, 2, X, X), np.float64)}

    def set_image(self, L):
        self.L = None if L is None else np.array(L)
        self.image_uploads += 1

    def set_dist_resident(self, on=True):
        self._dist_resident = bool(on)

    def set_click(self, *a):
        self.click = a

    def forward_host(self, L_mc, ab, mask, maskcent=0.0, glob=None, want_rgb=False, want_abq=False, out_ab=None,
                     out_rgb=None, out_abq=None, **kw):
        assert L_mc is None and self.L is not None        # the wrappers use the resident image
        self.calls += 1
        out_ab[...] = 0.25 * ab + 0.5 * mask + 0.01 * self.L + maskcent
        if out_rgb is not None:
            out_rgb[...] = (np.abs(out_ab[:, :1]).transpose(0, 2, 3, 1) * 50).astype(np.uint8)
        if out_abq is not None:
            out_abq[...] = np.round(out_ab)
        return {"ab": out_ab, "rgb": out_rgb, "abq": out_abq, "dist": None}

    def fetch_dist(self, img, y4, x4):
        return np.full(529, 1.0 / 529, np.float32)


class _FakeNet(object):
    dist, b200_device = True, 0

    def __init__(self, X):
        self.ctx = _FakeCtx(X)

    def _context(self, H, W, n):
        return self.ctx


def test_shared_trunk_bookkeeping_without_a_gpu():
    """ColorizeImageB200Dist.share_trunk: one forward per (image, hints) pair whichever model asks first; a changed
    image, changed hints or a different maskcent on one side always recompute; the image is uploaded once per photo."""
    X = 16
    rs = np.random.RandomState(0)
    cm = CI.ColorizeImageB200(Xd=X, maskcent=True, gpu_prepost=False)
    cd = CI.ColorizeImageB200Dist(Xd=X, maskcent=True)
    cd.gpu_prepost = False
    cm.net, cm.net_set = _FakeNet(X), True
    ctx = cm.net.ctx
    img = rs.randint(0, 256, (X, X, 3)).astype(np.uint8)
    cm.set_image(img); cd.set_image(img.copy())
    ab, m = np.zeros((2, X, X)), np.zeros((1, X, X))
    CI.put_point(ab, m, [5, 6], 1, [30, -20])
    cm.net_forward(ab, m)                                          # BEFORE sharing: this forward carried no distribution
    cd.share_trunk(cm)
    assert ctx._wrapper_shared and cd.net is cm.net and ctx._dist_resident
    cd.net_forward(ab, m)                                          # ... so the distribution model must not reuse it
    assert ctx.calls == 2
    ctx.calls = 0
    rgb = cm.net_forward(ab, m)                                    # same hints again: answered from the dist model's forward
    assert ctx.calls == 0 and ctx.image_uploads == 1
    CI.put_point(ab, m, [2, 12], 1, [-40, 15])
    rgb = cm.net_forward(ab, m)
    assert ctx.calls == 1 and ctx.image_uploads == 1
    ret = cd.net_forward(ab.copy(), m.copy())                      # same image (another array object), same hints
    assert ctx.calls == 1 and np.array_equal(ret, cm.output_ab_raw * 110.0) and cd.dist_ab_set
    CI.put_point(ab, m, [9, 3], 1, [-10, 44])
    ret2 = cd.net_forward(ab, m)                                   # new hints: the dist model pays ...
    assert ctx.calls == 2 and not np.array_equal(ret2, ret)
    rgb2 = cm.net_forward(ab.copy(), m.copy())                     # ... and the colour model rides along
    assert ctx.calls == 2 and ctx.image_uploads == 1 and not np.array_equal(rgb2, rgb)
    assert np.array_equal(cm.output_ab_raw * 110.0, ret2)
    cm.net_forward(ab, m)                                          # asking again recomputes nothing either
    assert ctx.calls == 2
    cd.set_image(img[::-1].copy())                                 # another photo on one side only
    ret3 = cd.net_forward(ab, m)
    assert ctx.calls == 3 and ctx.image_uploads == 2 and not np.array_equal(ret3, ret2)
    cm.net_forward(ab, m)                                          # the colour model still holds the first photo
    assert ctx.calls == 4 and ctx.image_uploads == 3
    cd.mask_cent = 0.0                                             # different centring -> different network input
    cd.set_image(img.copy())
    cd.net_forward(ab, m)
    assert ctx.calls == 5
    cd.hint_click(8, 4, K=9)
    assert ctx.click == (0, 2, 1, 9)
