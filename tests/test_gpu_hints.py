"""GPU: hint lists rasterised on the device (idc_set_hints) and the gamut map kernel (idc_gamut_ab).

A hint-mode forward must be bit-identical to the dense forward of the planes oracle/hints_ref.py rasterises from the
same list, on every path: the click graph (n <= 4, pinned and pageable buffers), the chunked large-batch path, the
resident image, the announced click, global hints, FAST_FP16 and the SIMT engine.  Editing the list never re-captures
the click graph."""
import numpy as np
import pytest

from interactive_deep_colorization_b200 import _lib
from interactive_deep_colorization_b200 import colorize_image as CI
from interactive_deep_colorization_b200 import prepost
from oracle import caffe_spec, gamut_ref, hints_ref, synth
from tests import util
from tests.test_hints_cpu import FakeUIControl, _golden_gamut, _ulps32, dense_gui_planes, fake_edits

pytestmark = pytest.mark.gpu


def _glob_sd():
    import torch
    sd = dict(synth.torch_state_dict(1234))
    sd.update({k: torch.from_numpy(v) for k, v in caffe_spec.synthetic_glob_state_dict().items()})
    return sd


def _rects(rs, n_hints, n_img, X):
    out = np.zeros(n_hints, _lib.HINT_DTYPE)
    for i in range(n_hints):
        y0, x0 = rs.randint(-4, X + 2, 2)
        h, w = rs.randint(-1, 9, 2)
        out[i] = (rs.randint(n_img), y0, x0, y0 + h, x0 + w, rs.uniform(-100, 100), rs.uniform(-100, 100))
    return out


def _dense(rects, n, X):
    ab, m = hints_ref.raster(rects, n, X, X)
    return np.ascontiguousarray(ab), np.ascontiguousarray(m)


def _check(ref, got, keys):
    for k in keys:
        assert np.array_equal(ref[k], got[k]), k


@pytest.mark.parametrize("n", [1, 2, 4, 8, 16])
def test_hint_mode_equals_dense(synth_sd, n):
    X = 64
    L, _, _ = synth.synthetic_batch(n, X, seed=20 + n, max_hints=0)
    ctx = util.make_ctx(synth_sd, X, X, max_n=n, dist=True)
    rs = np.random.RandomState(n)
    kw = dict(want_dist=True, want_rgb=True, want_abq=True)
    for trial in range(3):
        rects = _rects(rs, rs.randint(0, 40), n, X)
        ab, m = _dense(rects, n, X)
        ref = ctx.forward_host(L, ab, m, 0.5, **kw)
        ctx.set_hints(rects)
        got = ctx.forward_host(L, None, None, 0.5, n=n, **kw)
        _check(ref, got, ("ab", "dist", "rgb", "abq"))
        ctx.set_image(L)                                         # resident L + hints: only the hint block travels
        got = ctx.forward_host(None, None, None, 0.5, n=n, **kw)
        _check(ref, got, ("ab", "dist", "rgb", "abq"))
    ctx.close()


def test_click_graph_pinned_buffers_never_recapture(synth_sd):
    """20 sequential clicks (add, move, erase) through the pinned hint-mode click buffers, with the announced click:
    one graph instantiation, every click equal to the dense forward."""
    X = 128
    L, _, _ = synth.synthetic_batch(1, X, seed=3, max_hints=0)
    ctx = util.make_ctx(synth_sd, X, X, max_n=1, dist=True)
    plain = util.make_ctx(synth_sd, X, X, max_n=1, dist=True)
    ctx.set_dist_resident(True)
    plain.set_dist_resident(True)
    buf = ctx.click_buffers(1, hints=True)
    assert buf["ab"] is None and buf["mask"] is None
    buf["L_mc"][...] = L
    ctx.set_image(buf["L_mc"])
    rs = np.random.RandomState(4)
    pts = []
    captures = None
    for step in range(20):
        op = step % 4
        if op in (0, 1) or not pts:
            pts.append((rs.randint(0, X, 2), int(rs.randint(1, 5)), rs.uniform(-90, 90, 2)))   # add
        elif op == 2:
            i = rs.randint(len(pts))
            pts[i] = (rs.randint(0, X, 2), pts[i][1], pts[i][2])                                # move
        else:
            pts.pop(rs.randint(len(pts)))                                                       # erase
        loc = pts[-1][0] if pts else (0, 0)
        ctx.set_click(0, int(loc[0]) // 4, int(loc[1]) // 4, 5)
        plain.set_click(0, int(loc[0]) // 4, int(loc[1]) // 4, 5)
        rects = CI.hints_from_points(pts, X)
        ctx.set_hints(rects)
        r = ctx.forward_host(None, None, None, 0.5, n=1, want_rgb=True, want_abq=True, out_ab=buf["out_ab"],
                             out_rgb=buf["out_rgb"], out_abq=buf["out_abq"])
        ab, m = _dense(rects, 1, X)
        p = plain.forward_host(L, ab, m, 0.5, want_rgb=True, want_abq=True)
        _check(p, r, ("ab", "rgb", "abq"))
        y4, x4 = int(loc[0]) // 4, int(loc[1]) // 4
        assert np.array_equal(ctx.fetch_dist(0, y4, x4), plain.fetch_dist(0, y4, x4))
        c1, f1, _ = ctx.ab_reccs(0, y4, x4, K=5)
        c2, f2, _ = plain.ab_reccs(0, y4, x4, K=5)
        assert np.array_equal(c1, c2) and np.array_equal(f1, f2)
        if captures is None:
            captures = ctx.graph_captures()
        assert ctx.graph_captures() == captures, step
    assert captures == 1
    ctx.close()
    plain.close()


@pytest.mark.parametrize("kw", [dict(fast_fp16=True), dict(engine="simt"), dict(global_hints=True),
                                dict(use_graph=False), dict(options={"tanh_scale": 100})])
def test_hint_mode_equals_dense_engine_variants(kw):
    X = 64
    sd = _glob_sd() if kw.get("global_hints") else synth.torch_state_dict(1234)
    L, _, _ = synth.synthetic_batch(2, X, seed=8, max_hints=0)
    ctx = util.make_ctx(sd, X, X, max_n=2, **kw)
    glob = np.ascontiguousarray(np.random.RandomState(1).rand(2, 316).astype(np.float32)) if kw.get("global_hints") else None
    rects = _rects(np.random.RandomState(9), 25, 2, X)
    ab, m = _dense(rects, 2, X)
    ref = ctx.forward_host(L, ab, m, 0.0, glob=glob, want_rgb=True)
    ctx.set_hints(rects)
    got = ctx.forward_host(L, None, None, 0.0, glob=glob, want_rgb=True, n=2)
    _check(ref, got, ("ab", "rgb"))
    ctx.close()


def test_zero_hints_equal_zero_planes_and_errors(synth_sd):
    X = 64
    L, _, _ = synth.synthetic_batch(2, X, seed=2, max_hints=0)
    ctx = util.make_ctx(synth_sd, X, X, max_n=2)
    z_ab, z_m = np.zeros((2, 2, X, X), np.float32), np.zeros((2, 1, X, X), np.float32)
    with pytest.raises(_lib.IdcError) as e:                      # never set: a state error, not a zero-hint forward
        ctx.forward_host(L, None, None, n=2)
    assert e.value.code == -3
    ctx.set_hints([])
    _check(ctx.forward_host(L, z_ab, z_m), ctx.forward_host(L, None, None, n=2), ("ab",))
    for bad in (dict(ab=z_ab, mask=None), dict(ab=None, mask=z_m)):
        with pytest.raises(_lib.IdcError) as e:
            ctx.forward_host(L, bad["ab"], bad["mask"], n=2)
        assert e.value.code == -1
    ctx.set_hints([(1, 0, 0, 3, 3, 1.0, 2.0)])
    with pytest.raises(_lib.IdcError) as e:                      # img 1 of a 1-image forward
        ctx.forward_host(np.ascontiguousarray(L[:1]), None, None, n=1)
    assert e.value.code == -1
    ctx.set_hints([(-1, 0, 0, 3, 3, 1.0, 2.0)])
    with pytest.raises(_lib.IdcError):
        ctx.forward_host(L, None, None, n=2)
    lib = _lib.load()
    one = np.zeros(1, _lib.HINT_DTYPE)
    assert lib.idc_set_hints(ctx.h, -1, one.ctypes.data) == -1
    assert lib.idc_set_hints(ctx.h, _lib.MAX_HINTS + 1, one.ctypes.data) == -1
    assert lib.idc_set_hints(ctx.h, 1, None) == -1
    ctx.set_hints(np.zeros(_lib.MAX_HINTS, _lib.HINT_DTYPE))    # the maximum is accepted
    ctx.forward_host(L, None, None, n=2)
    ctx.close()


def _wrapper_pairs(sd, X):
    caffe_sd = dict(sd)
    glob_sd = _glob_sd()
    out = []
    for make in (lambda: CI.ColorizeImageB200(Xd=X, maskcent=True),
                 lambda: CI.ColorizeImageB200GlobDist(Xd=X),
                 lambda: CI.ColorizeImageB200Caffe(Xd=X)):
        a, b = make(), make()
        for m in (a, b):
            if isinstance(m, CI.ColorizeImageB200Caffe):
                m.prep_net(0, state_dict=caffe_sd)
            elif isinstance(m, CI.ColorizeImageB200GlobDist):
                m.prep_net(0, state_dict=glob_sd)
            else:
                m.prep_net(0, state_dict=sd)
        out.append((a, b))
    return out


def test_wrappers_hint_list_equals_dense(synth_sd):
    X = 64
    img = (np.random.RandomState(0).rand(X, X, 3) * 255).astype(np.uint8)
    pts = [((10, 12), 2, (20.5, -30.25)), ((40, 50), 3, (-60.0, 45.0)), ((-2, 30), 2, (5.0, 5.0)), ((33, 20), 1, (0.0, 0.0))]
    rects = CI.hints_from_points(pts, X)
    ab, mask = np.zeros((2, X, X)), np.zeros((1, X, X))
    for loc, p, val in pts:
        CI.put_point(ab, mask, loc, p, val)
    for dense, hinted in _wrapper_pairs(synth_sd, X):
        for m in (dense, hinted):
            m.set_image(img)
        r1 = dense.net_forward(ab, mask)
        r2 = hinted.net_forward_hints(rects)
        assert np.array_equal(r1, r2), type(dense).__name__
        assert np.array_equal(dense.output_ab, hinted.output_ab)
        for k in ("input_ab", "input_mask", "input_ab_mc", "input_mask_mult"):
            assert np.array_equal(np.asarray(getattr(dense, k)), getattr(hinted, k)), k
        assert np.array_equal(dense.get_input_img(), hinted.get_input_img())
        if isinstance(dense, CI.ColorizeImageB200GlobDist):
            gd = np.random.RandomState(3).rand(313)
            assert np.array_equal(dense.net_forward(ab, mask, gd), hinted.net_forward_hints(rects, gd))


def test_caffe_dist_hint_list_equals_dense():
    X = 64
    import torch
    sd = dict(synth.torch_state_dict(1234))
    csd = caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=prepost.pts_in_hull())
    sd.update({k: torch.from_numpy(v) for k, v in csd.items() if k != "caffe.pts_in_hull"})
    img = (np.random.RandomState(5).rand(X, X, 3) * 255).astype(np.uint8)
    pts = [((10, 12), 2, (20.5, -30.25)), ((40, 50), 3, (-60.0, 45.0))]
    a, b = CI.ColorizeImageB200CaffeDist(Xd=X), CI.ColorizeImageB200CaffeDist(Xd=X)
    for m in (a, b):
        m.prep_net(0, state_dict=sd)
        m.set_image(img)
    ab, mask = np.zeros((2, X, X)), np.zeros((1, X, X))
    for loc, p, val in pts:
        CI.put_point(ab, mask, loc, p, val)
    assert np.array_equal(a.net_forward(ab, mask), b.net_forward_hints(CI.hints_from_points(pts, X)))


def test_share_trunk_compares_hint_lists(synth_sd):
    X = 64
    img = (np.random.RandomState(1).rand(X, X, 3) * 255).astype(np.uint8)
    cm = CI.ColorizeImageB200(Xd=X)
    cm.prep_net(0, state_dict=synth_sd, dist=True)
    cm.set_image(img)
    dm = CI.ColorizeImageB200Dist(Xd=X).share_trunk(cm)
    dm.set_image(img)
    ref = CI.ColorizeImageB200Dist(Xd=X)
    ref.prep_net(0, state_dict=synth_sd)
    ref.set_image(img)
    pts = [((10, 12), 2, (20.5, -30.25)), ((40, 50), 3, (-60.0, 45.0))]
    ctx = cm.net._context(X, X, 1)
    for k in range(3):
        rects = CI.hints_from_points(pts[:k + 1] if k < 2 else pts[:1], X)
        cm.net_forward_hints(rects)
        captures = ctx.graph_captures()
        got = dm.net_forward_hints(rects)                          # answered from the colour model's forward
        want = ref.net_forward_hints(rects)
        assert np.array_equal(got, want)
        assert np.array_equal(np.asarray(dm.dist_ab[:, 20, 24]), np.asarray(ref.dist_ab[:, 20, 24]))
        assert ctx.graph_captures() == captures
    # a different list is not shared: it runs its own forward
    other = CI.hints_from_points([((30, 30), 2, (1.0, 2.0))], X)
    assert np.array_equal(dm.net_forward_hints(other), ref.net_forward_hints(other))


class FakeGUIDraw(object):
    """Qt-free stand-in for ui/gui_draw.py GUIDraw: the attributes compute_result / predict_color touch."""

    def __init__(self, model, dist_model, ui, l_win):
        self.model, self.dist_model, self.uiControl, self.l_win = model, dist_model, ui, l_win
        self.image_loaded = True
        self.win_w = self.win_h = l_win.shape[0]

    def update(self):
        pass


def test_fake_gui_compute_result_hook_matches_dense(synth_sd):
    from interactive_deep_colorization_b200 import launcher
    X = 256
    img = (np.random.RandomState(2).rand(X, X, 3) * 255).astype(np.uint8)
    cls = type("GUIDrawHinted", (FakeGUIDraw,), {})
    launcher.use_device_hints(cls)
    dense_model = CI.ColorizeImageB200(Xd=X)
    hint_model = CI.ColorizeImageB200(Xd=X)
    for m in (dense_model, hint_model):
        m.prep_net(0, state_dict=synth_sd)
        m.set_image(img)
    ui = FakeUIControl(fake_edits(np.random.RandomState(7), 15))
    gui = cls(hint_model, None, ui, np.full((X, X), 50.0))
    gui.compute_result()
    ab_d, mask_d = dense_gui_planes(ui)
    dense_model.net_forward(ab_d, mask_d)
    assert np.all(_ulps32(gui.im_ab0, ab_d) <= 1) and np.array_equal(gui.im_mask0, mask_d)
    assert np.max(np.abs(hint_model.output_ab_raw - dense_model.output_ab_raw)) <= 1e-3
    assert gui.result.shape == (X, X, 3)


def test_gamut_kernel_matches_oracle_and_golden():
    for L in np.arange(0.0, 100.0001, 0.5):
        rgb, mask = prepost.gamut_gpu(float(L))
        orgb, omask, r255, nrm = gamut_ref.update_gamut(float(L), details=True)
        diff = np.any(rgb != orgb, axis=2) | (mask != omask)
        assert not np.any(diff & ~gamut_ref.edge_cells(r255, nrm)), L
    g, gmask = _golden_gamut()
    for i, L in enumerate(g["L"]):
        rgb, mask = prepost.gamut_gpu(float(L), int(g["gamut_size"]), int(g["D"]))
        orgb, omask, r255, nrm = gamut_ref.update_gamut(float(L), details=True)
        diff = np.any(rgb != g["masked_rgb"][i], axis=2) | (mask != gmask[i])
        assert not np.any(diff & ~gamut_ref.edge_cells(r255, nrm)), L
    for D in (2, 3):
        rgb, mask = prepost.gamut_gpu(50.0, 110, D)
        orgb, omask, r255, nrm = gamut_ref.update_gamut(50.0, 110, D, details=True)
        assert rgb.shape == orgb.shape
        diff = np.any(rgb != orgb, axis=2) | (mask != omask)
        assert not np.any(diff & ~gamut_ref.edge_cells(r255, nrm))
