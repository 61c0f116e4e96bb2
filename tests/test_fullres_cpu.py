"""CPU: the full-resolution renders without a device -- the zoom rule render_planes_kernel restates (tests/zoom_ref.py)
against the installed scipy, the routing of the four getters (device under gpu_prepost with a net set and float planes,
ColorizeImageBase's statements otherwise) with a stubbed prepost.render_planes_gpu, and the argument checks of
idc_render_planes_u8."""
import ctypes
import types

import numpy as np
import pytest
from scipy.ndimage import zoom

from interactive_deep_colorization_b200 import _lib, prepost
from interactive_deep_colorization_b200 import colorize_image as CI
from tests import zoom_ref
from tests.test_host_logic import _FakeNet

N_IN = (8, 32, 64, 128, 176, 256, 512)
N_OUT = tuple(range(1, 700)) + (1080, 1920, 3456, 4000, 5184, 6000, 10000)
GETTERS = ("get_img_gray_fullres", "get_input_img_fullres", "get_img_mask_fullres", "get_sup_fullres")


def test_order0_index_ramp_equals_scipy():
    for n_in in N_IN:
        ramp = np.arange(1, n_in + 1, dtype=np.float64)        # 0 in the output can only be cval
        for n_out in N_OUT:
            got = zoom(ramp, n_out / n_in, order=0)
            assert got.shape == (n_out,), (n_in, n_out)
            assert np.array_equal(zoom_ref.zoom_1d(ramp, n_out, 0), got), (n_in, n_out)
            assert np.array_equal(got == 0, zoom_ref.overshoot(n_in, n_out)), (n_in, n_out)


def test_order1_equals_scipy():
    rs = np.random.RandomState(0)
    for n_in in N_IN:
        v = rs.uniform(-80, 80, n_in)
        for n_out in N_OUT:
            got = zoom(v, n_out / n_in, order=1)
            d = np.abs(zoom_ref.zoom_1d(v, n_out, 1) - got).max()
            assert d <= 1e-12 * np.abs(v).max(), (n_in, n_out, d)
            over = zoom_ref.overshoot(n_in, n_out)
            assert np.all(got[over] == 0.0) and np.all(got[~over] != 0.0), (n_in, n_out)


def test_plane_zoom_equals_scipy():
    """The 2-D restatement against scipy's zoom of a [2, h_in, w_in] plane pair, as _to_fullres calls it."""
    rs = np.random.RandomState(1)
    for n_in in (8, 64, 256):
        v = rs.uniform(-80, 80, (2, n_in, n_in))
        for (h, w) in ((507, 600), (12, 14), (23, 27), (45, 53), (75, 91), (1, 300), (300, 1), (100, 80), (n_in, n_in)):
            for order in (0, 1):
                got = zoom(v, (1, h / n_in, w / n_in), order=order)
                assert got.shape == (2, h, w)
                for c in range(2):
                    d = np.abs(zoom_ref.zoom_plane(v[c], h, w, order) - got[c]).max()
                    assert d <= 1e-12 * 80, (n_in, h, w, order, d)


def test_overshoot_sizes():
    """At n_in = 256 the float64 ratio rounds up for 1218 of the output sizes 2 ... 10000; the render sizes of the
    photos in the tests and tools are not among them."""
    assert sum(bool(zoom_ref.overshoot(256, n)[-1]) for n in range(2, 10001)) == 1218
    for n in (12, 14, 23, 27, 32, 45, 53):
        assert zoom_ref.overshoot(256, n)[-1] and zoom_ref.overshoot(256, n).sum() == 1
    for n in (256, 507, 600, 3456, 5184):
        assert not zoom_ref.overshoot(256, n).any()


def test_output_shapes_equal_scipy():
    full_sizes = (1, 13, 75, 91, 507, 600, 1080, 3456, 5184, 10000)
    for n_in in (1, 8, 64, 256):
        for like in (n_in, 64, 100, 256):
            for full in full_sizes:
                n = zoom_ref.out_len(n_in, full, like)
                assert zoom(np.zeros(n_in), 1. * full / like, order=0).shape == (n,), (n_in, like, full)
    cm = CI.ColorizeImageB200(Xd=16, gpu_prepost=False)
    cm.img_l_fullres = np.zeros((1, 3456, 5184))
    for hw_in, hw_like in (((256, 256), (256, 256)), ((256, 256), (100, 64)), ((64, 91), (256, 200))):
        plane, like = types.SimpleNamespace(shape=(1,) + hw_in), types.SimpleNamespace(shape=(2,) + hw_like)
        assert cm._fullres_hw(plane, like) == (zoom_ref.out_len(hw_in[0], 3456, hw_like[0]),
                                               zoom_ref.out_len(hw_in[1], 5184, hw_like[1]))


# ----- routing of the four getters -----
class _Stub(object):
    def __init__(self):
        self.calls = []

    def __call__(self, h, w, **kw):
        self.calls.append((h, w, kw))
        return np.full((h, w, 3), 7, np.uint8)


def _wrapper(cls, X=16, full=(75, 91), dtype=np.float64, seed=0):
    """A wrapper object whose image was prepared on the host (gpu_prepost off, no net), with a net stand-in and hint
    planes of `dtype` set afterwards, as a forward would leave them."""
    rs = np.random.RandomState(seed)
    cm = cls(Xd=X)
    cm.gpu_prepost = False
    cm._ingest(rs.randint(0, 256, full + (3,)).astype(np.uint8), rs.randint(0, 256, (X, X, 3)).astype(np.uint8))
    if cls is CI.ColorizeImageB200:
        cm.net = _FakeNet(X)
    else:
        cm._ctx = types.SimpleNamespace(device=0)
    cm.net_set = True
    ab, mask = np.zeros((2, X, X)), np.zeros((1, X, X))
    CI.put_point(ab, mask, [5, 6], 2, [23, -69])
    CI.put_point(ab, mask, [12, 2], 1, [-40, 15.5])
    cm.input_ab, cm.input_mask = ab.astype(dtype), mask.astype(dtype)
    cm.output_ab = rs.uniform(-60, 60, (2, X, X))
    return cm


def _same_outcome(fn_a, fn_b):
    """Both calls return equal arrays, or both raise the same exception."""
    try:
        a = fn_a()
    except Exception as e:
        with pytest.raises(type(e)) as eb:
            fn_b()
        assert str(eb.value) == str(e)
        return
    b = fn_b()
    assert a.dtype == b.dtype and np.array_equal(a, b)


CLASSES = [CI.ColorizeImageB200, CI.ColorizeImageB200Caffe, CI.ColorizeImageB200GlobDist]


@pytest.mark.parametrize("cls", CLASSES, ids=lambda c: c.__name__)
def test_getters_take_the_base_statements_without_the_gate(cls, monkeypatch):
    stub = _Stub()
    monkeypatch.setattr(prepost, "render_planes_gpu", stub)
    for gpu_prepost, net_set in ((False, True), (True, False), (False, False)):
        cm = _wrapper(cls)
        cm.gpu_prepost, cm.net_set = gpu_prepost, net_set
        for g in GETTERS:
            got, want = getattr(cm, g)(), getattr(CI.ColorizeImageBase, g)(cm)
            assert got.dtype == np.uint8 and np.array_equal(got, want), (gpu_prepost, net_set, g)
    assert stub.calls == []


@pytest.mark.parametrize("cls", CLASSES, ids=lambda c: c.__name__)
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_getters_route_float_planes_to_the_device(cls, dtype, monkeypatch):
    stub = _Stub()
    monkeypatch.setattr(prepost, "render_planes_gpu", stub)
    cm = _wrapper(cls, dtype=dtype)
    cm.gpu_prepost = True
    for g in GETTERS:
        assert np.array_equal(getattr(cm, g)(), np.full((75, 91, 3), 7, np.uint8)), g
    (gray, inp, mask, sup) = stub.calls
    assert gray[:2] == (75, 91) and gray[2]["L"] is cm.img_l_fullres and "ab" not in gray[2] and "mask" not in gray[2]
    assert inp[:2] == (75, 91) and inp[2]["ab"] is cm.input_ab and inp[2]["ab_order"] == 1
    assert inp[2]["L"] is cm.img_l_fullres
    assert mask[:2] == (75, 91) and mask[2]["mask"] is cm.input_mask and mask[2]["l_mode"] == _lib.RENDER_L_MASK
    assert "ab" not in mask[2] and "L" not in mask[2]
    assert sup[:2] == (75, 91) and sup[2]["mask"] is cm.input_mask and sup[2]["ab"] is cm.input_ab
    assert sup[2]["ab_order"] == 0 and sup[2]["l_mode"] == _lib.RENDER_L_SUP and "L" not in sup[2]
    assert all(c[2]["device"] == 0 for c in stub.calls)


@pytest.mark.parametrize("ab_dtype,mask_dtype", [(np.int64, np.float64), (np.float64, bool), (np.float64, np.uint8),
                                                 (np.float16, np.float16), (np.float64, np.int32)])
def test_non_float_planes_take_the_host_path(ab_dtype, mask_dtype, monkeypatch):
    stub = _Stub()
    monkeypatch.setattr(prepost, "render_planes_gpu", stub)
    cm = _wrapper(CI.ColorizeImageB200)
    cm.gpu_prepost = True
    cm.input_ab, cm.input_mask = cm.input_ab.astype(ab_dtype), cm.input_mask.astype(mask_dtype)
    ab_float = np.dtype(ab_dtype) in (np.float32, np.float64)
    mask_float = np.dtype(mask_dtype) in (np.float32, np.float64)
    # only a getter whose planes (and the plane its zoom factor comes from) are all float32 / float64 reaches the device
    device = {"get_input_img_fullres": ab_float, "get_img_mask_fullres": ab_float and mask_float,
              "get_sup_fullres": ab_float and mask_float}
    for g in GETTERS[1:]:
        n = len(stub.calls)
        if device[g]:
            assert np.array_equal(getattr(cm, g)(), np.full((75, 91, 3), 7, np.uint8)) and len(stub.calls) == n + 1, g
        else:
            _same_outcome(lambda: getattr(CI.ColorizeImageBase, g)(cm), getattr(cm, g))
            assert len(stub.calls) == n, g


def test_bool_mask_raises_where_the_host_statement_raises(monkeypatch):
    """The GUI hands net_forward a bool mask (`mask > 0`); the mask render keeps the host statement's outcome."""
    stub = _Stub()
    monkeypatch.setattr(prepost, "render_planes_gpu", stub)
    cm = _wrapper(CI.ColorizeImageB200)
    cm.gpu_prepost = True
    cm.input_mask = cm.input_mask > 0
    _same_outcome(lambda: CI.ColorizeImageBase.get_img_mask_fullres(cm), cm.get_img_mask_fullres)
    _same_outcome(lambda: CI.ColorizeImageBase.get_sup_fullres(cm), cm.get_sup_fullres)
    assert stub.calls == []


def test_device_renders_have_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    cm = _wrapper(CI.ColorizeImageB200)
    cm.gpu_prepost = True
    for g in GETTERS:
        with pytest.raises(_lib.IdcError):
            getattr(cm, g)()


def test_render_planes_argument_validation_without_gpu():
    """Every rejected call returns IDC_ERR_ARG before touching a device (the pointers are never dereferenced)."""
    lib = _lib.load()
    buf = np.zeros(64)
    p = ctypes.c_void_p(buf.ctypes.data)
    PLANE, MASK, SUP = _lib.RENDER_L_PLANE, _lib.RENDER_L_MASK, _lib.RENDER_L_SUP
    ok = dict(device=0, h_in=4, w_in=4, ab=p, ab_order=1, ab_f32=0, mask=p, mask_f32=0, l_mode=PLANE, L=p, h=8, w=8,
              rgb=p, stream=None)
    bad = [dict(ab_order=2), dict(ab_order=-1), dict(ab_f32=2), dict(mask_f32=-1), dict(l_mode=3), dict(l_mode=-1),
           dict(l_mode=PLANE, L=None), dict(l_mode=MASK, mask=None), dict(l_mode=SUP, mask=None),
           dict(h=0), dict(w=-3), dict(h_in=0), dict(w_in=0), dict(rgb=None), dict(h=1 << 30, w=1 << 30)]
    for b in bad:
        a = dict(ok, **b)
        assert lib.idc_render_planes_u8(*a.values()) == -1, b


@pytest.mark.parametrize("cls", CLASSES, ids=lambda c: c.__name__)
def test_get_img_fullres_is_the_input_render_of_the_output_ab(cls, monkeypatch):
    """Under the gate get_img_fullres renders through render_planes_gpu (scipy's zoom rule, cval rows included): the
    output ab with order 1 and the full-resolution L, which is handed over as is (a DeviceLab stays on the device)."""
    stub = _Stub()
    monkeypatch.setattr(prepost, "render_planes_gpu", stub)
    cm = _wrapper(cls)
    cm.gpu_prepost = True
    assert np.array_equal(cm.get_img_fullres(), np.full((75, 91, 3), 7, np.uint8))
    ((h, w, kw),) = stub.calls
    assert (h, w) == (75, 91) and kw["ab"] is cm.output_ab and kw["ab_order"] == 1 and kw["L"] is cm.img_l_fullres
    assert "mask" not in kw and kw.get("l_mode", _lib.RENDER_L_PLANE) == _lib.RENDER_L_PLANE and kw["device"] == 0


def test_zoom_lab2rgb_argument_validation_without_gpu():
    """idc_zoom_lab2rgb_u8 (get_img_fullres in the C ABI) rejects what idc_render_planes_u8 rejects, and a NULL ab,
    before touching a device."""
    lib = _lib.load()
    buf = np.zeros(64)
    p = ctypes.c_void_p(buf.ctypes.data)
    ok = dict(device=0, h_in=4, w_in=4, ab=p, h=8, w=8, L=p, rgb=p, stream=None)
    for b in (dict(ab=None), dict(L=None), dict(rgb=None), dict(h=0), dict(w=-1), dict(h_in=0), dict(w_in=0),
              dict(h=1 << 30, w=1 << 30)):
        assert lib.idc_zoom_lab2rgb_u8(*dict(ok, **b).values()) == -1, b
