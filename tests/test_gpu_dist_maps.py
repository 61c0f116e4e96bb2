"""GPU: whole-map reads of the two distribution models -- the 313-bin dist_ab_S map (dist313_map_kernel), the entropy
sum (negentropy_kernel) on both models, and the wrapper surface built on them: dist_ab as an array, dist_ab_full,
dist_ab_grid, compute_entropy, plot_dist_grid and plot_dist_entropy (reference data/colorize_image.py:297-372,
:487-561)."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import _lib, prepost
from interactive_deep_colorization_b200 import colorize_image as CI
from oracle import caffe_spec, synth
from tests import util

pytestmark = pytest.mark.gpu
X = 64
TOL_ENT = 5e-5       # both sides sum the bins in the same order; only logf and numpy's log differ
# pixels of image 1 compared bit for bit with the single-pixel lookup: the four corners, the last row and column (where
# the x4 upsample reads the zero padding beyond the last cell) and cells inside
PIX = [(0, 0), (0, 63), (63, 0), (63, 63), (63, 17), (40, 63), (62, 62), (61, 63), (13, 62), (31, 7), (1, 2), (4, 4),
       (35, 36), (50, 3), (22, 59), (60, 30), (3, 0), (0, 3)]


def _np_negentropy(d):
    """The reference statement (data/colorize_image.py:358, :547)."""
    d = np.asarray(d)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.sum(d * np.log(d), axis=0)


def _entropy_err(got, want):
    """NaN at the same pixels (a bin that underflowed to exactly 0: 0 * log 0), then max-abs over the others."""
    assert np.array_equal(np.isnan(got), np.isnan(want)), (np.isnan(got).sum(), np.isnan(want).sum())
    ok = ~np.isnan(want)
    return util.maxabs(got[ok], want[ok]), int((~ok).sum())


def _caffe_sd(synth_sd):
    pts = np.load(os.path.join(util.GOLDEN, "pts_in_hull.npy"))
    csd = caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=pts)
    sd = dict(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in csd.items()})
    return sd, csd


@pytest.fixture(scope="module")
def caffe_case(synth_sd):
    """As test_caffe313_head: 2 images at 64^2, maskcent 0.5, the FP32 spec oracle's dist_ab_S."""
    sd, csd = _caffe_sd(synth_sd)
    L, ab, m = util.small_batch(2, X, seed=500)
    _, inter = util.oracle_forward(synth_sd, L, ab, m, 0.5, intermediates=True)
    with torch.no_grad():
        _, dist_ref = caffe_spec.caffe313_head(csd, inter)
    return sd, (L, ab, m), dist_ref.numpy()


@pytest.mark.parametrize("engine", ["simt", "wgmma"])
def test_dist313_map(caffe_case, engine):
    sd, (L, ab, m), ref = caffe_case
    ctx = util.make_ctx(sd, X, X, max_n=2, engine=engine, caffe313=True)
    try:
        ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5)
        d = ctx.caffe313_dist_map(2).cpu().numpy()
        assert d.shape == (2, 313, X, X) and d.dtype == np.float32
        for (y, x) in PIX:
            px = ctx.caffe313_dist_pixel(1, y, x)
            assert np.array_equal(d[1, :, y, x].view(np.uint32), px.view(np.uint32)), (engine, y, x)
        err = util.maxabs(d, ref)
        s = np.abs(d.sum(1, dtype=np.float64) - 1.0).max()
        print("dist313 map %s: max|d - FP32 oracle| = %.3e over every pixel, max|sum - 1| = %.3e" % (engine, err, s))
        assert err < 1e-5 and s < 1e-5
        assert util.maxabs(ctx.caffe313_dist_map(2, S=0.5).cpu().numpy(), d) > 1e-3
        assert np.array_equal(ctx.caffe313_dist_map(1).cpu().numpy()[0], d[0])
        lib = _lib.load()
        out = torch.empty((3, 313, X, X), dtype=torch.float32, device="cuda")
        for n in (0, 3, -1):
            assert lib.idc_caffe313_dist_map(ctx.h, n, 0.2, out.data_ptr(), None) == -1, n
        assert lib.idc_caffe313_dist_map(ctx.h, 1, 0.2, None, None) == -1
    finally:
        ctx.close()


def test_dist313_map_needs_the_caffe_head(synth_sd):
    ctx = util.make_ctx(synth_sd, X, X, max_n=1)
    try:
        with pytest.raises(_lib.IdcError) as e:
            ctx.caffe313_dist_map(1)
        assert e.value.code == -3 and b"CAFFE313" in ctx.lib.idc_last_error(ctx.h)
    finally:
        ctx.close()


def test_negentropy_kernel(caffe_case):
    sd, (L, ab, m), _ = caffe_case
    ctx = util.make_ctx(sd, X, X, max_n=2, caffe313=True)
    try:
        ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5)
        dmap = ctx.caffe313_dist_map(2)
        neg = prepost.negentropy_gpu(dmap).cpu().numpy()
        d = dmap.cpu().numpy()
    finally:
        ctx.close()
    assert neg.shape == (2, X, X) and neg.dtype == np.float32
    for i in range(2):
        err, nans = _entropy_err(neg[i], _np_negentropy(d[i]))
        print("negentropy image %d: max|kernel - numpy| = %.3e (%d NaN pixels)" % (i, err, nans))
        assert err <= TOL_ENT
    # an exact zero bin: 0 * log(0) = 0 * -inf = NaN at that pixel, in numpy and in the kernel
    h = np.random.RandomState(0).dirichlet(np.ones(7), size=10).T.astype(np.float32)      # [7 bins, 10 pixels]
    h[3, 4] = 0.0
    got = prepost.negentropy_gpu(torch.from_numpy(h[None]).cuda()).cpu().numpy()[0]
    want = _np_negentropy(h)
    err, nans = _entropy_err(got, want)
    assert np.isnan(want[4]) and nans == 1 and err <= TOL_ENT
    lib = _lib.load()
    t = torch.from_numpy(h).cuda()
    o = torch.empty(10, device="cuda")
    for args in ((0, 7, 10), (1, 0, 10), (1, 7, 0)):
        assert lib.idc_negentropy(0, *args, t.data_ptr(), o.data_ptr(), None) == -1, args
    assert lib.idc_negentropy(0, 1, 7, 10, None, o.data_ptr(), None) == -1


def test_dist_negentropy_resident(synth_sd):
    L, ab, m = util.small_batch(2, X, seed=300)
    ctx = util.make_ctx(synth_sd, X, X, max_n=2, dist=True)
    try:
        with pytest.raises(_lib.IdcError) as e:              # no forward has kept a distribution yet
            ctx.dist_negentropy(0)
        assert e.value.code == -3
        ctx.set_dist_resident(True)
        ctx.forward_host(L, ab, m, 0.5)
        for img in (0, 1):
            neg = ctx.dist_negentropy(img)
            err, _ = _entropy_err(neg, _np_negentropy(ctx.fetch_dist(img)))
            print("resident negentropy image %d: max|kernel - numpy| = %.3e" % (img, err))
            assert neg.shape == (X // 4, X // 4) and neg.dtype == np.float32 and err <= TOL_ENT
        with pytest.raises(_lib.IdcError) as e:
            ctx.dist_negentropy(2)
        assert e.value.code == -3
        # the stand-alone entry on a forward's out_dist: the same kernel on the same distribution, the same bits
        r = ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5, want_dist=True)
        alone = prepost.negentropy_gpu(r["dist"]).cpu().numpy()
        ctx.forward_host(L, ab, m, 0.5)
        assert np.array_equal(alone[1], ctx.dist_negentropy(1))
    finally:
        ctx.close()


def _hints(X, seed):
    return synth.synthetic_hints(X, 4, seed)


def _check_dist529_views(dm):
    """dist_ab_full / dist_ab_grid of ColorizeImageB200Dist against dist_ab, as the reference builds them (:312-317)."""
    for (h, w) in ((0, 0), (5, 9), (X - 1, X - 1), (31, 40), (-1, 3)):
        col = np.asarray(dm.dist_ab[:, h % X, w % X]).astype(np.float64)
        f = dm.dist_ab_full[:, h, w]
        g = dm.dist_ab_grid[:, :, h, w]
        assert f.dtype == np.float64 and np.array_equal(f, col)
        assert g.shape == (23, 23) and np.array_equal(g, col.reshape(23, 23))
    d = np.asarray(dm.dist_ab)
    full = np.asarray(dm.dist_ab_full)
    assert full.dtype == np.float64 and full.shape == (529, X, X) and np.array_equal(full, d.astype(np.float64))
    assert np.array_equal(np.asarray(dm.dist_ab_grid), full.reshape(23, 23, X, X))
    dm.compute_entropy()
    e = dm.dist_entropy
    assert e.shape == (X, X) and e.dtype == np.float32
    assert np.array_equal(e, np.repeat(np.repeat(e[::4, ::4], 4, 0), 4, 1), equal_nan=True)   # constant on 4x4 blocks
    err, _ = _entropy_err(e, _np_negentropy(d))
    print("ColorizeImageB200Dist.compute_entropy: max|device - numpy| = %.3e" % err)
    assert err <= TOL_ENT
    return d, e


def test_dist529_wrapper_views(synth_sd):
    img = (np.random.RandomState(4).rand(X, X, 3) * 255).astype(np.uint8)
    a5, m5 = _hints(X, 1)
    alone = CI.ColorizeImageB200Dist(Xd=X, maskcent=True)
    alone.prep_net(state_dict=synth_sd)
    alone.set_image(img)
    alone.net_forward(a5, m5)
    d_alone, e_alone = _check_dist529_views(alone)
    # after share_trunk: the distribution comes from the colour model's forward
    cm = CI.ColorizeImageB200(Xd=X, maskcent=True)
    cm.prep_net(state_dict=synth_sd, dist=True)
    cm.set_image(img)
    dm = CI.ColorizeImageB200Dist(Xd=X, maskcent=True).share_trunk(cm)
    dm.set_image(img)
    cm.net_forward(a5, m5)
    dm.net_forward(a5, m5)
    d_shared, e_shared = _check_dist529_views(dm)
    assert np.array_equal(d_shared, d_alone) and np.array_equal(e_shared, e_alone, equal_nan=True)
    # materialize_full keeps the host arrays and the reference's host statement
    mf = CI.ColorizeImageB200Dist(Xd=X, maskcent=True, materialize_full=True)
    mf.prep_net(state_dict=synth_sd)
    mf.set_image(img)
    mf.net_forward(a5, m5)
    assert isinstance(mf.dist_ab_full, np.ndarray) and mf.dist_ab_grid.shape == (23, 23, X, X)
    assert util.maxabs(mf.dist_ab, d_alone) <= 1e-6
    mf.compute_entropy()
    assert np.array_equal(mf.dist_entropy, _np_negentropy(mf.dist_ab), equal_nan=True)
    assert _entropy_err(mf.dist_entropy, e_alone)[0] <= TOL_ENT


def _caffe_dist_model(synth_sd):
    sd, _ = _caffe_sd(synth_sd)
    sd = {k: v for k, v in sd.items() if k != "caffe.pts_in_hull"}      # prep_net adds the wrapper's own
    cd = CI.ColorizeImageB200CaffeDist(Xd=X)
    cd.prep_net(0, state_dict=sd)
    cd.set_image((np.random.RandomState(5).rand(X, X, 3) * 255).astype(np.uint8))
    return cd


def test_caffe_dist_wrapper_maps(synth_sd):
    cd = _caffe_dist_model(synth_sd)
    ab, mask = _hints(X, 2)
    cd.net_forward(ab, mask)
    d = np.asarray(cd.dist_ab)
    assert d.shape == (313, X, X) and d.dtype == np.float32
    for (y, x) in PIX:
        assert np.array_equal(d[:, y, x], cd.dist_ab[:, y, x]), (y, x)
    full = cd.dist_ab_full
    assert full.dtype == np.float64 and full.shape == (529, X, X)
    assert np.array_equal(full[cd.in_hull], d) and not np.any(full[~cd.in_hull])
    grid = cd.dist_ab_grid
    assert grid.shape == (23, 23, X, X) and np.array_equal(grid[:, :, 7, 11], full[:, 7, 11].reshape(23, 23))
    cd.compute_entropy()
    err, nans = _entropy_err(cd.dist_entropy, _np_negentropy(d))
    print("ColorizeImageB200CaffeDist.compute_entropy: max|device - numpy| = %.3e (%d NaN pixels)" % (err, nans))
    assert cd.dist_entropy.shape == (X, X) and cd.dist_entropy.dtype == np.float32 and err <= TOL_ENT
    # the next forward brings a new map
    ab2, mask2 = _hints(X, 3)
    cd.net_forward(ab2, mask2)
    d2 = np.asarray(cd.dist_ab)
    assert not np.array_equal(d2, d) and np.array_equal(cd.dist_ab_full[cd.in_hull], d2)


def _stub_pyplot(monkeypatch):
    calls = []
    plt = types.ModuleType("matplotlib.pyplot")
    for name in ("figure", "imshow", "colorbar", "xlabel", "ylabel"):
        setattr(plt, name, (lambda n: lambda *a, **k: calls.append((n, a, k)))(name))
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = plt
    monkeypatch.setitem(sys.modules, "matplotlib", mpl)
    monkeypatch.setitem(sys.modules, "matplotlib.pyplot", plt)
    return calls


def test_plot_methods_of_both_models(synth_sd, monkeypatch):
    calls = _stub_pyplot(monkeypatch)
    dm = CI.ColorizeImageB200Dist(Xd=X)
    dm.prep_net(state_dict=synth_sd)
    dm.set_image((np.random.RandomState(6).rand(X, X, 3) * 255).astype(np.uint8))
    ab, mask = _hints(X, 4)
    dm.net_forward(ab, mask)
    cd = _caffe_dist_model(synth_sd)
    cd.net_forward(ab, mask)
    for model in (dm, cd):
        del calls[:]
        model.plot_dist_grid(20, 33)
        shown = [c for c in calls if c[0] == "imshow"]
        assert len(shown) == 1 and np.array_equal(shown[0][1][0], model.dist_ab_grid[:, :, 20, 33])
        assert shown[0][2] == {"extent": [-110, 110, 110, -110], "interpolation": "nearest"}
        assert [c[0] for c in calls] == ["figure", "imshow", "colorbar", "ylabel", "xlabel"]
        del calls[:]
        model.compute_entropy()
        model.plot_dist_entropy()
        shown = [c for c in calls if c[0] == "imshow"]
        assert len(shown) == 1 and np.array_equal(shown[0][1][0], -model.dist_entropy, equal_nan=True)
