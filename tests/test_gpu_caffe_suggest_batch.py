"""GPU: batched colour suggestions of the Caffe 313-bin head (idc_caffe313_reccs_batch, LhnContext.caffe313_reccs_batch,
PhotoColorizer(caffe=True, caffe_dist=True).suggest).  The query pmf against idc_caffe313_dist_pixel at 256^2 and 72 x 88
with more queries than one launch carries; the batched k-means against idc_ab_reccs_pmf on the zero-padded pmf and bin
centres (what ColorizeImageB200CaffeDist.get_ab_reccs feeds it); the ABI's errors on a context; suggest against the
single-image Caffe pair on the exact-FP32 engine, and on the wgmma engine its colour result against caffe=True alone and
its answers against the single-pixel path on its own forward; batching, order and repeat runs; the command line; a
checkpoint without the head."""
import os

import cv2
import numpy as np
import pytest
import torch

import ideepcolor_b200 as cli
from interactive_deep_colorization_b200 import _lib, photos, prepost
from interactive_deep_colorization_b200 import colorize_image as CI
from oracle import caffe_spec, synth
from tests import util
from tests.test_gpu_reveal import SIZES, _photo
from tests.test_gpu_suggest_batch import _hints_and_points, _png_files

pytestmark = pytest.mark.gpu
PTS = prepost.pts_in_hull()
S = 0.2


@pytest.fixture(scope="module")
def csd(synth_sd):
    """A Caffe-scaled checkpoint with both heads: the regression trunk and the 313-bin hyper-column head."""
    sd = util.caffe_scaled(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=PTS).items()})
    return sd


@pytest.fixture(scope="module")
def photo_set():
    return [_photo(h, w, 120 + i) for i, (h, w) in enumerate(SIZES)]


def _forward(ctx, H, W, n, seed):
    """One forward of n synthetic images with a few hints, cropped to H x W."""
    X = max(H, W)
    L, ab, m = synth.synthetic_batch(n, X, seed=seed, max_hints=4)
    crop = lambda a: util.dev(a[:, :, :H, :W])
    ctx.forward_device(crop(L), crop(ab), crop(m), 0.0)
    torch.cuda.synchronize()


def _ctx(csd, H, W, n, seed=3, engine="wgmma"):
    ctx = util.make_ctx(csd, H, W, max_n=n, caffe313=True, engine=engine)
    _forward(ctx, H, W, n, seed)
    return ctx


def _padded(pmf313):
    """What get_ab_reccs(method='gpu') of the Caffe distribution model feeds the k-means: 529 slots, zero-padded."""
    p, q = np.zeros(529, np.float32), np.zeros((529, 2), np.float32)
    p[:313], q[:313] = pmf313, PTS
    return p, q


def _queries(H, W, n, count, seed):
    """The four corners of every image, every sub-position (y & 3, x & 3), the last row and column of the last image,
    then seeded pixels."""
    q = []
    for i in range(n):
        q += [(i, 0, 0), (i, 0, W - 1), (i, H - 1, 0), (i, H - 1, W - 1)]
    q += [(1 % n, 4 + ry, 8 + rx) for ry in range(4) for rx in range(4)]
    q += [(n - 1, H - 1, x) for x in range(W)] + [(n - 1, y, W - 1) for y in range(H)]
    rs = np.random.RandomState(seed)
    q += list(zip(rs.randint(0, n, count), rs.randint(0, H, count), rs.randint(0, W, count)))
    return np.array(q, np.int32)


def _batch(ctx, q, K, n_init=8, pmf=False):
    out_pmf = torch.full((len(q), 529), -1.0, dtype=torch.float32, device="cuda") if pmf else None
    c, f, it = ctx.caffe313_reccs_batch(q, K=K, S=S, n_init=n_init, out_pmf=out_pmf)
    torch.cuda.synchronize()
    return c.cpu().numpy(), f.cpu().numpy(), it.cpu().numpy(), None if out_pmf is None else out_pmf.cpu().numpy()


@pytest.mark.parametrize("H,W", [(256, 256), (72, 88)])
def test_query_pmf_equals_dist_pixel(csd, H, W):
    ctx = _ctx(csd, H, W, 3)
    q = _queries(H, W, 3, 2100, 1)
    assert len(q) > 2048                                  # more than one query launch
    pmf = _batch(ctx, q, 5, pmf=True)[3]
    assert not pmf[:, 313:].any()
    for i, (img, y, x) in enumerate(q):
        assert pmf[i, :313].tobytes() == ctx.caffe313_dist_pixel(int(img), int(y), int(x), S).tobytes(), (H, W, i)
    ctx.close()


@pytest.mark.parametrize("H,W", [(256, 256), (72, 88)])
def test_batched_kmeans_equals_padded_single_pmf_calls(csd, H, W):
    ctx = _ctx(csd, H, W, 3, seed=5)
    q = _queries(H, W, 3, 12, 2)[::7]
    pads = [_padded(ctx.caffe313_dist_pixel(int(img), int(y), int(x), S)) for img, y, x in q]
    for K in (1, 5, 9, 32):
        for n_init in (1, 8):
            c, f, it, _ = _batch(ctx, q, K, n_init)
            assert c.shape == (len(q), K, 2) and f.shape == (len(q), K) and it.shape == (len(q),)
            for i, (p, pts) in enumerate(pads):
                cs, fs, its = prepost.ab_reccs_pmf_gpu(p, K=K, n_init=n_init, pts=pts)
                assert c[i].tobytes() == cs.tobytes() and f[i].tobytes() == fs.tobytes() and it[i] == its, \
                    (H, W, K, n_init, i)
    ctx.close()


def test_abi_errors_on_a_context(csd):
    X = 64
    q = np.array([[0, 1, 2], [1, 63, 63]], np.int32)
    out = torch.full((2, 5, 2), 7.0, device="cuda")
    plain = util.make_ctx(csd, X, X, max_n=2)                     # no 313-bin head
    _forward(plain, X, X, 2, 1)
    with pytest.raises(_lib.IdcError) as e:
        plain.caffe313_reccs_batch(q, K=5, out=(out, None, None))
    assert e.value.code == _lib.ERR_STATE and "IDC_FLAG_CAFFE313" in str(e.value)
    plain.close()
    ctx = util.make_ctx(csd, X, X, max_n=2, caffe313=True)
    with pytest.raises(_lib.IdcError) as e:                       # no forward yet
        ctx.caffe313_reccs_batch(q, K=5, out=(out, None, None))
    assert e.value.code == _lib.ERR_STATE
    _forward(ctx, X, X, 2, 1)
    for bad in ([1, X, 0], [1, 0, X]):                            # y = H, x = W
        with pytest.raises(_lib.IdcError) as e:
            ctx.caffe313_reccs_batch(np.array([q[0], bad], np.int32), K=5, out=(out, None, None))
        assert e.value.code == _lib.ERR_ARG and "query 1" in str(e.value)
    with pytest.raises(_lib.IdcError) as e:
        ctx.caffe313_reccs_batch(q, K=5, S=float("nan"), out=(out, None, None))
    assert e.value.code == _lib.ERR_ARG
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())                               # nothing was written
    c, _, _ = ctx.caffe313_reccs_batch(q[1:], K=5)                # the context still answers after the errors
    torch.cuda.synchronize()
    p, pts = _padded(ctx.caffe313_dist_pixel(1, 63, 63, S))
    assert c.cpu().numpy()[0].tobytes() == prepost.ab_reccs_pmf_gpu(p, K=5, pts=pts)[0].tobytes()
    ctx.close()


@pytest.mark.parametrize("X", [64, 256])
def test_exact_engine_suggest_equals_single_image_caffe_pair(csd, photo_set, tmp_path, X):
    imgs = photo_set[:5]
    paths = _png_files(tmp_path, imgs)
    mixed = [paths[0], imgs[1], paths[2], imgs[3], paths[4]]       # paths and arrays in one run
    hints, points = _hints_and_points(X, len(imgs), 21)
    pc = photos.PhotoColorizer(csd, Xd=X, batch=3, engine="simt", caffe=True, caffe_dist=True)
    res = list(pc.suggest(mixed, hints, points, K=9))
    pc.close()
    cm = CI.ColorizeImageB200Caffe(Xd=X, engine="simt")
    cm.prep_net(state_dict=csd)
    dm = CI.ColorizeImageB200CaffeDist(Xd=X, engine="simt")
    dm.prep_net(state_dict=csd)
    for p, h, pts, r in zip(paths, hints, points, res):
        ab, m = CI.raster_hints(h, X)                             # the dense planes of the photo's hints
        cm.load_image(p)
        cm.net_forward(ab, m)
        assert r.result.ab.tobytes() == cm.output_ab_raw.astype(np.float32).tobytes(), (X, p)
        assert r.result.rgb.tobytes() == cm.output_rgb.tobytes(), (X, p)
        assert r.result.fullres.tobytes() == cm.get_img_fullres().tobytes(), (X, p)
        dm.load_image(p)
        dm.net_forward(ab, m)
        assert r.centers.dtype == np.float64 and r.centers.shape == (len(pts), 9, 2) and r.conf.shape == (len(pts), 9)
        for k, (hh, ww) in enumerate(pts):
            c, f = dm.get_ab_reccs(int(hh), int(ww), K=9, return_conf=True)
            assert r.centers[k].tobytes() == c.tobytes() and r.conf[k].tobytes() == f.tobytes(), (X, p, k)


@pytest.mark.parametrize("X", [64, 256])
def test_wgmma_colour_result_unchanged_and_answers_on_its_forward(csd, photo_set, X):
    imgs = photo_set
    n, batch = len(imgs), 5                                       # the last pass carries photos 5 and 6
    hints, points = _hints_and_points(X, n, 33)
    pc = photos.PhotoColorizer(csd, Xd=X, batch=batch, caffe=True, caffe_dist=True)
    res = list(pc.suggest(imgs, hints, points, K=5, psnr=True))
    plain = photos.PhotoColorizer(csd, Xd=X, batch=batch, caffe=True)
    want = list(plain.colorize(imgs, hints=hints, psnr=True))
    plain.close()
    for i, (r, w) in enumerate(zip(res, want)):
        assert r.result.fullres.tobytes() == w.fullres.tobytes() and r.result.rgb.tobytes() == w.rgb.tobytes(), (X, i)
        assert r.result.ab.tobytes() == w.ab.tobytes() and r.result.psnr == w.psnr, (X, i)
    # the last pass's answers, against the single-pixel path on the logits that pass left on the context
    torch.cuda.synchronize()
    ctx = pc._backend.ctx
    for j, i in enumerate(range(batch, n)):
        assert len(points[i])
        for k, (hh, ww) in enumerate(points[i]):
            p, pts = _padded(ctx.caffe313_dist_pixel(j, int(hh), int(ww), S))
            c, f, _ = prepost.ab_reccs_pmf_gpu(p, K=5, pts=pts)
            assert res[i].centers[k].tobytes() == c.astype(np.float64).tobytes(), (X, i, k)
            assert res[i].conf[k].tobytes() == f.astype(np.float64).tobytes(), (X, i, k)
    pc.close()


def test_more_photos_than_batch_order_and_runs(csd, photo_set):
    X = 64
    hints, points = _hints_and_points(X, len(photo_set), 44)
    runs = []
    for batch in (7, 2, 2):
        pc = photos.PhotoColorizer(csd, Xd=X, batch=batch, engine="simt", caffe=True, caffe_dist=True)
        runs.append(list(pc.suggest(photo_set, hints, points, K=7)))
        pc.close()
    for other in runs[1:]:
        assert len(other) == len(runs[0])
        for a, b in zip(runs[0], other):
            assert a.centers.tobytes() == b.centers.tobytes() and a.conf.tobytes() == b.conf.tobytes()
            assert a.result.ab.tobytes() == b.result.ab.tobytes() and a.result.fullres.shape == b.result.fullres.shape
    for img, r in zip(photo_set, runs[1]):
        assert r.result.fullres.shape == img.shape                # input order


def test_cli_caffe_dist_end_to_end(csd, photo_set, tmp_path):
    import json
    X = 64
    d, hd, out = tmp_path / "photos", tmp_path / "hints", tmp_path / "out"
    d.mkdir()
    hd.mkdir()
    names = ["a.png", "b.png", "c.png"]
    for name, a in zip(names, photo_set[:3]):
        cv2.imwrite(str(d / name), a[:, :, ::-1])
    ha = [{"loc": [10, 20], "size": 2, "ab": [23, -69]}, {"loc": [40, 5], "rgb": [200, 30, 60]}]
    hc = [{"loc": [63, 63], "size": 0, "ab": [-5.5, 7.25]}]
    (hd / "a.json").write_text(json.dumps(ha))
    (hd / "c.json").write_text(json.dumps(hc))
    torch.save(csd, str(tmp_path / "m.pth"))
    rc = cli.main(["--color_model", str(tmp_path / "m.pth"), "--image_dir", str(d), "--hints_dir", str(hd),
                   "--out", str(out), "--load_size", str(X), "--batch", "2", "--caffe", "--caffe_dist", "--suggest", "6"])
    assert rc == 0
    assert sorted(os.listdir(str(out))) == ["a.png", "a_suggestions.json", "b.png", "c.png", "c_suggestions.json"]
    pc = photos.PhotoColorizer(csd, Xd=X, batch=2, caffe=True, caffe_dist=True)
    lists = [ha, [], hc]
    res = list(pc.suggest([str(d / f) for f in names], [cli.hint_rects(h, X) for h in lists],
                          [np.array([h["loc"] for h in hl], np.int64).reshape(-1, 2) for hl in lists], K=6))
    pc.close()
    for name, hl, r in zip(names, lists, res):
        stem = os.path.splitext(name)[0]
        got = cv2.imread(str(out / (stem + ".png")))[:, :, ::-1]
        assert np.array_equal(got, r.result.fullres)
        if hl:
            want = tmp_path / (stem + "_api.json")
            cli.write_suggestions(str(want), hl, r.centers, r.conf)
            assert (out / (stem + "_suggestions.json")).read_text() == want.read_text()


def test_checkpoint_without_the_head_fails_at_construction(csd):
    sd = {k: v for k, v in csd.items() if k != "caffe.pred_313.weight"}
    with pytest.raises(ValueError) as e:
        photos.PhotoColorizer(sd, Xd=64, batch=2, caffe=True, caffe_dist=True)
    assert "caffe.pred_313.weight" in str(e.value)
