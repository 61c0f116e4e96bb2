"""GPU: batched colour suggestions (idc_ab_reccs_batch, LhnContext.ab_reccs_batch, PhotoColorizer.suggest) at 64^2
and 256^2 on ragged photos.  The query pmf against idc_fetch_dist of the resident map; the batched k-means against
idc_ab_reccs on the same forward for every K / n_init / gamut table, and its independence from the query's position,
duplicates and the run; the picked restart against the FP64 oracle's best inertia; PhotoColorizer.suggest against the
single-image wrapper pair on the exact-FP32 engine, against idc_ab_reccs on its own batched forward on the wgmma
engine, and its colour result against colorize(hints=...) without the head; the announced click; the command line."""
import json
import os

import cv2
import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import _lib, photos
from interactive_deep_colorization_b200 import colorize_image as CI
from interactive_deep_colorization_b200.engine import LhnContext
from oracle import reccs_ref as R, synth
from tests.test_gpu_reveal import SIZES, _photo

pytestmark = pytest.mark.gpu
GRID = R.torch_gamut_points().astype(np.float32)


@pytest.fixture(scope="module")
def sd():
    return synth.torch_state_dict(1234)


@pytest.fixture(scope="module")
def photo_set():
    return [_photo(h, w, 80 + i) for i, (h, w) in enumerate(SIZES)]


def _resident_ctx(sd, X, n, engine="wgmma", seed=3):
    """A dist context after one resident forward_host of n synthetic images with hints."""
    ctx = LhnContext(device=0, max_n=n, H=X, W=X, dist=True, engine=engine)
    ctx.load_state_dict(sd)
    ctx.set_dist_resident(True)
    L, ab, m = synth.synthetic_batch(n, X, seed=seed, max_hints=6)
    ctx.forward_host(L, ab, m, 0.5)
    return ctx


def _queries(X, n, count, seed):
    rs = np.random.RandomState(seed)
    G = X // 4
    q = np.stack([rs.randint(0, n, count), rs.randint(0, G, count), rs.randint(0, G, count)], 1)
    corners = [(0, 0, 0), (n - 1, G - 1, G - 1), (0, G - 1, 0), (n - 1, 0, G - 1)]
    return np.concatenate([np.array(corners), q]).astype(np.int32)


def _batch(ctx, q, K, n_init=8, pts=None, pmf=False):
    out_pmf = torch.empty((len(q), 529), dtype=torch.float32, device="cuda") if pmf else None
    c, f, it = ctx.ab_reccs_batch(q, K=K, n_init=n_init, pts=pts, out_pmf=out_pmf)
    torch.cuda.synchronize()
    return c.cpu().numpy(), f.cpu().numpy(), it.cpu().numpy(), None if out_pmf is None else out_pmf.cpu().numpy()


@pytest.mark.parametrize("X", [64, 256])
def test_query_pmf_equals_resident_dist(sd, X):
    ctx = _resident_ctx(sd, X, 3)
    q = _queries(X, 3, 60, 1)
    q = np.concatenate([q, q[::-1]])                      # duplicates, in another order
    pmf = _batch(ctx, q, 5, pmf=True)[3]
    for i, (img, y4, x4) in enumerate(q):
        assert pmf[i].tobytes() == ctx.fetch_dist(int(img), int(y4), int(x4)).tobytes(), (X, i)
    ctx.close()


@pytest.mark.parametrize("X,Ks,inits", [(64, (1, 5, 9, 32), (1, 8, 16)), (256, (5, 32), (8, 16))])
def test_batched_kmeans_equals_single_pixel_calls(sd, X, Ks, inits):
    ctx = _resident_ctx(sd, X, 3, seed=5)
    q = _queries(X, 3, 24, 2)
    perm = np.random.RandomState(4).permutation(len(q))
    shuffled = np.concatenate([q[perm], q[:5]])           # another order, and five queries twice
    rs = np.random.RandomState(9)
    custom = (GRID[:, ::-1] + rs.uniform(-3, 3, GRID.shape)).astype(np.float32)   # (a, b)-ordered, jittered
    for pts in (None, custom):
        for K in Ks:
            for n_init in inits:
                c, f, it, _ = _batch(ctx, q, K, n_init, pts)
                assert c.shape == (len(q), K, 2) and f.shape == (len(q), K) and it.shape == (len(q),)
                for i, (img, y4, x4) in enumerate(q):
                    cs, fs, its = ctx.ab_reccs(int(img), int(y4), int(x4), K=K, n_init=n_init, pts=pts)
                    assert c[i].tobytes() == cs.tobytes() and f[i].tobytes() == fs.tobytes() and it[i] == its, \
                        (X, K, n_init, pts is None, i)
                c2, f2, it2, _ = _batch(ctx, shuffled, K, n_init, pts)
                want = np.concatenate([perm, np.arange(5)])
                assert c2.tobytes() == c[want].tobytes() and f2.tobytes() == f[want].tobytes()
                assert np.array_equal(it2, it[want])
                c3, f3, _, _ = _batch(ctx, q, K, n_init, pts)  # the same call again
                assert c3.tobytes() == c.tobytes() and f3.tobytes() == f.tobytes()
    ctx.close()


def test_picked_restart_has_the_oracle_best_inertia(sd):
    """The restart rule, independently of the library's own pick: the answer's weighted inertia is the lowest the
    FP64 oracle reaches over the same n_init restarts (restarts within 1e-9 of each other are ties)."""
    X = 64
    ctx = _resident_ctx(sd, X, 2, seed=8)
    q = _queries(X, 2, 60, 6)
    for K in (3, 5, 9):
        c, f, _, pmf = _batch(ctx, q, K, 8, pmf=True)
        for i in range(len(q)):
            runs = [R._one_restart(pmf[i], GRID, K, 100, v) for v in range(8)]
            best = min(R.weighted_inertia(pmf[i], GRID, r[0]) for r in runs)
            e = R.weighted_inertia(pmf[i], GRID, c[i])
            assert abs(e - best) <= 1e-7 * best + 1e-12, (K, i, e, best)
    ctx.close()


def test_batch_abi_errors_on_a_context(sd):
    X = 64
    q = np.array([[0, 1, 2], [1, 3, 4]], np.int32)
    out = torch.full((2, 5, 2), 7.0, device="cuda")
    plain = LhnContext(device=0, max_n=2, H=X, W=X)               # no 529-bin head
    plain.load_state_dict(sd)
    with pytest.raises(_lib.IdcError) as e:
        plain.ab_reccs_batch(q, K=5, out=(out, None, None))
    assert e.value.code == _lib.ERR_STATE
    plain.close()
    ctx = LhnContext(device=0, max_n=2, H=X, W=X, dist=True)
    ctx.load_state_dict(sd)
    with pytest.raises(_lib.IdcError) as e:                       # no forward yet
        ctx.ab_reccs_batch(q, K=5, out=(out, None, None))
    assert e.value.code == _lib.ERR_STATE
    L, ab, m = synth.synthetic_batch(1, X, seed=1, max_hints=3)
    ctx.set_dist_resident(True)
    ctx.forward_host(L, ab, m, 0.5)                               # one image: query 1's image 1 is not in it
    with pytest.raises(_lib.IdcError) as e:
        ctx.ab_reccs_batch(q, K=5, out=(out, None, None))
    assert e.value.code == _lib.ERR_ARG and "query 1" in str(e.value)
    for K, n_init in ((0, 8), (33, 8), (5, 0), (5, 17)):
        with pytest.raises(_lib.IdcError):
            ctx.ab_reccs_batch(q[:1], K=K, n_init=n_init, out=(out, None, None))
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())                               # nothing was written
    c, _, _ = ctx.ab_reccs_batch(q[:1], K=5)                        # the context still answers after the errors
    torch.cuda.synchronize()
    assert c.cpu().numpy()[0].tobytes() == ctx.ab_reccs(0, 1, 2, K=5)[0].tobytes()
    ctx.close()


def test_announced_click_answer_equals_batched(sd):
    X = 256
    ctx = LhnContext(device=0, max_n=1, H=X, W=X, dist=True)
    ctx.load_state_dict(sd)
    ctx.set_dist_resident(True)
    L, ab, m = synth.synthetic_batch(1, X, seed=12, max_hints=5)
    for y4, x4, K in ((10, 20, 9), (63, 0, 5), (31, 47, 32)):
        ctx.set_click(0, y4, x4, K)
        ctx.forward_host(L, ab, m, 0.5)
        served = ctx.ab_reccs(0, y4, x4, K=K)                     # from the click graph's side branch
        c, f, it, pmf = _batch(ctx, np.array([[0, y4, x4]]), K, pmf=True)
        assert served[0].tobytes() == c[0].tobytes() and served[1].tobytes() == f[0].tobytes() and served[2] == it[0]
        assert pmf[0].tobytes() == ctx.fetch_dist(0, y4, x4).tobytes()
    ctx.close()


def _hints_and_points(X, n, seed):
    """Per photo a hint list (hints_from_points, as the command line makes it) and its query points: the hints' locs
    plus a few other pixels; photo 2 has no hints and no points."""
    rs = np.random.RandomState(seed)
    hints, points = [], []
    for i in range(n):
        if i == 2:
            hints.append(CI.hints_from_points([], X))
            points.append(np.zeros((0, 2), np.int64))
            continue
        k = int(rs.randint(1, 8))
        locs = rs.randint(0, X, (k, 2))
        hints.append(CI.hints_from_points([(l, int(rs.randint(0, 4)), rs.uniform(-90, 90, 2)) for l in locs], X))
        points.append(np.concatenate([locs, rs.randint(0, X, (3, 2)), [[0, 0], [X - 1, X - 1]]]).astype(np.int64))
    return hints, points


def _png_files(tmp_path, imgs):
    paths = []
    for i, a in enumerate(imgs):
        p = str(tmp_path / ("p%d.png" % i))
        cv2.imwrite(p, a[:, :, ::-1])
        paths.append(p)
    return paths


@pytest.mark.parametrize("X", [64, 256])
def test_exact_engine_suggest_equals_single_image_wrappers(sd, photo_set, tmp_path, X):
    imgs = photo_set[:4]
    paths = _png_files(tmp_path, imgs)
    hints, points = _hints_and_points(X, len(imgs), 21)
    pc = photos.PhotoColorizer(sd, Xd=X, batch=3, maskcent=True, engine="simt", suggest=True)
    res = list(pc.suggest(paths, hints, points, K=9))
    pc.close()
    cm = CI.ColorizeImageB200(Xd=X, maskcent=True, engine="simt")
    cm.prep_net(state_dict=sd, dist=True)
    dm = CI.ColorizeImageB200Dist(Xd=X, maskcent=True, engine="simt").share_trunk(cm)
    for p, h, pts, r in zip(paths, hints, points, res):
        cm.load_image(p)
        cm.net_forward_hints(h)
        dm.set_image(cm.img_rgb)
        dm.net_forward_hints(h)
        assert r.result.ab.tobytes() == cm.output_ab_raw.astype(np.float32).tobytes()
        assert r.centers.dtype == np.float64 and r.centers.shape == (len(pts), 9, 2) and r.conf.shape == (len(pts), 9)
        for k, (hh, ww) in enumerate(pts):
            c, f = dm.get_ab_reccs(int(hh), int(ww), K=9, return_conf=True)
            assert r.centers[k].tobytes() == c.tobytes() and r.conf[k].tobytes() == f.tobytes(), (X, p, k)


@pytest.mark.parametrize("X", [64, 256])
def test_wgmma_suggest_equals_single_pixel_calls_on_its_forward_and_colour_result(sd, photo_set, X):
    imgs = photo_set
    n = len(imgs)
    hints, points = _hints_and_points(X, n, 33)
    pc = photos.PhotoColorizer(sd, Xd=X, batch=n, suggest=True)
    res = list(pc.suggest(imgs, hints, points, K=5, psnr=True))
    # the colour result: bit for bit what colorize(hints=...) gives without the head
    plain = photos.PhotoColorizer(sd, Xd=X, batch=n)
    want = list(plain.colorize(imgs, hints=hints, psnr=True))
    plain.close()
    for r, w in zip(res, want):
        assert r.result.fullres.tobytes() == w.fullres.tobytes() and r.result.rgb.tobytes() == w.rgb.tobytes()
        assert r.result.ab.tobytes() == w.ab.tobytes() and r.result.psnr == w.psnr
    # the suggestions: idc_ab_reccs on the same batched forward (the planes the pass fed its forward, run again on the
    # same context with the distribution kept resident)
    b = pc._backend
    torch.cuda.synchronize()
    L, ab, m = (t[:n].cpu().numpy() for t in (b.L_mc, b.ab_in, b.mask))
    ctx = b.ctx
    ctx.set_dist_resident(True)
    out = ctx.forward_host(L, ab, m, b.maskcent)
    assert all(out["ab"][i].tobytes() == res[i].result.ab.tobytes() for i in range(n))
    for i, (pts, r) in enumerate(zip(points, res)):
        for k, (hh, ww) in enumerate(pts):
            c, f, _ = ctx.ab_reccs(i, int(hh) // 4, int(ww) // 4, K=5)
            assert r.centers[k].tobytes() == c.astype(np.float64).tobytes(), (X, i, k)
            assert r.conf[k].tobytes() == f.astype(np.float64).tobytes(), (X, i, k)
    pc.close()


def test_suggest_across_batches_and_runs(sd, photo_set):
    """Batch 2 over 7 photos (a short last pass, the query scratch reused and grown) equals batch 7 on the exact engine,
    and a second run equals the first."""
    X = 64
    hints, points = _hints_and_points(X, len(photo_set), 44)
    runs = []
    for batch in (7, 2, 2):
        pc = photos.PhotoColorizer(sd, Xd=X, batch=batch, engine="simt", suggest=True)
        runs.append(list(pc.suggest(photo_set, hints, points, K=7)))
        pc.close()
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert a.centers.tobytes() == b.centers.tobytes() and a.conf.tobytes() == b.conf.tobytes()
            assert a.result.ab.tobytes() == b.result.ab.tobytes()


def test_cli_hints_dir_suggestions_end_to_end(sd, photo_set, tmp_path):
    import ideepcolor_b200 as cli
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
    torch.save(sd, str(tmp_path / "m.pth"))
    rc = cli.main(["--color_model", str(tmp_path / "m.pth"), "--image_dir", str(d), "--hints_dir", str(hd),
                   "--out", str(out), "--load_size", str(X), "--batch", "2", "--suggest", "6", "--psnr"])
    assert rc == 0
    assert sorted(os.listdir(str(out))) == ["a.png", "a_suggestions.json", "b.png", "c.png", "c_suggestions.json",
                                            "psnr.csv"]
    pc = photos.PhotoColorizer(sd, Xd=X, batch=2, suggest=True)
    lists = [ha, [], hc]
    res = list(pc.suggest([str(d / f) for f in names], [cli.hint_rects(h, X) for h in lists],
                          [np.array([h["loc"] for h in hl], np.int64).reshape(-1, 2) for hl in lists], K=6))
    pc.close()
    for name, hl, r in zip(names, lists, res):
        stem = os.path.splitext(name)[0]
        got = cv2.imread(str(out / (stem + ".png")))[:, :, ::-1]
        assert np.array_equal(got, r.result.fullres)
        if hl:
            entries = json.loads((out / (stem + "_suggestions.json")).read_text())
            assert entries == [{"loc": h["loc"], "ab": np.round(c, 3).tolist(), "conf": np.round(f, 5).tolist()}
                               for h, c, f in zip(hl, r.centers, r.conf)]
