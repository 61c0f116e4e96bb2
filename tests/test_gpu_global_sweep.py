"""GPU: global-hints statistics of photo batches (idc_global_stats_batch, PhotoColorizer.global_stats), the global-hints
sweep (PhotoColorizer.global_sweep), the Caffe switch and histogram transfer, on the ragged photo set of the reveal
tests.  The kernel against the reference's own NNEncode, the numpy restatement of global_stats.prototxt and
idc_global_stats; the sweep against LhnContext.forward_device in the same batch layout, the FP32 oracle, the
single-image wrappers and get_result_PSNR; the command line end to end."""
import os

import cv2
import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import _lib, photos, prepost
from interactive_deep_colorization_b200 import colorize_image as CI
from oracle import caffe_spec, synth
from tests import util
from tests.test_gpu_reveal import SIZES, _photo

pytestmark = pytest.mark.gpu
TOL_AB = 1e-3
BATCH = 12                            # three photos per device pass of the four conditions, a short last pass
PTS = prepost.pts_in_hull()


@pytest.fixture(scope="module")
def photo_set():
    return [_photo(h, w, 60 + i) for i, (h, w) in enumerate(SIZES)]


@pytest.fixture(scope="module")
def sdg():
    """The synthetic network with synthetic global-hints weights (glob.*), and those weights alone."""
    gsd = caffe_spec.synthetic_glob_state_dict()
    sd = synth.torch_state_dict(1234)
    sd.update({k: torch.from_numpy(v) for k, v in gsd.items()})
    return sd, gsd


def _kernel(imgs):
    """idc_global_stats_batch on a list of equal-size uint8 images -> [n,316]."""
    a = np.ascontiguousarray(np.stack(imgs))
    n, h, w = a.shape[:3]
    d = torch.from_numpy(a).cuda()
    pts = torch.from_numpy(PTS).cuda()
    out = torch.full((n, 316), float("nan"), device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert _lib.load().idc_global_stats_batch(0, n, h, w, d.data_ptr(), pts.data_ptr(), out.data_ptr(), st) == 0
    return out.cpu().numpy()


def _near(rgb):
    """Per 4x4 cell of rgb: True where the cell's pooled ab lies within 1e-3 ab units of a bin boundary (the margin of
    tests/golden/make_glob_golden.py: second-nearest minus nearest Euclidean distance)."""
    from oracle import color_ref
    lab = color_ref.rgb2lab(rgb)
    H, W = lab.shape[:2]
    ab = lab[..., 1:].reshape(H // 4, 4, W // 4, 4, 2).mean(axis=(1, 3)).reshape(-1, 1, 2)
    d = np.sqrt(((ab - PTS.astype(np.float64)[None]) ** 2).sum(-1))
    d.sort(axis=1)
    return (d[:, 1] - d[:, 0]) < 1e-3


def _counts(row, cells):
    c = np.rint(row[:313].astype(np.float64) * cells).astype(np.int64)
    assert np.array_equal(np.float32(c / cells), row[:313])          # every value is float32(count / cells)
    return c


def test_kernel_vs_reference_nnenc():
    """Row f3 pinned: the histogram against the reference's own NNEncode(NN=1) output; only cells within 1e-3 ab units
    of a bin boundary may land in the other bin."""
    g = util.golden("glob_nnenc.npz")
    for name in ("mortar", "rand"):
        got = _kernel([g[name + "_rgb"]])[0]
        cells = g[name + "_bin"].size
        near = int((g[name + "_margin"] < 1e-3).sum())
        moved = np.abs(got[:313].astype(np.float64) - g[name + "_hist"]).sum() * cells / 2
        print("global_stats_batch %s: %.1f of %d cells differ from NNEncode (%d near a boundary)" % (name, moved, cells, near))
        assert moved <= near + 0.01
        assert got[313] == 1 and got[315] == 1


@pytest.mark.parametrize("X", [64, 256])
def test_kernel_vs_oracle_and_single_image_kernel(photo_set, X):
    imgs = [cv2.resize(a, (X, X)) for a in photo_set]
    got = _kernel(imgs)
    cells = (X // 4) ** 2
    for i, img in enumerate(imgs):
        ref = caffe_spec.global_stats(img, PTS)
        near = int(_near(img).sum())
        c_got = _counts(got[i], cells)
        c_ref = np.rint(ref[:313].astype(np.float64) * cells).astype(np.int64)
        moved = np.abs(c_got - c_ref).sum() // 2
        assert moved <= near, (X, i, moved, near)
        same = c_got == c_ref
        assert np.array_equal(got[i, :313][same], np.float32(c_ref[same] / cells)), (X, i)
        assert got[i, 313] == 1 and got[i, 315] == 1
        assert abs(float(got[i, 314]) - float(ref[314])) <= np.spacing(np.float32(ref[314])), (X, i)
        one = prepost.global_stats_gpu(img)                     # the single-image, many-CTA kernel
        assert one[:313].tobytes() == got[i, :313].tobytes(), (X, i)      # one cell routine: the same bins
        assert abs(float(got[i, 314]) - float(one[314])) <= 2 * np.spacing(np.float32(one[314])), (X, i)
        print("X=%d photo %d: %d cells moved against the oracle (%d near a boundary)" % (X, i, moved, near))


@pytest.mark.parametrize("X", [64, 256])
def test_kernel_is_deterministic_and_batch_independent(photo_set, X):
    imgs = [cv2.resize(a, (X, X)) for a in photo_set]
    p = imgs[0]
    rs = np.random.RandomState(7)
    others = [imgs[1 + k % (len(imgs) - 1)] if k % 3 else rs.randint(0, 256, (X, X, 3)).astype(np.uint8)
              for k in range(126)]
    alone = _kernel([p])[0]
    first = _kernel([p] + others + [p])
    again = _kernel([p] + others + [p])
    assert first.shape == (128, 316)
    for row in (first[0], first[127], again[0], again[127]):
        assert row.tobytes() == alone.tobytes()
    assert first.tobytes() == again.tobytes()


@pytest.mark.parametrize("X", [64, 256])
def test_global_stats_equals_kernel_on_resized_photo(photo_set, sdg, X):
    pc = photos.PhotoColorizer(sdg[0], Xd=X, batch=3, global_hints=True)
    rows = list(pc.global_stats(photo_set))
    pc.close()
    want = _kernel([cv2.resize(a, (X, X)) for a in photo_set])
    assert len(rows) == len(photo_set)
    for i, r in enumerate(rows):
        assert r.dtype == np.float32 and r.tobytes() == want[i].tobytes(), (X, i)


def _single(photo, X):
    small, lab, _ = prepost.load_image_gpu(photo, X)
    return np.float32(lab[0] - 50)[None], small


@pytest.mark.parametrize("X", [64, 256])
def test_sweep_equals_forward_oracle_and_wrappers(photo_set, sdg, X, tmp_path):
    sd, gsd = sdg
    conds = photos.GLOBAL_CONDITIONS
    C = len(conds)
    pc = photos.PhotoColorizer(sd, Xd=X, batch=BATCH, global_hints=True)
    res = list(pc.global_sweep(photo_set))
    assert len(res) == len(photo_set)
    ctx = pc._backend.ctx
    singles = [_single(a, X) for a in photo_set]
    stats = _kernel([cv2.resize(a, (X, X)) for a in photo_set])
    per = BATCH // C
    zeros_ab, zeros_m = np.zeros((2, X, X), np.float32), np.zeros((1, X, X), np.float32)
    for k in range(0, len(photo_set), per):                 # the passes global_sweep cut: 3, 3, 1 photos
        idx = list(range(k, min(k + per, len(photo_set))))
        Ls = [singles[i][0] for i in idx for _ in conds]
        globs = [photos.glob_vector(stats[i], c) for i in idx for c in conds]
        n = len(Ls)
        ref = ctx.forward_device(util.dev(np.stack(Ls)), util.dev(np.stack([zeros_ab] * n)),
                                 util.dev(np.stack([zeros_m] * n)), 0.0, glob=util.dev(np.stack(globs)), want_rgb=True)
        torch.cuda.synchronize()
        ref_ab, ref_rgb = ref["ab"].cpu().numpy(), ref["rgb"].cpu().numpy()
        for jj, i in enumerate(idx):
            r = res[i]
            assert r.ab.shape == (C, 2, X, X) and r.rgb.shape == (C, X, X, 3) and r.psnr.shape == (C,)
            assert r.stats.tobytes() == stats[i].tobytes(), (X, i)
            assert np.array_equal(r.ab, ref_ab[jj * C:(jj + 1) * C]), (X, i)
            assert np.array_equal(r.rgb, ref_rgb[jj * C:(jj + 1) * C]), (X, i)
            w = CI.ColorizeImageBase(Xd=X)
            w.img_rgb = singles[i][1]
            for j in range(C):
                assert r.psnr[j] == w.get_result_PSNR(r.rgb[j]), (X, i, conds[j])
    # the global hints reach the network: each condition changes every photo's result
    assert all(util.maxabs(r.ab[0], r.ab[j]) > 1e-2 for r in res for j in (1, 2, 3))
    # "none" is colorize() with a zero glob vector, bit for bit
    plain = list(pc.colorize(photo_set, glob=[np.zeros(316, np.float32)] * len(photo_set)))
    for i, p in enumerate(plain):
        assert np.array_equal(p.ab, res[i].ab[0]) and np.array_equal(p.rgb, res[i].rgb[0]), (X, i)
    pc.close()
    # FP32 oracle (global_hints_vector of the synthetic glob weights) and the GlobDist wrapper's histogram call
    cm = CI.ColorizeImageB200GlobDist(Xd=X)
    cm.prep_net(state_dict=sd)
    for i in (0, 4):
        p = str(tmp_path / ("photo%d.png" % i))
        cv2.imwrite(p, photo_set[i][:, :, ::-1])
        cm.load_image(p)
        for j, c in enumerate(conds):
            g = photos.glob_vector(stats[i], c)[None]
            ref = util.oracle_forward(sd, singles[i][0][None], zeros_ab[None], zeros_m[None], 0.0,
                                      glob_add=caffe_spec.global_hints_vector(gsd, g))
            assert util.maxabs(res[i].ab[j], ref[0]) <= TOL_AB, (X, i, c)
        cm.net_forward(np.zeros((2, X, X)), np.zeros((1, X, X)), stats[i][:313])
        assert util.maxabs(res[i].ab[2], cm.output_ab_raw) <= TOL_AB, (X, i)


def test_sweep_is_deterministic_and_batch_independent(photo_set, sdg):
    """Batch 4, 12 and 32 put a photo's conditions in passes of 1, 3 and 7 photos (8 at 32).  On the exact-FP32 engine
    the forward does not depend on the context's batch, so every result is identical bit for bit; the wgmma engine
    chooses its split-K plan from the context's batch, so there the statistics and layout are identical and ab agrees
    within the engine's tolerance."""
    X = 64
    imgs = photo_set[:6]
    out = {}
    for eng in ("simt", "wgmma"):
        for batch in (4, 12, 32):
            pc = photos.PhotoColorizer(sdg[0], Xd=X, batch=batch, global_hints=True, engine=eng)
            out[eng, batch] = list(pc.global_sweep(imgs))
            if batch == 12:
                again = list(pc.global_sweep(imgs))
                for r, s in zip(out[eng, batch], again):
                    assert np.array_equal(r.ab, s.ab) and np.array_equal(r.rgb, s.rgb) and np.array_equal(r.psnr, s.psnr)
            pc.close()
    for eng in ("simt", "wgmma"):
        for batch in (12, 32):
            for r, s in zip(out[eng, 4], out[eng, batch]):
                assert r.stats.tobytes() == s.stats.tobytes()
                if eng == "simt":
                    assert np.array_equal(r.ab, s.ab) and np.array_equal(r.rgb, s.rgb), (eng, batch)
                    assert np.array_equal(r.psnr, s.psnr), (eng, batch)
                else:
                    print("wgmma, batch 4 against %d: max |d ab| = %.3g" % (batch, util.maxabs(r.ab, s.ab)))
                    assert util.maxabs(r.ab, s.ab) <= TOL_AB, (eng, batch)
    for r, s in zip(out["simt", 12], out["wgmma", 12]):
        assert util.maxabs(r.ab, s.ab) <= TOL_AB


def test_caffe_colorize_and_sweep(photo_set, sdg, tmp_path):
    sd, gsd = sdg
    X = 64
    csd = util.caffe_scaled(sd)                               # Caffe-scaled weights of the same network
    pc = photos.PhotoColorizer(csd, Xd=X, batch=8, global_hints=True, caffe=True)
    imgs = photo_set[:3]
    res = list(pc.global_sweep(imgs, conditions=("none", "hist")))
    stats = [r.stats for r in res]
    hint = CI.hints_from_points([([30, 20], 2, [23.0, -40.0])], X)
    col = list(pc.colorize(imgs, hints=[hint] * 3, glob=[photos.glob_vector(s, "hist") for s in stats]))
    pc.close()
    cg = CI.ColorizeImageB200CaffeGlobDist(Xd=X)
    cg.prep_net(0, state_dict=csd)
    zeros_ab, zeros_m = np.zeros((2, X, X)), np.zeros((1, X, X))
    ab, m = np.zeros((2, X, X)), np.zeros((1, X, X))
    CI.put_point(ab, m, [30, 20], 2, [23.0, -40.0])
    for i, a in enumerate(imgs):
        p = str(tmp_path / ("c%d.png" % i))
        cv2.imwrite(p, a[:, :, ::-1])
        cg.load_image(p)
        L = cg.img_l_mc.astype(np.float32)[None]
        cg.net_forward(zeros_ab, zeros_m)
        assert util.maxabs(res[i].ab[0], cg.output_ab_raw) <= TOL_AB, i
        cg.net_forward(zeros_ab, zeros_m, stats[i][:313])
        assert util.maxabs(res[i].ab[1], cg.output_ab_raw) <= TOL_AB, i
        cg.net_forward(ab, m, stats[i][:313])
        assert util.maxabs(col[i].ab, cg.output_ab_raw) <= TOL_AB, i
        for j, c in enumerate(("none", "hist")):
            g = caffe_spec.global_hints_vector(gsd, photos.glob_vector(stats[i], c)[None])
            ref = util.oracle_forward(sd, L, zeros_ab[None].astype(np.float32), zeros_m[None].astype(np.float32), 0.0,
                                      glob_add=g)[0] * (100.0 / 110.0)
            assert util.maxabs(res[i].ab[j], ref) <= TOL_AB, (i, c)
        g = caffe_spec.global_hints_vector(gsd, photos.glob_vector(stats[i], "hist")[None])
        ref = util.oracle_forward(sd, L, ab[None].astype(np.float32), m[None].astype(np.float32), 0.0,
                                  glob_add=g)[0] * (100.0 / 110.0)
        assert util.maxabs(col[i].ab, ref) <= TOL_AB, i


def test_histogram_transfer(photo_set, sdg, tmp_path):
    sd, _ = sdg
    X = 64
    ref_photo = _photo(375, 500, 99)
    pc = photos.PhotoColorizer(sd, Xd=X, batch=4, global_hints=True)
    ref_stats = next(iter(pc.global_stats([ref_photo])))
    imgs = photo_set[:5]
    out = list(pc.colorize(imgs, glob=[photos.glob_vector(ref_stats, "hist")] * len(imgs)))
    pc.close()
    cm = CI.ColorizeImageB200GlobDist(Xd=X)
    cm.prep_net(state_dict=sd)
    hist = cm.get_global_histogram(ref_photo)                 # the wrapper's own statistics of the same photo
    assert np.abs(hist.astype(np.float64) - ref_stats[:313]).sum() * (X // 4) ** 2 / 2 <= int(_near(cv2.resize(ref_photo, (X, X))).sum())
    for i, a in enumerate(imgs):
        p = str(tmp_path / ("t%d.png" % i))
        cv2.imwrite(p, a[:, :, ::-1])
        cm.load_image(p)
        cm.net_forward(np.zeros((2, X, X)), np.zeros((1, X, X)), ref_stats[:313])
        assert util.maxabs(out[i].ab, cm.output_ab_raw) <= TOL_AB, i


def test_command_line(photo_set, sdg, tmp_path):
    import ideepcolor_b200 as cli
    sd, _ = sdg
    d = tmp_path / "photos"
    d.mkdir()
    names = ["p%d.png" % i for i in range(5)]
    for name, a in zip(names, photo_set[:5]):
        cv2.imwrite(str(d / name), a[:, :, ::-1])
    ckpt = str(tmp_path / "glob.pth")
    torch.save(sd, ckpt)
    out = tmp_path / "sweep"
    assert cli.main(["--color_model", ckpt, "--image_dir", str(d), "--out", str(out), "--global_hints", "--glob_sweep",
                     "--batch", "8", "--load_size", "64"]) == 0
    lines = (out / "glob_psnr.csv").read_text().splitlines()
    assert lines[0] == "image," + ",".join(photos.GLOBAL_CONDITIONS)
    pc = photos.PhotoColorizer(sd, Xd=64, batch=8, global_hints=True)
    api = [r.psnr for r in pc.global_sweep([str(d / n) for n in names])]
    pc.close()
    for line, name, want in zip(lines[1:], names, api):
        cells = line.split(",")
        assert cells[0] == name and np.array_equal(np.array([float(v) for v in cells[1:]]), want)
    assert np.array_equal(np.array([float(v) for v in lines[-1].split(",")[1:]]), np.mean(api, axis=0))
    ref = tmp_path / "ref.png"
    cv2.imwrite(str(ref), _photo(200, 300, 5))
    out2 = tmp_path / "transfer"
    assert cli.main(["--color_model", ckpt, "--image_dir", str(d), "--out", str(out2), "--global_hints",
                     "--glob_ref", str(ref), "--load_size", "64"]) == 0
    assert sorted(os.listdir(str(out2))) == names
    for name, a in zip(names, photo_set[:5]):
        assert cv2.imread(str(out2 / name)).shape == a.shape
