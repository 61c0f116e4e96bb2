"""GPU: the wgmma engine end to end -- the parity tests proper.  Everything goes through
the C ABI (engine.LhnContext -> libidc_b200.so)."""
import numpy as np
import pytest
import torch

from oracle import color_ref, synth
from tests import util

pytestmark = pytest.mark.gpu
TOL_AB = 1e-3        # BASELINE.json north_star: ab within 1e-3 max-abs of the reference


def _hints(case):
    ab, m = np.zeros((2, 256, 256)), np.zeros((1, 256, 256))
    if case == "kat":
        synth.put_point(ab, m, [135, 160], 3, [23, -69])
        synth.put_point(ab, m, [100, 160], 3, [0, 0])
    elif case == "rand5":
        ab, m = synth.synthetic_hints(256, 5, 0)
    return ab, m


@pytest.fixture(scope="module")
def ctx256(synth_sd):
    ctx = util.make_ctx(synth_sd, 256, 256, max_n=4, dist=True)
    yield ctx
    ctx.close()


@pytest.mark.parametrize("case,mc", [("zero", 0.0), ("rand5", 0.0), ("kat", 0.0), ("rand5", 0.5)])
def test_golden_256(ctx256, case, mc):
    """configs 1 and 2 of BASELINE.json: reference net output on mortar_pestle.jpg @256."""
    g = util.golden("lhn_256.npz")
    L = g["img_l_mc"].astype(np.float32)[None]
    ab, m = _hints(case)
    r = ctx256.forward_host(L, ab[None].astype(np.float32), m[None].astype(np.float32), mc, want_rgb=True)
    ref = g["mc%d_%s_ab_raw" % (1 if mc else 0, case)]
    err = util.maxabs(util.at_pix(g, r["ab"][0]), ref)
    print("golden %s mc=%s max|dab| = %.3e" % (case, mc, err))
    assert err <= TOL_AB, err
    if not mc:
        rgb_ref = g["mc0_%s_rgb" % case]
        d = np.abs(util.at_pix_hwc(g, r["rgb"][0]).astype(int) - rgb_ref.astype(int))
        assert d.max() <= 1 and (d > 0).mean() < 2e-3, (d.max(), (d > 0).mean())


def test_batch_64_oracle_and_layers(synth_sd):
    L, ab, m = util.small_batch(3, 64, seed=300)
    ctx = util.make_ctx(synth_sd, 64, 64, max_n=3, dist=True, keep_conv10=True)
    r = ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5, want_dist=True)
    torch.cuda.synchronize()
    (reg, dist), inter = util.oracle_forward(synth_sd, L, ab, m, 0.5, dist=True, intermediates=True)
    for name in ["a1_1", "conv1_2", "conv2_2", "conv3_3", "conv4_3", "conv5_3", "conv6_3", "conv7_3", "conv8_3",
                 "conv9_3", "a10_1", "conv10_2"]:
        err = util.maxabs(ctx.get_activation(name, 3), inter[name])
        assert err < 2e-4, (name, err)
    assert util.maxabs(r["ab"], reg) <= TOL_AB
    assert util.maxabs(r["dist"], dist) < 1e-5
    assert abs(float(r["dist"].sum(1).mean()) - 1.0) < 1e-5
    ctx.close()
    # fused-head variant (default) must agree with the unfused one
    ctx2 = util.make_ctx(synth_sd, 64, 64, max_n=3)
    r2 = ctx2.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5)
    torch.cuda.synchronize()
    assert util.maxabs(r2["ab"], r["ab"]) < 1e-4
    ctx2.close()


def test_dist_golden(ctx256):
    g = util.golden("lhn_256.npz")
    gd = util.golden("lhn_dist_256.npz")
    L = g["img_l_mc"].astype(np.float32)[None]
    ab, m = _hints("rand5")
    r = ctx256.forward_host(L, ab[None].astype(np.float32), m[None].astype(np.float32), 0.5, want_dist=True)
    d = r["dist"][0]
    assert util.maxabs(d[:, ::8, ::8], gd["dist_rows"]) < 1e-5
    assert util.maxabs(d.sum(0), gd["dist_sum64"]) < 1e-5
    assert util.maxabs(d.max(0), gd["dist_max64"]) < 1e-5
    assert (d.argmax(0) == gd["dist_argmax64"]).mean() > 0.999
    assert util.maxabs(r["ab"][0] * 110.0, gd["ret_quirk"]) < 0.15      # quirk q1: tanh*110*110


def test_lab2rgb_kernel_bit_exact():
    from interactive_deep_colorization_b200 import _lib
    lib = _lib.load()
    rs = np.random.RandomState(3)
    L = rs.uniform(0, 100, (2, 1, 64, 96)).astype(np.float32)
    ab = rs.uniform(-110, 110, (2, 2, 64, 96)).astype(np.float32)
    dL, dab = util.dev(L), util.dev(ab)
    out = torch.empty((2, 64, 96, 3), dtype=torch.uint8, device="cuda")
    rc = lib.idc_lab2rgb_u8(0, 2, 64, 96, dL.data_ptr(), dab.data_ptr(), out.data_ptr(), None)
    assert rc == 0
    torch.cuda.synchronize()
    for i in range(2):
        ref = color_ref.lab2rgb_transpose(L[i].astype(np.float64), ab[i].astype(np.float64))
        assert np.array_equal(out[i].cpu().numpy(), ref)


def test_wrapper_api_end_to_end(synth_sd):
    """ColorizeImageB200 / ...Dist used exactly like the reference notebook uses ColorizeImageTorch."""
    from interactive_deep_colorization_b200 import colorize_image as CI
    g = util.golden("lhn_256.npz")
    cm = CI.ColorizeImageB200(Xd=256)
    cm.prep_net(state_dict=synth_sd)
    cm.set_image(g["img_rgb"])
    ab, m = np.zeros((2, 256, 256)), np.zeros((1, 256, 256))
    CI.put_point(ab, m, [135, 160], 3, [23, -69])
    CI.put_point(ab, m, [100, 160], 3, [0, 0])
    rgb = cm.net_forward(ab, m)
    assert rgb.shape == (256, 256, 3) and rgb.dtype == np.uint8
    assert util.maxabs(util.at_pix(g, cm.output_ab_raw), g["mc0_kat_ab_raw"]) <= TOL_AB
    d = np.abs(util.at_pix_hwc(g, rgb).astype(int) - g["mc0_kat_rgb"].astype(int))
    assert d.max() <= 1 and (d > 0).mean() < 2e-3
    assert np.max(np.abs(util.at_pix(g, cm.output_ab) - g["mc0_kat_output_ab"])) < 1.5     # 1 uint8 step in ab units
    full = cm.get_img_fullres()                      # GPU zoom + Lab->RGB (row f1)
    assert full.shape == (256, 256, 3)
    d = np.abs(full.astype(int) - color_ref.lab2rgb_transpose(cm.img_l_fullres, cm.output_ab).astype(int))
    assert d.max() <= 1 and (d > 0).mean() < 1e-3
    cd = CI.ColorizeImageB200Dist(Xd=256, maskcent=True)
    cd.prep_net(state_dict=synth_sd)
    cd.set_image(g["img_rgb"])
    a5, m5 = synth.synthetic_hints(256, 5, 0)
    ret = cd.net_forward(a5, m5)
    gd = util.golden("lhn_dist_256.npz")
    assert util.maxabs(ret, gd["ret_quirk"]) < 0.15
    # the distribution stays on the device; single pixels are fetched on demand (529 floats)
    assert util.maxabs(np.asarray(cd.dist_ab[:, 64, 96]), gd["dist_rows"][:, 2, 3]) < 1e-5
    assert util.maxabs(np.asarray(cd.dist_ab[:, 67, 99]), gd["dist_rows"][:, 2, 3]) < 1e-5     # nearest x4 upsample
    full = np.asarray(cd.dist_ab)
    assert full.shape == (529, 256, 256) and util.maxabs(full[:, ::32, ::32], gd["dist_rows"]) < 1e-5
    np.random.seed(0)
    reccs = cd.get_ab_reccs(128, 128, K=9, N=25000)
    assert reccs.shape == (9, 2) and np.all(np.abs(reccs) <= 110)


def test_full_size_batch_properties(synth_sd):
    """BASELINE config 3 size (64 x 256^2): size-independent properties instead of an oracle run:
    (1) every image of the batch equals the same image run alone (no cross-image leakage),
    (2) batch permutation equivariance, (3) outputs bounded by tanh*110."""
    N = 64
    L, ab, m = synth.synthetic_batch(N, 256, seed=0, max_hints=10)
    ctx = util.make_ctx(synth_sd, 256, 256, max_n=N)
    dL, dab, dm = util.dev(L), util.dev(ab), util.dev(m)
    out = ctx.forward_device(dL, dab, dm, 0.5)["ab"].clone()
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(0)).cuda()
    out_p = ctx.forward_device(dL[perm].contiguous(), dab[perm].contiguous(), dm[perm].contiguous(), 0.5)["ab"]
    torch.cuda.synchronize()
    assert torch.equal(out_p, out[perm])
    assert float(out.abs().max()) <= 110.0
    for i in (0, 17, 63):
        single = ctx.forward_device(dL[i:i + 1].contiguous(), dab[i:i + 1].contiguous(), dm[i:i + 1].contiguous(), 0.5)["ab"]
        torch.cuda.synchronize()
        assert torch.equal(single[0], out[i])
    # spot parity against the oracle on two images of the batch
    ref = util.oracle_forward(synth_sd, L[[5, 40]], ab[[5, 40]], m[[5, 40]], 0.5)
    assert util.maxabs(out[[5, 40]], ref) <= TOL_AB
    ctx.close()


def test_global_hints_branch(synth_sd):
    """row a15: 4-layer global MLP + per-(image, channel) add on conv4_3 (Caffe spec; parity unpinned,
    checked against oracle/caffe_spec.py + the glob_add path of oracle/lhn_ref.py)."""
    from oracle import caffe_spec
    gsd = caffe_spec.synthetic_glob_state_dict()
    sd = dict(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in gsd.items()})
    L, ab, m = util.small_batch(3, 64, seed=300)
    glob_ab, sat = synth.synthetic_glob(3, seed=1)
    glob = np.ascontiguousarray(np.concatenate([glob_ab, sat], axis=1).astype(np.float32))      # [3,316]
    gvec = caffe_spec.global_hints_vector(gsd, glob)
    ref, inter = util.oracle_forward(synth_sd, L, ab, m, 0.5, glob_add=gvec, intermediates=True)
    ref_noglob = util.oracle_forward(synth_sd, L, ab, m, 0.5)
    assert util.maxabs(ref, ref_noglob) > 0.5                      # the branch actually matters
    for engine in ("simt", "wgmma"):
        ctx = util.make_ctx(sd, 64, 64, max_n=3, engine=engine, global_hints=True)
        r = ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5, glob=util.dev(glob))
        torch.cuda.synchronize()
        assert util.maxabs(ctx.get_activation("conv4_3", 3), inter["conv4_3"]) < 2e-4, engine
        assert util.maxabs(r["ab"], ref) <= TOL_AB, engine
        r0 = ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5)          # glob omitted -> plain network
        torch.cuda.synchronize()
        assert util.maxabs(r0["ab"], ref_noglob) <= TOL_AB, engine
        ctx.close()


def test_caffe313_head(synth_sd):
    """row a14 (Caffe spec, parity unpinned): hyper-column + pred_313 + bilinear x4 + annealed mean, against
    oracle/caffe_spec.caffe313_head (which uses the literal grouped Deconvolution kernels)."""
    from oracle import caffe_spec
    pts = np.load(util.os.path.join(util.GOLDEN, "pts_in_hull.npy"))
    csd = caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=pts)
    sd = dict(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in csd.items()})
    L, ab, m = util.small_batch(2, 64, seed=500)
    _, inter = util.oracle_forward(synth_sd, L, ab, m, 0.5, intermediates=True)
    with torch.no_grad():
        pred_ref, distS_ref, logits_ref, hyper_ref = caffe_spec.caffe313_head(csd, inter, return_logits=True)
        pred64, _, logits64, _ = caffe_spec.caffe313_head(csd, inter, return_logits=True, dtype=torch.float64)
    assert float(pred_ref.abs().max()) > 5.0
    ref32_vs_64 = util.maxabs(pred_ref, pred64)            # how far an FP32 evaluation of the spec is from exact arithmetic
    for engine in ("simt", "wgmma"):
        ctx = util.make_ctx(sd, 64, 64, max_n=2, engine=engine, caffe313=True)
        ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5)
        torch.cuda.synchronize()
        assert util.maxabs(ctx.get_activation("hyper", 2), hyper_ref) < 3e-4, engine
        pred = ctx.caffe313_pred_ab(2)
        torch.cuda.synchronize()
        err, err64 = util.maxabs(pred, pred_ref), util.maxabs(pred, pred64)
        d = (pred.cpu().double() - pred64).abs()
        w = int(d.argmax())
        n_, c_, y_, x_ = np.unravel_index(w, tuple(d.shape))
        top2 = torch.topk(logits64[n_, :, y_ // 4, x_ // 4], 2).values
        print("caffe313 %s: max|d pred_ab| vs FP32 oracle %.3e, vs FP64 evaluation %.3e (FP32 oracle vs FP64: %.3e); worst pixel "
              "(n=%d, c=%d, y=%d, x=%d), top-2 logit gap there %.3f (x T=2.6 in the softmax)"
              % (engine, err, err64, ref32_vs_64, n_, c_, y_, x_, float(top2[0] - top2[1])))
        # spec-only head (parity unpinned).  The bar is the north_star's 1e-3, measured against the FP64 evaluation
        # of the spec; where the FP32 oracle itself is further than that from exact arithmetic (the annealed-mean
        # softmax multiplies logit noise by T * |ab range|), twice the oracle's own distance is allowed.
        assert err64 <= max(1e-3, 2.0 * ref32_vs_64), (engine, err64, ref32_vs_64)
        for (y, x) in ((0, 0), (13, 62), (63, 63), (31, 7)):
            d = ctx.caffe313_dist_pixel(1, y, x)
            assert util.maxabs(d, distS_ref[1, :, y, x]) < 1e-5, (engine, y, x)
            assert abs(float(d.sum()) - 1.0) < 1e-5
        ctx.close()


def test_config4_512_global_hints(synth_sd):
    """BASELINE config 4: 512x512 with a global-hints histogram vector (2 of the 16 images, oracle-checked)."""
    from oracle import caffe_spec
    gsd = caffe_spec.synthetic_glob_state_dict()
    sd = dict(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in gsd.items()})
    L, ab, m = synth.synthetic_batch(2, 512, seed=40, max_hints=10)
    glob_ab, sat = synth.synthetic_glob(2, seed=3)
    glob = np.ascontiguousarray(np.concatenate([glob_ab, sat], axis=1).astype(np.float32))
    gvec = caffe_spec.global_hints_vector(gsd, glob)
    ref = util.oracle_forward(synth_sd, L, ab, m, 0.5, glob_add=gvec)
    ctx = util.make_ctx(sd, 512, 512, max_n=2, global_hints=True)
    r = ctx.forward_host(L, ab, m, 0.5, glob=glob, want_rgb=True)
    err = util.maxabs(r["ab"], ref)
    print("512x512 + global hints: max|d ab| = %.3e" % err)
    assert err <= TOL_AB
    assert r["rgb"].shape == (2, 512, 512, 3)
    ctx.close()


def test_prepost_gpu_kernels_match_numpy_scipy():
    """row f1: float64 GPU rgb2lab and zoom(order=1)+lab2rgb against the numpy/scipy restatements."""
    from scipy.ndimage import zoom
    from interactive_deep_colorization_b200 import prepost
    rs = np.random.RandomState(5)
    rgb = rs.randint(0, 256, (2, 37, 53, 3)).astype(np.uint8)
    lab = prepost.rgb2lab_gpu(rgb)
    for i in range(2):
        assert np.max(np.abs(lab[i] - color_ref.rgb2lab_transpose(rgb[i]))) < 1e-10
    ab = rs.uniform(-80, 80, (2, 32, 32))
    Lf = rs.uniform(0, 100, (1, 75, 91))
    got = prepost.fullres_rgb_gpu(ab, Lf)
    ref = color_ref.lab2rgb_transpose(Lf, zoom(ab, (1, 75 / 32., 91 / 32.), order=1))
    d = np.abs(got.astype(int) - ref.astype(int))
    assert d.max() <= 1 and (d > 0).mean() < 1e-3, (d.max(), (d > 0).mean())


def test_global_stats_kernel():
    """row f3: histogram / saturation extractor against the numpy restatement of global_stats.prototxt."""
    from oracle import caffe_spec
    from interactive_deep_colorization_b200 import prepost
    g = util.golden("lhn_256.npz")
    pts = np.load(util.os.path.join(util.GOLDEN, "pts_in_hull.npy"))
    assert np.array_equal(pts, prepost.pts_in_hull())
    for rgb in (g["img_rgb"], np.random.RandomState(2).randint(0, 256, (64, 96, 3)).astype(np.uint8)):
        got = prepost.global_stats_gpu(rgb)
        ref = caffe_spec.global_stats(rgb, pts)
        assert got.shape == (316,) and abs(got[:313].sum() - 1.0) < 1e-5
        assert np.abs(got - ref).max() < 2e-3, np.abs(got - ref).max()      # a cell on a bin boundary may flip
        assert np.abs(got[313:] - ref[313:]).max() < 1e-6


def test_globdist_wrapper(synth_sd):
    """ColorizeImageB200GlobDist used like the reference notebook uses ColorizeImageCaffeGlobDist."""
    from interactive_deep_colorization_b200 import colorize_image as CI
    from oracle import caffe_spec
    gsd = caffe_spec.synthetic_glob_state_dict()
    sd = dict(synth_sd)
    sd.update({k: torch.from_numpy(v) for k, v in gsd.items()})
    g = util.golden("lhn_256.npz")
    cid = CI.ColorizeImageB200GlobDist(Xd=256)
    cid.prep_net(state_dict=sd)
    cid.set_image(g["img_rgb"])
    ab, m = np.zeros((2, 256, 256)), np.zeros((1, 256, 256))
    plain = cid.net_forward(ab, m)                                  # glob_dist = -1 -> zeros
    raw_plain = cid.output_ab_raw.copy()
    ref_rgb = np.random.RandomState(4).randint(0, 256, (120, 160, 3)).astype(np.uint8)
    hist = cid.get_global_histogram(ref_rgb)
    assert hist.shape == (313,) and abs(hist.sum() - 1) < 1e-5
    out = cid.net_forward(ab, m, hist)
    assert out.shape == (256, 256, 3) and plain.shape == (256, 256, 3)
    glob = np.zeros((1, 316), np.float32); glob[0, :313] = hist; glob[0, 313] = 1
    L = g["img_l_mc"].astype(np.float32)[None]
    for gl, got in ((np.zeros((1, 316), np.float32), raw_plain), (glob, cid.output_ab_raw)):
        ref = util.oracle_forward(synth_sd, L, ab[None], m[None], 0.0, glob_add=caffe_spec.global_hints_vector(gsd, gl))
        assert util.maxabs(got, ref[0]) <= TOL_AB


@pytest.mark.parametrize("H,W,n", [(72, 88, 2), (128, 64, 3), (8, 8, 1)])
def test_odd_geometries(synth_sd, H, W, n):
    """Geometry is any multiple of 8 (three ::2 + three x2 stages): partial tiles, non-square images, tile
    counts that do not pair up, and the smallest legal size."""
    rs = np.random.RandomState(H * 1000 + W)
    L = (rs.rand(n, 1, H, W) * 100 - 50).astype(np.float32)
    ab = np.zeros((n, 2, H, W), np.float32)
    m = np.zeros((n, 1, H, W), np.float32)
    for i in range(n):
        y, x = rs.randint(0, H - 3), rs.randint(0, W - 3)
        ab[i, :, y:y + 3, x:x + 3] = rs.uniform(-80, 80, (2, 1, 1))
        m[i, :, y:y + 3, x:x + 3] = 1
    ref = util.oracle_forward(synth_sd, L, ab, m, 0.5, dist=True)
    for forced_pairs in (0, 2):
        ctx = util.make_ctx(synth_sd, H, W, max_n=n, dist=True, options={"pairs": forced_pairs})
        r = ctx.forward_host(L, ab, m, 0.5, want_dist=True, want_rgb=True)
        assert util.maxabs(r["ab"], ref[0]) <= TOL_AB, (H, W, forced_pairs)
        assert util.maxabs(r["dist"], ref[1]) < 1e-5
        ctx.close()


@pytest.mark.parametrize("n,pinned", [(20, False), (40, True), (9, True), (67, True)])
def test_host_pipeline_matches_device_path(synth_sd, n, pinned):
    """idc_forward_host cuts batches >= 8 into image chunks (H2D / conv1_1 and last op / D2H overlap); the result
    must be bit-identical to the single-shot device-pointer path, for pinned and pageable caller memory."""
    L, ab, m = synth.synthetic_batch(n, 64, seed=3, max_hints=4)
    ctx = util.make_ctx(synth_sd, 64, 64, max_n=n)
    ref = ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5, want_rgb=True)
    ref_ab, ref_rgb = ref["ab"].cpu().numpy(), ref["rgb"].cpu().numpy()
    if pinned:
        L, ab, m = (torch.from_numpy(a).pin_memory().numpy() for a in (L, ab, m))
        out_ab = torch.empty((n, 2, 64, 64), dtype=torch.float32).pin_memory().numpy()
    else:
        out_ab = None
    for _ in range(2):                                  # second call re-uses streams / events
        r = ctx.forward_host(L, ab, m, 0.5, want_rgb=True, out_ab=out_ab)
        assert np.array_equal(r["ab"], ref_ab) and np.array_equal(r["rgb"], ref_rgb)
    assert ctx.last_launch_count() > 27                 # conv1_1 and the last op ran once per chunk
    ctx.close()


def test_headless_cli_writes_the_gui_result_folder(synth_sd, tmp_path):
    """ideepcolor_b200.py (row f4): hint list in, the reference GUI's save_result artefacts out."""
    import json
    import cv2
    import ideepcolor_b200
    g = util.golden("lhn_256.npz")
    img = tmp_path / "in.png"
    cv2.imwrite(str(img), np.ascontiguousarray(g["img_rgb"][:, :, ::-1]))
    wts = tmp_path / "w.pth"
    torch.save(synth_sd, str(wts))
    hints = tmp_path / "hints.json"
    hints.write_text(json.dumps([{"loc": [135, 160], "size": 3, "ab": [23, -69]}, {"loc": [100, 160], "rgb": [255, 255, 255]}]))
    out = tmp_path / "res"
    rc = ideepcolor_b200.main(["--image_file", str(img), "--color_model", str(wts), "--hints", str(hints),
                               "--out", str(out), "--suggest", "5"])
    assert rc == 0
    for f in ("im_l.npy", "im_ab.npy", "im_mask.npy", "input_mask.png", "ours.png", "ours_fullres.png",
              "input_fullres.png", "input.png", "input_ab.png", "suggestions.json"):
        assert (out / f).exists(), f
    ab = np.load(str(out / "im_ab.npy"))
    assert ab.shape == (2, 256, 256) and np.allclose(ab[:, 135, 160], [23, -69]) and np.abs(ab[:, 100, 160]).max() < 0.5
    ours = cv2.imread(str(out / "ours.png"))
    assert ours.shape == (256, 256, 3)
    sug = json.load(open(str(out / "suggestions.json")))
    assert len(sug) == 2 and np.array(sug[0]["ab"]).shape == (5, 2) and abs(sum(sug[0]["conf"]) - 1) < 1e-3
