"""GPU: the regression, distribution and global-hints heads of the default network against FP64 (tests/head_ref.py)
on the engine's own inputs, on every path that runs them.

One real forward per case; then each head's input is read back (a10_1, or conv10_2 where it is stored; conv8_3; a4_2)
and the head is evaluated in FP64 on exactly that readback, so the trunk's error stays out of the heads' bars:

  * regression head: the fused model_out of the wgmma c10_2 epilogue (halo and per-tap tiles, ragged tiles, the host
    pipe's image chunks with img0 > 0), out_head_kernel<true> (IDC_FLAG_KEEP_CONV10), out_head_kernel<false> (SIMT
    engine), tanh x 110 and x 100;
  * distribution head: class + softmax529_kernel on the side branch (n <= 4) and on the main stream (n > 4, SIMT), and
    the two other kernels that call softmax529_row: click_pmf_kernel (the click graph's clicked pixel) and
    reccs_query_pmf_kernel (ab_reccs_batch's out_pmf), each against the per-bin FP32 interval of head_ref.dist_head; a
    peaked class head (max |0.2 z| = 100) sends bins to 0 and into the subnormal range, where the zero sets, the
    subnormal rule and dist_negentropy's NaN pixels must follow the interval;
  * global hints: conv4_3 of a forward with a glob vector against FP64 c4_3 + the FP64 vector (the per-op bar), and,
    isolating the MLP, conv4_3 minus conv4_3 of run_op("c4_3") straight after (same a4_2, no vector) against the FP64
    vector, per element; the batches mix the four GLOBAL_CONDITIONS (a zero row, hist only, sat only, full rows).

Every case prints the worst measured fraction of each bar and where it sits."""
import time

import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import photos
from oracle import caffe_spec
from tests import calibrated, gpu_cases, head_ref, op_ref, util

pytestmark = pytest.mark.gpu
TOL_AB = 1e-3        # BASELINE.json north_star: ab within 1e-3 max-abs, end to end
TOL_DIST = 1e-5      # the end-to-end pmf bar of the other tests, absolute


@pytest.fixture(scope="module")
def nets(synth_sd):
    rho = calibrated.trained_like(synth_sd, 0.3, gpu_cases.calibration_batch())
    gsd = {k: torch.from_numpy(v) for k, v in caffe_spec.synthetic_glob_state_dict().items()}
    peak = util.small_batch(2, 64, seed=300)
    out = {"synth": synth_sd, "rho0.3": rho, "peak": head_ref.peaked(rho, peak, 100.0),
           "peak_synth": head_ref.peaked(synth_sd, peak, 100.0)}
    out.update({k + "+glob": dict(v, **gsd) for k, v in list(out.items())})
    return out, gsd


def _batch(H, W, n, seed=300):
    X = max(H, W, 32)
    return tuple(np.ascontiguousarray(a[:, :, :H, :W]) for a in util.small_batch(n, X, seed=seed))


def _glob_rows(n):
    """n glob inputs cycling through the four GLOBAL_CONDITIONS of two real global_stats rows (images of 16 flat
    colour blocks): a zero row, sat only, hist only and the full row."""
    pts = util.golden("pts_in_hull.npy")
    rs = np.random.RandomState(5)
    rows = [caffe_spec.global_stats(np.kron(rs.randint(0, 256, (4, 4, 3)), np.ones((16, 16, 1))).astype(np.uint8), pts)
            for _ in range(2)]
    conds = photos.GLOBAL_CONDITIONS
    return np.stack([photos.glob_vector(rows[(i // 4) % 2], conds[i % 4]) for i in range(n)]).astype(np.float32)


def _forward(ctx, batch, glob, path):
    """One forward -> (ab, dist) numpy; path "device" (forward_device) or "host" (forward_host)."""
    if path == "device":
        r = ctx.forward_device(*(util.dev(a) for a in batch), 0.5, glob=None if glob is None else util.dev(glob),
                               want_dist=True)
        torch.cuda.synchronize()
        return r["ab"].cpu().numpy(), r["dist"].cpu().numpy()
    r = ctx.forward_host(*batch, 0.5, glob=glob, want_dist=True)
    return r["ab"].copy(), r["dist"].copy()


def _worst(frac):
    i = int(np.argmax(frac))
    return float(frac.reshape(-1)[i]), tuple(int(k) for k in np.unravel_index(i, frac.shape))


def check_ab(tag, sd, ctx, ab, n, engine, keep, scale):
    """The regression head against FP64 on its own input; -> worst fraction of the bar."""
    if engine == "wgmma" and not keep:
        ref, bound = head_ref.reg_from_a10_1(sd, ctx.get_activation("a10_1", n).cpu(), scale)
        kind = "fused c10_2 + model_out on a10_1"
    else:
        ref, bound = head_ref.reg_from_conv10(sd, ctx.get_activation("conv10_2", n).cpu(), scale)
        kind = "out_head_kernel on conv10_2"
    err = np.abs(ab.astype(np.float64) - ref.numpy())
    frac, where = _worst(err / bound.numpy())
    print("%s: ab (%s) vs FP64: worst %.3f of the bar at (n, c, y, x) = %s, max|err| %.2e; bar max %.2e = %.3f TOL_AB, "
          "median %.2e" % (tag, kind, frac, where, float(err.max()), float(bound.max()), float(bound.max()) / TOL_AB,
                           float(bound.median())))
    assert ab.shape == tuple(ref.shape) and frac <= 1.0, (tag, frac, where)
    return frac


def check_dist(tag, p, ref, what="dist"):
    """A pmf p [n,529,h,w] (or [Q,529] as [Q,529,1,1]) against head_ref.dist_head's ref at the same pixels."""
    r = head_ref.dist_check(p, ref)
    normal = ref["p64"] >= head_ref.FLT_MIN
    lp = torch.log(torch.as_tensor(p, dtype=torch.float64).clamp(min=1e-300))
    lfrac = ((lp - torch.log(ref["p64"])).abs() / ref["logbound"])[normal]
    # the logit term of the bar against TOL_DIST relative to the bin (TOL_DIST / p64 is the relative error it allows)
    rel = (ref["logbound"] * ref["p64"] / TOL_DIST)[normal]
    # what the logit term of the bar had to cover, in units of C_CLS
    lt = ref["logit_term"][normal]
    need = float((((lp - torch.log(ref["p64"])).abs()[normal] - (ref["logbound"][normal] - lt)).clamp(min=0) / lt).max())
    print("%s: %s vs FP64: worst %.3f of the interval at (n, bin, y4, x4) = %s (log space: %.3f of the bound), %d bins "
          "outside; max|sum-1| %.2e (bound %.2e); bar / (TOL_DIST / bin) max %.3f; %d bins 0 (%d must, %d may), %d "
          "subnormal; the logits needed %.3f of C_CLS"
          % (tag, what, r["frac"], r["where"], float(lfrac.max()), r["bad"], r["sum_err"], ref["sum_bound"],
             float(rel.max()), int(r["zero_got"].sum()), int(r["zero_must"].sum()), int(r["zero_may"].sum()),
             int(r["sub"].sum()), need))
    assert r["bad"] == 0 and r["frac"] <= 1.0, (tag, what, r["frac"], r["where"])
    assert r["sum_err"] <= ref["sum_bound"], (tag, what, r["sum_err"])
    return r


def check_glob(tag, sd, gsd, ctx, glob, n, engine):
    """(a) conv4_3 against FP64 c4_3 + the FP64 vector, per-op bar; (b) conv4_3 - conv4_3 of run_op("c4_3") (no
    vector) against the vector, per element."""
    vec, dvec = head_ref.glob_vector(gsd, glob)
    a42 = ctx.get_activation("a4_2", n).cpu()
    got = ctx.get_activation("conv4_3", n).cpu().double()
    want, _ = head_ref.c4_3_glob(sd, a42, vec)
    err_a, top = float((got - want).abs().max()), float(want.abs().max())
    ctx.run_op("c4_3", n)
    torch.cuda.synchronize()
    plain = ctx.get_activation("conv4_3", n).cpu().double()
    S = ctx.act_exponent("conv4_3") if engine == "wgmma" else None
    bar = head_ref.glob_diff_bound(sd, got, plain, vec, dvec, S)
    d = ((got - plain) - vec[:, :, None, None]).abs()
    frac, where = _worst((d / bar).numpy())
    print("%s: conv4_3 vs FP64 c4_3 + vector %.2e (bar %.2e, %.3f of it); conv4_3 - run_op(c4_3) vs the vector: worst "
          "%.3f of the bar at (n, c, y, x) = %s, max|err| %.2e, vector MLP bound max %.2e, |vector| max %.2f"
          % (tag, err_a, 2e-5 * max(1.0, top), err_a / (2e-5 * max(1.0, top)), frac, where, float(d.max()),
             float(dvec.max()), float(vec.abs().max())))
    assert err_a <= 2e-5 * max(1.0, top), (tag, err_a, top)
    assert frac <= 1.0, (tag, frac, where)


# name -> (engine, (H, W, n, max_n), network, path, extra): an explicit list
CASES = {
    "wgmma_64_n3": ("wgmma", (64, 64, 3, 3), "synth", "device", {}),             # dist on the side branch, no halo
    "wgmma_256": ("wgmma", (256, 256, 1, 1), "synth", "device", {}),             # halo c10_2 with the fused head
    "wgmma_72x88_n2": ("wgmma", (72, 88, 2, 2), "rho0.3", "device", {}),         # ragged tiles
    "wgmma_40x200": ("wgmma", (40, 200, 1, 1), "synth", "device", {}),
    "wgmma_200x40": ("wgmma", (200, 40, 1, 1), "rho0.3", "device", {}),
    "wgmma_8": ("wgmma", (8, 8, 1, 1), "synth", "device", {}),                   # one softmax CTA, 4 of its 32 pixels
    "wgmma_128x64_n3of4": ("wgmma", (128, 64, 3, 4), "rho0.3", "device", {}),    # n below max_n
    "wgmma_64_n6of8_glob": ("wgmma", (64, 64, 6, 8), "synth", "device", {"glob": True}),   # class on the main stream
    # 256 tiles of c4_3 on 132 persistent CTAs: a CTA's second tile has the same n-tile in another image
    "wgmma_256_n8_glob": ("wgmma", (256, 256, 8, 8), "synth", "device", {"glob": True, "glob_only": True}),
    "wgmma_host_n9_glob": ("wgmma", (64, 64, 9, 9), "synth", "host", {"glob": True}),      # host pipe: 2 image chunks
    "wgmma_keep10_64_n3": ("wgmma", (64, 64, 3, 3), "rho0.3", "device", {"keep": True}),
    "wgmma_tanh100_64_n3": ("wgmma", (64, 64, 3, 3), "rho0.3", "device", {"scale": 100}),
    "simt_64_n3": ("simt", (64, 64, 3, 3), "synth", "device", {}),
    "simt_72x88_n2": ("simt", (72, 88, 2, 2), "rho0.3", "device", {}),
    "simt_64_n4_glob": ("simt", (64, 64, 4, 4), "rho0.3", "device", {"glob": True}),
    "simt_tanh100_64_n3": ("simt", (64, 64, 3, 3), "rho0.3", "device", {"scale": 100}),
    "wgmma_peak_64_n3": ("wgmma", (64, 64, 3, 3), "peak", "host", {}),
    "simt_peak_64_n3": ("simt", (64, 64, 3, 3), "peak", "host", {}),
    "wgmma_peak_synth_64_n3": ("wgmma", (64, 64, 3, 3), "peak_synth", "host", {}),     # pixels with and without a 0 bin
}


@pytest.mark.parametrize("name", list(CASES))
def test_heads_against_fp64(nets, name):
    t0 = time.time()
    engine, (H, W, n, max_n), net, path, extra = CASES[name]
    allnets, gsd = nets
    glob = _glob_rows(n) if extra.get("glob") else None
    sd = allnets[net + ("+glob" if glob is not None else "")]
    keep, scale = bool(extra.get("keep")), float(extra.get("scale", 110))
    ctx = util.make_ctx(sd, H, W, max_n=max_n, dist=True, engine=engine, global_hints=glob is not None,
                        keep_conv10=keep, options={"tanh_scale": int(scale)} if scale != 110 else None)
    try:
        batch = _batch(H, W, n)
        chunked = path == "host" and n >= 8
        if chunked:
            ab_dev, _ = _forward(ctx, batch, glob, "device")
            dev_launches = ctx.last_launch_count()
        ab, dist = _forward(ctx, batch, glob, path)
        if chunked:
            # forward_host's pipe cut the batch into 2 image chunks: conv1_1 and the fused c10_2 (img0 = 0, then img0 > 0)
            # ran once per chunk, one launch more each than the single-shot device forward, with the same results
            print("%s: %d launches, %d on the device path" % (name, ctx.last_launch_count(), dev_launches))
            assert ctx.last_launch_count() == dev_launches + 2, (ctx.last_launch_count(), dev_launches)
            assert np.array_equal(ab, ab_dev)
        if extra.get("glob_only"):
            check_glob(name, sd, gsd, ctx, glob, n, engine)
            return
        check_ab(name, sd, ctx, ab, n, engine, keep, scale)
        ref = head_ref.dist_head(sd, ctx.get_activation("conv8_3", n).cpu(), engine)
        r = check_dist(name, dist, ref)
        if keep:
            # c10_2's own accumulation on the stored conv10_2: the constant C10 of head_ref
            v, mag = op_ref.run_op("c10_2", sd, {"a10_1": ctx.get_activation("a10_1", n).cpu().double()})
            got = ctx.get_activation("conv10_2", n).cpu().double()
            st = 2.0 ** -22 * v.abs() + 2.0 ** (-25 - ctx.act_exponent("conv10_2"))
            need = float(((got - v).abs() - st).clamp(min=0).div(head_ref.U * mag.clamp(min=1e-300)).max())
            print("%s: c10_2 accumulation needs C10 >= %.2f (head_ref.C10 = %g)" % (name, need, head_ref.C10))
            assert need <= head_ref.C10
        if net.startswith("peak"):
            # zero bins: every bin that must be 0 is, every bin that is 0 may be; NaN entropy exactly where a bin is 0
            assert bool((r["zero_must"] <= r["zero_got"]).all()) and bool((r["zero_got"] <= r["zero_may"]).all())
            assert int(r["zero_must"].sum()) > 0 and int(r["sub"].sum()) > 0, name
            for i in range(n):
                neg = ctx.dist_negentropy(i)
                must = r["zero_must"][i].any(dim=0).numpy()
                may = r["zero_may"][i].any(dim=0).numpy()
                nan = np.isnan(neg)
                assert np.array_equal(nan, r["zero_got"][i].any(dim=0).numpy()), (name, i)
                assert not np.any(must & ~nan) and not np.any(nan & ~may), (name, i)
                print("%s: image %d: dist_negentropy NaN at %d pixels (%d must, %d may)"
                      % (name, i, int(nan.sum()), int(must.sum()), int(may.sum())))
        if glob is not None:
            check_glob(name, sd, gsd, ctx, glob, n, engine)
    finally:
        ctx.close()
    print("%s: %.1f s" % (name, time.time() - t0))


def test_click_graph_256(nets):
    """The click graph at 256^2, n = 1: the whole resident plane (fetch_dist), the clicked pixel's pmf from the click
    tail (click_pmf_kernel) and every pixel's pmf through ab_reccs_batch(out_pmf=...) (reccs_query_pmf_kernel), each
    against the FP64 interval; the fused head's ab as well.

    The C ABI does not say whether fetch_dist(0, y4, x4) was answered from the click tail's block or from the resident
    plane: the launch count shows that the forward ran the click tail (click_pmf_kernel, the k-means and the restart
    pick, three launches more than the same forward without an announced click), and test_gpu_click pins the answered
    pixel to the device path bit for bit."""
    sd = nets[0]["synth"]
    y4, x4 = 37, 21
    ctx = util.make_ctx(sd, 256, 256, max_n=1, dist=True)
    try:
        ctx.set_dist_resident(True)
        batch = _batch(256, 256, 1)
        ctx.set_click(0, -1, 0, 0)
        ctx.forward_host(*batch, 0.5)
        plain = ctx.last_launch_count()
        ctx.set_click(0, y4, x4, K=9)
        ab = ctx.forward_host(*batch, 0.5)["ab"].copy()
        print("click_256: %d launches with the announced click, %d without" % (ctx.last_launch_count(), plain))
        assert ctx.last_launch_count() == plain + 3
        check_ab("click_256", sd, ctx, ab, 1, "wgmma", False, 110.0)
        ref = head_ref.dist_head(sd, ctx.get_activation("conv8_3", 1).cpu())
        check_dist("click_256", ctx.fetch_dist(0)[None], ref, "fetch_dist plane")
        px = {k: v[:, :, y4:y4 + 1, x4:x4 + 1] for k, v in ref.items() if torch.is_tensor(v)}
        px["sum_bound"] = ref["sum_bound"]
        check_dist("click_256", ctx.fetch_dist(0, y4, x4)[None, :, None, None], px, "clicked pixel (click tail)")
        yy, xx = np.meshgrid(np.arange(64), np.arange(64), indexing="ij")
        q = np.stack([np.zeros(64 * 64, np.int64), yy.reshape(-1), xx.reshape(-1)], axis=1)
        pmf = torch.empty((q.shape[0], 529), dtype=torch.float32, device="cuda")
        ctx.ab_reccs_batch(q, K=1, max_iter=1, n_init=1, out_pmf=pmf)
        torch.cuda.synchronize()
        rows = pmf.cpu().numpy().reshape(64, 64, 529).transpose(2, 0, 1)[None]
        check_dist("click_256", rows, ref, "ab_reccs_batch out_pmf")
    finally:
        ctx.close()


# Plan options.  Reading umma_plan_op: pdl and side_dist change only when kernels start; mt = 1 is the automatic plan
# at these geometries (no launch reaches the 2 x 132 tiles that mt = 2 needs), so all three keep the arithmetic and its
# order: bit-identical.  pairs = 2 and mt = 2 turn split-K off where the automatic plan splits (every launch below half
# the machine), halo = 3 does too and reorders the k-blocks (input group outer, tap inner), and halo = 0 reorders them
# where the automatic plan uses halo tiles (c10_2 at 256^2: 512 tiles); at 64^2 no launch reaches the halo threshold, so
# halo = 0 is the automatic plan there.  Those only have to meet the FP64 bars.
OPTIONS = {"pairs2": {"pairs": 2}, "halo0": {"halo": 0}, "halo3": {"halo": 3}, "mt1": {"mt": 1}, "mt2": {"mt": 2},
           "side_dist0": {"side_dist": 0}, "pdl0": {"pdl": 0}}
SAME_ORDER = {(64, 64, 3, 3): ("mt1", "side_dist0", "pdl0", "halo0"), (256, 256, 1, 1): ("mt1", "side_dist0", "pdl0")}


@pytest.mark.parametrize("geom", list(SAME_ORDER), ids=lambda g: "%dx%d_n%d" % g[:3])
def test_plan_options(nets, geom):
    sd = nets[0]["synth"]
    H, W, n, max_n = geom
    batch = _batch(H, W, n)
    outs = {}
    for name in ["auto"] + list(OPTIONS):
        ctx = util.make_ctx(sd, H, W, max_n=max_n, dist=True, options=OPTIONS.get(name), use_graph=False)
        try:
            ab, dist = _forward(ctx, batch, None, "device")
            tag = "%dx%d_n%d %s" % (H, W, n, name)
            check_ab(tag, sd, ctx, ab, n, "wgmma", False, 110.0)
            check_dist(tag, dist, head_ref.dist_head(sd, ctx.get_activation("conv8_3", n).cpu()))
            outs[name] = (ab, dist, ctx.get_activation("conv4_3", n).cpu().numpy())
        finally:
            ctx.close()
    for name in OPTIONS:
        same = all(np.array_equal(a, b) for a, b in zip(outs[name], outs["auto"]))
        print("%dx%d_n%d %s: %s the automatic plan" % (H, W, n, name, "bit-identical to" if same else "differs from"))
        if name in SAME_ORDER[geom]:
            assert same, name
