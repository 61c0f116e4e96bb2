"""Photos/s and suggestions/s of batched colour suggestions: PhotoColorizer(suggest=True).suggest against the
single-image wrapper loop on the same photos and hints -- per photo ColorizeImageB200.load_image + net_forward_hints +
get_img_fullres, then ColorizeImageB200Dist (share_trunk) net_forward_hints + one get_ab_reccs(h, w, K,
return_conf=True) per hint; then, in separate torch.profiler runs, the device time of one batched pass split by kernel
and the device time of the single-pixel k-means kernel against the host wall time of one get_ab_reccs call.

    python tools/suggest_batch_profile.py --out DIR [--Xd 256] [--batch 32] [--photos 96] [--K 9] [--caffe_dist]

--caffe_dist measures the Caffe pair instead, on a Caffe-scaled checkpoint that also holds the synthetic 313-bin head:
PhotoColorizer(caffe=True, caffe_dist=True).suggest against, per photo, ColorizeImageB200Caffe.load_image + net_forward
+ get_img_fullres, then ColorizeImageB200CaffeDist.load_image + net_forward + one get_ab_reccs per hint (both wrappers
fed the dense hint planes), and writes DIR/suggest_batch_profile_caffe_dist.json.

Seeded synthetic 500 x 375 photos written as PNG files (both legs read and decode them), 10 to 20 hints each
(put_point patches of 1 to 7 pixels, colours drawn uniformly), the suggestions asked at every hint's loc; the
synthetic network.  Host wall time of each leg ends in a device synchronise and follows one untimed warm-up pass over
the same photos.  The card's name, power limit and maximum SM clock are read in the same run and written with the
numbers to DIR/suggest_batch_profile.json.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from reveal_sweep_profile import H, W, card, photo, timed  # noqa: E402

STEPS = [("prep", "photo_prep_kernel"), ("raster", "hint_raster_kernel"), ("query_pmf", "query_pmf_kernel"),
         ("kmeans", "ab_reccs_kernel"), ("pick", "reccs_pick_kernel"), ("rgb2lab", "rgb2lab_kernel"),
         ("render", "photo_render_kernel")]
COPIES = ("Memcpy", "Memset", "copy_kernel", "elementwise_kernel")


def make_hints(X, n, seed):
    """Per photo: the hint list (hints_from_points) and the int [P,2] locs the suggestions are asked at."""
    from interactive_deep_colorization_b200 import colorize_image as CI
    rs = np.random.RandomState(seed)
    rects, locs = [], []
    for _ in range(n):
        k = int(rs.randint(10, 21))
        loc = rs.randint(0, X, (k, 2))
        rects.append(CI.hints_from_points([(l, int(rs.randint(0, 4)), rs.uniform(-80, 80, 2)) for l in loc], X))
        locs.append(loc.astype(np.int64))
    return rects, locs


def wrapper_loop(cm, dm, paths, rects, locs, K, reccs_s=None):
    out = []
    for p, r, loc in zip(paths, rects, locs):
        cm.load_image(p)
        cm.net_forward_hints(r)
        cm.get_img_fullres()
        dm.set_image(cm.img_rgb)
        dm.net_forward_hints(r)
        t0 = time.perf_counter()
        out.append([dm.get_ab_reccs(int(h), int(w), K=K, return_conf=True) for h, w in loc])
        if reccs_s is not None:
            reccs_s.append((time.perf_counter() - t0) / max(len(loc), 1))
    return out


def caffe_wrapper_loop(cm, dm, paths, rects, locs, K, reccs_s=None):
    """The single-image Caffe pair per photo: colour model + get_img_fullres, distribution model + get_ab_reccs."""
    from interactive_deep_colorization_b200 import colorize_image as CI
    out = []
    for p, r, loc in zip(paths, rects, locs):
        ab, m = CI.raster_hints(r, cm.Xd)
        cm.load_image(p)
        cm.net_forward(ab, m)
        cm.get_img_fullres()
        dm.load_image(p)
        dm.net_forward(ab, m)
        t0 = time.perf_counter()
        out.append([dm.get_ab_reccs(int(h), int(w), K=K, return_conf=True) for h, w in loc])
        if reccs_s is not None:
            reccs_s.append((time.perf_counter() - t0) / max(len(loc), 1))
    return out


def caffe_checkpoint(sd):
    """The synthetic network as a Caffe-scaled checkpoint with the synthetic 313-bin head."""
    import torch
    from interactive_deep_colorization_b200 import prepost
    from oracle import caffe_spec
    from tests import util
    out = util.caffe_scaled(sd)
    out.update({k: torch.from_numpy(v) for k, v in
                caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=prepost.pts_in_hull()).items()})
    return out


def device_split(fn):
    """torch.profiler over fn(): device microseconds per step, the forward, and copies."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {k: 0.0 for k, _ in STEPS}
    split.update(forward=0.0, copies=0.0)
    kernels = {}
    for e in prof.key_averages():
        if e.device_type != DeviceType.CUDA:
            continue
        us = float(e.self_device_time_total)
        if us <= 0:
            continue
        kernels[e.key] = {"us": us, "count": int(e.count)}
        step = next((k for k, pat in STEPS if pat in e.key), None)
        if step is None:
            step = "copies" if any(c in e.key for c in COPIES) else "forward"
        split[step] += us
    return split, kernels


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--Xd", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--photos", type=int, default=96)
    ap.add_argument("--K", type=int, default=9)
    ap.add_argument("--caffe_dist", action="store_true", help="the Caffe pair and its 313-bin head")
    args = ap.parse_args(argv)
    import cv2
    import torch
    from interactive_deep_colorization_b200 import colorize_image as CI
    from interactive_deep_colorization_b200.photos import PhotoColorizer
    from oracle import synth
    if not torch.cuda.is_available():
        raise SystemExit("suggest_batch_profile needs a GPU")
    X, K = args.Xd, args.K
    os.makedirs(args.out, exist_ok=True)
    tmp = tempfile.TemporaryDirectory()                    # the PNG files stay out of the result folder
    pdir = tmp.name
    paths = []
    for s in range(args.photos):
        p = os.path.join(pdir, "p%03d.png" % s)
        cv2.imwrite(p, photo(s)[:, :, ::-1])
        paths.append(p)
    rects, locs = make_hints(X, args.photos, 1)
    n_sugg = int(sum(len(l) for l in locs))
    sd = synth.torch_state_dict(1234)
    name, power = card()
    if args.caffe_dist:
        sd = caffe_checkpoint(sd)
        pc = PhotoColorizer(sd, Xd=X, batch=args.batch, caffe=True, caffe_dist=True)
        cm = CI.ColorizeImageB200Caffe(Xd=X)
        cm.prep_net(state_dict=sd)
        dm = CI.ColorizeImageB200CaffeDist(Xd=X)
        dm.prep_net(state_dict=sd)
        loop = caffe_wrapper_loop
    else:
        pc = PhotoColorizer(sd, Xd=X, batch=args.batch, suggest=True)
        cm = CI.ColorizeImageB200(Xd=X)
        cm.prep_net(state_dict=sd, dist=True)
        dm = CI.ColorizeImageB200Dist(Xd=X).share_trunk(cm)
        loop = wrapper_loop
    t_batch, res = timed(lambda: list(pc.suggest(paths, rects, locs, K=K)))
    reccs_s = []
    t_wrap, wres = timed(lambda: loop(cm, dm, paths, rects, locs, K, reccs_s))
    reccs_s = reccs_s[len(reccs_s) // 2:]                   # the timed pass, not the warm-up
    d_cen = max(float(np.abs(r.centers - np.array([c for c, _ in w])).max()) for r, w in zip(res, wres))
    d_conf = max(float(np.abs(r.conf - np.array([f for _, f in w])).max()) for r, w in zip(res, wres))
    report = {"card": name, "power_limit,max_sm_clock": power, "head": "caffe313" if args.caffe_dist else "dist529",
              "Xd": X, "batch": args.batch, "K": K,
              "photos": args.photos, "photo_size": [H, W], "suggestions": n_sugg,
              "suggest_photos_per_s": args.photos / t_batch, "suggest_suggestions_per_s": n_sugg / t_batch,
              "wrapper_photos_per_s": args.photos / t_wrap, "wrapper_suggestions_per_s": n_sugg / t_wrap,
              "suggest_wall_s": t_batch, "wrapper_wall_s": t_wrap,
              "wrapper_get_ab_reccs_wall_ms_per_call": 1e3 * float(np.mean(reccs_s)),
              "max_abs_center_diff_vs_wrapper": d_cen, "max_abs_conf_diff_vs_wrapper": d_conf}
    print(json.dumps(report), flush=True)
    split, kernels = device_split(lambda: list(pc.suggest(paths, rects, locs, K=K)))
    pc.close()
    total = sum(split.values())
    report["device_us_per_pass"] = split
    report["device_share"] = {k: v / total for k, v in split.items()} if total else {}
    report["kernels_us"] = kernels
    # four photos' get_ab_reccs calls: the device time of the single-pixel k-means against the host wall time per call
    _, wk = device_split(lambda: loop(cm, dm, paths[:4], rects[:4], locs[:4], K))
    calls = int(sum(len(l) for l in locs[:4]))
    km = sum(v["us"] for k, v in wk.items() if "ab_reccs_kernel" in k)
    report["wrapper_ab_reccs_kernel_device_ms_per_call"] = km / 1e3 / calls
    fname = "suggest_batch_profile_caffe_dist.json" if args.caffe_dist else "suggest_batch_profile.json"
    with open(os.path.join(args.out, fname), "w") as f:
        json.dump(report, f, indent=1)
    tmp.cleanup()
    print(json.dumps({k: report[k] for k in ("device_us_per_pass", "device_share",
                                              "wrapper_ab_reccs_kernel_device_ms_per_call",
                                              "wrapper_get_ab_reccs_wall_ms_per_call", "card", "power_limit,max_sm_clock")}))


if __name__ == "__main__":
    main()
