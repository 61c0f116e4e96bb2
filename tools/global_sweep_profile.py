"""Photos/s of a global-hints sweep (PSNR with no hints, the photo's own saturation, its own histogram, both):
PhotoColorizer.global_sweep against the same sweep done the way it can be done without it -- the statistics of each
photo by prepost.global_stats_gpu(cv2.resize(photo, (Xd, Xd))), one blocking call per photo, then colorize(glob=...)
with every photo repeated once per condition; then, in a separate torch.profiler run, the device time of one sweep
split by kernel.

    python tools/global_sweep_profile.py --out DIR [--Xd 256] [--batch 64] [--photos 128]

Seeded synthetic 500 x 375 photos, the synthetic network with synthetic global-hints weights.  Host wall time of each
leg ends in a device synchronise and follows one untimed warm-up pass over the same photos.  The card's name, power
limit and maximum SM clock are read in the same run and written with the numbers to DIR/global_sweep_profile.json.
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from reveal_sweep_profile import H, W, card, photo, timed  # noqa: E402

STEPS = [("prep", "photo_prep_kernel"), ("stats", "global_stats_batch_kernel"), ("raster", "hint_raster_kernel"),
         ("sse", "rgb_sse_kernel")]
COPIES = ("Memcpy", "Memset", "copy_kernel", "elementwise_kernel", "where_kernel")


def host_sweep(pc, imgs, conditions):
    """The sweep without global_sweep: per-photo statistics, one colorize() image per condition."""
    import cv2
    from interactive_deep_colorization_b200 import prepost
    from interactive_deep_colorization_b200.photos import glob_vector
    rep, globs = [], []
    for a in imgs:
        stats = prepost.global_stats_gpu(cv2.resize(a, (pc.Xd, pc.Xd)), pc.device)
        for c in conditions:
            rep.append(a)
            globs.append(glob_vector(stats, c))
    psnr = np.array([r.psnr for r in pc.colorize(rep, glob=globs, psnr=True)])
    return psnr.reshape(len(imgs), len(conditions))


def device_split(pc, imgs):
    """torch.profiler over one sweep: device microseconds per step, the forward, and copies."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in pc.global_sweep(imgs):
            pass
        torch.cuda.synchronize()
    split = {k: 0.0 for k, _ in STEPS}
    split.update(forward=0.0, copies=0.0)
    kernels = {}
    for e in prof.key_averages():
        if e.device_type != DeviceType.CUDA:      # the host ops that launched them carry the same time again
            continue
        us = float(e.self_device_time_total)
        if us <= 0:
            continue
        kernels[e.key] = us
        step = next((k for k, pat in STEPS if pat in e.key), None)
        if step is None:
            step = "copies" if any(c in e.key for c in COPIES) else "forward"
        split[step] += us
    return split, kernels


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--Xd", type=int, default=256)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--photos", type=int, default=128)
    args = ap.parse_args(argv)
    import torch
    from interactive_deep_colorization_b200.photos import GLOBAL_CONDITIONS, PhotoColorizer
    from oracle import caffe_spec, synth
    os.makedirs(args.out, exist_ok=True)
    if not torch.cuda.is_available():
        raise SystemExit("global_sweep_profile needs a GPU")
    X, conds = args.Xd, GLOBAL_CONDITIONS
    sd = synth.torch_state_dict(1234)
    sd.update({k: torch.from_numpy(v) for k, v in caffe_spec.synthetic_glob_state_dict().items()})
    name, power = card()
    imgs = [photo(s) for s in range(args.photos)]
    pc = PhotoColorizer(sd, Xd=X, batch=args.batch, global_hints=True)
    t_sweep, res = timed(lambda: list(pc.global_sweep(imgs)))
    t_host, psnr_host = timed(lambda: host_sweep(pc, imgs, conds))
    psnr = np.stack([r.psnr for r in res])
    report = {"card": name, "power_limit,max_sm_clock": power, "Xd": X, "batch": args.batch, "conditions": list(conds),
              "photos": args.photos, "photo_size": [H, W],
              "global_sweep_photos_per_s": args.photos / t_sweep,
              "stats_then_colorize_photos_per_s": args.photos / t_host,
              "forward_images_per_s": args.photos * len(conds) / t_sweep,
              "sweep_wall_s": t_sweep, "stats_then_colorize_wall_s": t_host,
              "mean_psnr": psnr.mean(axis=0).tolist(),
              "max_abs_psnr_diff_vs_colorize": float(np.abs(psnr - psnr_host).max())}
    print(json.dumps(report), flush=True)
    split, kernels = device_split(pc, imgs)
    pc.close()
    total = sum(split.values())
    report["device_us_per_sweep"] = split
    report["device_share"] = {k: v / total for k, v in split.items()} if total else {}
    report["kernels_us"] = kernels
    with open(os.path.join(args.out, "global_sweep_profile.json"), "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps({"device_us_per_sweep": split, "device_share": report["device_share"],
                      "card": name, "power_limit,max_sm_clock": power}))


if __name__ == "__main__":
    main()
