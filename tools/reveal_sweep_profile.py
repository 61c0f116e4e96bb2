"""Photos/s of a reveal sweep (PSNR against the number of revealed hint points): PhotoColorizer.reveal_sweep against
the same sweep done through colorize(hints=...), with patch means computed on the host and every photo repeated once
per level; then, in a separate torch.profiler run, the device time of one sweep split by kernel.

    python tools/reveal_sweep_profile.py --out DIR [--Xd 256] [--batch 60] [--photos 120]

Host wall time of each leg ends in a device synchronise and follows one untimed warm-up pass over the same photos.  The
card's name, power limit and maximum SM clock are read in the same run and written with the numbers to
DIR/reveal_sweep_profile.json.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, W = 375, 500                       # an ImageNet-like photo
# device kernels by step of the sweep; everything else on the device is the forward (or a copy, listed apart)
STEPS = [("prep", "photo_prep_kernel"), ("lab", "rgb2lab_kernel"), ("fill", "hint_fill_mean_kernel"),
         ("raster", "hint_raster_kernel"), ("sse", "rgb_sse_kernel")]
COPIES = ("Memcpy", "Memset", "copy_kernel", "elementwise_kernel")


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the number is still reported, marked as unknown
        q = "unknown (%s)" % e
    return name, q


def photo(seed):
    import cv2
    rs = np.random.RandomState(seed)
    coarse = rs.randint(0, 256, (H // 24, W // 24, 3)).astype(np.uint8)
    img = cv2.resize(coarse, (W, H), interpolation=cv2.INTER_CUBIC).astype(np.int16)
    img += rs.randint(-12, 13, (H, W, 3)).astype(np.int16)
    return np.clip(img, 0, 255).astype(np.uint8)


def timed(fn):
    import torch
    fn()                                 # warm-up: pinned buffers, plans, reveal buffers
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def host_sweep(pc, imgs, levels, seed):
    """The sweep without reveal_sweep: net-size Lab and patch means on the host, one colorize() image per level."""
    import cv2
    from interactive_deep_colorization_b200 import color
    from interactive_deep_colorization_b200.colorize_image import HINT_LIST_DTYPE
    from interactive_deep_colorization_b200.photos import reveal_points
    X, M = pc.Xd, max(levels)
    rep, lists = [], []
    for i, a in enumerate(imgs):
        lab = color.rgb2lab(cv2.resize(a, (X, X))).transpose((2, 0, 1))
        pts = reveal_points(X, M, seed, i)
        h = np.zeros(M, HINT_LIST_DTYPE)
        for k, (y0, x0, P) in enumerate(pts):
            h[k] = (0, y0, x0, y0 + P - 1, x0 + P - 1, lab[1, y0:y0 + P, x0:x0 + P].mean(), lab[2, y0:y0 + P, x0:x0 + P].mean())
        for m in levels:
            rep.append(a)
            lists.append(h[:m])
    psnr = np.array([r.psnr for r in pc.colorize(rep, hints=lists, psnr=True)])
    return psnr.reshape(len(imgs), len(levels))


def device_split(pc, imgs, levels):
    """torch.profiler over one sweep: device microseconds per step, the forward, and copies."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in pc.reveal_sweep(imgs, levels=levels):
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
    ap.add_argument("--batch", type=int, default=60)
    ap.add_argument("--photos", type=int, default=120)
    args = ap.parse_args(argv)
    import torch
    from interactive_deep_colorization_b200.photos import REVEAL_LEVELS, PhotoColorizer
    from oracle import synth
    os.makedirs(args.out, exist_ok=True)
    if not torch.cuda.is_available():
        raise SystemExit("reveal_sweep_profile needs a GPU")
    X, levels = args.Xd, REVEAL_LEVELS
    sd = synth.torch_state_dict(1234)
    name, power = card()
    imgs = [photo(s) for s in range(args.photos)]
    pc = PhotoColorizer(sd, Xd=X, batch=args.batch, maskcent=True)
    t_sweep, res = timed(lambda: list(pc.reveal_sweep(imgs, levels=levels)))
    t_host, psnr_host = timed(lambda: host_sweep(pc, imgs, levels, 0))
    psnr = np.stack([r.psnr for r in res])
    from interactive_deep_colorization_b200.photos import reveal_points
    t0 = time.perf_counter()                # host share of the sweep: the points it draws
    for i in range(args.photos):
        reveal_points(X, max(levels), 0, i)
    t_points = time.perf_counter() - t0
    report = {"card": name, "power_limit,max_sm_clock": power, "Xd": X, "batch": args.batch, "levels": list(levels),
              "photos": args.photos, "photo_size": [H, W],
              "reveal_sweep_photos_per_s": args.photos / t_sweep,
              "colorize_per_level_photos_per_s": args.photos / t_host,
              "forward_images_per_s": args.photos * len(levels) / t_sweep,
              "sweep_wall_s": t_sweep, "host_reveal_points_s": t_points,
              "mean_psnr": psnr.mean(axis=0).tolist(),
              "max_abs_psnr_diff_vs_colorize": float(np.abs(psnr - psnr_host).max())}
    print(json.dumps(report), flush=True)
    split, kernels = device_split(pc, imgs, levels)
    pc.close()
    total = sum(split.values())
    report["device_us_per_sweep"] = split
    report["device_share"] = {k: v / total for k, v in split.items()} if total else {}
    report["kernels_us"] = kernels
    with open(os.path.join(args.out, "reveal_sweep_profile.json"), "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps({"device_us_per_sweep": split, "device_share": report["device_share"],
                      "card": name, "power_limit,max_sm_clock": power}))


if __name__ == "__main__":
    main()
