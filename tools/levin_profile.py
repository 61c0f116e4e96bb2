"""The Levin baseline of reveal sweeps on seeded 500 x 375 photos: photos/s of reveal_sweep(method="levin") and of the
network sweep in the same run, the solver's iteration counts per level (median and maximum over photos and the two ab
channels), and, in a separate torch.profiler run, the device time of one baseline sweep split by kernel.

    python tools/levin_profile.py --out DIR [--Xd 256] [--batch 60] [--photos 24] [--max_iter 200000]

The baseline runs with the default tolerance and a generous iteration budget (--max_iter), so that the counts it reports
are the ones the solver needed, not a cap.  Host wall time of each leg ends in a device synchronise and follows one
untimed warm-up pass over the same photos.  The card's name and power limit are read in the same run and written with
the numbers to DIR/levin_profile.json.
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from reveal_sweep_profile import card, photo, timed  # noqa: E402

STEPS = [("prep", "photo_prep_kernel"), ("lab", "rgb2lab_kernel"), ("fill", "hint_fill_mean_kernel"),
         ("raster", "hint_raster_kernel"), ("weights", "levin_weights_kernel"), ("solve", "levin_solve_kernel"),
         ("render", "lab2rgb_kernel"), ("sse", "rgb_sse_kernel")]


def device_split(run):
    """torch.profiler over run(): device microseconds per step of STEPS and the rest."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    split = {k: 0.0 for k, _ in STEPS}
    split["other"] = 0.0
    for e in prof.key_averages():
        if e.device_type != DeviceType.CUDA:
            continue
        us = float(e.self_device_time_total)
        if us > 0:
            split[next((k for k, pat in STEPS if pat in e.key), "other")] += us
    return split


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--Xd", type=int, default=256)
    ap.add_argument("--batch", type=int, default=60)
    ap.add_argument("--photos", type=int, default=24)
    ap.add_argument("--max_iter", type=int, default=200000)
    args = ap.parse_args(argv)
    import torch
    from interactive_deep_colorization_b200.photos import LEVIN_MAX_ITER, LEVIN_TOL, REVEAL_LEVELS, PhotoColorizer
    from oracle import synth
    os.makedirs(args.out, exist_ok=True)
    if not torch.cuda.is_available():
        raise SystemExit("levin_profile needs a GPU")
    X, levels = args.Xd, REVEAL_LEVELS
    name, power = card()
    imgs = [photo(s) for s in range(args.photos)]
    pc = PhotoColorizer(synth.torch_state_dict(1234), Xd=X, batch=args.batch, maskcent=True)

    def levin():
        return list(pc.reveal_sweep(imgs, levels=levels, method="levin", levin_max_iter=args.max_iter))

    pc._backend.levin_log = []
    t_levin, res = timed(levin)
    iters = np.stack(pc._backend.levin_log[-args.photos:])          # [photos, levels, 2] of the timed run
    pc._backend.levin_log = None
    t_net, net = timed(lambda: list(pc.reveal_sweep(imgs, levels=levels)))
    per_level = {str(m): {"median": float(np.median(iters[:, j])), "max": int(iters[:, j].max())}
                 for j, m in enumerate(levels)}
    report = {"card": name, "power_limit,max_sm_clock": power, "Xd": X, "batch": args.batch, "levels": list(levels),
              "photos": args.photos, "photo_size": [375, 500], "tol": LEVIN_TOL, "max_iter_run": args.max_iter,
              "max_iter_default": LEVIN_MAX_ITER,
              "levin_photos_per_s": args.photos / t_levin, "network_photos_per_s": args.photos / t_net,
              "levin_wall_s": t_levin, "network_wall_s": t_net, "iterations_per_level": per_level,
              "max_iterations": int(iters.max()),
              "mean_psnr_levin": np.stack([r.psnr for r in res]).mean(axis=0).tolist(),
              "mean_psnr_network": np.stack([r.psnr for r in net]).mean(axis=0).tolist()}
    print(json.dumps(report), flush=True)
    split = device_split(levin)
    pc.close()
    total = sum(split.values())
    report["device_us_per_levin_sweep"] = split
    report["device_share"] = {k: v / total for k, v in split.items()} if total else {}
    with open(os.path.join(args.out, "levin_profile.json"), "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps({"device_us_per_levin_sweep": split, "device_share": report["device_share"], "card": name,
                      "power_limit,max_sm_clock": power}))


if __name__ == "__main__":
    main()
