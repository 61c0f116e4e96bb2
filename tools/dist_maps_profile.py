"""Cost of the whole-map distribution reads, before and after the device-side map and entropy kernels (writes JSON).

At Xd = 64, 256 and 512 (n = 1, seeded synthetic weights: oracle/synth + oracle/caffe_spec) it measures
  * host wall time, ending in a device synchronise, of
      - the per-pixel loop over caffe313_dist_pixel that built the 313-bin map before (`old_map_loop_s`),
      - np.asarray(dist_ab) of ColorizeImageB200CaffeDist now (one idc_caffe313_dist_map + one copy, `new_map_s`),
      - compute_entropy of both models before (the numpy statement on the host map; for the Caffe model after the
        per-pixel loop, for the PyTorch model after fetch_dist(0) and the x4 repeat) and now (`*_entropy_*_s`),
  * CUDA-event kernel times, mean over --launches warmed launches, of dist313_map_kernel and negentropy_kernel, with
    the bytes each must move and that over the time, next to the H100 SXM data sheet's 3.35 TB/s,
  * the card's name and power limit, read in the same run.

    python tools/dist_maps_profile.py --out DIR [--sizes 64,256,512] [--launches 50] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from interactive_deep_colorization_b200 import _lib, prepost  # noqa: E402
from interactive_deep_colorization_b200 import colorize_image as CI  # noqa: E402
from oracle import caffe_spec, synth  # noqa: E402

HBM_BPS = 3.35e12       # H100 SXM data sheet


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = [s.strip() for s in q.split(",")]
        return name, plim
    except Exception as e:                                     # the numbers stay valid; the label is then unknown
        return "unknown (%s)" % e, "unknown"


def wall(fn, reps):
    """median host seconds of fn() followed by a device synchronise (one untimed warm-up call first)."""
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def kernel_ms(launch, launches):
    for _ in range(5):
        rc = launch()
        if rc != _lib.IDC_OK:
            raise _lib.IdcError(rc, "kernel launch failed")
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        launch()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / launches


def old_map_loop(ctx, X, S):
    """The body _LazyDist313.__array__ had: one caffe313_dist_pixel call per pixel, then np.stack."""
    return np.stack([np.stack([ctx.caffe313_dist_pixel(0, y, x, S) for x in range(X)], -1) for y in range(X)], -2)


def np_negentropy(d):
    return np.sum(d * np.log(d), axis=0)


def caffe_model(X, sd313):
    cd = CI.ColorizeImageB200CaffeDist(Xd=X)
    cd.prep_net(0, state_dict=sd313)
    cd.set_image((np.random.RandomState(X).rand(X, X, 3) * 255).astype(np.uint8))
    ab, mask = synth.synthetic_hints(X, 5, 1)
    cd.net_forward(ab, mask)
    return cd


def dist_model(X, sd):
    dm = CI.ColorizeImageB200Dist(Xd=X, maskcent=True)
    dm.prep_net(state_dict=sd)
    dm.set_image((np.random.RandomState(X + 1).rand(X, X, 3) * 255).astype(np.uint8))
    ab, mask = synth.synthetic_hints(X, 5, 2)
    dm.net_forward(ab, mask)
    return dm


def one_size(X, sd, sd313, reps, launches):
    lib = _lib.load()
    res = {"Xd": X}
    cd = caffe_model(X, sd313)
    ctx, S = cd._ctx, cd.S
    # before: per-pixel map (timed once: seconds at 256^2 and up), then the numpy statement on it
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    d_old = old_map_loop(ctx, X, S)
    t1 = time.perf_counter()
    e_old = np_negentropy(d_old)
    t2 = time.perf_counter()
    res["old_map_loop_s"] = t1 - t0
    res["caffe_entropy_before_s"] = t2 - t0
    res["new_map_s"] = wall(lambda: np.asarray(CI._LazyDist313(ctx, X, S)), reps)
    res["caffe_entropy_after_s"] = wall(cd.compute_entropy, reps)
    d_new = np.asarray(cd.dist_ab)
    res["map_equals_old_loop"] = bool(np.array_equal(d_new, d_old))
    res["caffe_entropy_max_abs_diff"] = float(np.nanmax(np.abs(cd.dist_entropy.astype(np.float64) - e_old)))
    # kernels, on torch's stream with preallocated buffers
    st = torch.cuda.current_stream().cuda_stream
    dmap = torch.empty((1, 313, X, X), dtype=torch.float32, device="cuda")
    neg = torch.empty((1, X, X), dtype=torch.float32, device="cuda")
    map_ms = kernel_ms(lambda: lib.idc_caffe313_dist_map(ctx.h, 1, S, dmap.data_ptr(), st), launches)
    neg_ms = kernel_ms(lambda: lib.idc_negentropy(ctx.device, 1, 313, X * X, dmap.data_ptr(), neg.data_ptr(), st), launches)
    H4 = X // 4
    map_bytes = 313 * X * X * 4 + H4 * H4 * 313 * 4        # the map written once + the logits read once
    neg_bytes = 313 * X * X * 4 + X * X * 4
    res["dist313_map_kernel"] = {"ms": map_ms, "bytes": map_bytes, "GBps": map_bytes / map_ms * 1e-6,
                                 "floor_ms_at_3.35TBps": map_bytes / HBM_BPS * 1e3}
    res["negentropy_kernel_313"] = {"ms": neg_ms, "bytes": neg_bytes, "GBps": neg_bytes / neg_ms * 1e-6,
                                    "floor_ms_at_3.35TBps": neg_bytes / HBM_BPS * 1e3}
    cd._ctx.close()
    del cd, dmap, neg
    # the PyTorch 529-bin model, resident distribution
    dm = dist_model(X, sd)
    dctx = dm._dist_ctx

    def before529():
        d = np.asarray(CI._LazyUpsampledDist(fetch=lambda y4, x4: dctx.fetch_dist(0, y4, x4), shape64=(529, H4, H4)))
        return np_negentropy(d)
    res["dist529_entropy_before_s"] = wall(before529, reps)
    res["dist529_entropy_after_s"] = wall(dm.compute_entropy, reps)
    res["dist529_entropy_max_abs_diff"] = float(np.nanmax(np.abs(dm.dist_entropy.astype(np.float64) - before529())))
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--sizes", default="64,256,512")
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dist_maps_profile needs a CUDA device")
    name, plim = card()
    sd = synth.torch_state_dict(1234)
    csd = caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=prepost.pts_in_hull())
    sd313 = dict(sd)
    sd313.update({k: torch.from_numpy(v) for k, v in csd.items() if k != "caffe.pts_in_hull"})
    res = {"card": name, "power_limit": plim, "launches": args.launches,
           "sizes": [one_size(int(X), sd, sd313, args.reps, args.launches) for X in args.sizes.split(",")]}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "dist_maps_profile.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
