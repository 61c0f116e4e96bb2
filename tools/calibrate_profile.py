"""What activation-range calibration costs, and that it leaves the forward's speed alone (H100; fails without a GPU).

  python tools/calibrate_profile.py --out DIR [--Xd 256] [--images 8 16]

Measured after a warm-up pass, for each number of calibration images:
  * idc_act_absmax over all buffers of the measuring (exact-FP32) context: CUDA events around sweeps that cycle
    through the buffers (memset of the result word + act_absmax_kernel + 4-byte copy per call), three runs of --reps
    sweeps, and act_absmax_kernel alone from torch.profiler, with the bytes read computed from the buffer shapes -> achieved bytes/s and its share of the H100 SXM's 3.35 TB/s (a
    data-sheet figure, not a measurement); the same on a wgmma context (hi + lo FP16 planes: the same bytes);
  * wall time of engine.measure_act_ranges end to end (it ends synchronised), and of its parts run separately: context
    build + weight pack, SIMT forwards, reductions;
  * the wgmma forward with weight-derived against calibrated exponents, alternated in one session: a batch-8
    forward_device (CUDA events) and the one-image forward_host click (host clock, p50).
The card's name, power limit and max SM clock are read in the same run and written with the numbers to
DIR/calibrate_profile.json.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
HBM_PEAK = 3.35e12       # H100 SXM data sheet, bytes/s


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    return torch.cuda.get_device_name(0), q[0] if q else "unknown"


def absmax_times(ctx, n, reps):
    """(ms per sweep of idc_act_absmax over every buffer for the first n images: [min, max] of three runs of `reps`
    sweeps, bytes read per sweep, ms per call on the largest buffer alone).  The sweep cycles through the buffers, 738 MB
    at 256² and n = 4, so no buffer is still in the 50 MB L2 when its turn comes again; the largest buffer alone (134 MB)
    does not fit either."""
    import torch
    names = ctx.act_names()
    shapes = {b: ctx.activation_shape(b) for b in names}
    nbytes = {b: n * c * h * w * 4 for b, (c, h, w) in shapes.items()}    # FP32 plane, or FP16 hi + lo: 4 bytes / element

    def span(bufs, k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(k):
            for b in bufs:
                ctx.act_absmax(b, n)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / k
    span(names, 2)
    sweeps = [span(names, reps) for _ in range(3)]
    big = max(names, key=lambda b: nbytes[b])
    return [min(sweeps), max(sweeps)], sum(nbytes.values()), {"name": big, "bytes": nbytes[big], "ms": span([big], reps)}


def kernel_only_ms(ctx, n, reps):
    """Sum over the buffers of act_absmax_kernel's own mean duration (torch.profiler, CUDA activities): the event
    spans above also hold the idle time of each call's host round trip."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            for b in ctx.act_names():
                ctx.act_absmax(b, n)
    ks = [e for e in prof.key_averages() if "act_absmax_kernel" in e.key]
    if not ks:
        raise RuntimeError("the profiler recorded no act_absmax_kernel")
    return sum(getattr(e, "device_time_total", None) or e.cuda_time_total for e in ks) / reps / 1e3


def wall(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t0) * 1e3


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--Xd", type=int, default=256)
    ap.add_argument("--images", type=int, nargs="*", default=[8, 16])
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("calibrate_profile: no CUDA device; these are H100 measurements and there is no fallback")
    from interactive_deep_colorization_b200 import engine
    from oracle import synth
    from tests import calibrated
    X = args.Xd
    name, power = card()
    rep = {"card": name, "power_limit,max_sm_clock": power, "Xd": X, "runs": []}
    sd = calibrated.trained_like(synth.torch_state_dict(1234), 0.3, synth.synthetic_batch(4, 64, seed=0))
    N = engine.CALIBRATION_MAX_N
    for n_img in args.images:
        batch = tuple(torch.from_numpy(a).cuda() for a in synth.synthetic_batch(n_img, X, seed=40 + n_img))
        engine.measure_act_ranges(sd, batch, X, X, maskcent=0.5)                   # warm-up pass
        ranges, t_all = wall(lambda: engine.measure_act_ranges(sd, batch, X, X, maskcent=0.5))

        def build():
            c = engine.LhnContext(device=0, max_n=N, H=X, W=X, engine="simt")
            c.load_state_dict(sd)
            return c
        ctx, t_build = wall(build)
        chunks = [tuple(a[i:i + N] for a in batch) for i in range(0, n_img, N)]
        _, t_fwd = wall(lambda: [ctx.forward_device(*c, 0.5) for c in chunks])
        _, t_red = wall(lambda: [[ctx.act_absmax(b, c[0].shape[0]) for b in ctx.act_names()] for c in chunks])
        sweep_ms, nbytes, big = absmax_times(ctx, N, args.reps)
        k_ms = kernel_only_ms(ctx, N, 10)
        ctx.close()
        ms = sweep_ms[1]
        run = {"images": n_img, "measure_act_ranges_ms": t_all, "build_and_pack_ms": t_build, "simt_forwards_ms": t_fwd,
               "reductions_ms": t_red, "absmax_images_per_call": N, "absmax_all_buffers_ms_min_max": sweep_ms,
               "absmax_all_buffers_ms": ms, "absmax_all_buffers_bytes": nbytes, "absmax_bytes_per_s": nbytes / (ms * 1e-3),
               "absmax_share_of_3.35TB/s": nbytes / (ms * 1e-3) / HBM_PEAK,
               "absmax_kernel_only_all_buffers_ms": k_ms, "absmax_kernel_only_bytes_per_s": nbytes / (k_ms * 1e-3),
               "absmax_kernel_only_share_of_3.35TB/s": nbytes / (k_ms * 1e-3) / HBM_PEAK}
        big["bytes_per_s"] = big["bytes"] / (big["ms"] * 1e-3)
        big["share_of_3.35TB/s"] = big["bytes_per_s"] / HBM_PEAK
        run["largest_buffer"] = big
        rep["runs"].append(run)
        print(json.dumps({k: v for k, v in run.items() if not isinstance(v, dict) or k == "largest_buffer"}))

    # the product engine with and without measured ranges, alternated
    ctxs = {}
    for key, r in (("weights", None), ("calibrated", ranges)):
        c = engine.LhnContext(device=0, max_n=8, H=X, W=X)
        c.load_state_dict(sd, act_ranges=r)
        ctxs[key] = c
    w_ms, w_bytes, _ = absmax_times(ctxs["weights"], 4, args.reps)
    rep["wgmma_absmax_all_buffers_ms_4_images"] = w_ms
    rep["wgmma_absmax_all_buffers_bytes"] = w_bytes
    b8 = tuple(torch.from_numpy(a).cuda() for a in synth.synthetic_batch(8, X, seed=3))
    L1, ab1, m1 = synth.synthetic_batch(1, X, seed=31, max_hints=6)
    fwd = {k: [] for k in ctxs}
    click = {k: [] for k in ctxs}
    for rnd in range(7):
        for key in (("weights", "calibrated"), ("calibrated", "weights"))[rnd % 2]:      # neither arm always runs first
            c = ctxs[key]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                c.forward_device(*b8, 0.5)
            e1.record()
            torch.cuda.synchronize()
            ts = []
            for _ in range(40):
                t0 = time.perf_counter()
                c.forward_host(L1, ab1, m1, 0.5, want_rgb=True)
                ts.append((time.perf_counter() - t0) * 1e3)
            if rnd:                                                    # round 0 warms both contexts up
                fwd[key].append(e0.elapsed_time(e1) / 10)
                click[key].append(float(np.median(ts)))
    rep["forward_batch8_ms_per_round"] = fwd
    rep["click_forward_host_p50_ms_per_round"] = click
    rep["forward_batch8_images_per_s"] = {k: 8e3 / float(np.mean(v)) for k, v in fwd.items()}
    rep["click_p50_ms"] = {k: float(np.median(v)) for k, v in click.items()}
    rep["exponents_that_differ"] = sum(ctxs["weights"].act_exponent(b) != ctxs["calibrated"].act_exponent(b)
                                       for b in ctxs["weights"].act_names())
    for c in ctxs.values():
        c.close()
    print(json.dumps({k: rep[k] for k in ("card", "power_limit,max_sm_clock", "forward_batch8_images_per_s", "click_p50_ms",
                                          "forward_batch8_ms_per_round", "click_forward_host_p50_ms_per_round",
                                          "exponents_that_differ", "wgmma_absmax_all_buffers_ms_4_images")}))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "calibrate_profile.json"), "w") as f:
        json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
