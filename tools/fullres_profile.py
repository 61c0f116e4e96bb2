"""Cost of the full-resolution renders, host statements against render_planes_kernel (writes JSON).

On seeded synthetic photos at 507 x 600 and 3456 x 5184 (loaded with load_image, a dense net_forward of four hints at
256^2, seeded synthetic weights from oracle/synth) it measures
  * host wall time, median of --reps, ending with the uint8 result in host memory, of each of get_img_fullres,
    get_img_gray_fullres, get_input_img_fullres, get_img_mask_fullres and get_sup_fullres: ColorizeImageB200's device
    path (`device_s`) and the ColorizeImageBase statements on the same object (`host_s`, scipy zoom + float64 lab2rgb;
    the full-resolution L is already on the host for them: that one-time copy is `l_copy_to_host_s`), and how far the
    two results are apart,
  * the GUI's save sequence (ui/gui_draw.py save_result: get_img_fullres, get_input_img_fullres, get_input_img,
    get_sup_img) with the host and with the device input render,
  * CUDA-event kernel times, mean over --launches warmed launches, of render_planes_kernel in each mode (the input
    mode is also get_img_fullres's launch), with the bytes each moves,
  * the card's name and power limit, read in the same run.

    python tools/fullres_profile.py --out DIR [--sizes 507x600,3456x5184] [--reps 5] [--host-reps 3] [--launches 50]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from interactive_deep_colorization_b200 import _lib  # noqa: E402
from interactive_deep_colorization_b200 import colorize_image as CI  # noqa: E402
from oracle import synth  # noqa: E402

HBM_BPS = 3.35e12       # H100 SXM data sheet
GETTERS = ("get_img_fullres", "get_img_gray_fullres", "get_input_img_fullres", "get_img_mask_fullres",
           "get_sup_fullres")
POINTS = [([135, 160], 3, [23, -69]), ([100, 60], 5, [-40, 15.5]), ([250, 3], 2, [60, 60]), ([30, 200], 4, [-10, -80])]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = [s.strip() for s in q.split(",")]
        return name, plim
    except Exception as e:                                     # the numbers stay valid; the label is then unknown
        return "unknown (%s)" % e, "unknown"


def wall(fn, reps, warm=True):
    """median host seconds of fn() followed by a device synchronise (one untimed warm-up call first if warm)."""
    if warm:
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


def photo(H, W, seed):
    coarse = np.random.RandomState(seed).randint(0, 256, (max(H // 64, 2), max(W // 64, 2), 3)).astype(np.uint8)
    return cv2.resize(coarse, (W, H), interpolation=cv2.INTER_CUBIC)


def diff(a, b):
    d = np.abs(a.astype(int) - b.astype(int))
    return {"max_lsb": int(d.max()), "frac_differing": float((d > 0).mean())}


def one_size(H, W, sd, tmp, reps, host_reps, launches):
    res = {"photo": [H, W]}
    cm = CI.ColorizeImageB200(Xd=256)
    cm.prep_net(state_dict=sd)
    path = os.path.join(tmp, "photo_%dx%d.png" % (H, W))
    cv2.imwrite(path, np.ascontiguousarray(photo(H, W, H + W)[:, :, ::-1]))
    cm.load_image(path)
    ab, m = np.zeros((2, 256, 256)), np.zeros((1, 256, 256))
    for (loc, p, val) in POINTS:
        CI.put_point(ab, m, loc, p, val)
    cm.net_forward(ab, m)
    # device path first: the host statements below copy the full-resolution L to the host
    dev = {g: getattr(cm, g)() for g in GETTERS}
    res["device_l_stayed_on_device"] = cm.img_l_fullres._host is None
    for g in GETTERS:
        res[g] = {"device_s": wall(getattr(cm, g), reps)}
    res["device_l_stayed_on_device"] &= cm.img_l_fullres._host is None
    res["save_sequence_device_s"] = wall(lambda: (cm.get_img_fullres(), cm.get_input_img_fullres(), cm.get_input_img(),
                                                  cm.get_sup_img()), reps)
    t0 = time.perf_counter()
    np.asarray(cm.img_l_fullres)
    res["l_copy_to_host_s"] = time.perf_counter() - t0
    for g in GETTERS:
        base = getattr(CI.ColorizeImageBase, g)
        host = base(cm)
        res[g].update(diff(dev[g], host))
        res[g]["host_s"] = wall(lambda: base(cm), host_reps, warm=False)
    res["save_sequence_host_s"] = wall(lambda: (cm.get_img_fullres(), CI.ColorizeImageBase.get_input_img_fullres(cm),
                                                cm.get_input_img(), cm.get_sup_img()), host_reps, warm=False)
    # kernels, on torch's stream with preallocated buffers (the planes as the getters upload them)
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    d_ab = torch.from_numpy(ab).cuda()
    d_m = torch.from_numpy(m[0]).cuda()
    d_L = cm.img_l_fullres.device_plane(0)
    rgb = torch.empty((H, W, 3), dtype=torch.uint8, device="cuda")
    P, MASK, SUP = _lib.RENDER_L_PLANE, _lib.RENDER_L_MASK, _lib.RENDER_L_SUP
    modes = {"gray": (None, 1, None, P, d_L.data_ptr()), "input": (d_ab.data_ptr(), 1, None, P, d_L.data_ptr()),
             "mask": (None, 1, d_m.data_ptr(), MASK, None), "sup": (d_ab.data_ptr(), 0, d_m.data_ptr(), SUP, None)}
    kern = {}
    for name, (pa, order, pm, mode, pl) in modes.items():
        ms = kernel_ms(lambda: lib.idc_render_planes_u8(0, 256, 256, pa, order, 0, pm, 0, mode, pl, H, W, rgb.data_ptr(), st),
                       launches)
        # HBM traffic: the uint8 result written once, the full-resolution L read once; the 256^2 planes stay in cache
        nbytes = 3 * H * W + (8 * H * W if mode == P else 0)
        kern["render_planes_kernel_" + name] = {"ms": ms, "bytes": nbytes, "GBps": nbytes / ms * 1e-6,
                                                "floor_ms_at_3.35TBps": nbytes / HBM_BPS * 1e3}
    res["kernels"] = kern
    # bytes each device getter moves between host and device: its planes up (float64), the uint8 result down
    up = {"get_img_fullres": 2 * 8 * 256 * 256, "get_img_gray_fullres": 0, "get_input_img_fullres": 2 * 8 * 256 * 256,
          "get_img_mask_fullres": 8 * 256 * 256, "get_sup_fullres": 3 * 8 * 256 * 256}
    for g in GETTERS:
        res[g]["h2d_bytes"], res[g]["d2h_bytes"] = up[g], 3 * H * W
    res["l_copy_to_host_bytes"] = 8 * H * W
    del cm, d_ab, d_m, d_L, rgb
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--sizes", default="507x600,3456x5184")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fullres_profile needs a CUDA device")
    name, plim = card()
    sd = synth.torch_state_dict(1234)
    sizes = [tuple(int(v) for v in s.split("x")) for s in args.sizes.split(",")]
    with tempfile.TemporaryDirectory() as tmp:
        res = {"card": name, "power_limit": plim, "reps": args.reps, "host_reps": args.host_reps,
               "launches": args.launches,
               "sizes": [one_size(H, W, sd, tmp, args.reps, args.host_reps, args.launches) for (H, W) in sizes]}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "fullres_profile.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
