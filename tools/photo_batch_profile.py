"""Photos/s of automatic colorization: the per-photo wrapper loop (load_image + net_forward(zeros) + get_img_fullres)
against photos.PhotoColorizer, from in-memory arrays and from PNG files, plus the kernel times of idc_photo_prep and
idc_photo_render from CUDA events over many launches.

    python tools/photo_batch_profile.py --out DIR [--batch 32] [--Xd 256]

Host wall time of each leg ends in a device synchronise and follows one untimed warm-up pass over the same photos.  The
card's name and power limit are read in the same run and written with the numbers to DIR/photo_batch_profile.json.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (H, W, photos per leg): ImageNet-like, the repository's test photo size, full HD, an 18 MP camera frame
SIZES = [(375, 500, 128), (507, 600, 128), (1080, 1920, 64), (3456, 5184, 12)]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the number is still reported, marked as unknown
        q = "unknown (%s)" % e
    return name, q


def photo(H, W, seed):
    import cv2
    rs = np.random.RandomState(seed)
    coarse = rs.randint(0, 256, (max(H // 48, 2), max(W // 48, 2), 3)).astype(np.uint8)
    return cv2.resize(coarse, (W, H), interpolation=cv2.INTER_CUBIC)


def timed(fn):
    import torch
    fn()                                 # warm-up: contexts, pinned buffers, page cache of the files
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def kernel_ms(imgs, X, iters):
    """Mean device time of one idc_photo_prep and one idc_photo_render launch over the batch `imgs`."""
    import torch
    from interactive_deep_colorization_b200 import _lib, photos
    lib = _lib.load()
    n = len(imgs)
    table, src = photos.pack_photos(imgs)
    src = torch.from_numpy(src).cuda()
    out = torch.empty_like(src)
    L = torch.empty((n, 1, X, X), dtype=torch.float32, device="cuda")
    lab = torch.rand((n, 3, X, X), dtype=torch.float64, device="cuda") * 60 - 30
    st = torch.cuda.current_stream().cuda_stream
    calls = {"prep": lambda: lib.idc_photo_prep(0, n, table.ctypes.data, src.data_ptr(), X, L.data_ptr(), None, st),
             "render": lambda: lib.idc_photo_render(0, n, table.ctypes.data, src.data_ptr(), X, lab.data_ptr(),
                                                    out.data_ptr(), st)}
    res = {}
    for name, call in calls.items():
        for _ in range(3):
            assert call() == 0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            call()
        e1.record()
        e1.synchronize()
        res[name + "_ms"] = e0.elapsed_time(e1) / iters
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--Xd", type=int, default=256)
    args = ap.parse_args(argv)
    import cv2
    import torch
    from interactive_deep_colorization_b200 import colorize_image as CI
    from interactive_deep_colorization_b200.photos import PhotoColorizer
    from oracle import synth
    os.makedirs(args.out, exist_ok=True)
    if not torch.cuda.is_available():
        raise SystemExit("photo_batch_profile needs a GPU")
    X = args.Xd
    sd = synth.torch_state_dict(1234)
    name, power = card()
    report = {"card": name, "power_limit,max_sm_clock": power, "Xd": X, "batch": args.batch, "sizes": []}
    pc = PhotoColorizer(sd, Xd=X, batch=args.batch)
    cm = CI.ColorizeImageB200(Xd=X)
    cm.prep_net(state_dict=sd)
    zab, zm = np.zeros((2, X, X)), np.zeros((1, X, X))
    with tempfile.TemporaryDirectory() as tmp:
        for (H, W, count) in SIZES:
            imgs = [photo(H, W, s) for s in range(count)]
            paths = []
            for i, a in enumerate(imgs):
                p = os.path.join(tmp, "%dx%d_%03d.png" % (H, W, i))
                cv2.imwrite(p, a[:, :, ::-1])
                paths.append(p)

            def wrapper_arrays():
                for a in imgs:
                    cm._ingest(a, None)         # load_image after its cv2.imread + BGR -> RGB
                    cm.net_forward(zab, zm)
                    cm.get_img_fullres()

            def wrapper_files():
                for p in paths:
                    cm.load_image(p)
                    cm.net_forward(zab, zm)
                    cm.get_img_fullres()

            def batch_arrays():
                for _ in pc.colorize(imgs):
                    pass

            def batch_files():
                for _ in pc.colorize(paths):
                    pass

            row = {"H": H, "W": W, "photos": count}
            for leg, fn in (("wrapper_arrays", wrapper_arrays), ("batch_arrays", batch_arrays),
                            ("wrapper_files", wrapper_files), ("batch_files", batch_files)):
                row[leg + "_photos_per_s"] = count / timed(fn)
            # host decode alone (the thread pool of PhotoColorizer reads with 4 workers)
            t0 = time.perf_counter()
            for p in paths:
                cv2.cvtColor(cv2.imread(p, 1), cv2.COLOR_BGR2RGB)
            row["decode_1thread_photos_per_s"] = count / (time.perf_counter() - t0)
            kimgs = imgs[:min(count, args.batch)]
            row["kernel_batch"] = len(kimgs)
            row.update(kernel_ms(kimgs, X, iters=50 if H * W < 4e6 else 10))
            # PCIe bytes per photo each way (source in, full-resolution result out)
            row["bytes_per_photo_each_way"] = H * W * 3
            report["sizes"].append(row)
            print(json.dumps(row), flush=True)
    pc.close()
    with open(os.path.join(args.out, "photo_batch_profile.json"), "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps({"card": name, "power_limit,max_sm_clock": power}))


if __name__ == "__main__":
    main()
