#!/usr/bin/env python
"""Headless front end of the H100 backend (SURVEY row f4).

The reference's entry point (`ideepcolor.py:60-86`) builds a colour model + a distribution model and hands them
to a PyQt window; its `Save` button writes a result folder (`ui/gui_draw.py:222-244`).  PyQt is not part of this
package; this script drives the same two models from a hint list instead of mouse clicks and writes the same
result folder, plus the K colour suggestions per hint that the GUI shows in its palette.

    python ideepcolor_b200.py --image_file test_imgs/mortar_pestle.jpg --color_model caffemodel.pth \\
        --hints hints.json --out result_dir [--suggest 9] [--pytorch_maskcent] [--gpu 0] [--load_size 256]
        [--calibrate photos/ | ranges.json] [--save_act_ranges ranges.json]

Automatic colorization of a folder of photos, in batches on the device (photos.PhotoColorizer):

    python ideepcolor_b200.py --color_model caffemodel.pth --image_dir scans/ --out scans_color/ [--batch 32] [--psnr]

writes <out>/<stem>.png per photo (the full-resolution result, get_img_fullres) and, with --psnr, <out>/psnr.csv
(get_result_PSNR of each photo).  With --hints_dir HDIR a photo <stem>.<ext> is coloured with the hints of HDIR/<stem>.json
(the --hints format; no file = no hints), and --suggest K also writes <out>/<stem>_suggestions.json, in the format of
the single-image suggestions.json, for every photo that has hints:

    python ideepcolor_b200.py --color_model caffemodel.pth --image_dir scans/ --hints_dir scan_hints/ --out o/ --suggest 9

PSNR against the number of hint points revealed from each photo's own colours (photos.reveal_points), written to
<out>/reveal_psnr.csv with no images:

    python ideepcolor_b200.py --color_model caffemodel.pth --image_dir val/ --out sweep/ --reveal_sweep 0,1,2,5,10,20,50
        [--reveal_seed 0] [--batch 60]

With a global-hints checkpoint (--global_hints: the glob.* keys; --caffe: Caffe-scaled weights such as the global
model's), every photo of the folder coloured with a reference photo's ab histogram (DemoGlobalHistogramTransfer.ipynb),
or PSNR under the global-hints conditions taken from each photo itself (none, sat, hist, hist+sat) written to
<out>/glob_psnr.csv with no images:

    python ideepcolor_b200.py --color_model glob.pth --global_hints --caffe --image_dir scans/ --out o/ --glob_ref ref.jpg
    python ideepcolor_b200.py --color_model glob.pth --global_hints --image_dir val/ --out o/ --glob_sweep [none,hist]

hints.json: [{"loc": [row, col], "size": 3, "ab": [23, -69]}, {"loc": [100, 160], "rgb": [255, 255, 255]}, ...]
(`loc` in load_size x load_size network coordinates, `size` = p of the notebook's put_point: a (2p+1)^2 patch.)
"""
from __future__ import print_function

import argparse
import json
import os
import sys

import numpy as np


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="iDeepColor on the H100 backend, headless")
    ap.add_argument("--image_file", default="test_imgs/mortar_pestle.jpg", help="input image")
    ap.add_argument("--color_model", required=True, help="state_dict (.pth) of the reference PyTorch model")
    ap.add_argument("--hints", default="", help="JSON list of hints; empty = automatic colorization")
    ap.add_argument("--out", default="", help="result folder (default: <image>_b200)")
    ap.add_argument("--gpu", type=int, default=0, help="gpu id")
    ap.add_argument("--load_size", type=int, default=256, help="network resolution")
    ap.add_argument("--pytorch_maskcent", action="store_true", help="centre the mask (siggraph_pretrained weights)")
    ap.add_argument("--suggest", type=int, default=0, help="K colour suggestions per hint (0 = off)")
    ap.add_argument("--image_dir", default="", help="colorize every photo of this folder automatically (needs --out)")
    ap.add_argument("--batch", type=int, default=32, help="photos per device pass (--image_dir)")
    ap.add_argument("--psnr", action="store_true", help="also write psnr.csv (--image_dir)")
    ap.add_argument("--hints_dir", default="", metavar="HDIR",
                    help="with --image_dir: colour photo <stem>.<ext> with the hints of HDIR/<stem>.json (the --hints "
                         "format; a missing file means no hints); with --suggest K also write <out>/<stem>_suggestions.json")
    ap.add_argument("--calibrate", default="", metavar="DIR_OR_JSON",
                    help="set the activation storage exponents from measured ranges instead of the weights: a folder of "
                         "colour photos to measure on (a seeded sample of at most 16), or a JSON file saved earlier")
    ap.add_argument("--save_act_ranges", default="", metavar="FILE", help="write the ranges --calibrate used as JSON")
    ap.add_argument("--reveal_sweep", default="", metavar="M1,M2,...",
                    help="with --image_dir: PSNR of every photo against the number of hint points revealed from its own "
                         "colours, one column per level, into <out>/reveal_psnr.csv (no images are written)")
    ap.add_argument("--reveal_seed", type=int, default=None, help="seed of the revealed points (--reveal_sweep; default 0)")
    ap.add_argument("--global_hints", action="store_true",
                    help="the checkpoint has the global-hints branch (glob.* keys; --image_dir)")
    ap.add_argument("--caffe", action="store_true",
                    help="Caffe-scaled weights (mask x 110 and tanh x 100, as ColorizeImageCaffe; --image_dir)")
    ap.add_argument("--glob_ref", default="", metavar="REF",
                    help="with --global_hints: colour every photo with the ab histogram of photo REF (histogram transfer)")
    ap.add_argument("--glob_sweep", nargs="?", const="", default=None, metavar="C1,C2,...",
                    help="with --global_hints: PSNR of every photo under global hints from its own statistics, one "
                         "column per condition of none,sat,hist,hist+sat (default all four), into <out>/glob_psnr.csv "
                         "(no images are written)")
    args = ap.parse_args(argv)
    given = {"global_hints": args.global_hints, "caffe": args.caffe, "glob_ref": bool(args.glob_ref),
             "glob_sweep": args.glob_sweep is not None, "hints_dir": bool(args.hints_dir)}
    for flag in ("global_hints", "caffe", "glob_ref", "glob_sweep", "hints_dir"):
        if given[flag] and not args.image_dir:
            ap.error("--%s needs --image_dir" % flag)
    if args.hints_dir:
        for flag, on in (("reveal_sweep", bool(args.reveal_sweep)), ("glob_sweep", given["glob_sweep"]),
                         ("glob_ref", given["glob_ref"])):
            if on:
                ap.error("--hints_dir excludes --%s" % flag)
        if args.suggest > 0 and (args.caffe or args.global_hints):
            ap.error("--hints_dir with --suggest works with the 529-bin distribution head only, not with --%s"
                     % ("caffe" if args.caffe else "global_hints"))
    if args.caffe and args.pytorch_maskcent:
        ap.error("--caffe and --pytorch_maskcent exclude each other: the Caffe models do not centre the mask")
    args.glob_conditions = None
    if args.glob_ref or args.glob_sweep is not None:
        if not args.global_hints:
            ap.error("--%s needs --global_hints" % ("glob_ref" if args.glob_ref else "glob_sweep"))
    if args.glob_sweep is not None:
        if args.glob_ref or args.reveal_sweep:
            ap.error("--glob_sweep excludes --%s" % ("glob_ref" if args.glob_ref else "reveal_sweep"))
        try:
            args.glob_conditions = parse_conditions(args.glob_sweep, args.batch)
        except ValueError as e:
            ap.error("--glob_sweep: %s" % e)
    args.reveal_levels = None
    if args.reveal_sweep:
        if not args.image_dir:
            ap.error("--reveal_sweep needs --image_dir")
        try:
            args.reveal_levels = parse_levels(args.reveal_sweep, args.batch)
        except ValueError as e:
            ap.error("--reveal_sweep: %s" % e)
    elif args.reveal_seed is not None:
        ap.error("--reveal_seed needs --reveal_sweep")
    if args.reveal_seed is None:
        args.reveal_seed = 0
    args.calibrate_source = None
    if args.calibrate:
        from interactive_deep_colorization_b200 import engine
        try:
            args.calibrate_source = engine.calibration_source(args.calibrate)
        except ValueError as e:
            ap.error(str(e))
    elif args.save_act_ranges:
        ap.error("--save_act_ranges needs --calibrate")
    return args


def parse_levels(text, batch):
    """'0,1,2,5' -> (0, 1, 2, 5): the levels of --reveal_sweep, checked as PhotoColorizer.reveal_sweep checks them."""
    from interactive_deep_colorization_b200 import photos
    try:
        levels = [int(v) for v in text.split(",")]
    except ValueError:
        raise ValueError("%r is not a comma-separated list of integers" % text)
    return photos.check_levels(levels, batch)


def parse_conditions(text, batch):
    """'none,hist' -> ('none', 'hist'), '' -> all of photos.GLOBAL_CONDITIONS: the conditions of --glob_sweep, checked
    as PhotoColorizer.global_sweep checks them."""
    from interactive_deep_colorization_b200 import photos
    return photos.check_conditions(text.split(",") if text else photos.GLOBAL_CONDITIONS, batch)


def save_ranges(args, ranges):
    if args.save_act_ranges:
        from interactive_deep_colorization_b200 import engine
        engine.save_act_ranges(args.save_act_ranges, ranges)


def hint_ab(h):
    """ab value of one hint: given directly, or derived from an RGB colour the way the GUI's palette does
    (ui/gui_draw.py:97-99: rgb2lab of the picked colour, ab part)."""
    if "ab" in h:
        return [float(h["ab"][0]), float(h["ab"][1])]
    from interactive_deep_colorization_b200 import color
    rgb = np.array(h["rgb"], np.uint8).reshape(1, 1, 3)
    lab = color.rgb2lab(rgb)
    return [float(lab[0, 0, 1]), float(lab[0, 0, 2])]


def hint_rects(hints, X):
    """A --hints list -> the hint rectangles (colorize_image.HINT_LIST_DTYPE) the notebook's put_point calls paint."""
    from interactive_deep_colorization_b200 import colorize_image as CI
    return CI.hints_from_points([([int(h["loc"][0]), int(h["loc"][1])], int(h.get("size", 3)), hint_ab(h)) for h in hints], X)


def write_suggestions(path, hints, centers, conf):
    """suggestions.json: one entry per hint, {"loc": its loc, "ab": the K centres rounded to 3 places, "conf": their
    mass rounded to 5} -- the one format of the single-image and the folder mode."""
    out = [{"loc": h["loc"], "ab": np.round(c, 3).tolist(), "conf": np.round(f, 5).tolist()}
           for h, c, f in zip(hints, centers, conf)]
    with open(path, "w") as f:
        json.dump(out, f, indent=1)


def read_hints_dir(hdir, names):
    """--hints_dir: the hint list of each photo name, from HDIR/<stem>.json; [] where there is no such file."""
    out = []
    for name in names:
        p = os.path.join(hdir, os.path.splitext(name)[0] + ".json")
        if os.path.isfile(p):
            with open(p) as f:
                out.append(json.load(f))
        else:
            out.append([])
    return out


IMAGE_EXTS = (".jpg", ".jpeg", ".png", ".bmp", ".tif", ".tiff", ".webp")


def colorize_dir(args):
    """--image_dir: every photo of the folder (sorted by name) through PhotoColorizer -> OUT/<stem>.png (+ psnr.csv)."""
    import cv2
    import torch
    from interactive_deep_colorization_b200.photos import PhotoColorizer
    if not args.out:
        print("--image_dir needs --out")
        return 2
    names = sorted(f for f in os.listdir(args.image_dir) if os.path.splitext(f)[1].lower() in IMAGE_EXTS)
    stems = {}
    for f in names:
        stems.setdefault(os.path.splitext(f)[0], []).append(f)
    clash = [" / ".join(v) for v in stems.values() if len(v) > 1]
    if clash:             # OUT/<stem>.png would hold only one of them
        print("photos share a name and would overwrite each other's result: %s" % ", ".join(clash))
        return 2
    paths = [os.path.join(args.image_dir, f) for f in names]
    if not os.path.isdir(args.out):
        os.makedirs(args.out)
    hints = read_hints_dir(args.hints_dir, names) if args.hints_dir else None
    sd = torch.load(args.color_model, map_location="cpu")
    extra = {"suggest": True} if hints is not None and args.suggest > 0 else {}
    pc = PhotoColorizer(sd, Xd=args.load_size, batch=args.batch, device=args.gpu, maskcent=args.pytorch_maskcent,
                        calibrate=args.calibrate_source, global_hints=args.global_hints, caffe=args.caffe, **extra)
    save_ranges(args, pc.act_ranges)
    if hints is not None:
        return hinted_dir(args, pc, names, paths, hints)
    if args.reveal_levels is not None:
        return reveal_dir(args, pc, names, paths)
    if args.glob_conditions is not None:
        return glob_sweep_dir(args, pc, names, paths)
    glob = None
    if args.glob_ref:         # histogram transfer: every photo with REF's histogram (DemoGlobalHistogramTransfer.ipynb)
        from interactive_deep_colorization_b200 import photos
        ref = next(iter(pc.global_stats([args.glob_ref])))
        glob = [photos.glob_vector(ref, "hist")] * len(paths)
    rows = []
    for name, r in zip(names, pc.colorize(paths, glob=glob, psnr=args.psnr)):
        stem = os.path.splitext(name)[0]
        cv2.imwrite(os.path.join(args.out, stem + ".png"), np.ascontiguousarray(r.fullres[:, :, ::-1]))
        if args.psnr:
            rows.append("%s,%.17g" % (name, r.psnr))
    pc.close()
    if args.psnr:
        with open(os.path.join(args.out, "psnr.csv"), "w") as f:
            f.write("image,psnr\n" + "".join(row + "\n" for row in rows))
    print("colorized %d photos into <%s>" % (len(names), args.out))
    return 0


def hinted_dir(args, pc, names, paths, hints):
    """--hints_dir: colorize(hints=...) over the folder -> OUT/<stem>.png (+ psnr.csv); with --suggest K,
    PhotoColorizer.suggest at every hint's loc -> OUT/<stem>_suggestions.json for each photo that has hints."""
    import cv2
    X = args.load_size
    rects = [hint_rects(h, X) for h in hints]
    if args.suggest > 0:
        locs = [np.array([[int(h["loc"][0]), int(h["loc"][1])] for h in hl], np.int64).reshape(-1, 2) for hl in hints]
        results = pc.suggest(paths, rects, locs, K=args.suggest, psnr=args.psnr)
    else:
        results = pc.colorize(paths, hints=rects, psnr=args.psnr)
    rows = []
    for name, hl, r in zip(names, hints, results):
        stem = os.path.splitext(name)[0]
        if args.suggest > 0:
            if hl:
                write_suggestions(os.path.join(args.out, stem + "_suggestions.json"), hl, r.centers, r.conf)
            r = r.result
        cv2.imwrite(os.path.join(args.out, stem + ".png"), np.ascontiguousarray(r.fullres[:, :, ::-1]))
        if args.psnr:
            rows.append("%s,%.17g" % (name, r.psnr))
    pc.close()
    if args.psnr:
        with open(os.path.join(args.out, "psnr.csv"), "w") as f:
            f.write("image,psnr\n" + "".join(row + "\n" for row in rows))
    print("colorized %d photos with the hints of <%s> into <%s>" % (len(names), args.hints_dir, args.out))
    return 0


def reveal_dir(args, pc, names, paths):
    """--reveal_sweep: PhotoColorizer.reveal_sweep over the folder -> OUT/reveal_psnr.csv (a row per photo, a column per
    level, then the mean row), and the mean curve on stdout."""
    levels = args.reveal_levels
    rows, curves = [], []
    for name, r in zip(names, pc.reveal_sweep(paths, levels=levels, seed=args.reveal_seed)):
        rows.append([name] + ["%.17g" % v for v in r.psnr])
        curves.append(r.psnr)
    pc.close()
    mean = np.mean(curves, axis=0) if curves else np.full(len(levels), np.nan)
    rows.append(["mean"] + ["%.17g" % v for v in mean])
    with open(os.path.join(args.out, "reveal_psnr.csv"), "w") as f:
        f.write(",".join(["image"] + [str(m) for m in levels]) + "\n" + "".join(",".join(row) + "\n" for row in rows))
    print("reveal sweep of %d photos (seed %d), mean PSNR per number of revealed points:" % (len(names), args.reveal_seed))
    for m, v in zip(levels, mean):
        print("  %4d  %.3f dB" % (m, v))
    return 0


def glob_sweep_dir(args, pc, names, paths):
    """--glob_sweep: PhotoColorizer.global_sweep over the folder -> OUT/glob_psnr.csv (a row per photo, a column per
    condition, then the mean row), and the mean per condition on stdout."""
    conds = args.glob_conditions
    rows, curves = [], []
    for name, r in zip(names, pc.global_sweep(paths, conditions=conds)):
        rows.append([name] + ["%.17g" % v for v in r.psnr])
        curves.append(r.psnr)
    pc.close()
    mean = np.mean(curves, axis=0) if curves else np.full(len(conds), np.nan)
    rows.append(["mean"] + ["%.17g" % v for v in mean])
    with open(os.path.join(args.out, "glob_psnr.csv"), "w") as f:
        f.write(",".join(["image"] + list(conds)) + "\n" + "".join(",".join(row) + "\n" for row in rows))
    print("global-hints sweep of %d photos, mean PSNR per condition:" % len(names))
    for c, v in zip(conds, mean):
        print("  %-8s  %.3f dB" % (c, v))
    return 0


def main(argv=None):
    args = parse_args(argv)
    if args.image_dir:
        return colorize_dir(args)
    import cv2
    import torch
    from interactive_deep_colorization_b200 import colorize_image as CI

    X = args.load_size
    sd = torch.load(args.color_model, map_location="cpu")
    color_model = CI.ColorizeImageB200(Xd=X, maskcent=args.pytorch_maskcent)
    # one checkpoint, one trunk (ideepcolor.py:34-38 "same model used for both"): with suggestions on, the colour model
    # carries the distribution head and the distribution model below shares its context -> ONE forward for both
    color_model.prep_net(gpu_id=args.gpu, state_dict=sd, dist=args.suggest > 0, calibrate=args.calibrate_source)
    save_ranges(args, color_model.act_ranges)
    color_model.load_image(args.image_file)
    dist_model = None
    if args.suggest > 0:
        dist_model = CI.ColorizeImageB200Dist(Xd=X, maskcent=args.pytorch_maskcent)
        dist_model.share_trunk(color_model)             # before the forward: it then carries the distribution head

    hints = json.load(open(args.hints)) if args.hints else []
    # the notebook's put_point calls as a rectangle list: the engine rasterises it on the device
    rects = hint_rects(hints, X)
    result = color_model.net_forward_hints(rects)
    if isinstance(result, int):
        print("net_forward failed")
        return 1
    im_ab, im_mask = color_model.input_ab, color_model.input_mask      # the planes put_point would have painted

    suggestions = None
    if args.suggest > 0 and hints:
        dist_model.set_image(color_model.img_rgb)
        dist_model.net_forward_hints(rects)             # answered from the colour model's forward above
        suggestions = [dist_model.get_ab_reccs(int(h["loc"][0]), int(h["loc"][1]), K=args.suggest, return_conf=True)
                       for h in hints]

    out = args.out or (os.path.splitext(os.path.abspath(args.image_file))[0] + "_b200")
    if not os.path.isdir(out):
        os.makedirs(out)
    print("saving result to <%s>" % out)
    # same artefacts as the GUI's save_result (ui/gui_draw.py:232-244)
    np.save(os.path.join(out, "im_l.npy"), color_model.img_l)
    np.save(os.path.join(out, "im_ab.npy"), im_ab)
    np.save(os.path.join(out, "im_mask.npy"), im_mask)
    cv2.imwrite(os.path.join(out, "input_mask.png"), im_mask.transpose((1, 2, 0)).astype(np.uint8) * 255)
    for name, rgb in (("ours.png", result), ("ours_fullres.png", color_model.get_img_fullres()),
                      ("input_fullres.png", color_model.get_input_img_fullres()),
                      ("input.png", color_model.get_input_img()), ("input_ab.png", color_model.get_sup_img())):
        cv2.imwrite(os.path.join(out, name), np.ascontiguousarray(rgb[:, :, ::-1]))
    if suggestions is not None:
        write_suggestions(os.path.join(out, "suggestions.json"), hints, [c for c, _ in suggestions],
                          [f for _, f in suggestions])
    return 0


if __name__ == "__main__":
    sys.exit(main())
