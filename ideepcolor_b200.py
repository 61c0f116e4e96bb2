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

With a Caffe checkpoint that also holds the 313-bin distribution head (the caffe.* keys, as the Caffe GUI's colour and
distribution models share one checkpoint), --caffe --caffe_dist gives the suggestions of that head, the colours from the
regression head of the same forward:

    python ideepcolor_b200.py --color_model caffe.pth --caffe --caffe_dist --image_dir scans/ --hints_dir h/ --out o/ \
        --suggest 9

PSNR against the number of hint points revealed from each photo's own colours (photos.reveal_points), written to
<out>/reveal_psnr.csv with no images:

    python ideepcolor_b200.py --color_model caffemodel.pth --image_dir val/ --out sweep/ --reveal_sweep 0,1,2,5,10,20,50
        [--reveal_seed 0] [--batch 60] [--reveal_levin]

--reveal_levin also writes <out>/reveal_psnr_levin.csv, the same sweep with the network replaced by the classical
baseline, colorization by optimization (Levin et al. 2004) on the same revealed points (DESIGN.md §4b).

With a global-hints checkpoint (--global_hints: the glob.* keys; --caffe: Caffe-scaled weights such as the global
model's), every photo of the folder coloured with a reference photo's ab histogram (DemoGlobalHistogramTransfer.ipynb),
or PSNR under the global-hints conditions taken from each photo itself (none, sat, hist, hist+sat) written to
<out>/glob_psnr.csv with no images:

    python ideepcolor_b200.py --color_model glob.pth --global_hints --caffe --image_dir scans/ --out o/ --glob_ref ref.jpg
    python ideepcolor_b200.py --color_model glob.pth --global_hints --image_dir val/ --out o/ --glob_sweep [none,hist]

Under torchrun (WORLD_SIZE > 1 in the environment) the folder mode is one shard of a job per process: rank r takes
the contiguous slice parallel.shard_range(n, world, r) of the sorted photos on GPU LOCAL_RANK (--gpu is ignored),
writes its own photos' <stem>.png and <stem>_suggestions.json, and rank 0 gathers every rank's rows and writes
psnr.csv, reveal_psnr.csv or glob_psnr.csv and the mean rows, byte for byte what one process writes.  The checkpoint
is read, and --calibrate / --save_act_ranges run, on rank 0 only; the other ranks receive the packed weights with one
broadcast.  An error on any rank (a photo that fails to read, say) makes every rank exit with status 1 and its message.
--dist_backend gloo lets ranks share one GPU (NCCL refuses two ranks on one device):

    torchrun --nproc_per_node 8 ideepcolor_b200.py --color_model caffemodel.pth --image_dir val/ --out sweep/ \
        --reveal_sweep 0,1,2,5,10,20,50 --batch 60

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
    ap.add_argument("--reveal_levin", action="store_true",
                    help="with --reveal_sweep: also the classical baseline, colorization by optimization on the same "
                         "revealed points, into <out>/reveal_psnr_levin.csv")
    ap.add_argument("--global_hints", action="store_true",
                    help="the checkpoint has the global-hints branch (glob.* keys; --image_dir)")
    ap.add_argument("--caffe", action="store_true",
                    help="Caffe-scaled weights (mask x 110 and tanh x 100, as ColorizeImageCaffe; --image_dir)")
    ap.add_argument("--caffe_dist", action="store_true",
                    help="with --caffe --hints_dir --suggest K: the suggestions of the checkpoint's 313-bin distribution "
                         "head (caffe.* keys), as ColorizeImageCaffeDist")
    ap.add_argument("--glob_ref", default="", metavar="REF",
                    help="with --global_hints: colour every photo with the ab histogram of photo REF (histogram transfer)")
    ap.add_argument("--glob_sweep", nargs="?", const="", default=None, metavar="C1,C2,...",
                    help="with --global_hints: PSNR of every photo under global hints from its own statistics, one "
                         "column per condition of none,sat,hist,hist+sat (default all four), into <out>/glob_psnr.csv "
                         "(no images are written)")
    ap.add_argument("--dist_backend", default="nccl", choices=("nccl", "gloo"),
                    help="process-group backend of --image_dir under torchrun (gloo: ranks may share a GPU)")
    args = ap.parse_args(argv)
    given = {"global_hints": args.global_hints, "caffe": args.caffe, "glob_ref": bool(args.glob_ref),
             "glob_sweep": args.glob_sweep is not None, "hints_dir": bool(args.hints_dir), "caffe_dist": args.caffe_dist}
    for flag in ("global_hints", "caffe", "glob_ref", "glob_sweep", "hints_dir", "caffe_dist"):
        if given[flag] and not args.image_dir:
            ap.error("--%s needs --image_dir" % flag)
    if args.caffe_dist:
        if not args.caffe:
            ap.error("--caffe_dist needs --caffe: the 313-bin head belongs to a Caffe checkpoint")
        if args.global_hints:
            ap.error("--caffe_dist excludes --global_hints: the global model has no 313-bin head")
        if not (args.hints_dir and args.suggest > 0):
            ap.error("--caffe_dist serves --hints_dir HDIR --suggest K only")
    if args.hints_dir:
        for flag, on in (("reveal_sweep", bool(args.reveal_sweep)), ("glob_sweep", given["glob_sweep"]),
                         ("glob_ref", given["glob_ref"])):
            if on:
                ap.error("--hints_dir excludes --%s" % flag)
        if args.suggest > 0 and args.global_hints:
            ap.error("--hints_dir with --suggest works with a distribution head, and the global model has none")
        if args.suggest > 0 and args.caffe and not args.caffe_dist:
            ap.error("--hints_dir with --suggest and --caffe needs --caffe_dist: a Caffe checkpoint's suggestions come "
                     "from its 313-bin head")
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
    elif args.reveal_levin:
        ap.error("--reveal_levin needs --reveal_sweep")
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
    """--image_dir: every photo of the folder (sorted by name) through PhotoColorizer -> OUT/<stem>.png (+ psnr.csv);
    this process's shard of them under torchrun (colorize_dir_sharded)."""
    import torch
    from interactive_deep_colorization_b200 import parallel
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
    os.makedirs(args.out, exist_ok=True)
    args.world, args.rank = parallel.world_rank()
    sd = hints = error = None
    try:
        hints = read_hints_dir(args.hints_dir, names) if args.hints_dir else None
        if args.rank == 0:        # the other ranks of a job receive the packed weights
            sd = torch.load(args.color_model, map_location="cpu")
    except Exception as e:
        if args.world == 1:
            raise
        error = e
    if args.world > 1:
        parallel.agree(error, device=args.gpu)
    extra = {}
    if hints is not None and args.suggest > 0:
        extra = {"caffe_dist": True} if args.caffe_dist else {"suggest": True}
    pc = PhotoColorizer(sd, Xd=args.load_size, batch=args.batch, device=args.gpu, maskcent=args.pytorch_maskcent,
                        calibrate=args.calibrate_source if args.rank == 0 else None, global_hints=args.global_hints,
                        caffe=args.caffe, **extra)
    if args.rank == 0:
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
        # one copy of REF per rank, so that every rank's shard holds one; its statistics do not depend on the batch
        ref = next(iter(pc.global_stats([args.glob_ref] * args.world)))
        glob = [photos.glob_vector(ref, "hist")] * len(paths)
    write_photos(args, pc, names, pc.colorize(paths, glob=glob, psnr=args.psnr))
    if args.rank == 0:
        print("colorized %d photos into <%s>" % (len(names), args.out))
    return 0


class JobFailed(Exception):
    """A rank of a torchrun job failed; every rank raises this with the same message from the final gather."""


def final_gather(args, error, items):
    """The last collective of a folder-mode job, which every rank reaches once, whether its shard succeeded or not:
    its error text (None if none) and its items, in photo order -> every rank's items in rank order (which is photo
    order) on rank 0, None on the others.  Raises JobFailed on every rank if any rank sent an error."""
    import torch.distributed as dist
    args.gathered = True
    got = [None] * args.world
    dist.all_gather_object(got, (error, items))
    errors = [e for e, _ in got if e is not None]
    if errors:
        raise JobFailed("; ".join(errors))
    return [x for _, part in got for x in part] if args.rank == 0 else None


def merge_rows(args, items):
    """This process's rows -> the rows of every photo on the process that writes the CSVs, None on the others."""
    return items if args.world == 1 else final_gather(args, None, items)


def my_names(pc, names):
    """The names of the photos this process colours (PhotoColorizer.local_slice), in order."""
    start, count = pc.local_slice(len(names))
    return names[start:start + count]


def colorize_dir_sharded(args):
    """--image_dir under torchrun: the process group for the job's lifetime, and every failure carried into the final
    gather (final_gather), so that all ranks exit with status 1 and the failing rank's message instead of waiting."""
    import traceback
    import torch
    import torch.distributed as dist
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if args.gpu != local:
        print("note: --gpu %d is ignored under torchrun: this rank runs on GPU LOCAL_RANK = %d" % (args.gpu, local))
    args.gpu = local
    if args.dist_backend == "nccl":
        torch.cuda.set_device(local)
    dist.init_process_group(args.dist_backend)
    args.gathered = False
    try:
        try:
            return colorize_dir(args)
        except JobFailed as e:
            msg = str(e)
        except Exception as e:
            if args.gathered:
                raise
            traceback.print_exc()
            msg = "rank %d: %s: %s" % (dist.get_rank(), type(e).__name__, e)
            try:
                final_gather(args, msg, [])
            except JobFailed as f:        # with every rank's errors
                msg = str(f)
        print("the job failed: %s" % msg, file=sys.stderr)
        return 1
    finally:
        dist.destroy_process_group()


def write_photos(args, pc, names, results):
    """OUT/<stem>.png of each photo's PhotoResult (its full-resolution result) and, with --psnr, OUT/psnr.csv; then
    closes pc.  names: every photo's; results: those of this process's photos."""
    import cv2
    rows = []
    for name, r in zip(my_names(pc, names), results):
        stem = os.path.splitext(name)[0]
        cv2.imwrite(os.path.join(args.out, stem + ".png"), np.ascontiguousarray(r.fullres[:, :, ::-1]))
        if args.psnr:
            rows.append("%s,%.17g" % (name, r.psnr))
    pc.close()
    rows = merge_rows(args, rows)
    if args.psnr and rows is not None:
        with open(os.path.join(args.out, "psnr.csv"), "w") as f:
            f.write("image,psnr\n" + "".join(row + "\n" for row in rows))


def hinted_dir(args, pc, names, paths, hints):
    """--hints_dir: colorize(hints=...) over the folder -> OUT/<stem>.png (+ psnr.csv); with --suggest K,
    PhotoColorizer.suggest at every hint's loc -> OUT/<stem>_suggestions.json for each photo that has hints."""
    X = args.load_size
    rects = [hint_rects(h, X) for h in hints]
    if args.suggest > 0:
        locs = [np.array([[int(h["loc"][0]), int(h["loc"][1])] for h in hl], np.int64).reshape(-1, 2) for hl in hints]
        suggested = pc.suggest(paths, rects, locs, K=args.suggest, psnr=args.psnr)

        def results():
            start = pc.local_slice(len(names))[0]
            for name, hl, r in zip(names[start:], hints[start:], suggested):
                if hl:
                    write_suggestions(os.path.join(args.out, os.path.splitext(name)[0] + "_suggestions.json"), hl,
                                      r.centers, r.conf)
                yield r.result
        write_photos(args, pc, names, results())
    else:
        write_photos(args, pc, names, pc.colorize(paths, hints=rects, psnr=args.psnr))
    if args.rank == 0:
        print("colorized %d photos with the hints of <%s> into <%s>" % (len(names), args.hints_dir, args.out))
    return 0


def write_sweep(args, pc, names, csv, labels, results, title, line):
    """A sweep's PSNR, one result per photo -> OUT/<csv> (a row per photo, a column per label, then the mean row), and
    `title` and the mean per label (`line` % (label, mean)) on stdout; closes pc.  names: every photo's; results: those
    of this process's photos."""
    rows = sweep_rows(pc, names, results)
    pc.close()
    rows = merge_rows(args, rows)
    if rows is not None:
        write_sweep_csv(args, csv, labels, rows, title, line)
    return 0


def sweep_rows(pc, names, results):
    """A sweep's results for this process's photos -> its rows ([name, PSNR text...], psnr curve)."""
    return [([name] + ["%.17g" % v for v in r.psnr], r.psnr) for name, r in zip(my_names(pc, names), results)]


def write_sweep_csv(args, csv, labels, rows, title, line):
    """Every photo's sweep rows -> OUT/<csv> and the mean curve on stdout (write_sweep)."""
    curves = [c for _, c in rows]
    rows = [row for row, _ in rows]
    mean = np.mean(curves, axis=0) if curves else np.full(len(labels), np.nan)
    rows.append(["mean"] + ["%.17g" % v for v in mean])
    with open(os.path.join(args.out, csv), "w") as f:
        f.write(",".join(["image"] + [str(c) for c in labels]) + "\n" + "".join(",".join(row) + "\n" for row in rows))
    print(title)
    for c, v in zip(labels, mean):
        print(line % (c, v))


def reveal_dir(args, pc, names, paths):
    """--reveal_sweep: PhotoColorizer.reveal_sweep over the folder -> OUT/reveal_psnr.csv, and the mean curve on
    stdout; with --reveal_levin first the Levin baseline's sweep -> OUT/reveal_psnr_levin.csv."""
    levels = args.reveal_levels
    title = ("reveal sweep of %d photos (seed %d), mean PSNR per number of revealed points:"
             % (len(names), args.reveal_seed))
    if not args.reveal_levin:
        return write_sweep(args, pc, names, "reveal_psnr.csv", levels,
                           pc.reveal_sweep(paths, levels=levels, seed=args.reveal_seed), title, "  %4d  %.3f dB")
    # both sweeps' rows travel in one gather, the job's last collective
    rows = [(0, r) for r in sweep_rows(pc, names, pc.reveal_sweep(paths, levels=levels, seed=args.reveal_seed))]
    rows += [(1, r) for r in sweep_rows(pc, names, pc.reveal_sweep(paths, levels=levels, seed=args.reveal_seed,
                                                                    method="levin"))]
    pc.close()
    rows = merge_rows(args, rows)
    if rows is not None:
        write_sweep_csv(args, "reveal_psnr.csv", levels, [r for k, r in rows if k == 0], title, "  %4d  %.3f dB")
        write_sweep_csv(args, "reveal_psnr_levin.csv", levels, [r for k, r in rows if k == 1],
                        "Levin baseline (colorization by optimization) on the same points:", "  %4d  %.3f dB")
    return 0


def glob_sweep_dir(args, pc, names, paths):
    """--glob_sweep: PhotoColorizer.global_sweep over the folder -> OUT/glob_psnr.csv, and the mean per condition on
    stdout."""
    conds = args.glob_conditions
    return write_sweep(args, pc, names, "glob_psnr.csv", conds, pc.global_sweep(paths, conditions=conds),
                       "global-hints sweep of %d photos, mean PSNR per condition:" % len(names), "  %-8s  %.3f dB")


def main(argv=None):
    args = parse_args(argv)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.image_dir:
        return colorize_dir_sharded(args) if world > 1 else colorize_dir(args)
    if world > 1:
        print("--image_file colours one photo on one GPU: run it without torchrun (WORLD_SIZE = %d), or shard a folder "
              "with --image_dir" % world)
        return 2
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
