#!/usr/bin/env python
"""Headless front end of the H100 backend (SURVEY row f4).

The reference's entry point (`ideepcolor.py:60-86`) builds a colour model + a distribution model and hands them
to a PyQt window; its `Save` button writes a result folder (`ui/gui_draw.py:222-244`).  PyQt is not part of this
package; this script drives the same two models from a hint list instead of mouse clicks and writes the same
result folder, plus the K colour suggestions per hint that the GUI shows in its palette.

    python ideepcolor_b200.py --image_file test_imgs/mortar_pestle.jpg --color_model caffemodel.pth \\
        --hints hints.json --out result_dir [--suggest 9] [--pytorch_maskcent] [--gpu 0] [--load_size 256]

Automatic colorization of a folder of photos, in batches on the device (photos.PhotoColorizer):

    python ideepcolor_b200.py --color_model caffemodel.pth --image_dir scans/ --out scans_color/ [--batch 32] [--psnr]

writes <out>/<stem>.png per photo (the full-resolution result, get_img_fullres) and, with --psnr, <out>/psnr.csv
(get_result_PSNR of each photo).

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
    return ap.parse_args(argv)


def hint_ab(h):
    """ab value of one hint: given directly, or derived from an RGB colour the way the GUI's palette does
    (ui/gui_draw.py:97-99: rgb2lab of the picked colour, ab part)."""
    if "ab" in h:
        return [float(h["ab"][0]), float(h["ab"][1])]
    from interactive_deep_colorization_b200 import color
    rgb = np.array(h["rgb"], np.uint8).reshape(1, 1, 3)
    lab = color.rgb2lab(rgb)
    return [float(lab[0, 0, 1]), float(lab[0, 0, 2])]


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
    sd = torch.load(args.color_model, map_location="cpu")
    pc = PhotoColorizer(sd, Xd=args.load_size, batch=args.batch, device=args.gpu, maskcent=args.pytorch_maskcent)
    rows = []
    for name, r in zip(names, pc.colorize(paths, psnr=args.psnr)):
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
    color_model.prep_net(gpu_id=args.gpu, state_dict=sd, dist=args.suggest > 0)
    color_model.load_image(args.image_file)
    dist_model = None
    if args.suggest > 0:
        dist_model = CI.ColorizeImageB200Dist(Xd=X, maskcent=args.pytorch_maskcent)
        dist_model.share_trunk(color_model)             # before the forward: it then carries the distribution head

    hints = json.load(open(args.hints)) if args.hints else []
    # the notebook's put_point calls as a rectangle list: the engine rasterises it on the device
    rects = CI.hints_from_points([([int(h["loc"][0]), int(h["loc"][1])], int(h.get("size", 3)), hint_ab(h)) for h in hints], X)
    result = color_model.net_forward_hints(rects)
    if isinstance(result, int):
        print("net_forward failed")
        return 1
    im_ab, im_mask = color_model.input_ab, color_model.input_mask      # the planes put_point would have painted

    suggestions = None
    if args.suggest > 0 and hints:
        dist_model.set_image(color_model.img_rgb)
        dist_model.net_forward_hints(rects)             # answered from the colour model's forward above
        suggestions = []
        for h in hints:
            centers, conf = dist_model.get_ab_reccs(int(h["loc"][0]), int(h["loc"][1]), K=args.suggest, return_conf=True)
            suggestions.append({"loc": h["loc"], "ab": np.round(centers, 3).tolist(), "conf": np.round(conf, 5).tolist()})

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
        json.dump(suggestions, open(os.path.join(out, "suggestions.json"), "w"), indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
