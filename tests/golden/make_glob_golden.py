#!/usr/bin/env python
"""Pin the encode step of the global-statistics extractor (SURVEY row f3) to the reference's OWN code.

The Caffe net `models/global_model/global_stats.prototxt` cannot run here (no Caffe), but its Python layer
`NNEncLayer` (caffe_files/caffe_traininglayers.py:161-196) only wraps `NNEncode(NN=1, sigma=5)`
(caffe_files/color_quantization.py:6-38), which needs numpy + scikit-learn and runs on the CPU.
This script imports THAT class unmodified from the reference checkout, feeds it the 4x4-pooled ab map of the
golden test image (and a random image), and stores the inputs + its encodings.  Run where the reference checkout is available:

    python tests/golden/make_glob_golden.py        -> tests/golden/glob_nnenc.npz
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import color_ref, ref_shims  # noqa: E402


def pooled_ab(rgb):
    lab = color_ref.rgb2lab(rgb)
    H, W = lab.shape[:2]
    return lab[..., 1:].reshape(H // 4, 4, W // 4, 4, 2).mean(axis=(1, 3))          # [H/4, W/4, 2] float64


def main():
    cf = os.path.join(ref_shims.REF_ROOT, "caffe_files")
    sys.path.insert(0, cf)                       # color_quantization.py does `import util` (its sibling)
    import color_quantization as cq              # the reference's own module, unmodified
    enc = cq.NNEncode(1., 5., km_filepath=os.path.join(ref_shims.REF_ROOT, "data", "color_bins", "pts_in_hull.npy"))
    g = np.load(os.path.join(HERE, "lhn_256.npz"))
    out = {}
    imgs = {"mortar": g["img_rgb"], "rand": np.random.RandomState(2).randint(0, 256, (64, 96, 3)).astype(np.uint8)}
    for name, rgb in imgs.items():
        ab = pooled_ab(rgb)                                           # what the AvgPool layer hands to NNEncLayer
        blob = ab.transpose(2, 0, 1)[None]                            # Caffe blob N x 2 x X x Y
        e = enc.encode_points_mtx_nd(blob, axis=1)                    # N x 313 x X x Y, one-hot rows (NN = 1)
        assert np.allclose(e.sum(1), 1.0)
        out[name + "_rgb"] = rgb
        out[name + "_ab_pooled"] = ab.astype(np.float64)
        out[name + "_bin"] = e[0].argmax(0).astype(np.int16)          # nearest-bin index per pooled cell
        out[name + "_hist"] = e[0].mean(axis=(1, 2)).astype(np.float64)   # global average pool = the histogram
        # distance margin between the best and second-best bin (cells near a boundary may legitimately flip in FP32)
        cc = enc.cc.astype(np.float64)
        d = np.sqrt(((ab.reshape(-1, 1, 2) - cc[None]) ** 2).sum(-1))
        d.sort(axis=1)
        out[name + "_margin"] = (d[:, 1] - d[:, 0]).reshape(ab.shape[:2]).astype(np.float32)
    np.savez_compressed(os.path.join(HERE, "glob_nnenc.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
