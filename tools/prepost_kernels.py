#!/usr/bin/env python
"""GPU tool for ncu: ONE launch of every bandwidth-bound kernel either side of the conv trunk at a realistic size
(rows a10-a14, f1, f3), so that a profiler yields one row per kernel.

    rgb2lab_kernel          18 MP photo (3456 x 5184, bird_gray.jpg's size), uint8 -> float64 Lab
    resize_linear_u8_kernel 3456 x 5184 -> 256 x 256
    render_planes_kernel    256^2 ab -> 3456 x 5184 full-resolution render (get_img_fullres)
    cubic_lab2rgb_kernel    256^2 ab -> 512 x 512 display
    global_stats_kernel     256 x 256 reference image
    decode313_kernel        batch 16, 256^2 (Caffe-spec annealed mean), + hyper / pred313 GEMMs in the same forward
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import caffe_spec, synth  # noqa: E402
from tests import util  # noqa: E402
from interactive_deep_colorization_b200 import prepost  # noqa: E402

rs = np.random.RandomState(0)
big = rs.randint(0, 256, (3456, 5184, 3)).astype(np.uint8)
small, lab, dlab = prepost.load_image_gpu(big, 256)                      # rgb2lab (18 MP), resize, rgb2lab (256^2)
ab = rs.uniform(-60, 60, (2, 256, 256))
prepost.fullres_rgb_gpu(ab, dlab.view(slice(0, 1)))                      # zoom + lab2rgb at 18 MP
prepost.display_rgb_gpu(ab, rs.uniform(5, 95, (512, 512)))               # cubic + lab2rgb
prepost.global_stats_gpu(small)                                          # histogram + saturation
sd = synth.torch_state_dict(1234)
pts = np.load(os.path.join(ROOT, "tests", "golden", "pts_in_hull.npy"))
sd.update({k: torch.from_numpy(v) for k, v in caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=pts).items()})
n = 16
L, a, m = synth.synthetic_batch(n, 256, seed=0)
ctx = util.make_ctx(sd, 256, 256, max_n=n, caffe313=True, use_graph=False)
ctx.forward_device(util.dev(L), util.dev(a), util.dev(m), 0.5)
ctx.caffe313_pred_ab(n)
torch.cuda.synchronize()
ctx.close()
print("done")
