#!/usr/bin/env python
"""GPU tool: ab error and time of the wgmma engine as a function of the chunk_kb option (k-blocks summed
inside the tensor core before the FP32 round-to-nearest add).  Prints a small table."""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import synth  # noqa: E402
from tests import util  # noqa: E402


def main():
    sd = synth.torch_state_dict(1234)
    g = util.golden("lhn_256.npz")
    L = g["img_l_mc"].astype(np.float32)[None]
    ab, m = synth.synthetic_hints(256, 5, 0)
    ref = g["mc1_rand5_ab_raw"]
    Lb, abb, mb = synth.synthetic_batch(16, 256, seed=0)
    print("chunk_kb | max|d ab| golden rand5 | ms / 16-image forward")
    for chunk in (1, 2, 4, 8, 100000):
        ctx = util.make_ctx(sd, 256, 256, max_n=16, use_graph=False, options={"chunk_kb": chunk})
        r = ctx.forward_host(L, ab[None].astype(np.float32), m[None].astype(np.float32), 0.5)
        err = util.maxabs(r["ab"][0], ref)
        dL, dab, dm = util.dev(Lb), util.dev(abb), util.dev(mb)
        for _ in range(3):
            ctx.forward_device(dL, dab, dm, 0.5)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(5):
            ctx.forward_device(dL, dab, dm, 0.5)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) / 5 * 1e3
        print("%8s | %.3e | %.3f" % (chunk if chunk < 1000 else "all", err, ms))
        ctx.close()


if __name__ == "__main__":
    main()
