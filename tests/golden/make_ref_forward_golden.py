#!/usr/bin/env python
"""Pin the CPU oracle's network forward to the reference's OWN SIGGRAPHGenerator (models/pytorch/model.py).

Imports the reference network unmodified (through oracle/ref_shims.py; IDC_REFERENCE_ROOT names its checkout),
loads the seeded synthetic weights, runs one 64x64 image with dist=True and stores:
  reg              its regression return (with the dist=True quirk, model.py:166-168)
  dist_bins        a fixed, seeded sample of 64 of the 529 distribution bins
  dist_sampled     the distribution at those bins on the 16x16 grid it is computed on ([::4, ::4] of the
                   nearest-upsampled 64x64 map)
  state_dict_keys  the network's parameter / buffer names

    python tests/golden/make_ref_forward_golden.py        -> tests/golden/ref_forward_64.npz
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import ref_shims, synth  # noqa: E402
from tests import util  # noqa: E402


def main():
    model = ref_shims.import_reference_model()
    net = model.SIGGRAPHGenerator(dist=True)
    net.load_state_dict(synth.torch_state_dict(1234))
    net.eval()
    L, ab, m = util.small_batch(1, 64, seed=7)
    reg, dist = net.forward(L[0], ab[0], m[0], 0.5)
    dist = dist.detach().numpy()
    bins = np.sort(np.random.RandomState(529).choice(dist.shape[1], 64, replace=False)).astype(np.int32)
    out = {"reg": reg.detach().numpy().astype(np.float32),
           "dist_bins": bins,
           "dist_sampled": dist[:, bins, ::4, ::4].astype(np.float32),
           "state_dict_keys": np.array(sorted(net.state_dict().keys()))}
    np.savez_compressed(os.path.join(HERE, "ref_forward_64.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
