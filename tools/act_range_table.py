"""DESIGN §3's headroom table: for the synthetic network and its trained-like variants (tests/calibrated.py), every
stored buffer's magnitude estimate, bound and storage exponent S_b (as idc_finalize_weights chooses them), the largest
|a| of the FP32 oracle, and that value stored (max|a| * 2^S_b, which must stay below FP16's 65504).  CPU only.

  python tools/act_range_table.py [--rho 0 0.3 1.0]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import lhn_ref, synth  # noqa: E402
from tests import calibrated  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rho", type=float, nargs="*", default=[0.0, 0.3, 1.0])
    a = ap.parse_args()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    sd0 = synth.torch_state_dict(1234)
    cal = synth.synthetic_batch(4, 64, seed=0)                   # the calibration batch of the tests
    test = synth.synthetic_batch(3, 64, seed=1300, max_hints=4)  # a batch the network was not calibrated on
    nets = [("synthetic", sd0)] + [("rho=%g" % r, calibrated.trained_like(sd0, r, cal)) for r in a.rho]
    for name, sd in nets:
        est = calibrated.act_estimates(sd)
        old = calibrated.act_estimates(sd, with_bound=False)
        with torch.no_grad():
            mx = {}
            for batch in (cal, test):
                _, inter = lhn_ref.lhn_forward(sd, *batch, 0.5, ref_quirks=False, return_intermediates=True)
                for b in est:
                    mx[b] = max(mx.get(b, 0.0), float(inter[b].abs().max()))
        print("## %s" % name)
        print("| buffer | est | bound | max\\|a\\| | max/est | S | stored | S (2-norm only) | stored |")
        print("|---|---|---|---|---|---|---|---|---|")
        for b, (e, bd, s) in est.items():
            s_old = old[b][2]
            print("| %s | %.3g | %.3g | %.3g | %.2f | %d | %.3g | %d | %.3g |"
                  % (b, e, bd, mx[b], mx[b] / e, s, mx[b] * 2.0 ** s, s_old, mx[b] * 2.0 ** s_old))
        worst = max(est, key=lambda b: mx[b] * 2.0 ** est[b][2])
        worst_old = max(est, key=lambda b: mx[b] * 2.0 ** old[b][2])
        print("worst stored: %s %.3g; with the 2-norm estimate alone: %s %.3g\n"
              % (worst, mx[worst] * 2.0 ** est[worst][2], worst_old, mx[worst_old] * 2.0 ** old[worst_old][2]))


if __name__ == "__main__":
    main()
