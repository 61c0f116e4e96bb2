"""DESIGN §3's headroom table: for the synthetic network and its trained-like variants (tests/calibrated.py), every
stored buffer's magnitude estimate, bound and storage exponent S_b (as idc_finalize_weights chooses them), the largest
|a| of the FP32 oracle, and that value stored (max|a| * 2^S_b, which must stay below FP16's 65504).  CPU only.

  python tools/act_range_table.py [--rho 0 0.3 1.0]

With --device the max|a| and stored columns of a real checkpoint come from idc_act_absmax on the wgmma engine instead
(H100; seconds at 256²), on seeded synthetic inputs or on photos, and the calibrated exponent / stored pair is added:

  python tools/act_range_table.py --device --checkpoint model.pth [--photos DIR] [--Xd 256] [--pytorch_maskcent]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import lhn_ref, synth  # noqa: E402
from tests import calibrated  # noqa: E402


def device_table(a):
    """The table of one checkpoint from the engines themselves: ranges measured on the FP32 engine, max|a| and stored
    read back from the wgmma engine's own planes."""
    if not torch.cuda.is_available():
        raise SystemExit("act_range_table --device: no CUDA device (there is no fallback; drop --device for the oracle)")
    from interactive_deep_colorization_b200 import _lib, engine
    sd = torch.load(a.checkpoint, map_location="cpu") if a.checkpoint else synth.torch_state_dict(1234)
    X, mc = a.Xd, 0.5 if a.pytorch_maskcent else 0.0
    if a.photos:
        batch = engine.calibration_batch(engine.calibration_source(a.photos), X)
    else:
        batch = tuple(torch.from_numpy(t).cuda() for t in synth.synthetic_batch(4, X, seed=0))
    ranges = engine.measure_act_ranges(sd, batch, X, X, maskcent=mc)
    n = min(int(batch[0].shape[0]), engine.CALIBRATION_MAX_N)
    est = calibrated.act_estimates(sd)
    rows = {}
    for key, r in (("weights", None), ("calibrated", ranges)):
        ctx = engine.LhnContext(device=0, max_n=n, H=X, W=X)
        ctx.load_state_dict(sd, act_ranges=r)
        try:                                # the synchronous forward reports its own saturation
            ctx.forward_host(*(t[:n].cpu().numpy() for t in batch[:3]), mc)
        except _lib.IdcError as e:
            if e.code != _lib.ERR_RANGE:
                raise
            print("%s exponents: SATURATED, the max|a| and stored columns of the named buffers and of every buffer after "
                  "them are clamped values: %s" % (key, e))
        rows[key] = {b: (ctx.act_exponent(b), ctx.act_absmax(b, n)) for b in ctx.act_names()}
        ctx.close()
    print("| buffer | est | bound | max\\|a\\| (wgmma) | S | stored | calibrated S | stored |")
    print("|---|---|---|---|---|---|---|---|")
    for b, (s, mx) in rows["weights"].items():
        sc, mxc = rows["calibrated"][b]
        print("| %s | %.3g | %.3g | %.3g | %d | %.3g | %d | %.3g |"
              % (b, est[b][0], est[b][1], mxc, s, mx * 2.0 ** s, sc, mxc * 2.0 ** sc))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rho", type=float, nargs="*", default=[0.0, 0.3, 1.0])
    ap.add_argument("--device", action="store_true", help="measure on the GPU engines instead of the CPU oracle")
    ap.add_argument("--checkpoint", default="", help="--device: state_dict (.pth); default the synthetic weights")
    ap.add_argument("--photos", default="", help="--device: folder of colour photos; default seeded synthetic inputs")
    ap.add_argument("--Xd", type=int, default=256)
    ap.add_argument("--pytorch_maskcent", action="store_true")
    a = ap.parse_args()
    if a.device:
        return device_table(a)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    sd0 = synth.torch_state_dict(1234)
    cal = synth.synthetic_batch(4, 64, seed=0)                   # the calibration batch of the tests
    test = synth.synthetic_batch(3, 64, seed=1300, max_hints=4)  # a batch the network was not calibrated on
    nets = [("synthetic", sd0)] + [("rho=%g" % r, calibrated.trained_like(sd0, r, cal)) for r in a.rho]
    for name, sd in nets:
        est = calibrated.act_estimates(sd)
        old = calibrated.act_estimates(sd, with_bound=False)
        with torch.no_grad():
            mx, mx_cal = {}, {}
            for batch in (cal, test):
                _, inter = lhn_ref.lhn_forward(sd, *batch, 0.5, ref_quirks=False, return_intermediates=True)
                for b in est:
                    mx[b] = max(mx.get(b, 0.0), float(inter[b].abs().max()))
                    mx_cal.setdefault(b, mx[b])           # the calibration batch alone: what a calibration pass measures
        print("## %s" % name)
        print("| buffer | est | bound | max\\|a\\| | max/est | S | stored | S (2-norm only) | stored | calibrated S | stored |")
        print("|---|---|---|---|---|---|---|---|---|---|---|")
        for b, (e, bd, s) in est.items():
            s_old = old[b][2]
            s_cal = 10 - calibrated._ceil_log2(mx_cal[b])     # kActExpCal - ceil(log2 max|a| on the calibration batch)
            print("| %s | %.3g | %.3g | %.3g | %.2f | %d | %.3g | %d | %.3g | %d | %.3g |"
                  % (b, e, bd, mx[b], mx[b] / e, s, mx[b] * 2.0 ** s, s_old, mx[b] * 2.0 ** s_old, s_cal, mx[b] * 2.0 ** s_cal))
        worst = max(est, key=lambda b: mx[b] * 2.0 ** est[b][2])
        worst_old = max(est, key=lambda b: mx[b] * 2.0 ** old[b][2])
        print("worst stored: %s %.3g; with the 2-norm estimate alone: %s %.3g\n"
              % (worst, mx[worst] * 2.0 ** est[worst][2], worst_old, mx[worst_old] * 2.0 ** old[worst_old][2]))


if __name__ == "__main__":
    main()
