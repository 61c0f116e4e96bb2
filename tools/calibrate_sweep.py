"""What the calibration constant kActExpCal costs or gains, and where the calibrated stale-statistics network's ab
error comes from (H100; fails without a GPU).

  python tools/calibrate_sweep.py --out DIR

For the synthetic, rho = 0, rho = 0.6 and stale-statistics networks of the tests (64², the tests' batches): ab error
of the wgmma engine against the FP32 and FP64 oracles with the exponents kActExpCal = 8, 10 and 12 would give (set
through act_exp.<buffer> from the measured ranges, so one build serves all three), next to the weight-derived
exponents and to the exact-FP32 SIMT engine as the control for the network's own conditioning.  For the stale network
also: chunk_kb = 1, every stored buffer's error relative to its largest value against the FP64 oracle, and single ops
run on the oracle's inputs, to find the layer an error starts in.  Writes DIR/calibrate_sweep.json.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from interactive_deep_colorization_b200 import _lib, engine  # noqa: E402
from oracle import lhn_ref, synth  # noqa: E402
from tests import calibrate_ref, calibrated, util  # noqa: E402


def oracles(sd, batch):
    with torch.no_grad():
        reg32 = lhn_ref.lhn_forward(sd, *batch, 0.5, ref_quirks=False)
        reg64, inter64 = lhn_ref.lhn_forward(sd, *batch, 0.5, ref_quirks=False, return_intermediates=True,
                                             dtype=torch.float64)
    return reg32, reg64, inter64


def run(sd, batch, reg32, reg64, **kw):
    ctx = util.make_ctx(sd, 64, 64, max_n=batch[0].shape[0], **kw)
    try:
        r = ctx.forward_host(*batch, 0.5)
        out = {"vs_fp32": util.maxabs(r["ab"], reg32), "vs_fp64": util.maxabs(r["ab"], reg64)}
    except _lib.IdcError as e:
        out = {"error": str(e)[:120]}
    return ctx, out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("calibrate_sweep: no CUDA device; these are measurements on the engines, there is no fallback")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    sd0 = synth.torch_state_dict(1234)
    cal = synth.synthetic_batch(4, 64, seed=0)
    test = util.small_batch(3, 64, seed=1300)
    nets = {"synthetic": sd0, "rho=0": calibrated.trained_like(sd0, 0.0, cal), "rho=0.6": calibrated.trained_like(sd0, 0.6, cal)}
    nets["stale"] = calibrate_ref.stale_statistics(calibrated.trained_like(sd0, 0.3, cal), cal)
    rep = {"card": torch.cuda.get_device_name(0), "nets": {}}
    for name, sd in nets.items():
        reg32, reg64, inter64 = oracles(sd, test)
        ranges = engine.measure_act_ranges(sd, cal, 64, 64, maskcent=0.5)
        row = {"fp32_vs_fp64": util.maxabs(reg32, reg64)}
        for key, kw in (("simt", {"engine": "simt"}), ("weights", {})):
            ctx, row[key] = run(sd, test, reg32, reg64, **kw)
            ctx.close()
        variants = [(c, {}) for c in (8, 10, 12)] + ([(10, {"chunk_kb": 1}), (10, {"chunk_kb": 100000})] if name == "stale" else [])
        for c, extra in variants:
            opts = {"act_exp." + b: c - calibrated._ceil_log2(v) for b, v in ranges.items() if b != "conv10_2"}
            opts.update(extra)
            ctx, res = run(sd, test, reg32, reg64, options=opts)
            key = "cal=%d" % c + "".join(" %s=%d" % kv for kv in extra.items())
            row[key] = res
            if name == "stale" and c == 10 and not extra:
                rel = {}
                for b in ctx.act_names():
                    got = ctx.get_activation(b, 3).cpu().double()
                    rel[b] = float((got - inter64[b]).abs().max() / inter64[b].abs().max())
                row["buffer_error_over_max"] = rel
            ctx.close()
        if name == "stale":
            opts = {"act_exp." + b: 10 - calibrated._ceil_log2(v) for b, v in ranges.items()}
            iso = {}
            for eng in ("wgmma", "simt"):
                ctx = util.make_ctx(sd, 64, 64, max_n=3, keep_conv10=True, use_graph=False, engine=eng, options=opts)
                for op in ("c4_2", "c4_3", "c5_1", "c5_2", "c5_3"):
                    ins, out = util.OP_IO[op]
                    for nm in ins:
                        ctx.set_activation(nm, inter64[nm].float().cuda().contiguous())
                    ctx.run_op(op, 3)
                    torch.cuda.synchronize()
                    got = ctx.get_activation(out, 3).cpu().double()
                    iso["%s %s" % (eng, op)] = float((got - inter64[out]).abs().max() / inter64[out].abs().max())
                ctx.close()
            row["isolated_op_error_over_max"] = iso
        rep["nets"][name] = row
        print(name, json.dumps(row))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "calibrate_sweep.json"), "w") as f:
        json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
