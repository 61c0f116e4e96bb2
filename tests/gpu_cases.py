"""Networks, geometries, contexts and the per-op isolation loop shared by the GPU per-op tests (test infrastructure).

The references of tests/op_ref.py are evaluated on the CPU: float64 convolutions, frexp and rounding there do not
depend on a device math library, so the reference is the same numbers the CPU tests check."""
import numpy as np
import torch

from interactive_deep_colorization_b200 import engine
from oracle import lhn_ref, synth
from tests import calibrated, op_ref, util

U24 = 2.0 ** -24
C11_ANALYTIC = 2 * 3 + 3       # conv1_1's FAST accumulation bound (units of 2^-24 * mag): 3 MMA steps of K = 16 in
                               # one chunk, <= 2 each (tests/test_gpu_fast_fp16.analytic_c); bias add, ReLU, exact scale
GEOMS = {"64": (64, 64, 3), "72x88": (72, 88, 2), "8": (8, 8, 2)}      # H, W, n


def calibration_batch():
    return synth.synthetic_batch(4, 64, seed=0)


def make_nets(synth_sd, cal_batch):
    """The synthetic network and the trained-like networks rho = 0.3 and 1 (tests/calibrated.py)."""
    out = {"synthetic": synth_sd}
    out.update({rho: calibrated.trained_like(synth_sd, rho, cal_batch) for rho in (0.3, 1.0)})
    return out


def net_id(net):
    return ("rho%g" % net) if net != "synthetic" else "synth"


def make_batch(geom, seed=300):
    H, W, n = GEOMS[geom]
    X = max(H, W, 32)          # the hint generator wants room; smaller geometries are crops
    return tuple(np.ascontiguousarray(a[:, :, :H, :W]) for a in util.small_batch(n, X, seed=seed))


def oracle_inter(sd, batch):
    """The FP32 oracle's activations (CPU tensors): what the per-op tests inject as each op's inputs."""
    with torch.no_grad():
        return lhn_ref.lhn_forward(sd, *batch, 0.5, ref_quirks=False, return_intermediates=True)[1]


def make_ctx(sd, geom, calibrate=False, ranges_batch=None, **kw):
    """A context of the geometry; calibrate: the storage exponents from ranges measured on `ranges_batch` (the
    exact-FP32 engine, engine.measure_act_ranges) instead of the weight-derived ones."""
    H, W, n = GEOMS[geom]
    ranges = engine.measure_act_ranges(sd, ranges_batch, H, W, maskcent=0.5, keep_conv10=True) if calibrate else None
    ctx = engine.LhnContext(device=0, max_n=n, H=H, W=W, **kw)
    ctx.load_state_dict(sd, act_ranges=ranges)
    return ctx


def conv1_1_of_forward(ctx, sd, batch, maskcent, mode):
    """a1_1 after one forward_device, and op_ref.conv1_1 in `mode` and "exact" -> (got, ref, mag, exact), float64 CPU."""
    ctx.forward_device(*(util.dev(a) for a in batch), maskcent)
    torch.cuda.synchronize()
    got = ctx.get_activation("a1_1", batch[0].shape[0]).double().cpu()
    inputs = [torch.from_numpy(a) for a in batch]
    ref, mag = op_ref.conv1_1(sd, *inputs, maskcent, mode=mode)
    ex = ref if mode == "exact" else op_ref.conv1_1(sd, *inputs, maskcent)[0]
    return got, ref, mag, ex


def run_ops(ctx, sd, inter, n, mode, exps=None):
    """Every op of util.OP_IO in isolation: the FP32 oracle's activations injected as its inputs, ONE op run.
    -> {op: (engine output, reference out, reference mag, exact reference out)}, float64 CPU tensors."""
    out = {}
    for op, (ins, ob) in util.OP_IO.items():
        acts = {b: inter[b].contiguous() for b in ins}
        for b in ins:
            ctx.set_activation(b, acts[b].cuda())
        ctx.run_op(op, n)
        torch.cuda.synchronize()
        got = ctx.get_activation(ob, n).double().cpu()
        ref, mag = op_ref.OPS[op](sd, acts, mode=mode, exps=exps)
        ex = ref if mode == "exact" else op_ref.OPS[op](sd, acts)[0]
        out[op] = (got, ref, mag, ex)
    return out


def fast_check(got, ref, mag, S, c):
    """-> (worst |err| / bar, fraction of elements equal to fp16-RN of the reference, c needed): bar = half an FP16 ulp
    of the stored value + c * 2^-24 * mag, in value units (the stored value is x 2^S); c needed = the largest
    (|err| - half ulp) / (2^-24 * mag)."""
    got = got.double()
    half = 0.5 * op_ref.ulp16(torch.maximum(got.abs(), ref.abs()) * 2.0 ** S) * 2.0 ** -S
    err = (got - ref).abs()
    frac = float((err / (half + c * U24 * mag)).max())
    eq = float((got == op_ref.f16(ref * 2.0 ** S) * 2.0 ** -S).double().mean())
    need = float(((err - half).clamp(min=0) / (U24 * mag).clamp(min=1e-300)).max())
    return frac, eq, need
