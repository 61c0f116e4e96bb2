"""GPU: every op of the exact-FP32 SIMT engine in isolation against the FP64 reference of tests/op_ref.py: the FP32
oracle's activations are injected as the op's inputs, ONE op runs, and its output is compared with the FP64 evaluation
of the op on those inputs; conv1_1 through a forward's a1_1.  The SIMT engine is what engine.measure_act_ranges
calibrates with and the engine the others are debugged against, so each of its ops is held on its own.

Bar: SIMT_BAR * max(1, |out|max), SIMT_BAR 4x the worst case measured on an H100 over these networks and geometries."""
import pytest
import torch

from tests.gpu_cases import (GEOMS, calibration_batch, conv1_1_of_forward, make_batch, make_ctx, make_nets, net_id,
                             oracle_inter, run_ops)

pytestmark = pytest.mark.gpu
SIMT_BAR = 2e-5      # measured on an H100: up to 4.6e-6 x max(1, |out|max)


@pytest.fixture(scope="module")
def nets(synth_sd):
    return make_nets(synth_sd, calibration_batch())


CASES = [("synthetic", "64"), ("synthetic", "72x88"), ("synthetic", "8"), (0.3, "64"), (0.3, "8"), (1.0, "64"),
         (1.0, "72x88")]


@pytest.mark.parametrize("net,geom", CASES, ids=["%s-%s" % (net_id(n), g) for n, g in CASES])
def test_simt_ops_against_fp64(nets, net, geom):
    sd = nets[net]
    batch = make_batch(geom)
    n = GEOMS[geom][2]
    inter = oracle_inter(sd, batch)
    ctx = make_ctx(sd, geom, engine="simt", keep_conv10=True, use_graph=False)
    results = {"conv1_1": conv1_1_of_forward(ctx, sd, batch, 0.5, "exact")[:2]}
    results.update({op: v[:2] for op, v in run_ops(ctx, sd, inter, n, "exact").items()})
    ctx.close()
    rows, bad = [], {}
    for op, (got, ref) in results.items():
        scale = max(1.0, float(ref.abs().max()))
        frac = float((got - ref).abs().max()) / (SIMT_BAR * scale)
        rows.append("  %-7s worst/bar %.3f  (max|err| %.2e, |out|max %.3g)" % (op, frac, frac * SIMT_BAR * scale,
                                                                             float(ref.abs().max())))
        if frac > 1.0:
            bad[op] = frac
    print("SIMT %s %s (bar %.0e x max(1, |out|max)):\n%s" % (net, geom, SIMT_BAR, "\n".join(rows)))
    assert not bad, bad
