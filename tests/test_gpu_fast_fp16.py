"""GPU: IDC_FLAG_FAST_FP16 against an FP64 evaluation of the operands it feeds the tensor core (tests/op_ref.py, mode
"fp16"), op by op, and its end-to-end error against the FP64 oracle.

FP16 operands carry 2^-11 relative error, so a plain FP64 comparison needs a bar near 1e-3 relative, under which most
kernel bugs fit.  Against the same rounded operands only the accumulation is left: per element the engine's stored
value may differ from the reference by half an FP16 ulp of the stored value (its final rounding) plus
c * 2^-24 * sum |a*w| (op_ref's `mag`), where c = `analytic_c` of the op's chunk structure.  Measured on an H100
(80GB HBM3, 700 W) the largest c any element needs is printed per op next to that bound."""
import numpy as np
import pytest
import torch

from oracle import lhn_ref, synth
from tests import op_ref, util
from tests.gpu_cases import (C11_ANALYTIC, GEOMS, calibration_batch, conv1_1_of_forward, fast_check, make_batch,
                             make_ctx, make_nets, net_id, oracle_inter, run_ops)

pytestmark = pytest.mark.gpu
KBK = 64             # input channels per k-block
# op -> K (input channels x taps per output-parity class) of the wgmma conv: 3x3 convs 9 * cin, the up-sampling ops
# one 2x2 class of the transposed conv (4 * cin) plus the 3x3 shortcut
CIN = {"c1_2": 64, "c2_1": 64, "c2_2": 128, "c3_1": 128, "c3_2": 256, "c3_3": 256, "c4_1": 256, "c4_2": 512,
       "c4_3": 512, "c5_1": 512, "c5_2": 512, "c5_3": 512, "c6_1": 512, "c6_2": 512, "c6_3": 512, "c7_1": 512,
       "c7_2": 512, "c7_3": 512, "c8_2": 256, "c8_3": 256, "c9_2": 128, "c10_2": 128}
K_OP = dict({op: 9 * c for op, c in CIN.items()}, up8=4 * 512 + 9 * 256, up9=4 * 256 + 9 * 128, up10=4 * 128 + 9 * 64)

# (net, calibrated exponents, geometry, plan options)
CASES = [
    ("synthetic", False, "64", {}),
    ("synthetic", False, "72x88", {}),
    ("synthetic", False, "8", {}),
    ("synthetic", False, "64", {"mt": 2}),
    ("synthetic", False, "64", {"split_k": 1}),
    ("synthetic", False, "8", {"split_k": 1, "chunk_kb": 1}),
    ("synthetic", False, "64", {"chunk_kb": 2}),
    ("synthetic", True, "64", {}),
    (0.3, False, "64", {}),
    (0.3, True, "72x88", {"chunk_kb": 1}),
    (0.3, True, "8", {}),
    (1.0, False, "64", {"mt": 2, "chunk_kb": 2}),
    (1.0, True, "64", {}),
    (1.0, False, "72x88", {}),
]


def case_id(case):
    net, cal, geom, opts = case
    return "-".join([net_id(net), geom] + (["cal"] if cal else []) + ["%s%d" % kv for kv in sorted(opts.items())])


def analytic_c(op, chunk_kb):
    """The accumulation error bound of one output element in units of 2^-24 * mag, for a tensor core that forms the
    16 products of an MMA step exactly and adds them to the accumulator with one truncation to FP32: each in-core step
    of a chunk loses < 1 FP32 ulp of the accumulator (<= 2 units); every FP32 round-to-nearest add of a chunk or of a
    split-K slice (at most one per k-block) <= 1; the FP32 epilogue (bias sum and add, folded BatchNorm scale and shift,
    FMA, LeakyReLU slope) <= 6."""
    nkb = K_OP[op] // KBK
    return 2 * 4 * min(chunk_kb, nkb) + nkb + 6


@pytest.fixture(scope="module")
def cal_batch():
    return calibration_batch()


@pytest.fixture(scope="module")
def nets(synth_sd, cal_batch):
    return make_nets(synth_sd, cal_batch)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_fast_ops_against_fp16_reference(nets, cal_batch, case):
    """Per op, and conv1_1 through a forward's a1_1: within half an FP16 ulp + analytic_c * 2^-24 * sum|a*w| of the
    FP64 evaluation of the same FP16 operands, on a FAST context (keep_conv10, no graph)."""
    net, cal, geom, opts = case
    sd = nets[net]
    batch = make_batch(geom)
    n = GEOMS[geom][2]
    inter = oracle_inter(sd, batch)
    ctx = make_ctx(sd, geom, cal, cal_batch if geom == "64" else batch, fast_fp16=True, keep_conv10=True,
                   use_graph=False, options=opts)
    exps = ctx.act_exponents()
    chunk = opts.get("chunk_kb", 4)
    results = {"conv1_1": conv1_1_of_forward(ctx, sd, batch, 0.5, "fp16")}     # conv1_1_umma_kernel<false>
    results.update(run_ops(ctx, sd, inter, n, "fp16", exps))
    ctx.close()
    rows, bad = [], {}
    for op, (got, ref, mag, ex) in results.items():
        ob = "a1_1" if op == "conv1_1" else util.OP_IO[op][1]
        c = C11_ANALYTIC if op == "conv1_1" else analytic_c(op, chunk)
        assert float(ref.abs().max()) * 2.0 ** exps[ob] < op_ref.FP16_MAX, (op, "reference stores above 65504")
        frac, eq, need = fast_check(got, ref, mag, exps[ob], c)
        e_ex = float((got - ex).abs().max()) / max(1.0, float(ex.abs().max()))
        rows.append("  %-7s worst/bar %.3f  =RN16 %.4f  c needed %.2f of %d  |err vs exact|/max(1,|out|) %.2e"
                    % (op, frac, eq, need, c, e_ex))
        if frac > 1.0:
            bad[op] = (frac, need, c)
    print("FAST_FP16 %s:\n%s" % (case_id(case), "\n".join(rows)))
    assert not bad, bad


def test_fast_halo_and_pairs_are_off(synth_sd):
    """The plan turns the halo-tile A operand and CTA pairs off under FAST_FP16: a context asking for both on every
    op gives bit-identical output and activations to one without them."""
    batch = make_batch("64", seed=17)
    outs = []
    for opts in ({}, {"halo": 3, "pairs": 2}):
        ctx = make_ctx(synth_sd, "64", False, fast_fp16=True, dist=True, keep_conv10=True, use_graph=False,
                       options=opts)
        r = ctx.forward_host(*batch, 0.5, want_dist=True)
        outs.append([r["ab"].copy(), r["dist"].copy()] + [ctx.get_activation(b, 3).cpu().numpy() for b in ctx.act_names()])
        ctx.close()
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


# end-to-end: FAST forward against the FP64 oracle.  Bars: the measured worst case on an H100 with headroom.
E2E_AB = 0.3        # measured: up to 0.135 (256² click graph)
E2E_DIST = 6e-3      # measured: up to 2.6e-3 (golden 256² image)


def _e2e(ctx, sd, batch, maskcent, what, dist=True):
    r = ctx.forward_host(*batch, maskcent, want_dist=dist)
    with torch.no_grad():
        o = lhn_ref.lhn_forward(sd, *batch, maskcent, dist=dist, ref_quirks=False, dtype=torch.float64)
    reg, d = o if dist else (o, None)
    e_ab = util.maxabs(r["ab"], reg)
    e_d = util.maxabs(r["dist"], d) if dist else 0.0
    print("FAST_FP16 end to end %s: ab %.3e  dist %.3e" % (what, e_ab, e_d))
    return e_ab, e_d


@pytest.mark.parametrize("net", ["synthetic", 0.3, 1.0])
def test_fast_end_to_end_64(nets, net):
    batch = make_batch("64", seed=1300)
    ctx = make_ctx(nets[net], "64", False, fast_fp16=True, dist=True)
    e_ab, e_d = _e2e(ctx, nets[net], batch, 0.5, "64^2 n=3 %s" % net)
    ctx.close()
    assert e_ab <= E2E_AB and e_d <= E2E_DIST, (e_ab, e_d)


def test_fast_end_to_end_golden_256(synth_sd):
    g = util.golden("lhn_256.npz")
    L = g["img_l_mc"].astype(np.float32)[None]
    ab, m = synth.synthetic_hints(256, 5, 0)
    batch = (L, ab[None].astype(np.float32), m[None].astype(np.float32))
    from interactive_deep_colorization_b200.engine import LhnContext
    ctx = LhnContext(device=0, max_n=1, H=256, W=256, dist=True, fast_fp16=True)
    ctx.load_state_dict(synth_sd)
    e_ab, e_d = _e2e(ctx, synth_sd, batch, 0.5, "golden 256^2 image, 5 hints")
    ctx.close()
    assert e_ab <= E2E_AB and e_d <= E2E_DIST, (e_ab, e_d)


def test_fast_click_graph_256(synth_sd):
    """n = 1 at 256² through the click graph (forward_host replays a captured graph), twice."""
    from interactive_deep_colorization_b200.engine import LhnContext
    L, ab, m = synth.synthetic_batch(1, 256, seed=31, max_hints=6)
    ctx = LhnContext(device=0, max_n=1, H=256, W=256, fast_fp16=True)
    ctx.load_state_dict(synth_sd)
    e1 = _e2e(ctx, synth_sd, (L, ab, m), 0.5, "256^2 click graph", dist=False)[0]
    e2 = _e2e(ctx, synth_sd, (L, ab, m), 0.5, "256^2 click graph, replay", dist=False)[0]
    assert ctx.graph_captures() >= 1
    ctx.close()
    assert e1 == e2 and e1 <= E2E_AB, (e1, e2)
