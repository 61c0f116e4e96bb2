"""GPU: every wgmma op in isolation -- oracle activations are injected as the op's inputs,
ONE op runs, and its output is compared with the oracle's activation.  Localises a bug to
a layer / tap table / tensor map instead of letting it smear through the network."""
import numpy as np
import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=[(1, 0, 0), (2, 0, 0), (1, 2, 0), (2, 2, 0), (1, 0, 3), (1, 2, 3)],
                ids=["mt1", "mt2", "pairs", "pairs_mt2", "halo", "halo_pairs"])
def setup(request, synth_sd):
    """The plan-time options (mt, pairs, halo) are applied when the launch plan is built: the 128-pixel tiles, the 256-pixel
    tiles, the pair path (clusters of two CTAs sharing a multicast weight tile; forced, incl. the odd-tile-count dummy
    tile) and the halo-tile A operand (one TMA tile per 64 input channels + pixel-shifted wgmma descriptors, stride-1
    3x3 layers with <= 128 output columns) are exercised on every op that supports them."""
    L, ab, m = util.small_batch(3, 64, seed=300)
    _, inter = util.oracle_forward(synth_sd, L, ab, m, 0.5, dist=False, intermediates=True)
    ctx = util.make_ctx(synth_sd, 64, 64, max_n=3, engine="wgmma", keep_conv10=True, use_graph=False,
                        options={"mt": request.param[0], "pairs": request.param[1], "halo": request.param[2]})
    yield ctx, inter
    ctx.close()


@pytest.mark.parametrize("op", list(util.OP_IO.keys()))
def test_single_op(setup, op):
    ctx, inter = setup
    ins, out = util.OP_IO[op]
    for nm in ins:
        ctx.set_activation(nm, inter[nm].cuda().contiguous())
    ctx.run_op(op, 3)
    torch.cuda.synchronize()
    got = ctx.get_activation(out, 3)
    err = util.maxabs(got, inter[out])
    scale = float(inter[out].abs().max())
    print("op %-6s max|err| = %.3e  (|out|max %.2f)" % (op, err, scale))
    assert err < 2e-5 * max(1.0, scale), (op, err, scale)


def test_hi_lo_roundtrip(setup):
    ctx, inter = setup
    ctx.set_activation("conv3_3", inter["conv3_3"].cuda().contiguous())
    back = ctx.get_activation("conv3_3", 3)
    assert util.maxabs(back, inter["conv3_3"]) < 2e-6       # hi+lo carries ~22 bits
