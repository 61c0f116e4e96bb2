"""GPU: FP32 CUDA-core engine (IDC_FLAG_ENGINE_SIMT) against the oracle / golden vectors."""
import numpy as np
import pytest
import torch

from oracle import synth
from tests import util

pytestmark = pytest.mark.gpu


def test_simt_forward_64_all_layers(synth_sd):
    L, ab, m = util.small_batch(2, 64, seed=100)
    ctx = util.make_ctx(synth_sd, 64, 64, max_n=2, engine="simt", dist=True)
    r = ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5, want_dist=True, want_rgb=True)
    torch.cuda.synchronize()
    (reg, dist), inter = util.oracle_forward(synth_sd, L, ab, m, 0.5, dist=True, intermediates=True)
    for name in ["a1_1", "conv1_2", "a2_1", "conv2_2", "conv3_3", "conv4_3", "conv5_3", "conv6_3", "conv7_3",
                 "a8_1", "conv8_3", "a9_1", "conv9_3", "a10_1", "conv10_2"]:
        got = ctx.get_activation(name, 2)
        err = util.maxabs(got, inter[name])
        assert err < 2e-4, (name, err)
    assert util.maxabs(r["ab"], reg) < 2e-3
    assert util.maxabs(r["dist"], dist) < 1e-5
    g = util.golden("lhn_64.npz")
    for i in range(2):
        assert util.maxabs(r["ab"][i], g["reg_quirk_%d" % i] / 110.0) < 2e-3
    ctx.close()


def test_simt_golden_256(synth_sd):
    g = util.golden("lhn_256.npz")
    L = g["img_l_mc"].astype(np.float32)[None]
    ab, m = synth.synthetic_hints(256, 5, 0)
    ctx = util.make_ctx(synth_sd, 256, 256, engine="simt")
    r = ctx.forward_host(L, ab[None].astype(np.float32), m[None].astype(np.float32), 0.5)
    err = util.maxabs(util.at_pix(g, r["ab"][0]), g["mc1_rand5_ab_raw"])
    assert err < 1e-3, err
    ctx.close()
