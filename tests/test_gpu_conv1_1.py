"""GPU: conv1_1 (the input pack cat(L/100, ab/110, mask - maskcent) and model1.0 + ReLU) in isolation, on all four of
its kernels, against op_ref.conv1_1 in FP64: a1_1 after one forward.

  * split wgmma (conv1_1_umma_kernel<true>): hi/lo operands (2^-22 each) plus the in-core sums, then hi/lo storage;
  * FAST_FP16 wgmma (conv1_1_umma_kernel<false>): against the same FP16 operands (op_ref mode "fp16"), half an FP16
    ulp of the stored value plus the analytic accumulation bound of its 3 MMA steps, as in test_gpu_fast_fp16;
  * conv1_1_umma=0 (conv1_1_kernel<true>, FP32 FMAs, hi/lo storage) and the SIMT engine (conv1_1_kernel<false>, FP32
    storage): a K = 36 FP32 sum.

The inputs hit the edges of the pack: maskcent 0 and 0.5, non-binary masks, |ab| at 110 and at 300, L at 0 and 100
(L - 50 = -50 and 50), and batches whose 128-pixel tiles straddle two images (8x8 with n = 3, 72x88 with n = 2).  The
host pipeline's image chunks (n = 9 and 33: chunks that start at img0 > 0) must equal the device path bit for bit
on the wgmma kernels."""
import numpy as np
import pytest
import torch

from tests import util
from tests.gpu_cases import C11_ANALYTIC, conv1_1_of_forward, fast_check

pytestmark = pytest.mark.gpu
U24 = 2.0 ** -24
C_SPLIT = 16.0       # split mode: operand error 2^-22 per operand (8 units) + in-core steps, measured with headroom
C_FP32 = 36.0 + 4    # a K = 36 FP32 sum + the quotient and bias roundings

KERNELS = {"split": dict(), "fast": dict(fast_fp16=True), "fp32": dict(options={"conv1_1_umma": 0}),
           "simt": dict(engine="simt")}


def edge_inputs(n, H, W, seed):
    """L - 50, ab, mask with the pack's edge values in stripes: L at 0 / 100, ab at +-110 and +-300, masks that are
    binary on even images and fractional on odd ones."""
    rng = np.random.RandomState(seed)
    L = rng.uniform(-50, 50, (n, 1, H, W))
    ab = rng.uniform(-110, 110, (n, 2, H, W))
    mask = (rng.uniform(0, 1, (n, 1, H, W)) < 0.3).astype(np.float64)
    mask[1::2] = rng.uniform(0, 1, mask[1::2].shape)
    L[:, :, 0::5] = -50.0
    L[:, :, 1::5] = 50.0
    ab[:, 0, :, 0::4] = 110.0
    ab[:, 1, :, 1::4] = -110.0
    ab[:, 0, :, 2::4] = -300.0
    ab[:, 1, :, 3::4] = 300.0
    return tuple(np.ascontiguousarray(a.astype(np.float32)) for a in (L, ab, mask))


def _storage(kind, ref, S):
    """The storage error of a1_1: hi/lo planes of the value x 2^S carry 2^-22 relative and 2^-25 absolute error."""
    return 2.0 ** -22 * ref.abs() + 2.0 ** (-25 - S) if kind in ("split", "fp32") else torch.zeros_like(ref)


@pytest.mark.parametrize("geom", [(8, 8, 3), (72, 88, 2)], ids=["8x8n3", "72x88n2"])
@pytest.mark.parametrize("kind", list(KERNELS))
def test_conv1_1_against_fp64(synth_sd, kind, geom):
    H, W, n = geom
    ctx = util.make_ctx(synth_sd, H, W, max_n=n, use_graph=False, **KERNELS[kind])
    S = ctx.act_exponent("a1_1") if kind != "simt" else 0
    for maskcent in (0.0, 0.5):
        batch = edge_inputs(n, H, W, seed=H + n)
        if kind == "fast":
            got, ref, mag, _ = conv1_1_of_forward(ctx, synth_sd, batch, maskcent, "fp16")
            frac, eq, need = fast_check(got, ref, mag, S, C11_ANALYTIC)
            print("conv1_1 %s %dx%d n=%d maskcent=%g: worst/bar %.3f  =RN16 %.4f  c needed %.2f"
                  % (kind, H, W, n, maskcent, frac, eq, need))
        else:
            got, ref, mag, _ = conv1_1_of_forward(ctx, synth_sd, batch, maskcent, "exact")
            err, st = (got - ref).abs(), _storage(kind, ref, S)
            c = C_SPLIT if kind == "split" else C_FP32
            frac = float((err / (st + c * U24 * mag)).max())
            need = float(((err - st).clamp(min=0) / (U24 * mag).clamp(min=1e-300)).max())
            print("conv1_1 %s %dx%d n=%d maskcent=%g: worst/bar %.3f  max|err| %.2e  c needed %.2f"
                  % (kind, H, W, n, maskcent, frac, float(err.max()), need))
        assert frac <= 1.0, (kind, maskcent, frac)
    ctx.close()


@pytest.mark.parametrize("kind", ["split", "fast", "fp32"])
def test_conv1_1_host_chunks_equal_device(synth_sd, kind):
    """forward_host with n = 9 and n = 33 cuts the batch into image chunks whose conv1_1 launches start at img0 > 0;
    a1_1 and ab equal the single-shot device path bit for bit.  The wgmma kernels only: the SIMT engine's host path
    runs the batch in one piece."""
    ctx = util.make_ctx(synth_sd, 8, 8, max_n=33, **KERNELS[kind])
    for n in (9, 33):
        batch = edge_inputs(n, 8, 8, seed=n)
        r = ctx.forward_host(*batch, 0.5)
        a_host = ctx.get_activation("a1_1", n).cpu().numpy()
        ab_host = r["ab"].copy()
        ab_dev = ctx.forward_device(*(util.dev(a) for a in batch), 0.5)["ab"]
        torch.cuda.synchronize()
        a_dev = ctx.get_activation("a1_1", n).cpu().numpy()
        assert np.array_equal(a_host, a_dev), (kind, n)
        assert np.array_equal(ab_host, ab_dev.cpu().numpy()), (kind, n)
    ctx.close()
