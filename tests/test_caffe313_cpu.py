"""CPU: the closed-form x4 up-sample of tests/caffe313_ref.py (the rule decode313_kernel and dist313_row follow) against
oracle/caffe_spec.py's literal pair of grouped Deconvolutions, in float64, on cell grids from 1 x 1 up.  The edge the
kernels special-case -- the zero padding past the last cell row and column -- is exercised on every grid."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import caffe_spec
from tests import caffe313_ref, util

GRIDS = [(1, 1), (1, 5), (6, 1), (2, 2), (3, 4), (16, 16), (22, 18), (64, 64)]


def _spec_up4(logits):
    """pred_313_us + pred_313_rs as oracle/caffe_spec.caffe313_head evaluates them, in float64."""
    k = torch.from_numpy(caffe_spec.US_KERNEL).double()[None, None].repeat(313, 1, 1, 1)
    up = F.conv_transpose2d(torch.from_numpy(logits), k, None, stride=2, padding=1, groups=313)
    return F.conv_transpose2d(up, k, None, stride=2, padding=1, groups=313).numpy()


def _logits(h, w, seed):
    return (np.random.RandomState(seed).standard_normal((1, 313, h, w)) * 4.0).astype(np.float32).astype(np.float64)


@pytest.mark.parametrize("h,w", GRIDS, ids=["%dx%d" % g for g in GRIDS])
def test_up4_is_the_spec_deconv_pair(h, w):
    a = _logits(h, w, 10 * h + w)
    want = _spec_up4(a)
    got = caffe313_ref.up4(a)
    assert got.shape == want.shape == (1, 313, 4 * h, 4 * w)
    err = float(np.abs(got - want).max())
    print("up4 %dx%d cells: max|closed form - deconv pair| = %.3e" % (h, w, err))
    assert err <= 1e-12, err
    # the last output row and column read a[len] = 0: a quarter of the last cell, not all of it
    assert np.allclose(got[..., -1, :], 0.25 * caffe313_ref.up4_axis(a, -1)[..., -1, :], rtol=0, atol=1e-12)
    assert np.allclose(got[..., :, -1], 0.25 * caffe313_ref.up4_axis(a, -2)[..., :, -1], rtol=0, atol=1e-12)


@pytest.mark.parametrize("h,w", [(1, 1), (3, 4), (22, 18)])
def test_head_outputs_follow_the_spec(h, w):
    """dist_ab_S and the annealed mean of the restatement against the same quantities built on the spec's up-sample."""
    a = _logits(h, w, 7)
    pts = util.golden("pts_in_hull.npy")
    up = _spec_up4(a)
    dS = torch.softmax(torch.from_numpy(up) * 0.2, dim=1).numpy()
    pred = np.einsum("nbhw,bc->nchw", torch.softmax(torch.from_numpy(up) * 2.6, dim=1).numpy(), pts.astype(np.float64))
    got_dS = caffe313_ref.dist_ab_S(a)
    assert np.abs(got_dS - dS).max() <= 1e-12
    assert np.abs(got_dS.sum(1) - 1.0).max() <= 1e-12
    assert np.abs(caffe313_ref.pred_ab(a, pts) - pred).max() <= 1e-10        # |ab| <= 110
    ent = caffe313_ref.negentropy(got_dS[0])
    assert ent.shape == (4 * h, 4 * w) and np.all(ent < 0) and np.all(ent >= -np.log(313) - 1e-9)
