"""Row f2 on the GPU: ab_reccs_kernel (csrc/idc_heads.cu) through the C ABI vs oracle/reccs_ref.py."""
import numpy as np
import pytest

from oracle import reccs_ref as R, synth
from tests import util

pytestmark = pytest.mark.gpu

P = R.torch_gamut_points()


def _check(pmf, K, n_init, pts=None, tie_prone=False):
    from interactive_deep_colorization_b200.prepost import ab_reccs_pmf_gpu
    pmf = np.asarray(pmf, np.float32)
    pp = P if pts is None else pts
    c, mass, iters = ab_reccs_pmf_gpu(pmf, K=K, n_init=n_init, pts=pts)
    co, mo, io = R.weighted_kmeans_pmf(pmf, pp, K, n_init=n_init)
    assert c.shape == (K, 2) and abs(float(mass.sum()) - 1) < 1e-5 and np.all(np.diff(mass) <= 1e-7)
    e, eo = R.weighted_inertia(pmf, pp, c), R.weighted_inertia(pmf, pp, co)
    assert abs(e - eo) <= (2e-2 if tie_prone else 1e-6) * max(eo, 1e-3) + 1e-6, (e, eo)
    if not tie_prone:           # exact ties (symmetric pmfs) may resolve differently at the last ulp
        assert np.max(np.abs(c - co)) < 1e-4 and np.max(np.abs(mass - mo)) < 1e-6 and iters == io
    return c, mass


@pytest.mark.parametrize("K", [1, 3, 5, 9, 32])
@pytest.mark.parametrize("kind,seed", [("blobs", 0), ("softmax", 1), ("softmax", 2), ("softmax", 3), ("peaked", 4)])
def test_kernel_matches_oracle(kind, seed, K):
    # the flat floor of the near-one-hot pmf makes exactly symmetric configurations once K is large
    _check(R.synthetic_pmf(kind, seed), K, 8, tie_prone=(kind == "peaked" and K > 9))


@pytest.mark.parametrize("n_init", [1, 2, 16])
def test_restarts(n_init):
    _check(R.synthetic_pmf("softmax", 7), 6, n_init)


def test_uniform_pmf_ties():
    _check(R.synthetic_pmf("uniform"), 5, 8, tie_prone=True)


def test_custom_bin_table_and_unnormalised_pmf():
    pts = P[:, ::-1].copy()                                  # (a, b)-ordered grid (pts_grid.npy order, quirk q3)
    c, mass = _check(R.synthetic_pmf("blobs", 0) * 37.5, 4, 8, pts=pts)
    assert np.all(np.abs(c) <= 110)


def test_bad_arguments_are_rejected():
    from interactive_deep_colorization_b200 import _lib
    from interactive_deep_colorization_b200.prepost import ab_reccs_pmf_gpu
    for kw in ({"K": 0}, {"K": 33}, {"n_init": 17}, {"max_iter": 0}):
        with pytest.raises(_lib.IdcError):
            ab_reccs_pmf_gpu(np.ones(529, np.float32), **{"K": 5, **kw})


def test_resident_distribution_path_and_wrapper(synth_sd):
    """idc_ab_reccs reads the pixel's pmf straight from the resident distribution of the last forward."""
    from interactive_deep_colorization_b200 import colorize_image as CI
    g = util.golden("lhn_256.npz")
    gd = util.golden("lhn_dist_256.npz")
    cd = CI.ColorizeImageB200Dist(Xd=256, maskcent=True)
    cd.prep_net(state_dict=synth_sd)
    cd.set_image(g["img_rgb"])
    a5, m5 = synth.synthetic_hints(256, 5, 0)
    cd.net_forward(a5, m5)
    centers, conf = cd.get_ab_reccs(128, 128, K=9, return_conf=True)
    pmf = np.asarray(cd.dist_ab[:, 128, 128])
    co, mo, _ = R.weighted_kmeans_pmf(pmf, cd.pts_in_hull, 9)
    assert centers.shape == (9, 2) and np.max(np.abs(centers - co)) < 1e-3 and np.max(np.abs(conf - mo)) < 1e-5
    # at least as good a clustering of this pixel's pmf as the reference's own (sampled) answer in the golden file
    ref = gd["reccs_128_128_K9"]
    assert R.weighted_inertia(pmf, cd.pts_in_hull, centers) <= 1.01 * R.weighted_inertia(pmf, cd.pts_in_hull, ref)
    # a pixel whose 4x4 cell is shared returns the same suggestions (nearest x4 upsample)
    assert np.array_equal(cd.get_ab_reccs(131, 129, K=9), centers)
    # the wrapper that materialises the host distribution agrees
    cm = CI.ColorizeImageB200Dist(Xd=256, maskcent=True, materialize_full=True)
    cm.prep_net(state_dict=synth_sd)
    cm.set_image(g["img_rgb"])
    cm.net_forward(a5, m5)
    assert np.max(np.abs(cm.get_ab_reccs(128, 128, K=9) - centers)) < 1e-3
