"""CPU: the whole-map distribution surface without a device -- the C-ABI table, the package import without matplotlib,
and the lazy dist_ab_full / dist_ab_grid / compute_entropy / cached 313-bin map logic over fake contexts."""
import os
import re
import subprocess
import sys

import numpy as np
import torch

from interactive_deep_colorization_b200 import _lib
from interactive_deep_colorization_b200 import colorize_image as CI
from tests.test_host_logic import _FakeNet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("idc_caffe313_dist_map", "idc_negentropy", "idc_dist_negentropy")


def test_new_symbols_are_declared():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "idc_b200.h")).read(), flags=re.S)
    table = {s[0]: s for s in _lib.SYMBOLS}
    for name in NEW:
        assert re.search(r"\b%s\s*\(" % name, src), name
        assert name in table, name
    assert len(table["idc_caffe313_dist_map"][2]) == 5
    assert len(table["idc_negentropy"][2]) == 7
    assert len(table["idc_dist_negentropy"][2]) == 3


def test_package_imports_without_matplotlib():
    code = ("import sys\n"
            "class Block(object):\n"
            "    def find_spec(self, name, path=None, target=None):\n"
            "        if name.split('.')[0] == 'matplotlib':\n"
            "            raise ImportError('matplotlib blocked')\n"
            "sys.meta_path.insert(0, Block())\n"
            "import interactive_deep_colorization_b200\n"
            "from interactive_deep_colorization_b200 import colorize_image as CI\n"
            "m = CI.ColorizeImageB200Dist(Xd=16)\n"
            "assert 'matplotlib' not in sys.modules\n"
            "try:\n"
            "    m.plot_dist_entropy()\n"
            "except ImportError:\n"
            "    print('plot needs matplotlib')\n")
    r = subprocess.run([sys.executable, "-s", "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "plot needs matplotlib" in r.stdout


def _pmf_plane(X4, seed=0):
    d = np.random.RandomState(seed).rand(529, X4, X4).astype(np.float32)
    return d / d.sum(0, keepdims=True)


class _DistCtxCalls(object):
    """fetch_dist / dist_negentropy of a fake context over a host plane, counting what each read costs."""

    def __init__(self, d64):
        self.d64, self.pixels, self.planes, self.negent = d64, 0, 0, 0

    def fetch_dist(self, img, y4=None, x4=None):
        if y4 is None:
            self.planes += 1
            return self.d64.copy()
        self.pixels += 1
        return self.d64[:, y4, x4].copy()

    def dist_negentropy(self, img=0):
        self.negent += 1
        return np.sum(self.d64 * np.log(self.d64), axis=0)


def test_dist529_lazy_views_over_a_fake_context():
    X = 16
    net = _FakeNet(X)
    cd = CI.ColorizeImageB200Dist(Xd=X)
    cd.gpu_prepost = False
    cd.net, cd.net_set = net, True
    cd.set_image(np.random.RandomState(1).randint(0, 256, (X, X, 3)).astype(np.uint8))
    cd.net_forward(np.zeros((2, X, X)), np.zeros((1, X, X)))
    fake = _DistCtxCalls(_pmf_plane(X // 4))
    net.ctx.fetch_dist, net.ctx.dist_negentropy = fake.fetch_dist, fake.dist_negentropy
    assert cd.dist_ab_full.shape == (529, X, X) and cd.dist_ab_grid.shape == (23, 23, X, X)
    up = np.repeat(np.repeat(fake.d64, 4, 1), 4, 2)
    for (h, w) in ((0, 0), (7, 9), (15, 15), (-1, 2)):
        col = up[:, h, w].astype(np.float64)
        f, g = cd.dist_ab_full[:, h, w], cd.dist_ab_grid[:, :, h, w]
        assert f.dtype == np.float64 and np.array_equal(f, col)
        assert np.array_equal(g, col.reshape(23, 23))
        assert cd.dist_ab_grid[4, 5, h, w] == col[4 * 23 + 5]
    assert fake.planes == 0 and fake.pixels == 12            # one 529-float fetch per pixel read
    full = np.asarray(cd.dist_ab_full)
    assert full.dtype == np.float64 and np.array_equal(full, up.astype(np.float64))
    assert np.array_equal(np.asarray(cd.dist_ab_grid), full.reshape(23, 23, X, X))
    assert np.array_equal(cd.dist_ab_full[3], full[3]) and np.array_equal(cd.dist_ab_grid[1, :, 2:5], full.reshape(23, 23, X, X)[1, :, 2:5])
    cd.compute_entropy()
    assert fake.negent == 1 and cd.dist_entropy.shape == (X, X)
    assert np.array_equal(cd.dist_entropy, np.sum(up * np.log(up), axis=0))


def test_lazy_full_keeps_out_of_hull_bins_zero():
    d64 = _pmf_plane(2, seed=3)[:313]
    dist = CI._LazyUpsampledDist(d64)
    in_hull = np.zeros(529, bool)
    in_hull[np.random.RandomState(0).permutation(529)[:313]] = True
    full = CI._LazyDistFull(dist, in_hull, (529, 8, 8))
    ref = np.zeros((529, 8, 8))
    ref[in_hull] = np.asarray(dist)
    assert np.array_equal(np.asarray(full), ref)
    assert np.array_equal(full[:, 6, 1], ref[:, 6, 1])


class _Fake313Ctx(object):
    def __init__(self, X):
        self.map = np.random.RandomState(2).rand(1, 313, X, X).astype(np.float32)
        self.maps = 0

    def caffe313_dist_map(self, n=1, S=0.2):
        self.maps += 1
        return torch.from_numpy(self.map[:n].copy())

    def caffe313_dist_pixel(self, img, y, x, S=0.2):
        return self.map[img, :, y, x].copy()


def test_caffe_dist_map_is_fetched_once_per_forward():
    X = 8
    cd = CI.ColorizeImageB200CaffeDist.__new__(CI.ColorizeImageB200CaffeDist)
    cd.Xd, cd.AB, cd.A, cd.B = X, 529, 23, 23
    cd.in_hull = np.zeros(529, bool)
    cd.in_hull[:313] = True
    ctx = _Fake313Ctx(X)
    cd.dist_ab = CI._LazyDist313(ctx, X, 0.2)
    assert ctx.maps == 0
    assert np.array_equal(np.asarray(cd.dist_ab), ctx.map[0]) and np.array_equal(cd.dist_ab[5], ctx.map[0, 5])
    full = cd.dist_ab_full
    assert cd.dist_ab_full is full and ctx.maps == 1                  # one map per view, scattered once
    assert np.array_equal(full[:313], ctx.map[0]) and not np.any(full[313:])
    assert cd.dist_ab_grid.shape == (23, 23, X, X) and np.shares_memory(cd.dist_ab_grid, full)
    a = np.array(cd.dist_ab)
    a[:] = 0
    assert np.array_equal(np.asarray(cd.dist_ab), ctx.map[0])         # np.array copies the cached map
    assert np.array_equal(cd.dist_ab[:, 3, 4], ctx.map[0, :, 3, 4]) and ctx.maps == 1
