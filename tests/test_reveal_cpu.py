"""CPU: the reveal sweep's host side -- the point sampler (photos.reveal_points), the level checks, the batch layout on a
fake device, the argument checks of idc_hint_fill_mean (IDC_ERR_ARG before any device call) and the command line."""
import ctypes
import os

import numpy as np
import pytest

import ideepcolor_b200 as cli
from interactive_deep_colorization_b200 import _lib, photos


def _rule(X, m, seed, index):
    """The sampling rule of the docstring, restated draw by draw."""
    rng = np.random.default_rng([seed, index])
    out = []
    for _ in range(m):
        P = rng.integers(1, 10)
        cy, cx = rng.normal(X / 2, X / 4, 2)
        out.append((np.clip(np.floor(cy) - (P - 1) // 2, 0, X - P), np.clip(np.floor(cx) - (P - 1) // 2, 0, X - P), P))
    return np.array(out, np.int64).reshape(m, 3)


@pytest.mark.parametrize("X", [16, 64, 256])
def test_points_follow_the_rule_and_stay_inside(X):
    for seed, index in ((0, 0), (3, 17), (2 ** 40, 5)):
        p = photos.reveal_points(X, 1024, seed, index)
        assert p.dtype == np.int32 and p.shape == (1024, 3)
        assert np.array_equal(p, _rule(X, 1024, seed, index))
        y0, x0, P = p[:, 0], p[:, 1], p[:, 2]
        assert P.min() >= 1 and P.max() <= 9 and set(P.tolist()) == set(range(1, 10))
        assert (y0 >= 0).all() and (x0 >= 0).all() and (y0 + P <= X).all() and (x0 + P <= X).all()


def test_points_deterministic_prefixes_and_keyed_by_seed_and_index():
    a = photos.reveal_points(256, 500, 7, 3)
    photos.reveal_points(256, 10, 8, 4)                  # no hidden state between calls
    assert np.array_equal(a, photos.reveal_points(256, 500, 7, 3))
    for m in (0, 1, 2, 5, 10, 20, 50, 100, 200):
        assert np.array_equal(photos.reveal_points(256, m, 7, 3), a[:m])
    assert photos.reveal_points(256, 0, 7, 3).shape == (0, 3)
    assert not np.array_equal(a, photos.reveal_points(256, 500, 7, 4))
    assert not np.array_equal(a, photos.reveal_points(256, 500, 8, 3))
    with pytest.raises(ValueError):
        photos.reveal_points(8, 1, 0, 0)
    with pytest.raises(ValueError):
        photos.reveal_points(64, -1, 0, 0)


def test_check_levels():
    assert photos.check_levels([0, 1, 2, 5], 4) == (0, 1, 2, 5)
    assert photos.check_levels((np.int64(1024), 3), 8) == (1024, 3)
    assert photos.check_levels(photos.REVEAL_LEVELS, 10) == photos.REVEAL_LEVELS
    for bad in ([], [1, 1], [-1], [1025], [1.0], [True], ["3"], 5):
        with pytest.raises(ValueError):
            photos.check_levels(bad, 32)
    with pytest.raises(ValueError):
        photos.check_levels(range(11), 10)                # more levels than one pass holds


class FakeDevice(object):
    """Records the reveal batches it is given; the results carry the photo's tag and its points."""

    def __init__(self):
        self.log, self.pending = [], 0

    def submit_reveal(self, imgs, points, levels):
        self.log.append(("submit", [int(a[0, 0, 0]) for a in imgs], levels))
        self.pending += 1
        assert self.pending <= 2
        return imgs, points, levels

    def collect_reveal(self, token):
        imgs, points, levels = token
        self.pending -= 1
        return [photos.RevealResult(np.full(len(levels), float(a[0, 0, 0])), None, None, p) for a, p in zip(imgs, points)]

    def discard(self, token):
        self.pending -= 1

    def close(self):
        assert self.pending == 0


class FakeColorizer(photos.PhotoColorizer):
    def _make_backend(self, state_dict):
        return FakeDevice()


def _img(tag, h=20, w=30):
    a = np.zeros((h, w, 3), np.uint8)
    a[0, 0, 0] = tag
    return a


def test_sweep_layout_order_and_batch_independent_points():
    imgs = [_img(i) for i in range(7)]
    runs = {}
    for batch in (10, 21, 64):
        pc = FakeColorizer(None, Xd=64, batch=batch)
        res = list(pc.reveal_sweep(imgs, levels=(0, 3, 50), seed=5))
        per = batch // 3
        assert [e[1] for e in pc._backend.log] == [list(range(k, min(k + per, 7))) for k in range(0, 7, per)]
        assert all(e[2] == (0, 3, 50) for e in pc._backend.log)
        assert [int(r.psnr[0]) for r in res] == list(range(7))
        runs[batch] = [r.points for r in res]
        for i, r in enumerate(res):
            assert np.array_equal(r.points, photos.reveal_points(64, 50, 5, i))
        pc.close()
    for batch in (21, 64):
        assert all(np.array_equal(a, b) for a, b in zip(runs[10], runs[batch]))


def test_sweep_argument_errors_before_device_work():
    pc = FakeColorizer(None, Xd=64, batch=4)
    for kw in ({"levels": (0, 1, 2, 3, 4)}, {"levels": (1, 1)}, {"levels": (2000,)}, {"levels": ()}):
        with pytest.raises(ValueError):
            pc.reveal_sweep([_img(0)], **kw)
    for bad in ([np.zeros((4, 4), np.uint8)], [np.zeros((4, 4, 3), np.float32)], [3],
                [np.zeros((photos.XFULLRES_MAX + 1, 2, 3), np.uint8)]):
        with pytest.raises(ValueError):
            pc.reveal_sweep(bad, levels=(0, 1))
    assert pc._backend.log == []
    with pytest.raises(ValueError):
        FakeColorizer(None, Xd=8, batch=4).reveal_sweep([_img(0)], levels=(0,))


def test_fill_mean_abi_argument_checks():
    lib = _lib.load()
    P = ctypes.c_void_p(16)          # never dereferenced: every call below fails its checks first
    bad =[(0, 0, 3, 64, P, P, 44, None), (0, 65536, 3, 64, P, P, 44, None),      # n_blocks outside [1, 65535]
           (0, 6, 0, 64, P, P, 44, None),                                         # levels < 1
           (0, 6, 3, 0, P, P, 44, None), (0, 6, 3, _lib.MAX_PHOTO_X + 1, P, P, 44, None),
           (0, 6, 3, 64, None, P, 44, None), (0, 6, 3, 64, P, None, 44, None),    # NULL lab / blocks
           (0, 6, 3, 64, P, P, 12, None), (0, 6, 3, 64, P, P, 46, None),          # stride below the header / not x4
           (0, 6, 3, 64, P, ctypes.c_void_p(18), 44, None)]                       # blocks not 4-byte aligned
    for args in bad:
        assert lib.idc_hint_fill_mean(*args) == _lib.ERR_ARG, args


def test_cli_reveal_sweep_parsing(tmp_path):
    base = ["--color_model", "m.pth", "--image_dir", "d", "--out", "o"]
    a = cli.parse_args(base + ["--reveal_sweep", "0,1,2,5,500"])
    assert a.reveal_levels == (0, 1, 2, 5, 500) and a.reveal_seed == 0
    a = cli.parse_args(base + ["--reveal_sweep", "7", "--reveal_seed", "3"])
    assert a.reveal_levels == (7,) and a.reveal_seed == 3
    assert cli.parse_args(base).reveal_levels is None
    for bad in (["--reveal_sweep", "0,1,x"], ["--reveal_sweep", "0,1,1"], ["--reveal_sweep", "0,-1"],
                ["--reveal_sweep", "1025"], ["--reveal_sweep", "0,,1"],
                ["--reveal_sweep", ",".join(map(str, range(5))), "--batch", "4"],
                ["--reveal_seed", "1"]):
        with pytest.raises(SystemExit):
            cli.parse_args(base + bad)
    with pytest.raises(SystemExit):
        cli.parse_args(["--color_model", "m.pth", "--reveal_sweep", "0,1"])       # needs --image_dir


def test_cli_reveal_csv(tmp_path, monkeypatch, capsys):
    import cv2
    import torch
    d = tmp_path / "photos"
    d.mkdir()
    for i, name in enumerate(("b.png", "a.png", "c.jpg")):
        cv2.imwrite(str(d / name), _img(10 * (i + 1)))
    torch.save({}, str(tmp_path / "m.pth"))
    seen = {}

    class Fake(FakeColorizer):
        def __init__(self, sd, **kw):
            seen.update(kw)
            FakeColorizer.__init__(self, sd, **kw)

        def reveal_sweep(self, paths, levels, seed):
            seen["paths"], seen["levels"], seen["seed"] = [os.path.basename(p) for p in paths], levels, seed
            return iter(photos.RevealResult(np.array([i + 10.0 * j for j in range(len(levels))]), None, None, None)
                        for i in range(len(paths)))

    monkeypatch.setattr(photos, "PhotoColorizer", Fake)
    out = tmp_path / "out"
    rc = cli.main(["--color_model", str(tmp_path / "m.pth"), "--image_dir", str(d), "--out", str(out),
                   "--reveal_sweep", "0,5,20", "--reveal_seed", "9", "--batch", "6", "--load_size", "64"])
    assert rc == 0
    assert seen["paths"] == ["a.png", "b.png", "c.jpg"] and seen["levels"] == (0, 5, 20) and seen["seed"] == 9
    assert seen["batch"] == 6 and seen["Xd"] == 64
    lines = (out / "reveal_psnr.csv").read_text().splitlines()
    assert lines[0] == "image,0,5,20"
    assert [l.split(",")[0] for l in lines[1:]] == ["a.png", "b.png", "c.jpg", "mean"]
    assert [float(v) for v in lines[1].split(",")[1:]] == [0.0, 10.0, 20.0]
    assert [float(v) for v in lines[-1].split(",")[1:]] == [1.0, 11.0, 21.0]
    assert sorted(os.listdir(str(out))) == ["reveal_psnr.csv"]                   # no images
    assert "21.000" in capsys.readouterr().out
