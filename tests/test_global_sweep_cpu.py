"""CPU: the global-hints sweep's host side -- the condition vectors (photos.glob_vector), the condition checks, the
batch layout on a fake device, the argument checks of idc_global_stats_batch (IDC_ERR_ARG before any device call),
the Caffe switch and the command line."""
import ctypes
import os

import numpy as np
import pytest

import ideepcolor_b200 as cli
from interactive_deep_colorization_b200 import _lib, photos


def _stats(seed=0):
    rs = np.random.RandomState(seed)
    hist = rs.randint(0, 50, 313).astype(np.float64)
    return np.r_[hist / hist.sum(), 1.0, rs.uniform(0.05, 0.9), 1.0].astype(np.float32)


def test_glob_vector_layouts():
    s = _stats()
    z = np.zeros(316, np.float32)
    want = {"none": z,
            "sat": np.r_[np.zeros(314), s[314], 1.0],
            "hist": np.r_[s[:313], 1.0, 0.0, 0.0],
            "hist+sat": s}
    for c in photos.GLOBAL_CONDITIONS:
        v = photos.glob_vector(s, c)
        assert v.dtype == np.float32 and v.shape == (316,)
        assert np.array_equal(v, np.asarray(want[c], np.float32)), c
        assert np.array_equal(v.view(np.uint32) == 0, ~np.isin(np.arange(316), np.nonzero(v)[0])), c   # +0, not -0
    assert photos.glob_vector(s.tolist(), "hist+sat").tobytes() == s.tobytes()
    with pytest.raises(ValueError):
        photos.glob_vector(s, "histogram")
    with pytest.raises(ValueError):
        photos.glob_vector(s[:313], "hist")


def test_check_conditions():
    assert photos.check_conditions(photos.GLOBAL_CONDITIONS, 4) == photos.GLOBAL_CONDITIONS
    assert photos.check_conditions(["hist", "none"], 2) == ("hist", "none")
    for bad in ([], ["none", "none"], ["hist", "sat", "hist"], ["bogus"], ["Hist"], [3], "none", None, 5):
        with pytest.raises(ValueError):
            photos.check_conditions(bad, 32)
    with pytest.raises(ValueError):
        photos.check_conditions(photos.GLOBAL_CONDITIONS, 3)     # more conditions than one pass holds


def test_global_stats_batch_abi_argument_checks():
    lib = _lib.load()
    P = ctypes.c_void_p(16)          # never dereferenced: every call below fails its checks first
    X1 = _lib.MAX_PHOTO_X + 4
    bad = [(0, 0, 64, 64, P, P, P, None), (0, 65536, 64, 64, P, P, P, None),      # n outside [1, 65535]
           (0, 2, 0, 64, P, P, P, None), (0, 2, 64, 0, P, P, P, None),            # h, w below 4
           (0, 2, 2, 64, P, P, P, None), (0, 2, 64, -4, P, P, P, None),
           (0, 2, 66, 64, P, P, P, None), (0, 2, 64, 62, P, P, P, None),          # not a multiple of 4
           (0, 2, X1, 64, P, P, P, None), (0, 2, 64, X1, P, P, P, None),          # above IDC_MAX_PHOTO_X
           (0, 2, 64, 64, None, P, P, None), (0, 2, 64, 64, P, None, P, None),    # NULL rgb / pts313 / out
           (0, 2, 64, 64, P, P, None, None)]
    for args in bad:
        assert lib.idc_global_stats_batch(*args) == _lib.ERR_ARG, args


class FakeDevice(object):
    """Records the batches it is given; a photo's statistics row carries its tag, its results the tag per condition."""

    def __init__(self):
        self.log, self.pending = [], 0

    def _tags(self, imgs):
        return [int(a[0, 0, 0]) for a in imgs]

    def submit_glob(self, imgs, conditions):
        self.log.append(("glob", self._tags(imgs), conditions))
        self.pending += 1
        assert self.pending <= 2
        return self._tags(imgs), conditions

    def collect_glob(self, token):
        tags, conditions = token
        self.pending -= 1
        return [photos.GlobalSweepResult(np.array([t + 0.25 * j for j in range(len(conditions))]), None, None,
                                         np.full(316, t, np.float32)) for t in tags]

    def submit_stats(self, imgs):
        self.log.append(("stats", self._tags(imgs)))
        self.pending += 1
        assert self.pending <= 2
        return self._tags(imgs)

    def collect_stats(self, tags):
        self.pending -= 1
        return [np.full(316, t, np.float32) for t in tags]

    def discard(self, token):
        self.pending -= 1

    def close(self):
        assert self.pending == 0


class FakeColorizer(photos.PhotoColorizer):
    def _make_backend(self, state_dict):
        self.loaded = state_dict
        return FakeDevice()


def _img(tag, h=20, w=30):
    a = np.zeros((h, w, 3), np.uint8)
    a[0, 0, 0] = tag
    return a


def test_sweep_layout_order_and_batch_independence():
    imgs = [_img(i) for i in range(7)]
    runs = {}
    for batch, conds in ((4, photos.GLOBAL_CONDITIONS), (12, photos.GLOBAL_CONDITIONS), (32, photos.GLOBAL_CONDITIONS),
                         (5, ("hist", "none", "sat"))):
        pc = FakeColorizer(None, Xd=64, batch=batch, global_hints=True)
        res = list(pc.global_sweep(imgs, conditions=conds))
        per = batch // len(conds)
        assert [e[1] for e in pc._backend.log] == [list(range(k, min(k + per, 7))) for k in range(0, 7, per)]
        assert all(e[0] == "glob" and e[2] == conds for e in pc._backend.log)
        assert [int(r.stats[0]) for r in res] == list(range(7))
        assert all(r.psnr.shape == (len(conds),) for r in res)
        runs[batch, conds] = [r.psnr for r in res]
        pc.close()
    a = runs[4, photos.GLOBAL_CONDITIONS]
    for batch in (12, 32):
        assert all(np.array_equal(x, y) for x, y in zip(a, runs[batch, photos.GLOBAL_CONDITIONS]))
    # global_stats: batches of `batch` photos, rows in input order
    pc = FakeColorizer(None, Xd=64, batch=3)
    rows = list(pc.global_stats(imgs))
    assert [int(r[0]) for r in rows] == list(range(7))
    assert [e[1] for e in pc._backend.log] == [[0, 1, 2], [3, 4, 5], [6]]
    pc.close()


def test_sweep_argument_errors_before_device_work():
    pc = FakeColorizer(None, Xd=64, batch=4, global_hints=True)
    for kw in ({"conditions": ("none", "sat", "hist", "hist+sat", "none")}, {"conditions": ("hist", "hist")},
               {"conditions": ("all",)}, {"conditions": ()}):
        with pytest.raises(ValueError):
            pc.global_sweep([_img(0)], **kw)
    for bad in ([np.zeros((4, 4), np.uint8)], [np.zeros((4, 4, 3), np.float32)], [3],
                [np.zeros((photos.XFULLRES_MAX + 1, 2, 3), np.uint8)]):
        with pytest.raises(ValueError):
            pc.global_sweep(bad)
        with pytest.raises(ValueError):
            pc.global_stats(bad)
    assert pc._backend.log == []
    with pytest.raises(ValueError):              # the sweep needs the global-hints branch
        FakeColorizer(None, Xd=64, batch=4).global_sweep([_img(0)])


def test_caffe_switch():
    import torch
    with pytest.raises(ValueError):
        FakeColorizer({}, Xd=64, batch=4, caffe=True, maskcent=True)
    w = torch.ones((64, 4, 3, 3))
    pc = FakeColorizer({"model1.0.weight": w}, Xd=64, batch=4, caffe=True)
    assert pc.options == {"tanh_scale": 100}
    scale = pc.loaded["model1.0.weight"][0, :, 0, 0].tolist()
    assert scale == [100.0, 110.0, 110.0, 110.0]                    # caffe_scaled_state_dict's conv1_1 scaling
    assert torch.equal(w, torch.ones((64, 4, 3, 3)))                # the caller's weights are left as they are
    pc = FakeColorizer({"model1.0.weight": w}, Xd=64, batch=4)
    assert pc.options is None and pc.loaded["model1.0.weight"] is w


def test_cli_global_parsing():
    base = ["--color_model", "m.pth", "--image_dir", "d", "--out", "o"]
    a = cli.parse_args(base + ["--global_hints", "--glob_sweep"])
    assert a.glob_conditions == photos.GLOBAL_CONDITIONS and a.global_hints and not a.caffe
    a = cli.parse_args(base + ["--global_hints", "--caffe", "--glob_sweep", "hist,none", "--batch", "2"])
    assert a.glob_conditions == ("hist", "none") and a.caffe
    a = cli.parse_args(base + ["--global_hints", "--glob_ref", "ref.jpg"])
    assert a.glob_ref == "ref.jpg" and a.glob_conditions is None
    assert cli.parse_args(base).glob_conditions is None
    for bad in (["--glob_sweep"], ["--glob_ref", "r.jpg"],                               # need --global_hints
                ["--global_hints", "--glob_sweep", "hist,bogus"], ["--global_hints", "--glob_sweep", "hist,hist"],
                ["--global_hints", "--glob_sweep", "none,hist,sat", "--batch", "2"],
                ["--global_hints", "--glob_sweep", "--glob_ref", "r.jpg"],
                ["--global_hints", "--glob_sweep", "--reveal_sweep", "0,1"],
                ["--caffe", "--pytorch_maskcent"]):
        with pytest.raises(SystemExit):
            cli.parse_args(base + bad)
    for flag in (["--global_hints"], ["--caffe"], ["--global_hints", "--glob_ref", "r.jpg"],
                 ["--global_hints", "--glob_sweep"]):
        with pytest.raises(SystemExit):                                            # need --image_dir
            cli.parse_args(["--color_model", "m.pth"] + flag)


def _folder(tmp_path):
    import cv2
    import torch
    d = tmp_path / "photos"
    d.mkdir()
    for i, name in enumerate(("b.png", "a.png", "c.jpg")):
        cv2.imwrite(str(d / name), _img(10 * (i + 1)))
    torch.save({"model1.0.weight": torch.ones((64, 4, 3, 3))}, str(tmp_path / "m.pth"))
    return d


def test_cli_glob_sweep_csv(tmp_path, monkeypatch, capsys):
    d = _folder(tmp_path)
    seen = {}

    class Fake(FakeColorizer):
        def __init__(self, sd, **kw):
            seen.update(kw)
            FakeColorizer.__init__(self, sd, **kw)

        def global_sweep(self, paths, conditions):
            seen["paths"], seen["conditions"] = [os.path.basename(p) for p in paths], conditions
            return iter(photos.GlobalSweepResult(np.array([i + 10.0 * j for j in range(len(conditions))]), None, None,
                                                 None) for i in range(len(paths)))

    monkeypatch.setattr(photos, "PhotoColorizer", Fake)
    out = tmp_path / "out"
    rc = cli.main(["--color_model", str(tmp_path / "m.pth"), "--image_dir", str(d), "--out", str(out),
                   "--global_hints", "--glob_sweep", "--batch", "8", "--load_size", "64"])
    assert rc == 0
    assert seen["paths"] == ["a.png", "b.png", "c.jpg"] and seen["conditions"] == photos.GLOBAL_CONDITIONS
    assert seen["batch"] == 8 and seen["Xd"] == 64 and seen["global_hints"] and not seen["caffe"]
    lines = (out / "glob_psnr.csv").read_text().splitlines()
    assert lines[0] == "image,none,sat,hist,hist+sat"
    assert [l.split(",")[0] for l in lines[1:]] == ["a.png", "b.png", "c.jpg", "mean"]
    assert [float(v) for v in lines[1].split(",")[1:]] == [0.0, 10.0, 20.0, 30.0]
    assert [float(v) for v in lines[-1].split(",")[1:]] == [1.0, 11.0, 21.0, 31.0]
    assert sorted(os.listdir(str(out))) == ["glob_psnr.csv"]                     # no images
    assert "31.000" in capsys.readouterr().out


def test_cli_glob_ref_transfer(tmp_path, monkeypatch):
    d = _folder(tmp_path)
    ref = tmp_path / "ref.png"
    import cv2
    cv2.imwrite(str(ref), _img(99))
    seen = {}

    class Fake(FakeColorizer):
        def global_stats(self, paths):
            seen["ref"] = list(paths)
            return iter([_stats(3)])

        def colorize(self, paths, glob=None, psnr=False):
            seen["glob"], seen["psnr"] = glob, psnr
            return iter(photos.PhotoResult(np.zeros((20, 30, 3), np.uint8), None, None, 1.5) for _ in paths)

    monkeypatch.setattr(photos, "PhotoColorizer", Fake)
    out = tmp_path / "out"
    rc = cli.main(["--color_model", str(tmp_path / "m.pth"), "--image_dir", str(d), "--out", str(out),
                   "--global_hints", "--caffe", "--glob_ref", str(ref), "--psnr"])
    assert rc == 0
    assert seen["ref"] == [str(ref)] and seen["psnr"]
    want = photos.glob_vector(_stats(3), "hist")
    assert len(seen["glob"]) == 3 and all(np.array_equal(g, want) for g in seen["glob"])
    assert sorted(os.listdir(str(out))) == ["a.png", "b.png", "c.png", "psnr.csv"]
