"""CPU: batched colour suggestions' host side -- the argument checks of idc_ab_reccs_batch (the same code through its
host-only hook, so nothing reaches a device), PhotoColorizer(suggest=True) and PhotoColorizer.suggest's checks and
batch layout on a fake device, and the command line's --hints_dir (file matching, missing files, rejected
combinations, and one suggestions formatter for the folder and the single-image mode)."""
import ctypes
import json
import os

import numpy as np
import pytest

import ideepcolor_b200 as cli
from interactive_deep_colorization_b200 import _lib, photos
from interactive_deep_colorization_b200 import colorize_image as CI


def _check(q, K=5, max_iter=100, n_init=8, head=1, n_img=3, h=64, w=48):
    lib = _lib.load()
    qa = np.ascontiguousarray(q, np.int32).reshape(-1, 3)
    msg = ctypes.create_string_buffer(256)
    rc = lib.idc_ab_reccs_batch_check(head, n_img, h, w, qa.shape[0], qa.ctypes.data if qa.size else None, K, max_iter,
                                      n_init, msg, 256)
    return rc, msg.value.decode()


def test_abi_argument_checks():
    good = [(0, 0, 0), (2, 15, 11), (1, 7, 3)]                   # 64 x 48 -> a 16 x 12 grid, 3 images
    assert _check(good) == (_lib.IDC_OK, "")
    assert _check(good, K=1, n_init=1, max_iter=1)[0] == _lib.IDC_OK
    assert _check(good, K=32, n_init=16)[0] == _lib.IDC_OK
    for kw in ({"K": 0}, {"K": 33}, {"n_init": 0}, {"n_init": 17}, {"max_iter": 0}):
        rc, msg = _check(good, **kw)
        assert rc == _lib.ERR_ARG and "K <= 32" in msg, kw
    for bad, what in (((3, 0, 0), "image 3"), ((-1, 0, 0), "image -1"), ((0, 16, 0), "pixel (16,0)"),
                      ((0, -1, 0), "pixel (-1,0)"), ((0, 0, 12), "pixel (0,12)"), ((0, 0, -1), "pixel (0,-1)")):
        rc, msg = _check(good + [bad] + good)
        assert rc == _lib.ERR_ARG and "query 3" in msg and what in msg, (bad, msg)
    rc, msg = _check(good, head=0)                                 # a context without the 529-bin head
    assert rc == _lib.ERR_STATE and "IDC_FLAG_DIST" in msg
    assert _check(good, n_img=0)[0] == _lib.ERR_STATE              # no forward yet
    assert _check(good, n_img=2)[0] == _lib.ERR_ARG                # image 2 is not in a 2-image forward
    assert _check(np.zeros((0, 3)))[0] == _lib.ERR_ARG             # q = 0
    assert _check(np.zeros((_lib.MAX_RECCS_QUERIES + 1, 3)))[0] == _lib.ERR_ARG
    assert _check(np.zeros((_lib.MAX_RECCS_QUERIES, 3)))[0] == _lib.IDC_OK
    P = ctypes.c_void_p(16)                                        # never dereferenced
    assert _lib.load().idc_ab_reccs_batch(None, 1, P, 5, 100, 8, None, P, None, None, None, None) == _lib.ERR_ARG


def _loc_answer(loc, K):
    """A deterministic stand-in for get_ab_reccs at loc: (centres [K,2], conf [K]) float64 with many digits."""
    h, w = int(loc[0]), int(loc[1])
    k = np.arange(K, dtype=np.float64)
    centers = np.stack([h / 7.0 + k * 1.0000123456, -w / 3.0 - k * 0.98765432], 1)
    conf = (K - k) / (K * (K + 1) / 2.0) + 1e-7 * h
    return centers, conf


class FakeDevice(object):
    """Records what it is given; a photo's result carries its tag, its suggestions _loc_answer of each point."""

    def __init__(self):
        self.log, self.pending = [], 0

    def submit(self, imgs, hints, glob, psnr, points=None, K=0):
        tags = [int(a[0, 0, 0]) for a in imgs]
        self.log.append((tags, None if hints is None else [None if h is None else len(h) for h in hints],
                         None if points is None else [p.tolist() for p in points], K, psnr))
        self.pending += 1
        assert self.pending <= 2
        return tags, points, K

    def collect(self, token):
        tags, points, K = token
        self.pending -= 1
        out = []
        for t, p in zip(tags, points):
            r = photos.PhotoResult(np.full((2, 3, 3), t, np.uint8), None, None, None)
            ans = [_loc_answer(l, K) for l in p]
            out.append(photos.SuggestResult(r, np.array([a for a, _ in ans]).reshape(-1, K, 2),
                                            np.array([c for _, c in ans]).reshape(-1, K)))
        return out

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


def test_suggest_switch_and_argument_errors_before_device_work():
    with pytest.raises(ValueError):
        FakeColorizer(None, Xd=64, batch=4, suggest=True, caffe=True)
    with pytest.raises(ValueError):
        FakeColorizer(None, Xd=64, batch=4, suggest=True, global_hints=True)
    with pytest.raises(ValueError):                                # suggest needs suggest=True
        FakeColorizer(None, Xd=64, batch=4).suggest([_img(0)], None, [np.zeros((1, 2), int)])
    pc = FakeColorizer(None, Xd=64, batch=4, suggest=True)
    assert pc.dist
    imgs = [_img(1), _img(2)]
    ok = [np.array([[0, 0], [63, 63]]), np.zeros((0, 2), int)]
    for kw in ({"K": 0}, {"K": 33}, {"K": 2.0}, {"K": True},
               {"points": ok[:1]},                                                     # one list per photo
               {"points": [np.array([[0, 64]]), ok[1]]}, {"points": [np.array([[-1, 0]]), ok[1]]},
               {"points": [np.array([[0.5, 1.0]]), ok[1]]}, {"points": [np.array([1, 2, 3]), ok[1]]},
               {"hints": [None]}):
        args = {"hints": None, "points": ok, "K": 5}
        args.update(kw)
        with pytest.raises(ValueError):
            pc.suggest(imgs, **args)
    with pytest.raises(ValueError):
        pc.suggest([np.zeros((4, 4), np.uint8), _img(2)], None, ok)
    assert pc._backend.log == []
    pc.close()


def test_suggest_layout_and_order():
    imgs = [_img(i) for i in range(7)]
    rs = np.random.RandomState(3)
    points = [rs.randint(0, 64, (int(rs.randint(0, 5)), 2)) for _ in imgs]
    hints = [None if i == 2 else CI.hints_from_points([((5, 6), 1, (10., -20.))] * (i + 1), 64) for i in range(7)]
    pc = FakeColorizer(None, Xd=64, batch=3, suggest=True)
    res = list(pc.suggest(imgs, hints, points, K=4, psnr=True))
    assert [e[0] for e in pc._backend.log] == [[0, 1, 2], [3, 4, 5], [6]]
    assert [e[1] for e in pc._backend.log] == [[1, 2, None], [4, 5, 6], [7]]
    assert all(e[3] == 4 and e[4] is True for e in pc._backend.log)
    assert [p for e in pc._backend.log for p in e[2]] == [p.tolist() for p in points]
    for i, r in enumerate(res):
        assert isinstance(r, photos.SuggestResult) and int(r.result.fullres[0, 0, 0]) == i
        assert r.centers.shape == (len(points[i]), 4, 2) and r.conf.shape == (len(points[i]), 4)
        for k, loc in enumerate(points[i]):
            c, f = _loc_answer(loc, 4)
            assert np.array_equal(r.centers[k], c) and np.array_equal(r.conf[k], f)
    pc.close()


def test_cli_hints_dir_parsing():
    base = ["--color_model", "m.pth", "--image_dir", "d", "--out", "o"]
    a = cli.parse_args(base + ["--hints_dir", "h", "--suggest", "9"])
    assert a.hints_dir == "h" and a.suggest == 9
    assert cli.parse_args(base).hints_dir == ""
    for bad in (["--hints_dir", "h", "--reveal_sweep", "0,1"], ["--hints_dir", "h", "--global_hints", "--glob_sweep"],
                ["--hints_dir", "h", "--global_hints", "--glob_ref", "r.jpg"],
                ["--hints_dir", "h", "--suggest", "5", "--global_hints"], ["--hints_dir", "h", "--suggest", "5", "--caffe"]):
        with pytest.raises(SystemExit):
            cli.parse_args(base + bad)
    with pytest.raises(SystemExit):                                 # needs --image_dir
        cli.parse_args(["--color_model", "m.pth", "--hints_dir", "h"])


HINTS_A = [{"loc": [10, 20], "size": 2, "ab": [23, -69]}, {"loc": [40, 5], "rgb": [200, 30, 60]}]
HINTS_C = [{"loc": [63, 0], "size": 0, "ab": [-5.5, 7.25]}]


def _folder(tmp_path):
    import cv2
    import torch
    d, hd = tmp_path / "photos", tmp_path / "hints"
    d.mkdir()
    hd.mkdir()
    for i, name in enumerate(("b.png", "a.png", "c.jpg")):
        cv2.imwrite(str(d / name), _img(10 * (i + 1)))
    (hd / "a.json").write_text(json.dumps(HINTS_A))
    (hd / "c.json").write_text(json.dumps(HINTS_C))
    (hd / "b.png.json").write_text(json.dumps(HINTS_C))         # not <stem>.json: b has no hints
    torch.save({"model1.0.weight": torch.ones((64, 4, 3, 3))}, str(tmp_path / "m.pth"))
    return d, hd


def test_cli_hints_dir_matching_and_suggestions(tmp_path, monkeypatch):
    d, hd = _folder(tmp_path)
    seen = {}

    class Fake(FakeColorizer):
        def __init__(self, sd, **kw):
            seen["kw"] = kw
            FakeColorizer.__init__(self, sd, **kw)

        def colorize(self, paths, hints=None, glob=None, psnr=False):
            seen["colorize"] = ([os.path.basename(p) for p in paths], hints, glob, psnr)
            return iter(photos.PhotoResult(np.zeros((20, 30, 3), np.uint8), None, None, 2.5) for _ in paths)

    monkeypatch.setattr(photos, "PhotoColorizer", Fake)
    out = tmp_path / "out"
    base = ["--color_model", str(tmp_path / "m.pth"), "--image_dir", str(d), "--hints_dir", str(hd), "--load_size", "64"]
    # without --suggest: colorize(hints=...), the lists matched by stem, [] where HDIR has no <stem>.json
    assert cli.main(base + ["--out", str(out), "--psnr"]) == 0
    names, hints, glob, psnr = seen["colorize"]
    assert names == ["a.png", "b.png", "c.jpg"] and glob is None and psnr
    assert "suggest" not in seen["kw"]
    want = [cli.hint_rects(HINTS_A, 64), cli.hint_rects([], 64), cli.hint_rects(HINTS_C, 64)]
    assert len(hints) == 3 and all(np.array_equal(h, w) for h, w in zip(hints, want))
    assert hints[1].shape == (0,)
    assert sorted(os.listdir(str(out))) == ["a.png", "b.png", "c.png", "psnr.csv"]
    # with --suggest: PhotoColorizer(suggest=True).suggest at every hint's loc; JSON only for photos with hints
    out2 = tmp_path / "out2"
    assert cli.main(base + ["--out", str(out2), "--suggest", "3"]) == 0
    assert seen["kw"]["suggest"] is True
    assert sorted(os.listdir(str(out2))) == ["a.png", "a_suggestions.json", "b.png", "c.png", "c_suggestions.json"]
    got = json.loads((out2 / "a_suggestions.json").read_text())
    assert [e["loc"] for e in got] == [h["loc"] for h in HINTS_A]
    c, f = _loc_answer(HINTS_A[1]["loc"], 3)
    assert got[1]["ab"] == np.round(c, 3).tolist() and got[1]["conf"] == np.round(f, 5).tolist()


class _FakeWrapper(object):
    """The single-image wrappers, as far as the command line's single-image mode uses them; get_ab_reccs answers
    _loc_answer, like the fake folder device."""
    X = 64

    def __init__(self, Xd=256, maskcent=False):
        self.act_ranges = None

    def prep_net(self, **kw):
        pass

    def load_image(self, path):
        X = self.X
        self.img_rgb, self.img_l = np.zeros((X, X, 3), np.uint8), np.zeros((1, X, X))
        self.input_ab, self.input_mask = np.zeros((2, X, X)), np.zeros((1, X, X))

    def share_trunk(self, other):
        return self

    def set_image(self, rgb):
        pass

    def net_forward_hints(self, rects):
        return np.zeros((self.X, self.X, 3), np.uint8)

    def get_ab_reccs(self, h, w, K=5, return_conf=False):
        return _loc_answer((h, w), K)

    get_img_fullres = get_input_img_fullres = get_input_img = get_sup_img = \
        lambda self: np.zeros((self.X, self.X, 3), np.uint8)


def test_folder_and_single_image_json_share_one_formatter(tmp_path, monkeypatch):
    d, hd = _folder(tmp_path)
    monkeypatch.setattr(photos, "PhotoColorizer", FakeColorizer)
    monkeypatch.setattr(CI, "ColorizeImageB200", _FakeWrapper)
    monkeypatch.setattr(CI, "ColorizeImageB200Dist", _FakeWrapper)
    calls = []
    real = cli.write_suggestions

    def spy(path, hints, centers, conf):
        calls.append(os.path.basename(path))
        return real(path, hints, centers, conf)

    monkeypatch.setattr(cli, "write_suggestions", spy)
    m = str(tmp_path / "m.pth")
    assert cli.main(["--color_model", m, "--image_dir", str(d), "--hints_dir", str(hd), "--out", str(tmp_path / "o"),
                     "--load_size", "64", "--suggest", "4"]) == 0
    one = tmp_path / "one"
    assert cli.main(["--color_model", m, "--image_file", str(d / "a.png"), "--hints", str(hd / "a.json"),
                     "--out", str(one), "--load_size", "64", "--suggest", "4"]) == 0
    assert calls == ["a_suggestions.json", "c_suggestions.json", "suggestions.json"]
    folder = (tmp_path / "o" / "a_suggestions.json").read_text()
    assert folder == (one / "suggestions.json").read_text()
    # the format itself: loc as given, ab to 3 places, conf to 5, indent 1
    c, f = _loc_answer(HINTS_A[0]["loc"], 4)
    assert json.loads(folder)[0] == {"loc": [10, 20], "ab": np.round(c, 3).tolist(), "conf": np.round(f, 5).tolist()}
    assert folder.startswith('[\n {\n  "loc": [\n   10,')
