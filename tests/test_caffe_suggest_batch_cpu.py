"""CPU: batched suggestions of the Caffe 313-bin head, host side -- the argument checks of idc_caffe313_reccs_batch
(the same code through its host-only hook, so nothing reaches a device), PhotoColorizer(caffe=True, caffe_dist=True)
and its suggest checks on a fake device, the query builder of both heads, and the command line's --caffe_dist."""
import ctypes

import numpy as np
import pytest
import torch

import ideepcolor_b200 as cli
from interactive_deep_colorization_b200 import _lib, photos
from tests.test_suggest_batch_cpu import FakeColorizer, _img, _loc_answer


def _check(q, S=0.2, K=5, max_iter=100, n_init=8, head=1, n_img=3, h=64, w=48):
    lib = _lib.load()
    qa = np.ascontiguousarray(q, np.int32).reshape(-1, 3)
    msg = ctypes.create_string_buffer(256)
    rc = lib.idc_caffe313_reccs_batch_check(head, n_img, h, w, qa.shape[0], qa.ctypes.data if qa.size else None, S, K,
                                            max_iter, n_init, msg, 256)
    return rc, msg.value.decode()


def test_abi_checks_use_the_full_resolution_grid():
    good = [(0, 0, 0), (2, 63, 47), (1, 17, 5)]                  # 64 x 48: the corner (63, 47) is a pixel
    assert _check(good) == (_lib.IDC_OK, "")
    for bad, what in (((0, 64, 0), "pixel (64,0)"), ((0, 0, 48), "pixel (0,48)"), ((0, -1, 0), "pixel (-1,0)"),
                      ((0, 0, -1), "pixel (0,-1)"), ((3, 0, 0), "image 3"), ((-1, 0, 0), "image -1")):
        rc, msg = _check(good + [bad])
        assert rc == _lib.ERR_ARG and "idc_caffe313_reccs_batch: query 3" in msg and what in msg, msg
        if what.startswith("pixel"):
            assert "64x48 grid" in msg, msg
    # the 529-bin check reads the same queries on the 16 x 12 grid of 4 x 4 cells and rejects both
    msg = ctypes.create_string_buffer(256)
    for t in ((0, 63, 0), (0, 0, 47)):
        qa = np.array([t], np.int32)
        assert _lib.load().idc_ab_reccs_batch_check(1, 3, 64, 48, 1, qa.ctypes.data, 5, 100, 8, msg, 256) == _lib.ERR_ARG


def test_abi_state_and_argument_errors():
    good = [(0, 1, 2)]
    rc, msg = _check(good, head=0)
    assert rc == _lib.ERR_STATE and "IDC_FLAG_CAFFE313" in msg
    rc, msg = _check(good, n_img=0)
    assert rc == _lib.ERR_STATE and "no forward" in msg
    for S in (float("nan"), float("inf"), float("-inf")):
        rc, msg = _check(good, S=S)
        assert rc == _lib.ERR_ARG and "S" in msg, S
    assert _check(good, S=0.0)[0] == _lib.IDC_OK
    assert _check(np.zeros((0, 3)))[0] == _lib.ERR_ARG
    assert _check(np.zeros((_lib.MAX_RECCS_QUERIES + 1, 3)))[0] == _lib.ERR_ARG
    assert _check(np.zeros((_lib.MAX_RECCS_QUERIES, 3)))[0] == _lib.IDC_OK
    for kw in ({"K": 0}, {"K": 33}, {"n_init": 0}, {"n_init": 17}, {"max_iter": 0}):
        rc, msg = _check(good, **kw)
        assert rc == _lib.ERR_ARG and "K <= 32" in msg, kw
    assert _check(good, K=32, n_init=16, max_iter=1)[0] == _lib.IDC_OK
    P = ctypes.c_void_p(16)                                        # never dereferenced
    assert _lib.load().idc_caffe313_reccs_batch(None, 1, P, 0.2, 5, 100, 8, P, None, None, None, None) == _lib.ERR_ARG


def test_query_builder_of_both_heads():
    points = [np.array([[0, 0], [63, 47], [5, 9]]), np.zeros((0, 2), np.int64), np.array([[17, 30]])]
    q313 = photos.reccs_queries(points, True)
    q529 = photos.reccs_queries(points, False)
    assert q313.dtype == q529.dtype == np.int32
    assert q313.tolist() == [[0, 0, 0], [0, 63, 47], [0, 5, 9], [2, 17, 30]]
    assert q529.tolist() == [[0, 0, 0], [0, 15, 11], [0, 1, 2], [2, 4, 7]]
    assert photos.reccs_queries([np.zeros((0, 2), np.int64)], True).shape == (0, 3)


def _caffe_sd(drop=None):
    sd = {"model1.0.weight": torch.ones((64, 4, 3, 3))}
    sd.update({k: torch.zeros(1) for k in photos.CAFFE313_KEYS if k != drop})
    return sd


def test_caffe_dist_switch_and_checkpoint():
    for kw in ({"caffe_dist": True}, {"caffe_dist": True, "global_hints": True},
               {"caffe_dist": True, "caffe": True, "global_hints": True}):
        with pytest.raises(ValueError):
            FakeColorizer(_caffe_sd(), Xd=64, batch=4, **kw)
    with pytest.raises(ValueError) as e:                           # suggest with caffe points to caffe_dist
        FakeColorizer(None, Xd=64, batch=4, suggest=True, caffe=True)
    assert "caffe_dist=True" in str(e.value)
    for key in ("caffe.pred_313.weight", "caffe.conv3_pred.bias"):
        with pytest.raises(ValueError) as e:
            FakeColorizer(_caffe_sd(drop=key), Xd=64, batch=4, caffe=True, caffe_dist=True)
        assert key in str(e.value)
    sd = _caffe_sd()
    pc = FakeColorizer(sd, Xd=64, batch=4, caffe=True, caffe_dist=True)
    assert pc.caffe_dist and not pc.dist
    assert "caffe.pts_in_hull" not in sd                            # the caller's checkpoint is left as it was
    pc.close()
    with pytest.raises(ValueError) as e:                           # suggest needs a head
        FakeColorizer(_caffe_sd(), Xd=64, batch=4, caffe=True).suggest([_img(0)], None, [np.zeros((1, 2), int)])
    assert "caffe_dist" in str(e.value)


def test_caffe_dist_suggest_errors_before_device_work_and_points_unchanged():
    pc = FakeColorizer(_caffe_sd(), Xd=64, batch=3, caffe=True, caffe_dist=True)
    imgs = [_img(1), _img(2)]
    ok = [np.array([[0, 0], [63, 63]]), np.zeros((0, 2), int)]
    for kw in ({"K": 0}, {"K": 33}, {"K": 2.0}, {"points": ok[:1]}, {"points": [np.array([[0, 64]]), ok[1]]},
               {"points": [np.array([[-1, 0]]), ok[1]]}, {"points": [np.array([[0.5, 1.0]]), ok[1]]},
               {"hints": [None]}):
        args = {"hints": None, "points": ok, "K": 5}
        args.update(kw)
        with pytest.raises(ValueError):
            pc.suggest(imgs, **args)
    assert pc._backend.log == []
    rs = np.random.RandomState(8)
    imgs = [_img(i) for i in range(5)]
    points = [rs.randint(0, 64, (int(rs.randint(0, 6)), 2)) for _ in imgs]
    res = list(pc.suggest(imgs, None, points, K=6))
    assert [p for e in pc._backend.log for p in e[2]] == [p.tolist() for p in points]   # full-resolution (h, w) as given
    for i, r in enumerate(res):
        assert int(r.result.fullres[0, 0, 0]) == i and r.centers.shape == (len(points[i]), 6, 2)
        for k, loc in enumerate(points[i]):
            assert np.array_equal(r.centers[k], _loc_answer(loc, 6)[0])
    pc.close()


def test_cli_caffe_dist_parsing():
    base = ["--color_model", "m.pth", "--image_dir", "d", "--out", "o"]
    a = cli.parse_args(base + ["--caffe", "--caffe_dist", "--hints_dir", "h", "--suggest", "9"])
    assert a.caffe_dist and a.caffe and a.suggest == 9
    assert not cli.parse_args(base).caffe_dist
    for bad in (["--caffe_dist", "--hints_dir", "h", "--suggest", "9"],                      # no --caffe
                ["--caffe", "--caffe_dist", "--hints_dir", "h"],                             # no --suggest
                ["--caffe", "--caffe_dist", "--suggest", "9"],                               # no --hints_dir
                ["--caffe", "--caffe_dist"],
                ["--caffe", "--caffe_dist", "--global_hints", "--hints_dir", "h", "--suggest", "9"],
                ["--caffe", "--hints_dir", "h", "--suggest", "9"]):                          # --caffe alone, as before
        with pytest.raises(SystemExit):
            cli.parse_args(base + bad)
    with pytest.raises(SystemExit):                                 # needs --image_dir
        cli.parse_args(["--color_model", "m.pth", "--caffe", "--caffe_dist", "--hints_dir", "h", "--suggest", "9"])


def test_cli_caffe_dist_builds_the_313_head_colorizer(tmp_path, monkeypatch):
    import json
    import cv2
    d, hd = tmp_path / "photos", tmp_path / "hints"
    d.mkdir()
    hd.mkdir()
    cv2.imwrite(str(d / "a.png"), _img(10))
    hints = [{"loc": [10, 20], "size": 2, "ab": [23, -69]}, {"loc": [63, 1], "ab": [5, 5]}]
    (hd / "a.json").write_text(json.dumps(hints))
    torch.save(_caffe_sd(), str(tmp_path / "m.pth"))
    seen = {}

    class Fake(FakeColorizer):
        def __init__(self, sd, **kw):
            seen["kw"] = kw
            FakeColorizer.__init__(self, sd, **kw)

    monkeypatch.setattr(photos, "PhotoColorizer", Fake)
    out = tmp_path / "out"
    assert cli.main(["--color_model", str(tmp_path / "m.pth"), "--image_dir", str(d), "--hints_dir", str(hd),
                     "--out", str(out), "--load_size", "64", "--caffe", "--caffe_dist", "--suggest", "4"]) == 0
    assert seen["kw"]["caffe"] is True and seen["kw"]["caffe_dist"] is True and "suggest" not in seen["kw"]
    got = json.loads((out / "a_suggestions.json").read_text())
    assert [e["loc"] for e in got] == [h["loc"] for h in hints]
    c, f = _loc_answer(hints[1]["loc"], 4)
    assert got[1]["ab"] == np.round(c, 3).tolist() and got[1]["conf"] == np.round(f, 5).tolist()
