"""CPU: the batch logic of PhotoColorizer (cutting, order, bounded read-ahead, input checks) on a fake device, and the
argument checks of the batched-photo C ABI entries, which return IDC_ERR_ARG before any device call."""
import ctypes
import os

import numpy as np
import pytest

from interactive_deep_colorization_b200 import _lib, photos
from interactive_deep_colorization_b200.colorize_image import HINT_LIST_DTYPE


class FakeDevice(object):
    """Records the batches it is given; the 'results' identify each photo by its first pixel."""

    def __init__(self, log):
        self.log, self.pending = log, 0

    def submit(self, imgs, hints, glob, psnr):
        self.log.append(("submit", [a.shape for a in imgs], None if hints is None else [None if h is None else len(h) for h in hints]))
        self.pending += 1
        assert self.pending <= 2, "more than two batches in flight"
        return imgs, psnr

    def collect(self, token):
        imgs, psnr = token
        self.pending -= 1
        self.log.append(("collect", len(imgs)))
        return [photos.PhotoResult(a, None, None, 1.0 if psnr else None) for a in imgs]

    def discard(self, token):
        self.pending -= 1
        self.log.append(("discard", len(token[0])))

    def close(self):
        assert self.pending == 0


class FakeColorizer(photos.PhotoColorizer):
    def _make_backend(self, state_dict):
        self.log = []
        return FakeDevice(self.log)


def _img(h, w, tag):
    a = np.zeros((h, w, 3), np.uint8)
    a[0, 0, 0] = tag
    return a


def _hints(k):
    return np.zeros(k, HINT_LIST_DTYPE)


def test_cut_by_count_bytes_and_hints():
    items = [(10, 0, i) for i in range(7)]
    assert list(photos.cut_batches(items, 3, 1000)) == [[0, 1, 2], [3, 4, 5], [6]]
    # byte budget 25: 10 + 10 fits, a third does not; a 40-byte item over the budget goes alone
    items = [(10, 0, 0), (10, 0, 1), (10, 0, 2), (40, 0, 3), (5, 0, 4)]
    assert list(photos.cut_batches(items, 8, 25)) == [[0, 1], [2], [3], [4]]
    # hint budget 1024 per batch
    items = [(1, 600, 0), (1, 424, 1), (1, 1, 2), (1, 1024, 3), (1, 0, 4)]
    assert list(photos.cut_batches(items, 8, 100)) == [[0, 1], [2], [3, 4]]
    assert list(photos.cut_batches([], 4, 10)) == []


def test_results_in_input_order_and_batches():
    pc = FakeColorizer(None, Xd=64, batch=3, max_batch_bytes=1 << 20, workers=3)
    imgs = [_img(5 + i, 7 + 2 * i, i) for i in range(8)]
    out = list(pc.colorize(imgs, psnr=True))
    assert [int(r.fullres[0, 0, 0]) for r in out] == list(range(8))
    assert all(r.psnr == 1.0 for r in out)
    subs = [e for e in pc.log if e[0] == "submit"]
    assert [len(e[1]) for e in subs] == [3, 3, 2]
    # batch k-1 is collected after batch k was submitted: the device always has the next batch queued
    assert [e[0] for e in pc.log] == ["submit", "submit", "collect", "submit", "collect", "collect"]


def test_hint_budget_cuts_batches():
    pc = FakeColorizer(None, Xd=64, batch=8)
    imgs = [_img(8, 8, i) for i in range(4)]
    out = list(pc.colorize(imgs, hints=[_hints(600), _hints(500), None, _hints(3)]))
    assert len(out) == 4
    subs = [e for e in pc.log if e[0] == "submit"]
    assert [e[2] for e in subs] == [[600], [500, None, 3]]


def test_byte_budget_and_oversized_photo():
    pc = FakeColorizer(None, Xd=64, batch=8, max_batch_bytes=3 * 100 * 3)
    imgs = [_img(10, 10, 0), _img(10, 10, 1), _img(10, 10, 2), _img(40, 40, 3), _img(10, 10, 4)]
    out = list(pc.colorize(imgs))
    assert [int(r.fullres[0, 0, 0]) for r in out] == [0, 1, 2, 3, 4]
    assert [len(e[1]) for e in pc.log if e[0] == "submit"] == [3, 1, 1]


def test_read_ahead_is_bounded():
    loaded, consumed = [], []

    def load(i):
        loaded.append(i)
        return i

    for r in photos.read_ahead(range(1000), load, depth=5, workers=3):
        consumed.append(r)
        assert len(loaded) <= len(consumed) + 5
        if len(consumed) == 20:
            break
    assert consumed == list(range(20))
    assert len(loaded) <= 25


def test_pipeline_reads_a_bounded_number_of_photos(tmp_path):
    cv2 = pytest.importorskip("cv2")
    paths = []
    for i in range(12):
        p = str(tmp_path / ("p%02d.png" % i))
        cv2.imwrite(p, _img(6, 9, i)[:, :, ::-1])
        paths.append(p)
    pc = FakeColorizer(None, Xd=64, batch=2, readahead=3, workers=2)
    reads = []
    real = photos.read_photo
    photos.read_photo = lambda p: (reads.append(p), real(p))[1]
    try:
        it = pc.colorize(paths)
        first = next(it)
        # first result: batches 0 and 1 submitted (4 photos) + at most readahead (3) more decoded
        assert len(reads) <= 4 + 3
        rest = list(it)
    finally:
        photos.read_photo = real
    got = [first] + rest
    assert [int(r.fullres[0, 0, 0]) for r in got] == list(range(12))   # written as BGR, read back as RGB


def test_abandoned_iteration_leaves_no_batch_in_flight(tmp_path):
    """A peek, a break or a photo that fails to read part way through: the batch in flight is waited for, so the next
    colorize() on the same colorizer never has more than two batches in flight."""
    pc = FakeColorizer(None, Xd=64, batch=2)
    imgs = [_img(6, 6, i) for i in range(9)]
    assert int(next(pc.colorize(imgs)).fullres[0, 0, 0]) == 0
    assert pc._backend.pending == 0 and pc.log[-1][0] == "discard"
    for r in pc.colorize(imgs):
        if int(r.fullres[0, 0, 0]) == 4:
            break
    assert pc._backend.pending == 0
    out = list(pc.colorize(imgs))
    assert [int(r.fullres[0, 0, 0]) for r in out] == list(range(9))
    pytest.importorskip("cv2")
    bad = imgs[:5] + [str(tmp_path / "missing.png")] + imgs[5:]
    got = []
    with pytest.raises(IOError):
        for r in pc.colorize(bad):
            got.append(int(r.fullres[0, 0, 0]))
    # photo 5 is read while batch [2, 3] is in flight: that batch is discarded, the error surfaces after [0, 1]
    assert got == [0, 1] and pc._backend.pending == 0 and pc.log[-1] == ("discard", 2)
    assert [int(r.fullres[0, 0, 0]) for r in pc.colorize(imgs)] == list(range(9))


def _folder(tmp_path, names):
    cv2 = pytest.importorskip("cv2")
    d = tmp_path / "in"
    d.mkdir()
    for i, name in enumerate(names):
        cv2.imwrite(str(d / name), _img(5 + i, 9, 10 + i)[:, :, ::-1])
    return d


def _front_end(monkeypatch, tmp_path, d, *extra):
    import torch
    import ideepcolor_b200
    sd = tmp_path / "sd.pth"
    torch.save({}, str(sd))
    monkeypatch.setattr(photos, "PhotoColorizer", FakeColorizer)
    out = tmp_path / "out"
    return ideepcolor_b200.main(["--color_model", str(sd), "--image_dir", str(d), "--out", str(out), "--load_size", "64"]
                                + list(extra)), out


def test_image_dir_front_end(monkeypatch, tmp_path):
    """--image_dir writes OUT/<stem>.png per photo (the fake device returns each photo unchanged) and psnr.csv."""
    cv2 = pytest.importorskip("cv2")
    d = _folder(tmp_path, ["b.png", "a.png", "c.bmp"])
    (d / "notes.txt").write_text("not a photo")
    rc, out = _front_end(monkeypatch, tmp_path, d, "--batch", "2", "--psnr")
    assert rc == 0
    assert sorted(os.listdir(str(out))) == ["a.png", "b.png", "c.png", "psnr.csv"]
    for name in ("a.png", "b.png", "c.bmp"):
        want = cv2.imread(str(d / name), 1)
        got = cv2.imread(str(out / (os.path.splitext(name)[0] + ".png")), 1)
        assert np.array_equal(got, want), name
    assert (out / "psnr.csv").read_text().splitlines() == ["image,psnr", "a.png,1", "b.png,1", "c.bmp,1"]


def test_image_dir_refuses_shared_stems(monkeypatch, tmp_path):
    d = _folder(tmp_path, ["a.png", "a.bmp", "b.png"])
    rc, out = _front_end(monkeypatch, tmp_path, d)
    assert rc == 2 and not out.exists()


def test_rejections_before_device_work():
    pc = FakeColorizer(None, Xd=64, batch=4)
    good = _img(8, 8, 0)
    bad = [np.zeros((8, 8, 3), np.float32), np.zeros((8, 8), np.uint8), np.zeros((8, 8, 4), np.uint8),
           np.zeros((0, 8, 3), np.uint8), np.zeros((10001, 2, 3), np.uint8), np.zeros((2, 10001, 3), np.uint8), 7]
    for b in bad:
        with pytest.raises(ValueError):
            pc.colorize([good, b])
    with pytest.raises(ValueError):
        pc.colorize([good], hints=[_hints(1025)])
    with pytest.raises(ValueError):
        pc.colorize([good, good], hints=[_hints(1)])
    with pytest.raises(ValueError):
        pc.colorize([good], glob=[np.zeros(316)])               # global_hints=False
    assert pc.log == []
    assert max(photos.check_photo(np.zeros((10000, 3, 3), np.uint8)).shape) == 10000
    with pytest.raises(ValueError):
        FakeColorizer(None, Xd=60)
    with pytest.raises(ValueError):
        FakeColorizer(None, batch=_lib.MAX_PHOTOS + 1)


def test_unreadable_path_raises(tmp_path):
    pytest.importorskip("cv2")
    pc = FakeColorizer(None, Xd=64, batch=4)
    with pytest.raises(IOError):
        list(pc.colorize([str(tmp_path / "missing.png")]))
    assert pc.log == []


# ---- C ABI argument checks (no GPU needed: IDC_ERR_ARG comes before any device call) ----
def _table(*hw, offs=None):
    t = np.zeros(len(hw), _lib.PHOTO_DTYPE)
    off = 0
    for i, (h, w) in enumerate(hw):
        t[i] = (off if offs is None else offs[i], h, w)
        off += h * w
    return t


def test_photo_abi_argument_checks():
    lib = _lib.load()
    P = ctypes.c_void_p(16)          # never dereferenced: every call below fails its checks first
    t = _table((10, 12), (5, 7))
    tp = t.ctypes.data
    assert lib.idc_photo_prep(0, 0, tp, P, 64, P, None, None) == -1                    # n < 1
    assert lib.idc_photo_prep(0, _lib.MAX_PHOTOS + 1, tp, P, 64, P, None, None) == -1
    assert lib.idc_photo_prep(0, 2, None, P, 64, P, None, None) == -1                  # NULL table
    assert lib.idc_photo_prep(0, 2, tp, None, 64, P, None, None) == -1                 # NULL src
    assert lib.idc_photo_prep(0, 2, tp, P, 64, None, None, None) == -1                 # NULL L_mc
    assert lib.idc_photo_prep(0, 2, tp, P, 60, P, None, None) == -1                    # X not a multiple of 8
    assert lib.idc_photo_prep(0, 2, tp, P, 0, P, None, None) == -1
    assert lib.idc_photo_prep(0, 2, tp, P, _lib.MAX_PHOTO_X + 8, P, None, None) == -1   # X * X * 3 past 32 bits
    assert lib.idc_photo_render(0, 2, tp, P, _lib.MAX_PHOTO_X + 8, P, P, None) == -1
    for side in ((1, _lib.MAX_PHOTO_SIDE + 1), (_lib.MAX_PHOTO_SIDE + 1, 1)):
        big = _table(side)
        assert lib.idc_photo_prep(0, 1, big.ctypes.data, P, 64, P, None, None) == -1
        assert lib.idc_photo_render(0, 1, big.ctypes.data, P, 64, P, P, None) == -1
    assert lib.idc_hint_raster(0, 1, 65536, 32768, 0, P, P, P, None) == -1             # h * w past the int index
    for bad in (_table((0, 12), (5, 7)), _table((10, 12), (5, 0)), _table((10, 12), (5, 7), offs=[0, 119]),
                _table((10, 12), (5, 7), offs=[-1, 200])):
        assert lib.idc_photo_prep(0, 2, bad.ctypes.data, P, 64, P, None, None) == -1
        assert lib.idc_photo_render(0, 2, bad.ctypes.data, P, 64, P, P, None) == -1
    assert lib.idc_photo_render(0, 0, tp, P, 64, P, P, None) == -1
    assert lib.idc_photo_render(0, 2, tp, None, 64, P, P, None) == -1
    assert lib.idc_photo_render(0, 2, tp, P, 64, None, P, None) == -1                  # NULL lab
    assert lib.idc_photo_render(0, 2, tp, P, 64, P, None, None) == -1                  # NULL out
    assert lib.idc_photo_render(0, 2, tp, P, 12, P, P, None) == -1
    assert lib.idc_hint_raster(0, 0, 64, 64, 0, P, P, P, None) == -1
    assert lib.idc_hint_raster(0, 1, 0, 64, 0, P, P, P, None) == -1
    assert lib.idc_hint_raster(0, 1, 64, 0, 0, P, P, P, None) == -1
    assert lib.idc_hint_raster(0, 1, 64, 64, _lib.MAX_HINTS + 1, P, P, P, None) == -1
    assert lib.idc_hint_raster(0, 1, 64, 64, -1, P, P, P, None) == -1
    for k in range(3):
        args = [P, P, P]
        args[k] = None
        assert lib.idc_hint_raster(0, 1, 64, 64, 0, *args, None) == -1
    assert lib.idc_rgb_sse(0, 0, 8, 8, P, P, P, None) == -1
    assert lib.idc_rgb_sse(0, 1, 0, 8, P, P, P, None) == -1
    assert lib.idc_rgb_sse(0, 1, 8, 0, P, P, P, None) == -1
    for k in range(3):
        args = [P, P, P]
        args[k] = None
        assert lib.idc_rgb_sse(0, 1, 8, 8, *args, None) == -1


def test_photo_dtype_matches_header():
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "idc_b200.h")).read()
    assert "typedef struct { int64_t off; int32_t h, w; } idc_photo;" in src
    assert "#define IDC_MAX_PHOTOS %d" % _lib.MAX_PHOTOS in src
    assert "#define IDC_MAX_PHOTO_SIDE %d" % _lib.MAX_PHOTO_SIDE in src
    assert "#define IDC_MAX_PHOTO_X %d" % _lib.MAX_PHOTO_X in src
    assert _lib.PHOTO_DTYPE.itemsize == 16
