"""GPU: batched photo colorization (photos.PhotoColorizer; idc_photo_prep / idc_photo_render / idc_hint_raster /
idc_rgb_sse) on ragged photo sets, against the single-image path: load_image_gpu, LhnContext.forward_device on the
same stacked inputs, get_img_fullres (prepost.fullres_rgb_gpu, scipy zoom + oracle/color_ref), the wrapper end to end,
and get_result_PSNR."""
import cv2
import numpy as np
import pytest
import torch
from scipy.ndimage import zoom

from interactive_deep_colorization_b200 import _lib, photos, prepost
from interactive_deep_colorization_b200 import colorize_image as CI
from oracle import color_ref, synth
from tests import util
from tests.test_gpu_configs import _glob_sd

pytestmark = pytest.mark.gpu
TOL_AB = 1e-3
# every resize path of prep (identity, exact-2x area, down- and up-sampling, single rows / columns), with the large
# photo last so that it forms the final, short batch of its own at batch = 4
SIZES = [(507, 600), (600, 507), (256, 256), (512, 512), (513, 1023), (8, 8), (1, 300), (300, 1), (3456, 5184)]
BATCH = 4


def _photo(H, W, seed):
    """A seeded synthetic photo: a cubic up-sample of coarse noise plus fine noise, so both smooth and busy regions."""
    rs = np.random.RandomState(seed)
    coarse = rs.randint(0, 256, (max(H // 48, 2), max(W // 48, 2), 3)).astype(np.uint8)
    img = cv2.resize(coarse, (W, H), interpolation=cv2.INTER_CUBIC).astype(np.int16)
    img += rs.randint(-12, 13, (H, W, 3)).astype(np.int16)
    return np.clip(img, 0, 255).astype(np.uint8)


@pytest.fixture(scope="module")
def photo_set():
    return [_photo(h, w, 10 + i) for i, (h, w) in enumerate(SIZES)]


@pytest.fixture(scope="module")
def sd():
    return synth.torch_state_dict(1234)


def _single(photo, X):
    """load_image_gpu of one photo: (L_mc float32 [1,X,X], img_rgb [X,X,3], DeviceLab of the full-resolution photo)."""
    small, lab, dlab = prepost.load_image_gpu(photo, X)
    return np.float32(lab[0] - 50)[None], small, dlab


def _pack(imgs):
    table = np.zeros(len(imgs), _lib.PHOTO_DTYPE)
    off = 0
    for i, a in enumerate(imgs):
        table[i] = (off, a.shape[0], a.shape[1])
        off += a.shape[0] * a.shape[1]
    return table, torch.from_numpy(np.concatenate([a.reshape(-1) for a in imgs])).cuda()


@pytest.mark.parametrize("X", [64, 256])
def test_photo_prep_equals_load_image(photo_set, X):
    lib = _lib.load()
    table, src = _pack(photo_set)
    n = len(photo_set)
    L = torch.empty((n, 1, X, X), dtype=torch.float32, device="cuda")
    rgb = torch.empty((n, X, X, 3), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert lib.idc_photo_prep(0, n, table.ctypes.data, src.data_ptr(), X, L.data_ptr(), rgb.data_ptr(), st) == 0
    L, rgb = L.cpu().numpy(), rgb.cpu().numpy()
    for i, a in enumerate(photo_set):
        l_ref, small, _ = _single(a, X)
        assert np.array_equal(rgb[i], cv2.resize(a, (X, X))), (i, a.shape)
        assert np.array_equal(small, rgb[i])
        assert np.array_equal(L[i], l_ref), (i, a.shape)


@pytest.mark.parametrize("X", [64, 256])
def test_batches_equal_single_image_path(photo_set, sd, X, tmp_path):
    pc = photos.PhotoColorizer(sd, Xd=X, batch=BATCH, maskcent=True)
    res = list(pc.colorize(photo_set, psnr=True))
    assert len(res) == len(photo_set)
    ctx = pc._backend.ctx
    singles = [_single(a, X) for a in photo_set]
    for k in range(0, len(photo_set), BATCH):            # batches of 4, 4 and a final 1, as colorize cut them
        idx = list(range(k, min(k + BATCH, len(photo_set))))
        n = len(idx)
        L = util.dev(np.stack([singles[i][0] for i in idx]))
        zero_ab, zero_m = torch.zeros((n, 2, X, X), device="cuda"), torch.zeros((n, 1, X, X), device="cuda")
        ref = ctx.forward_device(L, zero_ab, zero_m, 0.5, want_rgb=True)
        torch.cuda.synchronize()
        for j, i in enumerate(idx):
            assert np.array_equal(res[i].ab, ref["ab"][j].cpu().numpy()), (X, i)
            assert np.array_equal(res[i].rgb, ref["rgb"][j].cpu().numpy()), (X, i)
    for i, (a, r) in enumerate(zip(photo_set, res)):
        _, small, dlab = singles[i]
        assert r.fullres.shape == a.shape and r.fullres.dtype == np.uint8
        abq = prepost.rgb2lab_gpu(r.rgb)[1:]
        want = prepost.fullres_rgb_gpu(abq, dlab)
        assert np.array_equal(r.fullres, want), (X, i, a.shape, int((r.fullres != want).sum()))
        # get_result_PSNR on the pipeline's own img_rgb / output_rgb
        w = CI.ColorizeImageBase(Xd=X)
        w.img_rgb, w.output_rgb = small, r.rgb
        assert r.psnr == w.get_result_PSNR(), (X, i)
    # the render against scipy zoom + the colour oracle for two photos
    for i in (0, 4):
        a, r = photo_set[i], res[i]
        L_full = color_ref.rgb2lab_transpose(a)[[0]]
        abq = color_ref.rgb2lab_transpose(r.rgb)[1:]
        ab_full = zoom(abq, (1, a.shape[0] / X, a.shape[1] / X), order=1)
        rgb255 = np.clip(color_ref.lab2rgb(np.concatenate((L_full, ab_full)).transpose((1, 2, 0))), 0, 1) * 255
        util.assert_render_exact(r.fullres, rgb255.astype(np.uint8), rgb255, ("photo render", X, a.shape))
    # a few photos against the FP32 oracle network
    for i in (0, 5):
        ref = util.oracle_forward(sd, singles[i][0][None], np.zeros((1, 2, X, X), np.float32),
                                  np.zeros((1, 1, X, X), np.float32), 0.5)
        assert util.maxabs(res[i].ab, ref[0]) <= TOL_AB, (X, i)
    # end to end from PNG files against the wrapper's load_image + net_forward + get_img_fullres (batch-1 click plan)
    pick = [0, 4, 6, 7]
    paths = []
    for i in pick:
        p = str(tmp_path / ("photo%d.png" % i))
        cv2.imwrite(p, photo_set[i][:, :, ::-1])
        paths.append(p)
    from_files = list(pc.colorize(paths))
    cm = CI.ColorizeImageB200(Xd=X, maskcent=True)
    cm.prep_net(state_dict=sd)
    for p, i, r in zip(paths, pick, from_files):
        assert np.array_equal(r.fullres, res[i].fullres)                  # PNG is lossless: the same photo
        cm.load_image(p)
        cm.net_forward(np.zeros((2, X, X)), np.zeros((1, X, X)))
        want = cm.get_img_fullres()
        d = np.abs(r.fullres.astype(int) - want.astype(int))
        assert d.max() <= 1 and (d > 0).mean() < 1e-3, (X, i, int(d.max()), float((d > 0).mean()))
        assert util.maxabs(r.ab, cm.output_ab_raw) <= TOL_AB
    pc.close()


def test_hints_and_glob_equal_dense_forward(sd):
    X = 64
    sdg, _ = _glob_sd(sd)
    rs = np.random.RandomState(7)
    imgs = [_photo(h, w, 50 + i) for i, (h, w) in enumerate([(90, 70), (64, 64), (33, 200), (128, 128), (17, 5)])]
    hint_lists = []
    for i in range(len(imgs)):
        if i == 2:
            hint_lists.append(None)
            continue
        k = rs.randint(1, 12)
        h = np.zeros(k, CI.HINT_LIST_DTYPE)
        y0, x0 = rs.randint(-3, X, k), rs.randint(-3, X, k)
        h["y0"], h["x0"] = y0, x0
        h["y1"], h["x1"] = y0 + rs.randint(0, 6, k), x0 + rs.randint(0, 6, k)
        h["a"], h["b"] = rs.uniform(-100, 100, k), rs.uniform(-100, 100, k)
        hint_lists.append(h)
    globs = [rs.rand(316).astype(np.float32) for _ in imgs]
    pc = photos.PhotoColorizer(sdg, Xd=X, batch=3, maskcent=True, global_hints=True)
    res = list(pc.colorize(imgs, hints=hint_lists, glob=globs))
    ctx = pc._backend.ctx
    for k in (0, 3):
        idx = list(range(k, min(k + 3, len(imgs))))
        L = np.stack([_single(imgs[i], X)[0] for i in idx])
        planes = [CI.raster_hints(hint_lists[i] if hint_lists[i] is not None else [], X) for i in idx]
        ab = np.stack([p[0] for p in planes]).astype(np.float32)
        m = np.stack([p[1] for p in planes]).astype(np.float32)
        ref = ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5, glob=util.dev(np.stack([globs[i] for i in idx])),
                                 want_rgb=True)
        torch.cuda.synchronize()
        for j, i in enumerate(idx):
            assert np.array_equal(res[i].ab, ref["ab"][j].cpu().numpy()), i
            assert np.array_equal(res[i].rgb, ref["rgb"][j].cpu().numpy()), i
    # the hints and the vectors reach the network: without them the result differs
    plain = list(pc.colorize(imgs))
    assert all(util.maxabs(a.ab, b.ab) > 1e-2 for a, b in zip(res, plain))
    pc.close()


def test_abandoned_interleaved_and_oversized_batches(photo_set, sd):
    """An iteration left early never corrupts the next one; an iterator whose buffers a later run reused raises rather
    than return another batch's pixels; a photo over the byte budget grows its slot for that batch only."""
    X = 64
    imgs = photo_set[:8]
    pc = photos.PhotoColorizer(sd, Xd=X, batch=2)
    want = list(pc.colorize(imgs))
    assert np.array_equal(next(pc.colorize(imgs)).fullres, want[0].fullres)         # peek, then drop
    for i, r in enumerate(pc.colorize(imgs)):
        if i == 4:
            break
    it = pc.colorize(imgs)
    assert np.array_equal(next(it).fullres, want[0].fullres)
    for a, b in zip(pc.colorize(imgs), want):                                      # runs while `it` is suspended
        assert np.array_equal(a.fullres, b.fullres) and np.array_equal(a.ab, b.ab)
    with pytest.raises(RuntimeError):
        list(it)
    for a, b in zip(pc.colorize(imgs), want):
        assert np.array_equal(a.fullres, b.fullres) and np.array_equal(a.ab, b.ab)
    pc.close()

    budget = 1 << 20
    pc = photos.PhotoColorizer(sd, Xd=X, batch=4, max_batch_bytes=budget)
    seq = [photo_set[0], photo_set[-1], photo_set[1], photo_set[2]]     # 0.9 MB, 54 MB alone, then two one-photo batches
    res = list(pc.colorize(seq))
    assert [s["cap"] for s in pc._backend.slots] == [budget, budget]
    for a, r in zip(seq, res):
        want = prepost.fullres_rgb_gpu(prepost.rgb2lab_gpu(r.rgb)[1:], _single(a, X)[2])
        assert np.array_equal(r.fullres, want), a.shape
    pc.close()
