"""GPU: reveal sweeps (photos.PhotoColorizer.reveal_sweep; idc_hint_fill_mean + idc_hint_raster) on ragged photo sets.
The hint planes against numpy painting of the same points (put_point's slice assignment) with sequential float64
means, the sweep against LhnContext.forward_device in the same batch layout, against the FP32 oracle and the
single-image wrapper, and get_result_PSNR."""
import cv2
import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import _lib, photos, prepost
from interactive_deep_colorization_b200 import colorize_image as CI
from oracle import color_ref, synth
from tests import util

pytestmark = pytest.mark.gpu
TOL_AB = 1e-3
SIZES = [(507, 600), (256, 256), (8, 8), (1, 300), (513, 1023), (300, 1), (600, 507)]
LEVELS = (0, 1, 2, 5, 50, 1024)       # 1024 points overlap heavily at 64^2
BATCH = 12                            # two photos per device pass, a short last pass


def _photo(H, W, seed):
    """A seeded synthetic photo: a cubic up-sample of coarse noise plus fine noise, so both smooth and busy regions."""
    rs = np.random.RandomState(seed)
    coarse = rs.randint(0, 256, (max(H // 48, 2), max(W // 48, 2), 3)).astype(np.uint8)
    img = cv2.resize(coarse, (W, H), interpolation=cv2.INTER_CUBIC).astype(np.int16)
    img += rs.randint(-12, 13, (H, W, 3)).astype(np.int16)
    return np.clip(img, 0, 255).astype(np.uint8)


@pytest.fixture(scope="module")
def photo_set():
    return [_photo(h, w, 30 + i) for i, (h, w) in enumerate(SIZES)]


@pytest.fixture(scope="module")
def sd():
    return synth.torch_state_dict(1234)


def _mean32(plane, y0, x0, P):
    """float32 of the float64 mean of plane[y0:y0+P, x0:x0+P] summed sequentially in row-major order, and that mean."""
    v = plane[y0:y0 + P, x0:x0 + P].ravel()
    m = np.cumsum(v)[-1] / v.size
    return np.float32(m), m


def _paint(lab, pts):
    """put_point for each point in order: (ab [2,X,X], mask [1,X,X]) float32, (a, b) float64 means per point."""
    X = lab.shape[-1]
    ab, mask = np.zeros((2, X, X), np.float32), np.zeros((1, X, X), np.float32)
    means = np.zeros((len(pts), 2))
    for k, (y0, x0, P) in enumerate(pts):
        (a, ma), (b, mb) = _mean32(lab[1], y0, x0, P), _mean32(lab[2], y0, x0, P)
        ab[0, y0:y0 + P, x0:x0 + P], ab[1, y0:y0 + P, x0:x0 + P] = a, b
        mask[0, y0:y0 + P, x0:x0 + P] = 1
        means[k] = ma, mb
    return ab, mask, means


def _single(photo, X):
    """load_image_gpu: (L_mc float32 [1,X,X], img_rgb [X,X,3], ground-truth Lab [3,X,X] of img_rgb)."""
    small, lab, _ = prepost.load_image_gpu(photo, X)
    return np.float32(lab[0] - 50)[None], small, lab


@pytest.mark.parametrize("X", [64, 256])
def test_fill_and_raster_equal_numpy_painting(photo_set, X):
    lib = _lib.load()
    imgs = photo_set[:4]
    n, L = len(imgs), len(LEVELS)
    table, src = photos.pack_photos(imgs)
    src = torch.from_numpy(src).cuda()
    L_mc = torch.empty((n, 1, X, X), device="cuda")
    rgb = torch.empty((n, X, X, 3), dtype=torch.uint8, device="cuda")
    lab = torch.empty((n, 3, X, X), dtype=torch.float64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert lib.idc_photo_prep(0, n, table.ctypes.data, src.data_ptr(), X, L_mc.data_ptr(), rgb.data_ptr(), st) == 0
    assert lib.idc_rgb2lab_f64(0, n, X, X, rgb.data_ptr(), lab.data_ptr(), st) == 0
    # blocks in the sweep's layout, with a stride that is not a multiple of 16 and stale colours to be overwritten
    pts = [photos.reveal_points(X, 1024, 11, i) for i in range(n)]
    stride = _lib.HINT_HDR_BYTES + 1024 * _lib.HINT_DTYPE.itemsize + 4
    host = np.zeros(n * L * stride, np.uint8)
    rects = np.zeros((n, 1024), _lib.HINT_DTYPE)
    p = np.stack(pts)
    rects["y0"], rects["x0"] = p[..., 0], p[..., 1]
    rects["y1"], rects["x1"] = p[..., 0] + p[..., 2] - 1, p[..., 1] + p[..., 2] - 1
    rects["a"], rects["b"] = 77.0, -77.0
    assert photos.pack_hints(rects, host, LEVELS, stride) == stride
    blocks = torch.from_numpy(host).cuda()
    N = n * L
    ab = torch.full((N, 2, X, X), 5.0, device="cuda")
    mask = torch.full((N, 1, X, X), 5.0, device="cuda")
    assert lib.idc_hint_fill_mean(0, N, L, X, lab.data_ptr(), blocks.data_ptr(), stride, st) == 0
    for b in range(N):
        assert lib.idc_hint_raster(0, 1, X, X, LEVELS[b % L], blocks.data_ptr() + b * stride, ab[b].data_ptr(),
                                   mask[b].data_ptr(), st) == 0
    torch.cuda.synchronize()
    ab, mask, filled = ab.cpu().numpy(), mask.cpu().numpy(), blocks.cpu().numpy().reshape(N, stride)
    lab, rgb = lab.cpu().numpy(), rgb.cpu().numpy()
    for i, a in enumerate(imgs):
        ref_lab = color_ref.rgb2lab_transpose(cv2.resize(a, (X, X)))
        for j, c in enumerate(LEVELS):
            b = i * L + j
            want_ab, want_mask, means = _paint(lab[i], pts[i][:c])
            assert np.array_equal(ab[b], want_ab), (X, i, c)
            assert np.array_equal(mask[b], want_mask), (X, i, c)
            got = filled[b, 16:16 + c * 28].view(_lib.HINT_DTYPE)
            assert np.array_equal(got["a"], np.float32(means[:, 0])) and np.array_equal(got["b"], np.float32(means[:, 1]))
            ref_means = np.array([[_mean32(ref_lab[k], y0, x0, P)[1] for k in (1, 2)] for y0, x0, P in pts[i][:c]])
            assert c == 0 or np.abs(means - ref_means).max() <= 1e-9, (X, i, c)
        assert np.array_equal(rgb[i], cv2.resize(a, (X, X)))
    # the 1024-point level paints many pixels more than once, so the order of painting mattered above
    assert (pts[0][:, 2].astype(int) ** 2).sum() > 1.3 * mask[L - 1].sum()


@pytest.mark.parametrize("X", [64, 256])
def test_sweep_equals_forward_on_painted_planes(photo_set, sd, X, tmp_path):
    pc = photos.PhotoColorizer(sd, Xd=X, batch=BATCH, maskcent=True)
    res = list(pc.reveal_sweep(photo_set, levels=LEVELS, seed=3))
    assert len(res) == len(photo_set)
    L = len(LEVELS)
    ctx = pc._backend.ctx
    singles = [_single(a, X) for a in photo_set]
    painted = {}
    per = BATCH // L
    for k in range(0, len(photo_set), per):                 # the batches reveal_sweep cut: 2, 2, 2, 1 photos
        idx = list(range(k, min(k + per, len(photo_set))))
        Ls, abs_, ms = [], [], []
        for i in idx:
            pts = photos.reveal_points(X, max(LEVELS), 3, i)
            assert np.array_equal(res[i].points, pts)
            for c in LEVELS:
                ab, m, _ = _paint(singles[i][2], pts[:c])
                painted[i, c] = ab, m
                Ls.append(singles[i][0])
                abs_.append(ab)
                ms.append(m)
        ref = ctx.forward_device(util.dev(np.stack(Ls)), util.dev(np.stack(abs_)), util.dev(np.stack(ms)), 0.5,
                                 want_rgb=True)
        torch.cuda.synchronize()
        ref_ab, ref_rgb = ref["ab"].cpu().numpy(), ref["rgb"].cpu().numpy()
        for jj, i in enumerate(idx):
            r = res[i]
            assert r.ab.shape == (L, 2, X, X) and r.rgb.shape == (L, X, X, 3) and r.psnr.shape == (L,)
            assert np.array_equal(r.ab, ref_ab[jj * L:(jj + 1) * L]), (X, i)
            assert np.array_equal(r.rgb, ref_rgb[jj * L:(jj + 1) * L]), (X, i)
            w = CI.ColorizeImageBase(Xd=X)
            w.img_rgb = singles[i][1]
            for j in range(L):
                assert r.psnr[j] == w.get_result_PSNR(r.rgb[j]), (X, i, LEVELS[j])
    # the hints reach the network: 50 points change every photo's result
    assert all(util.maxabs(r.ab[0], r.ab[4]) > 1e-2 for r in res)
    # two photos at levels 0 and 50 against the FP32 oracle and the single-image wrapper (batch-1 click plan)
    cm = CI.ColorizeImageB200(Xd=X, maskcent=True)
    cm.prep_net(state_dict=sd)
    for i in (0, 4):
        p = str(tmp_path / ("photo%d.png" % i))
        cv2.imwrite(p, photo_set[i][:, :, ::-1])
        cm.load_image(p)
        for j in (0, 4):
            ab, m = painted[i, LEVELS[j]]
            ref = util.oracle_forward(sd, singles[i][0][None], ab[None], m[None], 0.5)
            assert util.maxabs(res[i].ab[j], ref[0]) <= TOL_AB, (X, i, LEVELS[j])
            cm.net_forward(ab.astype(np.float64), m.astype(np.float64))
            assert util.maxabs(res[i].ab[j], cm.output_ab_raw) <= TOL_AB, (X, i, LEVELS[j])
            d = np.abs(res[i].rgb[j].astype(int) - cm.output_rgb.astype(int))
            assert d.max() <= 1 and (d > 0).mean() < 1e-3, (X, i, int(d.max()), float((d > 0).mean()))
    pc.close()


def test_sweep_is_deterministic_and_batch_independent(photo_set, sd):
    X, levels = 64, (0, 10, 100)
    imgs = photo_set[:5]
    pc = photos.PhotoColorizer(sd, Xd=X, batch=6)
    a = list(pc.reveal_sweep(imgs, levels=levels, seed=21))
    b = list(pc.reveal_sweep(imgs, levels=levels, seed=21))
    for r, s in zip(a, b):
        assert np.array_equal(r.psnr, s.psnr) and np.array_equal(r.ab, s.ab) and np.array_equal(r.rgb, s.rgb)
        assert np.array_equal(r.points, s.points)
    # colorize on the same colorizer still gives the zero-hint result of level 0
    plain = list(pc.colorize(imgs[:2]))
    assert util.maxabs(plain[0].ab, a[0].ab[0]) <= TOL_AB
    pc.close()
    pc = photos.PhotoColorizer(sd, Xd=X, batch=9)
    c = list(pc.reveal_sweep(imgs, levels=levels, seed=21))
    for r, s in zip(a, c):
        assert np.array_equal(r.points, s.points)
        assert util.maxabs(r.ab, s.ab) <= TOL_AB
    d = list(pc.reveal_sweep(imgs, levels=levels, seed=22))
    assert not np.array_equal(a[0].points, d[0].points)
    pc.close()
