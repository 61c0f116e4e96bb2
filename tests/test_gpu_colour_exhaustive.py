"""GPU: every kernel that converts colour, on every 8-bit colour and on dense Lab grids, against the float64 colour
oracle (oracle/color_ref.py).

  a  all 2^24 colours through idc_rgb2lab_f64 (rgb_u8_to_lab), in ulps against the oracle
  b  the same 64 images through idc_photo_prep at the identity size: rgb passes through, L_mc = float32(L - 50)
  c  Lab grids (L knees and ends, ab past the gamut clip and the fz < 0 clamp, linear RGB at the 0.0031308 knee)
     through idc_lab2rgb_u8, idc_render_planes_u8, idc_cubic_lab2rgb_u8 and the quantised output_ab of a forward
  d  the round trip rgb -> Lab -> idc_photo_render, what colorize does with the quantised ab
  e  idc_global_stats and idc_global_stats_batch: the same histogram bit for bit, equal to a host evaluation of the
     cell rule on the device's own Lab, and the same bytes on every run

The oracle's matmul (numpy / BLAS) and CUDA's pow / cbrt round differently from the device in the last bits, so Lab
is compared in ulps; a uint8 render must equal the oracle's except where the oracle's float64 value lies within 1e-9
of a truncation edge (util.assert_render_exact).  The fixtures are plain functions of this file (tests/
test_colour_fixtures_cpu.py checks them without a device).  Host memory stays below ~2 GB: the oracle runs in chunks
of 2^22 pixels."""
import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import _lib, photos, prepost
from oracle import color_ref, synth
from tests import util

pytestmark = pytest.mark.gpu

N_IMG, SIDE = 64, 512                  # 2^24 colours = 64 images of 512 x 512
CHUNK_IMG = 16                         # oracle chunks of 16 images = 2^22 pixels
PTS = prepost.pts_in_hull()
# Lab is compared in ulps of each channel's scale (the factor in front of its last operation: L = 116 fy - 16,
# a = 500 (fx - fy), b = 200 (fy - fz)).  One ulp of fx moves a by 500 ulps of a value near 0, so ulps of |value|
# would measure the cancellation, not the arithmetic.  The bar holds a few last-bit differences of pow / cbrt and of
# the matrix sums.
LAB_SCALE = np.array([116.0, 500.0, 200.0])
LAB_ULPS = 8
# a colour whose X, Y or Z / white lies within this many ulps of lab_f's 0.008856 knee, or whose channel / 255 lies
# this close to srgb_inv_gamma's 0.04045 knee, could take the other branch on the device; such colours are listed
KNEE_ULPS = 64
GAMMA_KNEE, LINEAR_KNEE, FINV_KNEE = 0.0031308, 0.008856, 0.2068966
KNEE_SIDE_ULPS = 4                     # the linear-RGB knee points lie within 4 ulps either side of 0.0031308


# ---------------------------------------------------------------------------------------------------------------
# fixtures (plain functions, shared with the CPU test)
# ---------------------------------------------------------------------------------------------------------------
def all_colours():
    """uint8 [64,512,512,3]: colour i = r<<16 | g<<8 | b at image i >> 18, row (i >> 9) & 511, column i & 511."""
    i = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(i >> 16) & 255, (i >> 8) & 255, i & 255], axis=-1).astype(np.uint8)
    return rgb.reshape(N_IMG, SIDE, SIDE, 3)


def oracle_rgb2lab(imgs):
    """color_ref.rgb2lab of uint8 images [n,h,w,3], CHUNK_IMG images per call -> float64 [n,h,w,3]."""
    out = np.empty(imgs.shape, np.float64)
    for k in range(0, imgs.shape[0], CHUNK_IMG):
        out[k:k + CHUNK_IMG] = color_ref.rgb2lab(imgs[k:k + CHUNK_IMG])
    return out


def lab_ulps(got, want):
    """|got - want| in ulps of each channel's scale (LAB_SCALE), channel last."""
    return np.abs(np.asarray(got, np.float64) - want) / np.spacing(LAB_SCALE)


def grid_L():
    """L values of the Lab grid: both ends, the lab_finv knee (L = 116 * 0.2068966 - 16 = 8.0000056) and its
    neighbourhood, 99.999, and every 0.5 step of [0, 100]."""
    special = [0.0, 1e-6, 7.9999, 116.0 * FINV_KNEE - 16.0, 8.001, 99.999, 100.0]
    return np.unique(np.concatenate([special, np.arange(0, 201) * 0.5]))


def grid_ab():
    """a and b of the grid: [-128, 127.5] in 0.5 steps, past the gamut clip and deep into the fz < 0 clamp."""
    return np.arange(-256, 256) * 0.5


def grid_image(L):
    """Lab planes [3,512,512] float64 of one grid L: row i <-> a = grid_ab()[i], column j <-> b = grid_ab()[j]."""
    g = grid_ab()
    return np.stack([np.full((SIDE, SIDE), L), np.broadcast_to(g[:, None], (SIDE, SIDE)),
                     np.broadcast_to(g[None, :], (SIDE, SIDE))])


def knee_lab(n_base=48, seed=5):
    """float64 Lab points [K,3] whose linear RGB (color_ref.lab2linear) has one channel within KNEE_SIDE_ULPS ulps of
    0.0031308, on both sides, for each of R, G and B; the other channels are dark (< 0.02 linear).  Built from target
    linear colours: their Lab, then every offset of -3 ... 3 ulps in each of L, a and b, keeping the offsets that land
    within the window."""
    rs = np.random.RandomState(seed)
    t = np.spacing(GAMMA_KNEE)
    out = []
    for ch in range(3):
        lin = rs.uniform(0, 0.02, (n_base, 3))
        lin[:, ch] = GAMMA_KNEE
        xyz = (lin @ color_ref.XYZ_FROM_RGB.T) / color_ref.WHITE_D65_2
        f = np.where(xyz > LINEAR_KNEE, np.cbrt(xyz), 7.787 * xyz + 16.0 / 116.0)
        base = np.stack([116.0 * f[:, 1] - 16.0, 500.0 * (f[:, 0] - f[:, 1]), 200.0 * (f[:, 1] - f[:, 2])], -1)
        k = np.arange(-3, 4)
        off = np.stack(np.meshgrid(k, k, k, indexing="ij"), -1).reshape(-1, 3)
        pts = base[:, None, :] + off[None] * np.spacing(base)[:, None, :]
        pts = pts.reshape(-1, 3)
        v = color_ref.lab2linear(pts)[:, ch]
        out.append(pts[np.abs(v - GAMMA_KNEE) <= KNEE_SIDE_ULPS * t])
    return np.concatenate(out)


def stats_cells_host(lab, pts=PTS):
    """The cell rule of global_stats_kernel / global_stats_batch_kernel on the host, from Lab planes [n,3,h,w] float64
    (the device's own, from idc_rgb2lab_f64): a cell's ab = the float64 row-major sum of its 16 pixels from -0.0 / 16,
    rounded to float32; its bin = the first minimum of float32 (da * da) + (db * db), each operation rounded (numpy
    float32).  -> bins [n, cells] int."""
    n, _, h, w = lab.shape
    cells = lab[:, 1:].reshape(n, 2, h // 4, 4, w // 4, 4)
    s = np.full((n, 2, h // 4, w // 4), -0.0)
    for dy in range(4):
        for dx in range(4):
            s = s + cells[:, :, :, dy, :, dx]
    ab = (s / 16.0).astype(np.float32).transpose(0, 2, 3, 1).reshape(n, -1, 2)
    out = np.empty(ab.shape[:2], np.int64)
    for i in range(n):
        for c in range(0, ab.shape[1], 4096):
            blk = ab[i, c:c + 4096]
            da = blk[:, None, 0] - pts[None, :, 0]
            db = blk[:, None, 1] - pts[None, :, 1]
            out[i, c:c + 4096] = np.argmin(da * da + db * db, axis=1)
    return out


# ---------------------------------------------------------------------------------------------------------------
# device helpers
# ---------------------------------------------------------------------------------------------------------------
def _st():
    return torch.cuda.current_stream().cuda_stream


def _rgb2lab_dev(imgs):
    """idc_rgb2lab_f64 of uint8 images [n,h,w,3] -> float64 [n,3,h,w] (host)."""
    n, h, w = imgs.shape[:3]
    d = torch.from_numpy(np.ascontiguousarray(imgs)).cuda()
    lab = torch.empty((n, 3, h, w), dtype=torch.float64, device="cuda")
    assert _lib.load().idc_rgb2lab_f64(0, n, h, w, d.data_ptr(), lab.data_ptr(), _st()) == 0
    return lab.cpu().numpy()


def _stats_single(img):
    out = torch.full((316,), float("nan"), device="cuda")
    d = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    pts = torch.from_numpy(PTS).cuda()
    assert _lib.load().idc_global_stats(0, img.shape[0], img.shape[1], d.data_ptr(), pts.data_ptr(), out.data_ptr(),
                                        _st()) == 0
    return out.cpu().numpy()


def _stats_batch(imgs):
    a = np.ascontiguousarray(np.stack(imgs))
    n, h, w = a.shape[:3]
    d = torch.from_numpy(a).cuda()
    pts = torch.from_numpy(PTS).cuda()
    out = torch.full((n, 316), float("nan"), device="cuda")
    assert _lib.load().idc_global_stats_batch(0, n, h, w, d.data_ptr(), pts.data_ptr(), out.data_ptr(), _st()) == 0
    return out.cpu().numpy()


def _render_check(got, lab, what, totals):
    """got uint8 [..., 3] against 255 * clip(color_ref.lab2rgb(lab)) under assert_render_exact (values within 1e-9 of
    255 before the clip count as edges); adds to totals."""
    raw = color_ref.lab2rgb(lab) * 255
    rgb255 = np.clip(raw, 0, 255)
    n_edge, n_flip = util.assert_render_exact(got, rgb255.astype(np.uint8), rgb255, what, unclipped=raw)
    t = totals.setdefault(what.split(" ")[0], [0, 0, 0])
    t[0] += n_edge
    t[1] += n_flip
    t[2] += got.size


@pytest.fixture(scope="module")
def colours():
    """(uint8 [64,512,512,3] every colour, oracle Lab [64,512,512,3], device Lab [64,3,512,512])."""
    rgb = all_colours()
    return rgb, oracle_rgb2lab(rgb), _rgb2lab_dev(rgb)


# ---------------------------------------------------------------------------------------------------------------
# a. all 2^24 colours, RGB -> Lab
# ---------------------------------------------------------------------------------------------------------------
def test_rgb2lab_all_colours(colours):
    rgb, ref, dev = colours
    got = dev.transpose(0, 2, 3, 1)
    u = lab_ulps(got, ref)
    not_equal = int((got != ref).any(-1).sum())
    print("rgb2lab_kernel: max ulps (of 116 / 500 / 200) L %.0f a %.0f b %.0f; %d of %d colours not bit-equal"
          % (*u.reshape(-1, 3).max(0), not_equal, 1 << 24))
    bad = np.argwhere(u.max(-1) > LAB_ULPS)
    assert len(bad) == 0, [(tuple(rgb[tuple(i)]), ref[tuple(i)], got[tuple(i)]) for i in bad[:5]]
    # knees: the colours where the device could take the other branch.  A colour on the wrong side of lab_f's knee
    # is ~4e-5 from the oracle in L (cbrt and the linear piece differ by 3.3e-7 there), far past the bar checked above,
    # so every listed colour has taken the oracle's branch.
    xyz = np.concatenate([color_ref.rgb2xyz_white(rgb[k:k + CHUNK_IMG]).reshape(-1, 3)
                          for k in range(0, N_IMG, CHUNK_IMG)])
    near = np.nonzero((np.abs(xyz - LINEAR_KNEE) <= KNEE_ULPS * np.spacing(LINEAR_KNEE)).any(-1))[0]
    for i in near:
        c = rgb.reshape(-1, 3)[i]
        print("  near the 0.008856 knee: rgb %s  X/Xn, Y, Z/Zn = %r  L a b ulps %s"
              % (tuple(int(v) for v in c), tuple(xyz[i]), lab_ulps(got.reshape(-1, 3)[i], ref.reshape(-1, 3)[i])))
    c255 = np.arange(256) / 255.0
    near_g = np.nonzero(np.abs(c255 - 0.04045) <= KNEE_ULPS * np.spacing(0.04045))[0]
    print("  %d colours within %d ulps of the 0.008856 knee, %d channel values within %d ulps of 0.04045"
          % (near.size, KNEE_ULPS, near_g.size, KNEE_ULPS))
    assert near_g.size == 0            # 10 / 255 = 0.0392 and 11 / 255 = 0.0431: no uint8 value is near


# ---------------------------------------------------------------------------------------------------------------
# b. photo prep at the identity size
# ---------------------------------------------------------------------------------------------------------------
def _f32_midpoint_dist(x):
    """Distance of float64 x to the nearest midpoint between two adjacent float32 values."""
    f = x.astype(np.float32)
    up = np.nextafter(f, np.float32(np.inf)).astype(np.float64)
    dn = np.nextafter(f, np.float32(-np.inf)).astype(np.float64)
    f = f.astype(np.float64)
    return np.minimum(np.abs(x - (f + up) / 2), np.abs(x - (f + dn) / 2))


def test_photo_prep_identity_all_colours(colours):
    rgb, ref, _ = colours
    lib = _lib.load()
    table, src = photos.pack_photos(list(rgb))
    d_src = torch.from_numpy(src).cuda()
    L = torch.empty((N_IMG, 1, SIDE, SIDE), dtype=torch.float32, device="cuda")
    out = torch.empty((N_IMG, SIDE, SIDE, 3), dtype=torch.uint8, device="cuda")
    assert lib.idc_photo_prep(0, N_IMG, table.ctypes.data, d_src.data_ptr(), SIDE, L.data_ptr(), out.data_ptr(),
                              _st()) == 0
    assert np.array_equal(out.cpu().numpy(), rgb)
    L = L.cpu().numpy()[:, 0]
    x = ref[..., 0] - 50.0
    want = x.astype(np.float32)
    edge = _f32_midpoint_dist(x) <= LAB_ULPS * np.spacing(LAB_SCALE[0])
    diff = L != want
    print("photo_prep_kernel L_mc: %d of %d values within %d ulps (of 116) of a float32 rounding midpoint, "
          "%d of them differ" % (int(edge.sum()), x.size, LAB_ULPS, int((diff & edge).sum())))
    assert not (diff & ~edge).any(), np.argwhere(diff & ~edge)[:5]


# ---------------------------------------------------------------------------------------------------------------
# c. Lab -> RGB on dense grids
# ---------------------------------------------------------------------------------------------------------------
def _lab2rgb_u8(L32, ab32):
    """idc_lab2rgb_u8: L [n,h,w], ab [n,2,h,w] float32 -> uint8 [n,h,w,3]."""
    n, h, w = L32.shape
    dL = torch.from_numpy(np.ascontiguousarray(L32)).cuda()
    dab = torch.from_numpy(np.ascontiguousarray(ab32)).cuda()
    out = torch.empty((n, h, w, 3), dtype=torch.uint8, device="cuda")
    assert _lib.load().idc_lab2rgb_u8(0, n, h, w, dL.data_ptr(), dab.data_ptr(), out.data_ptr(), _st()) == 0
    return out.cpu().numpy()


def _planes_u8(lab):
    """idc_render_planes_u8 (IDC_RENDER_L_PLANE, order-1 zoom at the identity size, float64 planes) and
    idc_cubic_lab2rgb_u8 (identity size) of Lab planes [3,H,W] -> (uint8 [H,W,3], uint8 [H,W,3])."""
    lib = _lib.load()
    _, H, W = lab.shape
    dL = torch.from_numpy(np.ascontiguousarray(lab[0])).cuda()
    dab = torch.from_numpy(np.ascontiguousarray(lab[1:])).cuda()
    r1 = torch.empty((H, W, 3), dtype=torch.uint8, device="cuda")
    r2 = torch.empty((H, W, 3), dtype=torch.uint8, device="cuda")
    assert lib.idc_render_planes_u8(0, H, W, dab.data_ptr(), 1, 0, None, 0, _lib.RENDER_L_PLANE, dL.data_ptr(), H, W,
                                    r1.data_ptr(), _st()) == 0
    assert lib.idc_cubic_lab2rgb_u8(0, H, W, dab.data_ptr(), H, W, dL.data_ptr(), r2.data_ptr(), _st()) == 0
    return r1.cpu().numpy(), r2.cpu().numpy()


def test_lab2rgb_dense_grid():
    Ls = grid_L()
    totals = {}
    per = 8                                          # L values per chunk: 8 images of 512 x 512
    for k in range(0, len(Ls), per):
        chunk = Ls[k:k + per]
        lab = np.stack([grid_image(L) for L in chunk])                     # [m,3,512,512] float64
        what = "L %g..%g" % (chunk[0], chunk[-1])
        tall = lab.transpose(1, 0, 2, 3).reshape(3, -1, SIDE)              # [3, m*512, 512]
        r_planes, r_cubic = _planes_u8(tall)
        _render_check(r_planes, tall.transpose(1, 2, 0), "render_planes_kernel " + what, totals)
        _render_check(r_cubic, tall.transpose(1, 2, 0), "cubic_lab2rgb_kernel " + what, totals)
        # lab2rgb_kernel reads float32 L and ab: its reference is the oracle on float64(float32 L) (ab is exact)
        L32, ab32 = lab[:, 0].astype(np.float32), lab[:, 1:].astype(np.float32)
        assert np.array_equal(ab32.astype(np.float64), lab[:, 1:])
        lab32 = np.concatenate([L32[:, None].astype(np.float64), lab[:, 1:]], axis=1)
        _render_check(_lab2rgb_u8(L32, ab32), lab32.transpose(0, 2, 3, 1), "lab2rgb_kernel " + what, totals)
    for name, (n_edge, n_flip, size) in totals.items():
        print("%s over the grid (%d L x 512 x 512): %d of %d values excluded, %d of them differ"
              % (name, len(Ls), n_edge, size, n_flip))


def test_lab2rgb_gamma_knee():
    """Lab points whose linear R, G or B lies within 4 ulps either side of 0.0031308, through the float64 renders
    (which see the points as they are) and idc_lab2rgb_u8 (on their float32 rounding, against the oracle on that)."""
    pts = knee_lab()
    m = pts.shape[0]
    H = -(-m // SIDE)
    lab = np.zeros((H * SIDE, 3))
    lab[:m] = pts
    tall = lab.reshape(H, SIDE, 3).transpose(2, 0, 1)
    r_planes, r_cubic = _planes_u8(tall)
    totals = {}
    _render_check(r_planes.reshape(-1, 3)[:m], pts, "render_planes_kernel knee", totals)
    _render_check(r_cubic.reshape(-1, 3)[:m], pts, "cubic_lab2rgb_kernel knee", totals)
    lab32 = tall.astype(np.float32)
    got = _lab2rgb_u8(lab32[0][None], lab32[1:][None])[0]
    _render_check(got.reshape(-1, 3)[:m], lab32.astype(np.float64).transpose(1, 2, 0).reshape(-1, 3)[:m],
                  "lab2rgb_kernel knee", totals)
    print("gamma knee: %d points" % m)


def test_lab2rgb_abq_forward():
    """The quantised output_ab of a forward (lab2rgb_kernel's abq branch) = rgb2lab of its own uint8 RGB."""
    sd = synth.torch_state_dict(1234)
    L, ab, m = synth.synthetic_batch(2, 64, seed=21, max_hints=4)
    ctx = util.make_ctx(sd, 64, 64, max_n=2)
    r = ctx.forward_host(L, ab, m, 0.5, want_abq=True)
    ctx.close()
    for i in range(2):
        lab = np.concatenate([L[i].astype(np.float64) + 50.0, r["ab"][i].astype(np.float64)]).transpose(1, 2, 0)
        _render_check(r["rgb"][i], lab, "lab2rgb_kernel forward %d" % i, {})
        ref = color_ref.rgb2lab(r["rgb"][i])
        u = lab_ulps(np.concatenate([ref[..., :1], r["abq"][i].transpose(1, 2, 0)], -1), ref)
        print("lab2rgb_kernel abq %d: max ulps a %.0f b %.0f" % (i, u[..., 1].max(), u[..., 2].max()))
        assert u.max() <= LAB_ULPS


# ---------------------------------------------------------------------------------------------------------------
# d. round trip through idc_photo_render
# ---------------------------------------------------------------------------------------------------------------
def test_photo_render_round_trip(colours):
    rgb, ref, dev = colours
    lib = _lib.load()
    table, src = photos.pack_photos(list(rgb))
    d_src = torch.from_numpy(src).cuda()
    d_lab = torch.from_numpy(dev).cuda()
    out = torch.empty_like(d_src)
    assert lib.idc_photo_render(0, N_IMG, table.ctypes.data, d_src.data_ptr(), SIDE, d_lab.data_ptr(), out.data_ptr(),
                                _st()) == 0
    got = out.cpu().numpy().reshape(rgb.shape)
    moved_k = moved_o = flipped = n_edge = 0
    for k in range(0, N_IMG, CHUNK_IMG):
        g, c = got[k:k + CHUNK_IMG], rgb[k:k + CHUNK_IMG]
        raw = color_ref.lab2rgb(ref[k:k + CHUNK_IMG]) * 255
        rgb255 = np.clip(raw, 0, 255)
        want = rgb255.astype(np.uint8)
        e, _ = util.assert_render_exact(g, want, rgb255, "photo_render_kernel images %d-%d" % (k, k + CHUNK_IMG - 1),
                                        unclipped=raw)
        n_edge += e
        assert np.abs(g.astype(int) - c).max() <= 1                 # a round trip moves a channel by at most 1
        moved_k += int((g != c).any(-1).sum())
        moved_o += int((want != c).any(-1).sum())
        flipped += int((g != want).any(-1).sum())
    # the round trip lands within ~1e-13 of the colour itself, so nearly every value is a truncation edge and which
    # side it lands on is the last bit of pow / cbrt: the counts differ by at most the colours that differ, all of
    # them on an edge (assert_render_exact above)
    print("photo_render round trip: %d colours do not map back to themselves (kernel), %d (oracle); %d values on an "
          "edge, %d colours differ" % (moved_k, moved_o, n_edge, flipped))
    assert abs(moved_k - moved_o) <= flipped


# ---------------------------------------------------------------------------------------------------------------
# e. global statistics
# ---------------------------------------------------------------------------------------------------------------
def _check_stats(imgs, what, lab=None):
    """Both kernels on images [n,h,w,3]: histograms bit-identical to each other and to the host cell rule on the
    device's Lab; saturation within 2 float32 ulps of each other.  -> number of cells."""
    imgs = np.ascontiguousarray(imgs)
    n, h, w = imgs.shape[:3]
    cells = (h // 4) * (w // 4)
    batch = _stats_batch(list(imgs))
    lab = _rgb2lab_dev(imgs) if lab is None else lab
    bins = stats_cells_host(lab)
    worst = 0.0
    for i in range(n):
        one = _stats_single(imgs[i])
        want = (np.bincount(bins[i], minlength=313) / cells).astype(np.float32)
        assert one[:313].tobytes() == want.tobytes(), (what, i, np.nonzero(one[:313] != want)[0][:5])
        assert batch[i, :313].tobytes() == want.tobytes(), (what, i)
        assert one[313] == 1 and one[315] == 1 and batch[i, 313] == 1 and batch[i, 315] == 1
        ulps = abs(float(one[314]) - float(batch[i, 314])) / np.spacing(np.float32(batch[i, 314]))
        worst = max(worst, ulps)
        assert ulps <= 2, (what, i, one[314], batch[i, 314])
    print("global stats %s: %d images, histograms bit-identical (kernel, batch kernel, host rule); s_avg within "
          "%.0f float32 ulps" % (what, n, worst))
    return cells


def test_global_stats_all_colours(colours):
    rgb, _, dev = colours
    _check_stats(rgb, "all colours", dev)


@pytest.mark.parametrize("X", [64, 256])
def test_global_stats_photos(X):
    import cv2
    from tests.test_gpu_photos import SIZES, _photo
    imgs = np.stack([cv2.resize(_photo(h, w, 10 + i), (X, X)) for i, (h, w) in enumerate(SIZES)])
    _check_stats(imgs, "photos X=%d" % X)


def test_global_stats_run_to_run(colours):
    img = colours[0][37]
    a = _stats_single(img)
    b = _stats_single(img)
    assert a.tobytes() == b.tobytes()
