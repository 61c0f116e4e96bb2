"""GPU versions of the steps either side of the network (SURVEY 8f row f1).

    rgb2lab_gpu        skimage color.rgb2lab on uint8 RGB  (reference data/colorize_image.py:31-36,172-178,196-198)
    fullres_rgb_gpu    get_img_fullres (:123-131): scipy zoom(order=1) of the output ab + Lab->RGB at full resolution
    render_planes_gpu  the grey, input, mask and supervision renders at full resolution (:119-158)

float64 arithmetic on the device, like the reference's numpy path.  torch supplies device memory only.
"""
import numpy as np

from . import _lib


def _torch():
    """torch supplies device memory / streams only.  No GPU -> fail loudly (there is no CPU fallback: a wrapper built
    with gpu_prepost=False uses the host numpy path by explicit choice, nothing switches silently)."""
    import torch
    if not torch.cuda.is_available():
        raise _lib.IdcError(-5, "no CUDA device: the GPU pre/post-processing path (row f1) needs an sm_90 GPU")
    return torch


def rgb2lab_gpu(rgb_u8, device=0):
    """HxWx3 (or NxHxWx3) uint8 -> 3xHxW (or Nx3xHxW) float64 numpy, == color.rgb2lab(...).transpose."""
    torch = _torch()
    a = np.ascontiguousarray(rgb_u8)
    assert a.dtype == np.uint8 and a.shape[-1] == 3
    single = a.ndim == 3
    if single:
        a = a[None]
    n, h, w = a.shape[:3]
    d_rgb = torch.from_numpy(a).to("cuda:%d" % device)
    d_lab = torch.empty((n, 3, h, w), dtype=torch.float64, device=d_rgb.device)
    st = torch.cuda.current_stream(d_rgb.device).cuda_stream
    rc = _lib.load().idc_rgb2lab_f64(device, n, h, w, d_rgb.data_ptr(), d_lab.data_ptr(), st)
    if rc != _lib.IDC_OK:
        raise _lib.IdcError(rc, "idc_rgb2lab_f64 failed")
    out = d_lab.cpu().numpy()
    return out[0] if single else out


class DeviceLab(object):
    """Lab planes [3,H,W] float64 that live in HBM (row f1: `load_image` on the GPU).  Behaves like the numpy array
    the reference keeps (`img_lab_fullres`, data/colorize_image.py:161-170: 432 MB of float64 for an 18 MP photo) but is
    only copied to the host if somebody actually reads it; the GPU consumers (get_img_fullres) take `.tensor`."""

    def __init__(self, tensor, planes=slice(0, 3)):
        self.tensor, self._planes, self._host = tensor, planes, None
        n = len(range(*planes.indices(3)))
        self.shape = (n,) + tuple(tensor.shape[1:])
        self.dtype = np.dtype(np.float64)
        self.ndim = 3

    def view(self, planes):
        return DeviceLab(self.tensor, planes)

    def device_plane(self, idx):
        return self.tensor[idx]

    def __array__(self, dtype=None, copy=None):
        if self._host is None:
            self._host = self.tensor[self._planes].cpu().numpy()
        return self._host.astype(dtype) if dtype is not None else self._host

    def __getitem__(self, idx):
        return self.__array__()[idx]

    def __len__(self):
        return self.shape[0]


def load_image_gpu(rgb_full_u8, Xd, device=0):
    """`load_image` (data/colorize_image.py:52-66) after cv2.imread: full-resolution rgb2lab (skimage, float64) and the
    cv2.resize(im, (Xd, Xd)) + rgb2lab of the network-size copy, all on the device: one H2D of the uint8 image, three
    kernels, D2H of the Xd x Xd results only.  -> (img_rgb uint8 [Xd,Xd,3] host, img_lab float64 [3,Xd,Xd] host,
    DeviceLab of the full-resolution image)."""
    torch = _torch()
    lib = _lib.load()
    a = np.ascontiguousarray(rgb_full_u8)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3
    H, W = a.shape[:2]
    d_full = torch.from_numpy(a).to("cuda:%d" % device)
    st = torch.cuda.current_stream(d_full.device).cuda_stream
    d_lab_full = torch.empty((1, 3, H, W), dtype=torch.float64, device=d_full.device)
    d_small = torch.empty((Xd, Xd, 3), dtype=torch.uint8, device=d_full.device)
    d_lab = torch.empty((1, 3, Xd, Xd), dtype=torch.float64, device=d_full.device)
    for rc, what in ((lib.idc_rgb2lab_f64(device, 1, H, W, d_full.data_ptr(), d_lab_full.data_ptr(), st), "idc_rgb2lab_f64"),
                     (lib.idc_resize_u8_linear(device, H, W, d_full.data_ptr(), Xd, Xd, d_small.data_ptr(), st), "idc_resize_u8_linear"),
                     (lib.idc_rgb2lab_f64(device, 1, Xd, Xd, d_small.data_ptr(), d_lab.data_ptr(), st), "idc_rgb2lab_f64")):
        if rc != _lib.IDC_OK:
            raise _lib.IdcError(rc, what + " failed")
    return d_small.cpu().numpy(), d_lab[0].cpu().numpy(), DeviceLab(d_lab_full[0])


def resize_u8_linear_gpu(rgb_u8, h, w, device=0):
    """cv2.resize(rgb_u8, (w, h)) (INTER_LINEAR, 8-bit fixed point) on the device; bit-identical to cv2."""
    torch = _torch()
    a = np.ascontiguousarray(rgb_u8)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3
    d = torch.from_numpy(a).to("cuda:%d" % device)
    o = torch.empty((h, w, 3), dtype=torch.uint8, device=d.device)
    rc = _lib.load().idc_resize_u8_linear(device, a.shape[0], a.shape[1], d.data_ptr(), h, w, o.data_ptr(),
                                          torch.cuda.current_stream(d.device).cuda_stream)
    if rc != _lib.IDC_OK:
        raise _lib.IdcError(rc, "idc_resize_u8_linear failed")
    return o.cpu().numpy()


def display_rgb_gpu(ab, l_win, device=0):
    """The GUI's per-click display step (ui/gui_draw.py:280-283): cv2.resize(ab.transpose(1,2,0), (win_w, win_h),
    INTER_CUBIC) + concatenate with l_win + lab2rgb + clip * 255 -> uint8.  ab [2,h,w], l_win [H,W] (float64)."""
    torch = _torch()
    ab = np.ascontiguousarray(ab, dtype=np.float64)
    L = np.ascontiguousarray(l_win, dtype=np.float64)
    H, W = L.shape
    d_ab = torch.from_numpy(ab).to("cuda:%d" % device)
    d_L = torch.from_numpy(L).to(d_ab.device)
    d_rgb = torch.empty((H, W, 3), dtype=torch.uint8, device=d_ab.device)
    rc = _lib.load().idc_cubic_lab2rgb_u8(device, ab.shape[1], ab.shape[2], d_ab.data_ptr(), H, W, d_L.data_ptr(),
                                          d_rgb.data_ptr(), torch.cuda.current_stream(d_ab.device).cuda_stream)
    if rc != _lib.IDC_OK:
        raise _lib.IdcError(rc, "idc_cubic_lab2rgb_u8 failed")
    return d_rgb.cpu().numpy()


def fullres_rgb_gpu(ab, l_fullres, device=0):
    """get_img_fullres: ab [2,h,w] float32 / float64, l_fullres [1,H,W] or [H,W] float64 (numpy or DeviceLab) -> uint8
    [H,W,3].  The input render of render_planes_gpu with the output ab, so the zoom is scipy's, edge rule included."""
    H, W = l_fullres.shape[-2:]
    return render_planes_gpu(H, W, ab=ab, ab_order=1, L=l_fullres, device=device)


def render_planes_gpu(h, w, ab=None, ab_order=1, mask=None, l_mode=_lib.RENDER_L_PLANE, L=None, device=0):
    """The full-resolution renders (get_img_gray_fullres, get_input_img_fullres, get_img_mask_fullres, get_sup_fullres,
    data/colorize_image.py:119-158) -> uint8 [h,w,3]; include/idc_b200.h: idc_render_planes_u8.
    ab [2,h_in,w_in] float32 / float64 or None (ab = 0), zoomed to [h,w] with ab_order as scipy.ndimage.zoom does;
    mask [1,h_in,w_in] (or [h_in,w_in]) float32 / float64, zoomed with order 0, for l_mode RENDER_L_MASK / RENDER_L_SUP;
    L [1,h,w] (or [h,w]) float64 numpy or DeviceLab for RENDER_L_PLANE (a DeviceLab plane never leaves the device).
    A float32 plane gives scipy's / numpy's float32 results, as the host statements would."""
    torch = _torch()
    dev = torch.device("cuda:%d" % device)
    planes = [p for p in (ab, mask) if p is not None]
    h_in, w_in = planes[0].shape[-2:] if planes else (h, w)
    d_ab = d_mask = d_L = None
    ab_f32 = mask_f32 = 0
    if ab is not None:
        ab_f32 = int(ab.dtype == np.float32)
        d_ab = torch.from_numpy(np.ascontiguousarray(ab, dtype=np.float64).reshape(2, h_in, w_in)).to(dev)
    if mask is not None:
        mask_f32 = int(mask.dtype == np.float32)
        d_mask = torch.from_numpy(np.ascontiguousarray(mask, dtype=np.float64).reshape(h_in, w_in)).to(dev)
    if L is not None:
        if isinstance(L, DeviceLab):
            d_L = L.device_plane(0).contiguous()
        else:
            d_L = torch.from_numpy(np.ascontiguousarray(np.asarray(L, dtype=np.float64).reshape(h, w))).to(dev)
        assert tuple(d_L.shape) == (h, w), (tuple(d_L.shape), h, w)
    ptr = lambda t: None if t is None else t.data_ptr()
    d_rgb = torch.empty((h, w, 3), dtype=torch.uint8, device=dev)
    rc = _lib.load().idc_render_planes_u8(device, int(h_in), int(w_in), ptr(d_ab), int(ab_order), ab_f32, ptr(d_mask),
                                          mask_f32, int(l_mode), ptr(d_L), int(h), int(w), d_rgb.data_ptr(),
                                          torch.cuda.current_stream(dev).cuda_stream)
    if rc != _lib.IDC_OK:
        raise _lib.IdcError(rc, "idc_render_planes_u8 failed")
    return d_rgb.cpu().numpy()


def gamut_gpu(L, gamut_size=110, D=1, device=0):
    """The GUI's gamut map on the device: `abGrid(gamut_size, D).update_gamut(L)` (data/lab_gamut.py:66-78) ->
    (masked_rgb uint8 [A,B,3], mask bool [A,B]); row <-> a, column <-> b (include/idc_b200.h: idc_gamut_ab)."""
    torch = _torch()
    A = len(np.arange(-gamut_size, gamut_size + D, D))
    d_rgb = torch.empty((A, A, 3), dtype=torch.uint8, device="cuda:%d" % device)
    d_mask = torch.empty((A, A), dtype=torch.uint8, device=d_rgb.device)
    rc = _lib.load().idc_gamut_ab(device, float(L), int(gamut_size), int(D), d_rgb.data_ptr(), d_mask.data_ptr(),
                                  torch.cuda.current_stream(d_rgb.device).cuda_stream)
    if rc != _lib.IDC_OK:
        raise _lib.IdcError(rc, "idc_gamut_ab failed")
    return d_rgb.cpu().numpy(), d_mask.cpu().numpy().astype(bool)


def negentropy_gpu(dist):
    """`np.sum(d * np.log(d), axis=0)` per image (compute_entropy, data/colorize_image.py:356-358) on the device:
    dist is a CUDA float32 tensor [n, bins, ...] (e.g. a forward's out_dist or LhnContext.caffe313_dist_map) ->
    device tensor [n, ...].  float32, bins summed in order, NaN where a bin is exactly 0 (include/idc_b200.h:
    idc_negentropy)."""
    torch = _torch()
    assert dist.is_cuda and dist.dtype == torch.float32 and dist.dim() >= 2
    d = dist.contiguous()
    n, bins = d.shape[0], d.shape[1]
    out = torch.empty((n,) + tuple(d.shape[2:]), dtype=torch.float32, device=d.device)
    hw = out[0].numel() if n else 0
    rc = _lib.load().idc_negentropy(d.device.index, n, bins, hw, d.data_ptr(), out.data_ptr(),
                                    torch.cuda.current_stream(d.device).cuda_stream)
    if rc != _lib.IDC_OK:
        raise _lib.IdcError(rc, "idc_negentropy failed")
    return out


def pts_in_hull():
    """The 313 in-gamut ab bin centres (data fixture of the reference: data/color_bins/pts_in_hull.npy)."""
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "pts_in_hull.npy")).astype(np.float32)


def global_stats_gpu(rgb_u8, device=0):
    """Reference image uint8 [H,W,3] (H, W multiples of 4) -> glob vector [316] =
    [313-bin ab histogram, 1, mean saturation, 1] (row f3; global_stats.prototxt)."""
    torch = _torch()
    a = np.ascontiguousarray(rgb_u8)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3
    d_rgb = torch.from_numpy(a).to("cuda:%d" % device)
    d_pts = torch.from_numpy(pts_in_hull()).to(d_rgb.device)
    d_out = torch.empty((316,), dtype=torch.float32, device=d_rgb.device)
    st = torch.cuda.current_stream(d_rgb.device).cuda_stream
    rc = _lib.load().idc_global_stats(device, a.shape[0], a.shape[1], d_rgb.data_ptr(), d_pts.data_ptr(), d_out.data_ptr(), st)
    if rc != _lib.IDC_OK:
        raise _lib.IdcError(rc, "idc_global_stats failed")
    return d_out.cpu().numpy()


def ab_reccs_pmf_gpu(pmf, K=5, max_iter=100, n_init=8, pts=None, device=0):
    """Colour suggestions for one 529-bin pmf (host array): the deterministic weighted-k-means form of the
    reference's get_ab_reccs (data/colorize_image.py:322-354), see include/idc_b200.h: idc_ab_reccs_pmf.
    Returns (centres [K,2], mass [K], Lloyd iterations)."""
    import ctypes
    p = np.ascontiguousarray(pmf, np.float32)
    assert p.shape == (529,)
    q = None if pts is None else np.ascontiguousarray(pts, np.float32)
    assert q is None or q.shape == (529, 2)
    centers, conf, iters = np.empty((K, 2), np.float32), np.empty((K,), np.float32), ctypes.c_int(0)
    vp = lambda a: ctypes.c_void_p(a.ctypes.data)
    rc = _lib.load().idc_ab_reccs_pmf(device, vp(p), int(K), int(max_iter), int(n_init), None if q is None else vp(q),
                                      vp(centers), vp(conf), ctypes.byref(iters))
    if rc != _lib.IDC_OK:
        raise _lib.IdcError(rc, "idc_ab_reccs_pmf failed")
    return centers, conf, iters.value
