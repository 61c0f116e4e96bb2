"""Host-side mirror of the reference wrapper classes, backed by the H100 engine.

API kept verbatim from /root/reference/data/colorize_image.py so `ideepcolor.py:62-72`, the Qt
GUI (`ui/gui_draw.py:109-113,258-286`) and the notebooks work unchanged:

    ColorizeImageBase      (:39-198)   image prep, getters, full-res zoom
    ColorizeImageB200      <-> ColorizeImageTorch      (:201-276)
    ColorizeImageB200Dist  <-> ColorizeImageTorchDist  (:279-372)
    ColorizeImageB200GlobDist <-> ColorizeImageCaffeGlobDist (:445-463) semantics on the torch scaling

Differences, all deliberate: no scikit-image import (colour math in .color) and matplotlib only inside the
plot_dist_* methods;
`prep_net` also accepts an in-memory `state_dict`; the network forward, the 529-bin softmax
and the Lab->RGB post-process run in libidc_b200.so.  There is no CPU fallback.
"""
import numpy as np

from . import color, engine
from .color import lab2rgb_transpose, rgb2lab_transpose  # noqa: F401  (re-exported like the reference)


def put_point(input_ab, mask, loc, p, val):
    """Notebook helper (DemoInteractiveColorization.ipynb:131-139): paint a (2p+1)^2 hint."""
    input_ab[:, loc[0] - p:loc[0] + p + 1, loc[1] - p:loc[1] + p + 1] = np.array(val)[:, np.newaxis, np.newaxis]
    mask[:, loc[0] - p:loc[0] + p + 1, loc[1] - p:loc[1] + p + 1] = 1
    return (input_ab, mask)


# A hint list on the wrapper side: the fields of the C ABI's idc_hint (engine.as_hints), with a / b kept in float64 so
# that the host planes rasterised from it equal the planes put_point paints.  The engine rounds a / b to float32, as it
# rounds the dense ab plane.
HINT_LIST_DTYPE = np.dtype([("img", "<i4"), ("y0", "<i4"), ("x0", "<i4"), ("y1", "<i4"), ("x1", "<i4"),
                            ("a", "<f8"), ("b", "<f8")])


def hints_from_points(points, X, img=0):
    """put_point(input_ab, mask, loc, p, val) calls on X x X planes -> the equivalent hint list (HINT_LIST_DTYPE), in
    call order.  Row / column ranges follow numpy's slice semantics exactly (`slice(loc - p, loc + p + 1).indices(X)`):
    a negative start wraps around and, as in put_point, usually leaves the slice empty.  points: (loc, p, val) each."""
    out = np.zeros(len(points), HINT_LIST_DTYPE)
    for i, (loc, p, val) in enumerate(points):
        y0, y1, _ = slice(int(loc[0]) - int(p), int(loc[0]) + int(p) + 1).indices(X)
        x0, x1, _ = slice(int(loc[1]) - int(p), int(loc[1]) + int(p) + 1).indices(X)
        out[i] = (img, y0, x0, y1 - 1, x1 - 1, float(val[0]), float(val[1]))
    return out


def raster_hints(rects, X, img=0):
    """Host raster of a hint list (the idc_set_hints semantics) -> (ab [2,X,X], mask [1,X,X]) float64, the planes a
    dense net_forward would have received."""
    ab, mask = np.zeros((2, X, X)), np.zeros((1, X, X))
    for h in rects:
        if int(h["img"]) != img:
            continue
        y0, x0 = max(int(h["y0"]), 0), max(int(h["x0"]), 0)
        y1, x1 = min(int(h["y1"]), X - 1), min(int(h["x1"]), X - 1)
        if y1 >= y0 and x1 >= x0:
            ab[0, y0:y1 + 1, x0:x1 + 1] = h["a"]
            ab[1, y0:y1 + 1, x0:x1 + 1] = h["b"]
            mask[:, y0:y1 + 1, x0:x1 + 1] = 1
    return ab, mask


def _lazy_hint_plane(name):
    """input_ab / input_mask / input_ab_mc / input_mask_mult: plain attributes after a dense net_forward; after
    net_forward_hints they are rasterised on the host on first read (a click itself never needs them)."""
    key = "_" + name

    def get(self):
        d = self.__dict__
        if key not in d and d.get("_hint_rects") is not None:
            self._rasterise_hints()
        if key not in d:
            raise AttributeError(name)
        return d[key]

    def set(self, v):
        self.__dict__[key] = v
        self.__dict__["_hint_rects"] = None      # dense planes given: no hint list behind them

    return property(get, set)


def _zoom(a, factors, order):
    from scipy.ndimage import zoom
    return zoom(a, factors, order=order)


class ColorizeImageBase(object):
    """Image state + getters.  Attribute and method names are the reference's public surface
    (data/colorize_image.py:39-198); the bodies are organised around three helpers:
    `_ingest` (RGB -> Lab planes), `_to_fullres` (scipy zoom to the full-resolution grid) and
    `_render` (Lab planes -> uint8 RGB)."""

    def __init__(self, Xd=256, Xfullres_max=10000):
        self.Xd, self.Xfullres_max = Xd, Xfullres_max
        self.img_l_set = self.net_set = self.img_just_set = False

    def prep_net(self):
        raise Exception("Should be implemented by base class")

    # ----- image prep: reference load_image :52-66, set_image :68-77 -----
    def _ingest(self, rgb_full, rgb_net):
        self.img_rgb_fullres = rgb_full
        self._set_img_lab_fullres_()
        self.img_rgb = rgb_net
        self._set_img_lab_()
        self._set_img_lab_mc_()

    def load_image(self, input_path):
        import cv2
        bgr = cv2.imread(input_path, 1)
        if bgr is None:
            raise IOError("cannot read image %r" % (input_path,))
        full = cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB)
        self._ingest(full.copy(), cv2.resize(full, (self.Xd, self.Xd)).copy())   # cv2 default = bilinear

    def set_image(self, input_image):
        self._ingest(input_image.copy(), input_image)

    input_ab = _lazy_hint_plane("input_ab")
    input_mask = _lazy_hint_plane("input_mask")
    input_ab_mc = _lazy_hint_plane("input_ab_mc")
    input_mask_mult = _lazy_hint_plane("input_mask_mult")

    # ----- forward preconditions + hint normalisation: reference :79-96 -----
    def net_forward(self, input_ab, input_mask):
        hints = self.__dict__.pop("_hints_next", None)      # set by net_forward_hints for this one call
        for ok, what in ((self.img_l_set, 'an image'), (self.net_set, 'a net')):
            if not ok:
                print('I need to have %s!' % what)
                return -1
        if hints is not None:
            for k in ("_input_ab", "_input_mask", "_input_ab_mc", "_input_mask_mult"):
                self.__dict__.pop(k, None)
            self._hint_rects = hints                          # the four planes now derive from the list, lazily
            return 0
        self.input_ab, self.input_mask = input_ab, input_mask
        # reference :92-93.  With the PyTorch constants (ab_mean 0, ab_norm 1, mask_mult 1) both statements are exact
        # identities; skipping the two float64 temporaries (2.5 MB of numpy traffic) is worth ~0.1 ms per click
        self.input_ab_mc = input_ab if (self.ab_mean == 0 and self.ab_norm == 1) else (input_ab - self.ab_mean) / self.ab_norm
        self.input_mask_mult = input_mask if self.mask_mult == 1 else input_mask * self.mask_mult
        return 0

    def net_forward_hints(self, rects, glob_dist=-1):
        """net_forward with the hints given as a list of rectangles (HINT_LIST_DTYPE, e.g. from hints_from_points)
        instead of dense ab / mask planes.  The result equals net_forward(*raster_hints(rects, Xd)); where the engine's
        click path runs, the list itself travels to the device and is rasterised there.  input_ab / input_mask /
        input_ab_mc / input_mask_mult read as the dense call would have set them (computed on first read)."""
        self._hints_next = np.array(rects, dtype=HINT_LIST_DTYPE).reshape(-1)
        try:
            if np.array(glob_dist).flatten()[0] != -1:
                return self.net_forward(None, None, glob_dist)
            return self.net_forward(None, None)
        finally:
            self.__dict__.pop("_hints_next", None)

    def _rasterise_hints(self):
        ab, mask = raster_hints(self._hint_rects, self.img_l_mc.shape[-1])
        d = self.__dict__
        d["_input_ab"], d["_input_mask"] = ab, mask
        d["_input_ab_mc"] = ab if (self.ab_mean == 0 and self.ab_norm == 1) else (ab - self.ab_mean) / self.ab_norm
        d["_input_mask_mult"] = mask if self.mask_mult == 1 else mask * self.mask_mult

    def get_result_PSNR(self, result=-1, return_SE_map=False):
        use_own = np.array((result)).flatten()[0] == -1
        err2 = (1. * self.img_rgb - (self.get_img_forward() if use_own else result.copy())) ** 2
        psnr = 20 * np.log10(255. / np.sqrt(np.mean(err2)))
        return (psnr, err2) if return_SE_map else psnr

    # ----- rendering helpers -----
    @staticmethod
    def _render(l_plane, ab_planes=None):
        if ab_planes is None:
            ab_planes = np.zeros((2,) + tuple(l_plane.shape[1:]))
        return lab2rgb_transpose(l_plane, ab_planes)

    def _to_fullres(self, planes, like, order):
        fh = 1. * self.img_l_fullres.shape[1] / like.shape[1]
        fw = 1. * self.img_l_fullres.shape[2] / like.shape[2]
        return _zoom(planes, (1, fh, fw), order)

    # ----- getters: reference :111-158 -----
    def get_img_forward(self):
        return self.output_rgb

    def get_img_gray(self):
        return self._render(self.img_l)

    def get_img_gray_fullres(self):
        return self._render(self.img_l_fullres)

    def get_img_fullres(self):       # bilinear up-zoom of the (quantised) output ab, then Lab->RGB
        return self._render(self.img_l_fullres, self._to_fullres(self.output_ab, self.output_ab, 1))

    def get_input_img_fullres(self):
        return self._render(self.img_l_fullres, self._to_fullres(self.input_ab, self.input_ab, 1))

    def get_input_img(self):
        return self._render(self.img_l, self.input_ab)

    def get_img_mask(self):
        return self._render(100. * (1 - self.input_mask))

    def get_img_mask_fullres(self):
        return self._render(100. * (1 - self._to_fullres(self.input_mask, self.input_ab, 0)))

    def get_sup_img(self):
        return self._render(50 * self.input_mask, self.input_ab)

    def get_sup_fullres(self):
        return self._render(50 * self._to_fullres(self.input_mask, self.output_ab, 0),
                            self._to_fullres(self.input_ab, self.output_ab, 0))

    # ----- Lab planes: reference :161-198 -----
    @staticmethod
    def _lab_planes(rgb):
        lab = color.rgb2lab(rgb).transpose((2, 0, 1))
        return lab, lab[[0]], lab[1:]

    def _set_img_lab_fullres_(self):
        big = max(self.img_rgb_fullres.shape[:2])
        if big > self.Xfullres_max:          # cap the longest side
            z = 1. * self.Xfullres_max / big
            self.img_rgb_fullres = _zoom(self.img_rgb_fullres, (z, z, 1), 1)
        self.img_lab_fullres, self.img_l_fullres, self.img_ab_fullres = self._lab_planes(self.img_rgb_fullres)

    def _set_img_lab_(self):
        self.img_lab, self.img_l, self.img_ab = self._lab_planes(self.img_rgb)

    def _set_img_lab_mc_(self):
        div = np.array((self.l_norm, self.ab_norm, self.ab_norm), dtype=np.float64).reshape(3, 1, 1)
        sub = np.array((self.l_mean, self.ab_mean, self.ab_mean), dtype=np.float64).reshape(3, 1, 1) / div
        self.img_lab_mc = self.img_lab / div - sub
        self._set_img_l_()

    def _set_img_l_(self):
        self.img_l_mc = self.img_lab_mc[[0]]
        self.img_l_set = True

    def _set_img_ab_(self):
        self.img_ab_mc = self.img_lab_mc[[1, 2]]

    def _set_out_ab_(self):
        # output_ab is re-derived from the uint8 RGB, i.e. quantised (reference :196-198, SURVEY q2)
        self.output_lab = rgb2lab_transpose(self.output_rgb)
        self.output_ab = self.output_lab[1:]


class ColorizeImageB200(ColorizeImageBase):
    """<-> ColorizeImageTorch (reference :201-276)."""

    def __init__(self, Xd=256, maskcent=False, engine="wgmma", fast_fp16=False, gpu_prepost=True):
        print('ColorizeImageB200 instantiated')
        self.gpu_prepost = gpu_prepost    # quantised output_ab and the full-res render on the GPU (row f1)
        ColorizeImageBase.__init__(self, Xd)
        self.l_norm = 1.
        self.ab_norm = 1.
        self.l_mean = 50.
        self.ab_mean = 0.
        self.mask_mult = 1.
        self.mask_cent = .5 if maskcent else 0
        self.engine = engine
        self.fast_fp16 = fast_fp16
        # torch-path bin grid (reference :213; (b,a)-ordered meshgrid, SURVEY q3)
        self.pts_in_hull = np.array(np.meshgrid(np.arange(-110, 120, 10), np.arange(-110, 120, 10))).reshape((2, 529)).T

    def _calibrate(self, calibrate, sd, device, **flags):
        """prep_net's calibrate= argument -> self.act_ranges, {buffer: max_abs} or None.  calibrate: None (exponents
        from the weights); a list of colour photos (paths or uint8 RGB arrays) to measure the activation ranges of
        this checkpoint on now (engine.calibration_batch + engine.measure_act_ranges); or such a measurement, as a dict
        or the path of a JSON file written by engine.save_act_ranges."""
        from . import engine
        X = self.Xd
        self.act_ranges = engine.resolve_calibration(calibrate, lambda photos: engine.measure_act_ranges(
            sd, engine.calibration_batch(photos, X, device=device, global_hints=flags.get("global_hints", False)),
            X, X, device=device, maskcent=float(self.mask_cent), **flags))
        return self.act_ranges

    def prep_net(self, gpu_id=None, path='', dist=False, state_dict=None, calibrate=None):
        import torch
        from .model import SIGGRAPHGeneratorB200
        print('path = %s' % path)
        print('Model set! dist mode? ', dist)
        self.net = SIGGRAPHGeneratorB200(dist=dist, device=0 if gpu_id is None else int(gpu_id), engine=self.engine,
                                         fast_fp16=self.fast_fp16)
        if state_dict is None:
            state_dict = torch.load(path, map_location='cpu')
        if hasattr(state_dict, '_metadata'):
            del state_dict._metadata
        self.net.load_state_dict(state_dict)
        self.net.cuda()
        self.net.eval()
        self.net.set_act_ranges(self._calibrate(calibrate, self.net.state_dict(), self.net.b200_device))
        self.net_set = True

    def net_forward(self, input_ab, input_mask):
        if ColorizeImageBase.net_forward(self, input_ab, input_mask) == -1:
            return -1
        ctx = self.net._context(self.img_l_mc.shape[-2], self.img_l_mc.shape[-1], 1)
        # ONE C-ABI call and one round trip: H2D, forward, fused Lab->RGB post-process (reference :263-264) and the
        # quantised output_ab = rgb2lab(output_rgb)[1:] (reference :267 -> :196-198) in the same kernel, D2H
        self._click(ctx, float(self.mask_cent))
        return self.output_rgb

    def _click(self, ctx, maskcent, glob=None, mask_div=1.0, want_rgb=True, publish_rgb=None, need_dist=False):
        """Stage the reference's float64 arrays into the context's page-locked click buffers (the float64 -> float32
        conversion IS the only CPU copy; L is re-staged only when the image changed), run idc_forward_host_q with
        the pinned buffers (zero-copy graph path) and publish copies of the results as the reference's attributes."""
        buf = self._click_buffers(ctx, glob is not None)
        want_q = bool(want_rgb and self.gpu_prepost)
        rects = self.__dict__.get("_hint_rects")            # net_forward_hints: the list goes to the device, not planes
        if ctx._wrapper_shared and glob is None and \
                self._same_as_last_forward(ctx, buf, maskcent, mask_div, want_rgb, want_q, need_dist):
            # share_trunk: the other model of the pair just ran this very forward; its results are still in the buffers
            r = {"ab": buf["out_ab"], "rgb": buf["out_rgb"], "abq": buf["out_abq"]}
        else:
            self._stage_image(ctx, buf)
            if rects is not None:
                hints = engine.as_hints(rects)
                ctx.set_hints(hints)
                ab_in = mask_in = None
            else:
                np.copyto(buf["ab"][0], self.input_ab_mc, casting='unsafe')
                if mask_div == 1.0:
                    np.copyto(buf["mask"][0], self.input_mask_mult, casting='unsafe')
                else:
                    np.divide(self.input_mask_mult, mask_div, out=buf["mask"][0], casting='unsafe')
                ab_in, mask_in = buf["ab"], buf["mask"]
            if glob is not None:
                buf["glob"][...] = glob
            ctx._wrapper_last = None
            # L_mc = None: the image uploaded by _stage_image (idc_set_image) -- a click moves only the hints
            r = ctx.forward_host(None, ab_in, mask_in, maskcent, glob=buf["glob"], want_rgb=want_rgb, n=1,
                                 want_abq=want_q, out_ab=buf["out_ab"], out_rgb=buf["out_rgb"] if want_rgb else None,
                                 out_abq=buf["out_abq"] if want_q else None)
            ctx._wrapper_hints = None if rects is None else hints
            ctx._wrapper_last = (float(maskcent), float(mask_div), glob is not None, bool(want_rgb), want_q,
                                 bool(getattr(ctx, "_dist_resident", False)))
        self.output_ab_raw = r["ab"][0].copy()   # raw net output (the parity quantity, SURVEY q2)
        if want_rgb and (publish_rgb is None or publish_rgb):
            self.output_rgb = r["rgb"][0].copy()
            if want_q:
                self.output_ab = r["abq"][0].copy()
                self._output_lab = None          # output_lab (L plane included) is derived on demand
            else:
                ColorizeImageBase._set_out_ab_(self)
        return r

    @staticmethod
    def _click_buffers(ctx, with_glob):
        buf = getattr(ctx, "_wrapper_click", None)
        if buf is None or with_glob != (buf["glob"] is not None):
            buf = ctx.click_buffers(1, glob=with_glob)
            ctx._wrapper_click = buf
            ctx._wrapper_staged_l = []
            ctx._wrapper_last = None
        return buf

    def _same_as_last_forward(self, ctx, buf, maskcent, mask_div, want_rgb, want_q, need_dist=False):
        """Did the (shared) context just run exactly this image + these hints (float32, as staged), producing at least
        the outputs asked for (RGB, quantised ab, the resident distribution)?"""
        last = ctx._wrapper_last
        if last is None or last[:3] != (float(maskcent), float(mask_div), False) or (want_rgb and not last[3]) or \
                (want_q and not last[4]) or (need_dist and not last[5]):
            return False
        if not any(a is self.img_l_mc for a in ctx._wrapper_staged_l):
            l32 = np.ascontiguousarray(self.img_l_mc, dtype=np.float32).reshape(buf["L_mc"].shape)
            if not (ctx._wrapper_staged_l and np.array_equal(buf["L_mc"], l32)):
                return False
            ctx._wrapper_staged_l = ctx._wrapper_staged_l[-3:] + [self.img_l_mc]
        last_hints = getattr(ctx, "_wrapper_hints", None)
        rects = self.__dict__.get("_hint_rects")
        if rects is not None:                    # hint lists: compare the lists (as the engine received them), not planes
            return last_hints is not None and np.array_equal(last_hints, engine.as_hints(rects))
        if last_hints is not None:               # the last forward rasterised a list; the plane buffers are stale
            return False
        mask32 = np.asarray(self.input_mask_mult, dtype=np.float32)
        if mask_div != 1.0:
            mask32 = mask32 / np.float32(mask_div)
        return (np.array_equal(buf["ab"][0], np.asarray(self.input_ab_mc, dtype=np.float32)) and
                np.array_equal(buf["mask"][0], mask32))

    def _stage_image(self, ctx, buf):
        """The L plane goes to the device once per image (reference: set_image / load_image, :68-77), not once per
        click.  `_wrapper_staged_l` lists the img_l_mc arrays known to equal the resident plane (several wrapper
        objects may share one context, see ColorizeImageB200Dist.share_trunk)."""
        if any(a is self.img_l_mc for a in ctx._wrapper_staged_l):
            return
        l32 = np.ascontiguousarray(self.img_l_mc, dtype=np.float32).reshape(buf["L_mc"].shape)
        if ctx._wrapper_staged_l and np.array_equal(buf["L_mc"], l32):
            ctx._wrapper_staged_l = ctx._wrapper_staged_l[-3:] + [self.img_l_mc]
            return
        buf["L_mc"][...] = l32
        ctx.set_image(buf["L_mc"])
        ctx._wrapper_staged_l = [self.img_l_mc]
        ctx._wrapper_last = None

    @property
    def output_lab(self):
        """reference :197 (`self.output_lab = rgb2lab_transpose(self.output_rgb)`); nothing in the reference reads it
        besides `_set_out_ab_` itself, so the fused path computes it lazily."""
        if getattr(self, "_output_lab", None) is None:
            self._output_lab = rgb2lab_transpose(self.output_rgb)
        return self._output_lab

    @output_lab.setter
    def output_lab(self, v):
        self._output_lab = v

    def get_img_forward(self):
        return self.output_rgb

    def get_img_gray(self):
        return lab2rgb_transpose(self.img_l, np.zeros((2, self.Xd, self.Xd)))

    # ----- row f1, image-load side: reference load_image :52-66 on the GPU when a net is set -----
    def _ingest(self, rgb_full, rgb_net):
        """Full-resolution rgb2lab (the reference spends seconds of float64 numpy on an 18 MP photo, :161-170) stays in
        HBM as a DeviceLab; only the Xd x Xd planes come back.  `rgb_net` None = resize here with the cv2-exact kernel."""
        big = max(rgb_full.shape[:2])
        if not (self.gpu_prepost and self.net_set) or big > self.Xfullres_max or rgb_full.dtype != np.uint8:
            if rgb_net is None:
                import cv2
                rgb_net = cv2.resize(rgb_full, (self.Xd, self.Xd)).copy()
            return ColorizeImageBase._ingest(self, rgb_full, rgb_net)
        from . import prepost
        small, lab, dlab = prepost.load_image_gpu(rgb_full, self.Xd, self._device())
        self.img_rgb_fullres = rgb_full
        self.img_lab_fullres, self.img_l_fullres, self.img_ab_fullres = dlab, dlab.view(slice(0, 1)), dlab.view(slice(1, 3))
        if rgb_net is None:
            self.img_rgb = small
            self.img_lab = lab
        else:                                             # set_image: the caller pre-resized (reference :68-77)
            self.img_rgb = rgb_net
            self.img_lab = prepost.rgb2lab_gpu(rgb_net, self._device()) if rgb_net.dtype == np.uint8 else self._lab_planes(rgb_net)[0]
        self.img_l, self.img_ab = self.img_lab[[0]], self.img_lab[1:]
        self._set_img_lab_mc_()

    def load_image(self, input_path):
        import cv2
        bgr = cv2.imread(input_path, 1)
        if bgr is None:
            raise IOError("cannot read image %r" % (input_path,))
        self._ingest(np.ascontiguousarray(cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB)), None)

    # ----- row f1: the numpy/scipy steps either side of the network, on the GPU when a net is set -----
    def _device(self):
        """CUDA device ordinal of the engine behind this wrapper (the Torch-named classes hold a module in
        `self.net`, the GlobDist / Caffe-named ones an LhnContext in `self._ctx`)."""
        ctx = getattr(self, "_ctx", None)
        return ctx.device if ctx is not None else self.net.b200_device

    def _set_out_ab_(self):
        if not (self.gpu_prepost and self.net_set):
            return ColorizeImageBase._set_out_ab_(self)
        from . import prepost
        self.output_lab = prepost.rgb2lab_gpu(self.output_rgb, self._device())
        self.output_ab = self.output_lab[1:]

    def get_img_fullres(self):
        if not (self.gpu_prepost and self.net_set):
            return ColorizeImageBase.get_img_fullres(self)
        from . import prepost
        return prepost.fullres_rgb_gpu(self.output_ab, self.img_l_fullres, self._device())

    # ----- row f1, the other full-resolution renders (reference :119-158) on the GPU under the same gate -----
    def _device_render(self, *planes):
        """float32 / float64 planes of three dimensions render on the device; anything else (a bool GUI mask, integer
        planes) takes the ColorizeImageBase statements, which then raise or convert exactly as they always did."""
        return self.gpu_prepost and self.net_set and all(
            getattr(p, "dtype", None) in (np.float32, np.float64) and getattr(p, "ndim", 0) == 3 for p in planes)

    def _fullres_hw(self, plane, like):
        """(h, w) of `_to_fullres(plane, like, order)`: scipy's int(round(n * factor)) per axis."""
        H, W = self.img_l_fullres.shape[1:]
        return (int(round(plane.shape[1] * (1. * H / like.shape[1]))), int(round(plane.shape[2] * (1. * W / like.shape[2]))))

    def get_img_gray_fullres(self):
        L = self.img_l_fullres
        if not self._device_render(L) or L.shape[0] != 1:
            return ColorizeImageBase.get_img_gray_fullres(self)
        from . import prepost
        return prepost.render_planes_gpu(L.shape[1], L.shape[2], L=L, device=self._device())

    def get_input_img_fullres(self):
        L, ab = self.img_l_fullres, self.input_ab
        if not self._device_render(L, ab) or L.shape[0] != 1 or ab.shape[0] != 2 or \
                self._fullres_hw(ab, ab) != tuple(L.shape[1:]):
            return ColorizeImageBase.get_input_img_fullres(self)
        from . import prepost
        return prepost.render_planes_gpu(L.shape[1], L.shape[2], ab=ab, ab_order=1, L=L, device=self._device())

    def get_img_mask_fullres(self):
        mask, like = self.input_mask, self.input_ab
        if not self._device_render(mask, like) or mask.shape[0] != 1:
            return ColorizeImageBase.get_img_mask_fullres(self)
        from . import _lib, prepost
        h, w = self._fullres_hw(mask, like)
        return prepost.render_planes_gpu(h, w, mask=mask, l_mode=_lib.RENDER_L_MASK, device=self._device())

    def get_sup_fullres(self):
        mask, ab, like = self.input_mask, self.input_ab, self.output_ab
        if not self._device_render(mask, ab, like) or mask.shape[0] != 1 or ab.shape[0] != 2 or \
                mask.shape[1:] != ab.shape[1:]:
            return ColorizeImageBase.get_sup_fullres(self)
        from . import _lib, prepost
        h, w = self._fullres_hw(mask, like)
        return prepost.render_planes_gpu(h, w, ab=ab, ab_order=0, mask=mask, l_mode=_lib.RENDER_L_SUP,
                                         device=self._device())


class _LazyUpsampledDist(object):
    """[529, X, X] view of the [529, X/4, X/4] distribution.  The reference materialises the nearest x4
    upsample (139 MB at 256^2, model.py:160) and copies it to the host; its consumers only index single
    pixels (`dist_ab[:, h, w]`, data/colorize_image.py:329).  Here the distribution stays on the device
    (`fetch` pulls 529 floats per lookup) or is a host [529, X/4, X/4] array; either way it is
    replicated on read."""

    def __init__(self, d64=None, fetch=None, shape64=None, negentropy=None):
        """negentropy: callable -> [X/4, X/4] sum_k d log d of the device-resident plane (compute_entropy)."""
        self.d64, self._fetch, self._negentropy = d64, fetch, negentropy
        s = d64.shape if d64 is not None else shape64
        self.shape = (s[0], s[1] * 4, s[2] * 4)
        self.dtype = np.dtype(np.float32)

    def _plane(self):
        if self.d64 is None:
            self.d64 = self._fetch(None, None)
        return self.d64

    def __getitem__(self, idx):
        if isinstance(idx, tuple) and len(idx) == 3 and all(isinstance(i, (int, np.integer)) for i in idx[1:]):
            if self.d64 is None:
                return self._fetch(int(idx[1]) // 4, int(idx[2]) // 4)[idx[0]]
            return self.d64[idx[0], idx[1] // 4, idx[2] // 4]
        return self.__array__()[idx]

    def __array__(self, dtype=None, copy=None):
        a = np.repeat(np.repeat(self._plane(), 4, axis=1), 4, axis=2)
        return a.astype(dtype) if dtype is not None else a


class _LazyDistFull(object):
    """`dist_ab_full` [AB, X, X] or `dist_ab_grid` [A, B, X, X] (float64, zero outside `in_hull`; reference :312-317)
    over a lazy `dist_ab`.  Indexing one pixel (`[:, h, w]`, `[:, :, h, w]`) reads that pixel's column of `dist_ab`
    only; np.asarray materialises the reference's float64 array."""

    def __init__(self, dist, in_hull, shape):
        self._dist, self._in_hull = dist, in_hull
        self.shape = tuple(shape)
        self.ndim = len(self.shape)
        self.dtype = np.dtype(np.float64)

    def __getitem__(self, idx):
        k = self.ndim - 2
        if isinstance(idx, tuple) and len(idx) == self.ndim and all(isinstance(i, (int, np.integer)) for i in idx[k:]):
            h, w = range(self.shape[-2])[int(idx[k])], range(self.shape[-1])[int(idx[k + 1])]
            col = np.zeros(self._in_hull.shape[0])
            col[self._in_hull] = np.asarray(self._dist[:, h, w])
            return col.reshape(self.shape[:k])[idx[:k]]
        return self.__array__()[idx]

    def __array__(self, dtype=None, copy=None):
        full = np.zeros((self._in_hull.shape[0],) + self.shape[-2:])
        full[self._in_hull] = np.asarray(self._dist)
        full = full.reshape(self.shape)
        return full.astype(dtype) if dtype is not None else full


class _DistPlots(object):
    """plot_dist_grid / plot_dist_entropy of both distribution models (reference :360-372, :549-561).  matplotlib is
    imported on call, so the package imports without it."""

    def plot_dist_grid(self, h, w):
        import matplotlib.pyplot as plt
        plt.figure()
        plt.imshow(self.dist_ab_grid[:, :, h, w], extent=[-110, 110, 110, -110], interpolation='nearest')
        plt.colorbar()
        plt.ylabel('a')
        plt.xlabel('b')

    def plot_dist_entropy(self):
        import matplotlib.pyplot as plt
        plt.figure()
        plt.imshow(-self.dist_entropy, interpolation='nearest')
        plt.colorbar()


class ColorizeImageB200Dist(_DistPlots, ColorizeImageB200):
    """<-> ColorizeImageTorchDist (reference :279-372)."""

    def __init__(self, Xd=256, maskcent=False, engine="wgmma", fast_fp16=False, materialize_full=False):
        ColorizeImageB200.__init__(self, Xd, engine=engine, fast_fp16=fast_fp16)
        self.dist_ab_set = False
        self.pts_grid = np.array(np.meshgrid(np.arange(-110, 120, 10), np.arange(-110, 120, 10))).reshape((2, 529)).T
        self.in_hull = np.ones(529, dtype=bool)
        self.AB = self.pts_grid.shape[0]
        self.A = int(np.sqrt(self.AB))
        self.B = int(np.sqrt(self.AB))
        self.materialize_full = materialize_full
        self.dist_entropy = np.zeros((self.Xd, self.Xd))
        self.mask_cent = .5 if maskcent else 0

    def prep_net(self, gpu_id=None, path='', dist=True, S=.2, state_dict=None, calibrate=None):
        ColorizeImageB200.prep_net(self, gpu_id=gpu_id, path=path, dist=dist, state_dict=state_dict, calibrate=calibrate)

    def share_trunk(self, color_model):
        """ONE forward per click instead of two.  The PyTorch backend loads the same checkpoint into both models
        (ideepcolor.py:34-38 "same model used for both") and the GUI feeds both the same hints, one after the other
        (ui/gui_draw.py:250-258 predict_color, :272-279 compute_result); the distribution head hangs off conv8_3 of
        the very trunk the colour model just ran.  After `share_trunk(color_model)` -- color_model prepared with
        `prep_net(..., dist=True)` -- this object uses the colour model's network: when net_forward sees the image and
        hints the shared context ran last, it publishes that forward's outputs (the resident distribution, the raw ab
        map) without launching anything; otherwise it runs the forward itself -- and the colour model's next
        net_forward with the same hints is answered from THAT forward (the sharing is symmetric, whichever model the
        GUI calls first pays).  Replaces prep_net."""
        net = getattr(color_model, "net", None)
        if not getattr(color_model, "net_set", False) or net is None or not getattr(net, "dist", False):
            raise ValueError("share_trunk: prepare the colour model with prep_net(..., dist=True) first")
        self.net = net
        self.net_set = True
        self._trunk = color_model
        Xd = self.Xd
        ctx = net._context(Xd, Xd, 1)
        ctx.set_dist_resident(True)          # every forward of the shared context keeps its distribution
        ctx._wrapper_shared = True           # _click may now answer from the other model's forward
        return self

    def hint_click(self, h, w, K=9):
        """Announce the pixel the GUI is about to ask suggestions for (ui/gui_draw.py:184 `suggest_color(h=y, w=x, K=9)`)
        BEFORE the forward: its pmf and the K suggestions then come back with the click itself (idc_set_click), and
        `dist_ab[:, h, w]` / `get_ab_reccs(h, w, K)` cost no device work.  h = None switches it off."""
        ctx = self.net._context(self.Xd, self.Xd, 1)
        if h is None:
            ctx.set_click(0, -1, 0, 0)
        else:
            ctx.set_click(0, int(h) // 4, int(w) // 4, int(K))

    def net_forward(self, input_ab, input_mask):
        if ColorizeImageBase.net_forward(self, input_ab, input_mask) == -1:
            return -1
        Xh, Xw = self.img_l_mc.shape[-2], self.img_l_mc.shape[-1]
        ctx = self.net._context(Xh, Xw, 1)
        if self.materialize_full:
            A = np.ascontiguousarray(self.img_l_mc, dtype=np.float32)[None]
            B = np.ascontiguousarray(self.input_ab_mc, dtype=np.float32)[None]
            M = np.ascontiguousarray(self.input_mask_mult, dtype=np.float32)[None]
            r = ctx.forward_host(A, B, M, float(self.mask_cent), want_dist=True)
            self.dist_ab_64 = r["dist"][0]                   # [529, X/4, X/4]
            self.output_ab_raw = r["ab"][0]
        else:
            ctx.set_dist_resident(True)                      # dist stays in HBM; pixels are fetched on demand
            # on a shared context keep the colour model's graph (same outputs requested -> no re-capture); the
            # distribution model itself publishes no RGB (reference :297-320 never sets output_rgb)
            self._click(ctx, float(self.mask_cent), want_rgb=getattr(self, "_trunk", None) is not None, publish_rgb=False,
                        need_dist=True)
        if self.materialize_full:
            self.dist_ab = np.repeat(np.repeat(self.dist_ab_64, 4, axis=1), 4, axis=2)
            self.dist_ab_full = np.zeros((self.AB, self.Xd, self.Xd))
            self.dist_ab_full[self.in_hull, :, :] = self.dist_ab
            self.dist_ab_grid = self.dist_ab_full.reshape((self.A, self.B, self.Xd, self.Xd))
        else:
            self.dist_ab = _LazyUpsampledDist(fetch=lambda y4, x4: ctx.fetch_dist(0, y4, x4),
                                              shape64=(529, Xh // 4, Xw // 4),
                                              negentropy=lambda: ctx.dist_negentropy(0))
            self.dist_ab_full = _LazyDistFull(self.dist_ab, self.in_hull, (self.AB, Xh, Xw))
            self.dist_ab_grid = _LazyDistFull(self.dist_ab, self.in_hull, (self.A, self.B, Xh, Xw))
        self._dist_ctx = ctx
        self.dist_ab_set = True
        # reference returns the regression output scaled by 110 twice (model.py:166-168, q1)
        return self.output_ab_raw * 110.0

    def get_ab_reccs(self, h, w, K=5, N=25000, return_conf=False, method='gpu'):
        """Colour suggestions at pixel (h, w) (reference :322-354).  The reference draws N samples from the
        529-bin distribution by inverse-CDF lookup, k-means them and orders the clusters by occupancy.
        method='gpu' (default): the N -> infinity limit of that, weighted k-means on the device over the
        resident distribution (idc_ab_reccs; deterministic, N unused).  method='sampled': the reference's
        stochastic procedure on the host (np.random + sklearn), for side-by-side comparison."""
        if not self.dist_ab_set:
            print('Need to set prediction first')
            return 0
        if method == 'gpu':                                  # the distribution of the last forward is still on the device
            centers, conf, _ = self._dist_ctx.ab_reccs(0, int(h) // 4, int(w) // 4, K=K, pts=self.pts_in_hull)
            centers, conf = centers.astype(np.float64), conf.astype(np.float64)
            return (centers, conf) if return_conf else centers
        if method != 'sampled':
            raise ValueError("method must be 'gpu' or 'sampled'")
        from sklearn.cluster import KMeans
        cdf = np.cumsum(np.asarray(self.dist_ab[:, h, w]))
        cdf /= cdf[-1]
        u = np.random.uniform(low=0, high=1.0, size=N)
        samples = self.pts_in_hull[np.searchsorted(cdf, u, side='right'), :]   # == np.digitize(u, cdf)
        km = KMeans(n_clusters=K).fit(samples)
        mass = np.bincount(km.labels_, minlength=K)
        order = np.argsort(mass)[::-1]
        centers, conf = km.cluster_centers_[order, :], mass[order] / float(N)
        return (centers, conf) if return_conf else centers

    def compute_entropy(self):
        neg = getattr(self.dist_ab, "_negentropy", None)
        if neg is not None:
            # the resident distribution: sum_k d log d at (X/4)^2 on the device, replicated x4 like the map itself
            # (replicated pixels have identical distributions, so this is the reference's value at every pixel)
            self.dist_entropy = np.repeat(np.repeat(neg(), 4, axis=0), 4, axis=1)
            return
        d = np.asarray(self.dist_ab)
        self.dist_entropy = np.sum(d * np.log(d), axis=0)


class ColorizeImageB200GlobDist(ColorizeImageB200):
    """<-> ColorizeImageCaffeGlobDist (reference :445-463): colorization conditioned on a global ab histogram.
    The global-hints branch of models/global_model/deploy_nodist.prototxt:38-172,501-527 is bolted onto the
    local-hints network (a superset of the Caffe global model, whose conv1_1 ignores the local hints); its
    weights arrive as extra state_dict keys `glob.{0..3}.*` (include/idc_b200.h).  Spec-only: no reference
    weights or vectors exist for it offline."""

    def __init__(self, Xd=256, maskcent=False, engine="wgmma"):
        ColorizeImageB200.__init__(self, Xd, maskcent=maskcent, engine=engine)
        self.glob_mask_mult = 1.

    def prep_net(self, gpu_id=None, path='', state_dict=None, calibrate=None):
        import torch
        from .engine import LhnContext
        if state_dict is None:
            state_dict = torch.load(path, map_location='cpu')
        device = 0 if gpu_id is None else int(gpu_id)
        ranges = self._calibrate(calibrate, state_dict, device, global_hints=True)
        self._ctx = LhnContext(device=device, max_n=1, H=self.Xd, W=self.Xd, engine=self.engine, global_hints=True)
        self._ctx.load_state_dict(state_dict, act_ranges=ranges)
        self.net_set = True

    def get_global_histogram(self, ref_rgb_u8):
        """DemoGlobalHistogramTransfer.ipynb:176-182: the reference image is resized to Xd x Xd, then
        global_stats.prototxt -> the first 313 entries are `glob_dist`."""
        import cv2
        from . import prepost
        img = cv2.resize(ref_rgb_u8, (self.Xd, self.Xd))
        self.glob_vec = prepost.global_stats_gpu(img, self._ctx.device)
        return self.glob_vec[:313].copy()

    def net_forward(self, input_ab, input_mask, glob_dist=-1):
        if ColorizeImageBase.net_forward(self, input_ab, input_mask) == -1:
            return -1
        glob = np.zeros((1, 316), np.float32)            # "run without this, zero it out" (reference :454-456)
        if np.array(glob_dist).flatten()[0] != -1:
            glob[0, :313] = np.asarray(glob_dist, dtype=np.float32)
            glob[0, 313] = self.glob_mask_mult             # reference :458-459; the s_avg input stays 0 as in the reference
        self._click(self._ctx, float(self.mask_cent), glob=glob)
        return self.output_rgb


# =============================================================================================
# Caffe-named wrapper surface (reference :375-442, :445-463, :466-561).  The notebooks and ideepcolor.py:60-65
# instantiate ColorizeImageCaffe / ColorizeImageCaffeDist / ColorizeImageCaffeGlobDist; these classes keep those
# names' semantics on the H100 engine:
#   * Caffe scaling (SURVEY q4): the deploy nets feed RAW L-50, raw ab and mask x 110 into conv1_1 and scale the
#     regression head by 100 (deploy_nodist.prototxt:19-51, :812-822; `self.mask_mult = 110.`, :383), where the
#     PyTorch model feeds L/100, ab/110, mask and scales by 110.  The engine normalises the PyTorch way inside
#     conv1_1_kernel, so a Caffe-scaled weight set is mapped exactly at load time (conv1_1 input channels x 100, x 110,
#     x 110; `tanh_scale` = 100) -- see `caffe_scaled_state_dict`.
#   * 313-bin head (deploy_nopred.prototxt:651-850): `dist_ab` = softmax(S * logits) over the in-gamut bins,
#     `pred_ab` = annealed mean (T = 2.6); `get_ab_reccs` works on `pts_in_hull` (313 bins).
# There is no .caffemodel parser offline (no Caffe, no caffe.proto): `caffemodel_path` is a torch state_dict file
# holding the Caffe blobs under the reference state_dict key names (+ the `caffe.*` keys of include/idc_b200.h), or an
# in-memory `state_dict`.  Spec-only: no Caffe weights or vectors exist offline (parity unpinned, oracle/caffe_spec.py).
# =============================================================================================
def caffe_scaled_state_dict(state_dict):
    """Caffe-scaled weights (conv1_1 trained on raw L-50 / ab / mask*110) -> the engine's PyTorch-scaled convention.
    Exact: w' . (L/100, ab/110, mask) == w . (L, ab, mask*110) with w' = w * (100, 110, 110, 110) per input channel."""
    import torch
    sd = dict(state_dict)
    w = sd["model1.0.weight"]
    w = w.detach().cpu().numpy() if hasattr(w, "detach") else np.asarray(w)
    scale = np.array([100.0, 110.0, 110.0, 110.0], dtype=np.float64).reshape(1, 4, 1, 1)
    sd["model1.0.weight"] = torch.from_numpy((w.astype(np.float64) * scale).astype(np.float32))
    return sd


class ColorizeImageB200Caffe(ColorizeImageB200):
    """<-> ColorizeImageCaffe (reference :375-442): regression model with the Caffe input / output scaling."""
    _caffe313 = False
    _global_hints = False

    def __init__(self, Xd=256, engine="wgmma"):
        ColorizeImageB200.__init__(self, Xd, maskcent=False, engine=engine)
        self.mask_mult = 110.                     # reference :383
        self.pred_ab_layer = 'pred_ab'
        from . import prepost
        self.pts_in_hull = prepost.pts_in_hull().astype(np.float64)       # 313 x 2, in-gamut (reference :388-389)

    def prep_net(self, gpu_id=0, prototxt_path='', caffemodel_path='', state_dict=None, calibrate=None):
        import torch
        from .engine import LhnContext
        print('gpu_id = %d, net_path = %s, model_path = %s' % (-1 if gpu_id is None else gpu_id, prototxt_path, caffemodel_path))
        if state_dict is None:
            state_dict = torch.load(caffemodel_path, map_location='cpu')
        self.gpu_id = gpu_id
        sd = caffe_scaled_state_dict(state_dict)
        if self._caffe313:
            sd["caffe.pts_in_hull"] = torch.from_numpy(self.pts_in_hull.astype(np.float32))   # reference :405-407
        device = 0 if gpu_id in (None, -1) else int(gpu_id)
        flags = dict(global_hints=self._global_hints, caffe313=self._caffe313, options={"tanh_scale": 100})
        ranges = self._calibrate(calibrate, sd, device, **flags)
        self._ctx = LhnContext(device=device, max_n=1, H=self.Xd, W=self.Xd, engine=self.engine, **flags)
        self._ctx.load_state_dict(sd, act_ranges=ranges)
        self.net_set = True

    def _engine_inputs(self):
        A = np.ascontiguousarray(self.img_l_mc, dtype=np.float32)[None]
        B = np.ascontiguousarray(self.input_ab_mc, dtype=np.float32)[None]
        M = np.ascontiguousarray(self.input_mask_mult / self.mask_mult, dtype=np.float32)[None]   # x110 lives in the weights
        return A, B, M

    def net_forward(self, input_ab, input_mask):
        if ColorizeImageBase.net_forward(self, input_ab, input_mask) == -1:
            return -1
        self._click(self._ctx, 0.0, mask_div=self.mask_mult)     # the x110 of the mask lives in the conv1_1 weights
        return self.output_rgb                                    # output_ab_raw = the `pred_ab` blob (tanh * 100)


class ColorizeImageB200CaffeGlobDist(ColorizeImageB200Caffe):
    """<-> ColorizeImageCaffeGlobDist (reference :445-463): additional 313-bin global histogram input."""
    _global_hints = True

    def __init__(self, Xd=256, engine="wgmma"):
        ColorizeImageB200Caffe.__init__(self, Xd, engine=engine)
        self.glob_mask_mult = 1.
        self.glob_layer = 'glob_ab_313_mask'

    def get_global_histogram(self, ref_rgb_u8):
        """DemoGlobalHistogramTransfer.ipynb:176-182 (gt_glob_net = global_stats.prototxt on the resized reference image)."""
        import cv2
        from . import prepost
        self.glob_vec = prepost.global_stats_gpu(cv2.resize(ref_rgb_u8, (self.Xd, self.Xd)), self._ctx.device)
        return self.glob_vec[:313].copy()

    def net_forward(self, input_ab, input_mask, glob_dist=-1):
        if ColorizeImageBase.net_forward(self, input_ab, input_mask) == -1:
            return -1
        glob = np.zeros((1, 316), np.float32)            # "run without this, zero it out" (reference :454-456)
        if np.array(glob_dist).flatten()[0] != -1:
            glob[0, :313] = np.asarray(glob_dist, dtype=np.float32)
            glob[0, 313] = self.glob_mask_mult             # reference :458-459
        self._click(self._ctx, 0.0, glob=glob, mask_div=self.mask_mult)
        return self.output_rgb


class _LazyDist313(object):
    """[313, X, X] view of `dist_ab_S`: one pixel (313 floats) is computed on demand from the resident 313-bin logits
    (idc_caffe313_dist_pixel); the reference materialises 313 x X x X floats per forward and reads one pixel of it per
    click (reference :505, :521).  The whole map (np.asarray, any other index) is one idc_caffe313_dist_map launch and
    one copy to the host, kept on this view: net_forward makes a new view, so the copy lives for one forward."""

    def __init__(self, ctx, X, S):
        self._ctx, self._S = ctx, S
        self.shape = (313, X, X)
        self.dtype = np.dtype(np.float32)
        self._host = self._full = None

    def __getitem__(self, idx):
        if isinstance(idx, tuple) and len(idx) == 3 and all(isinstance(i, (int, np.integer)) for i in idx[1:]):
            return self._ctx.caffe313_dist_pixel(0, int(idx[1]), int(idx[2]), self._S)[idx[0]]
        return self.__array__()[idx]

    def __array__(self, dtype=None, copy=None):
        if self._host is None:
            self._host = self._ctx.caffe313_dist_map(1, self._S)[0].cpu().numpy()
        a = self._host
        if dtype is not None:
            return a.astype(dtype)
        return a.copy() if copy else a

    def full(self, in_hull):
        """dist_ab_full [529, X, X] float64 (reference :503): the cached map scattered to the in-gamut bins, once."""
        if self._full is None:
            self._full = np.zeros((in_hull.shape[0],) + self.shape[1:])
            self._full[in_hull] = self.__array__()
        return self._full

    def negentropy(self):
        """compute_entropy's sum_k d log d [X, X] float32: map and sum on the device, only [X, X] is copied back."""
        from . import prepost
        return prepost.negentropy_gpu(self._ctx.caffe313_dist_map(1, self._S))[0].cpu().numpy()


class ColorizeImageB200CaffeDist(_DistPlots, ColorizeImageB200Caffe):
    """<-> ColorizeImageCaffeDist (reference :466-561): the 313-bin distribution model.  `pred_ab` is the annealed
    mean of the 313-bin head (deploy_nopred.prototxt:827-850), `dist_ab` the S-softened distribution (:808-820)."""
    _caffe313 = True

    def __init__(self, Xd=256, engine="wgmma"):
        ColorizeImageB200Caffe.__init__(self, Xd, engine=engine)
        self.dist_ab_set = False
        self.scale_S_layer = 'scale_S'
        self.dist_ab_S_layer = 'dist_ab_S'
        g = np.arange(-110, 120, 10)
        # pts_grid.npy is (a, b)-ordered with a slowest (SURVEY q3): pts_grid[i] = (g[i // 23], g[i % 23])
        self.pts_grid = np.stack([np.repeat(g, 23), np.tile(g, 23)], axis=1)
        hull = set(map(tuple, self.pts_in_hull.astype(int).tolist()))
        self.in_hull = np.array([tuple(p) in hull for p in self.pts_grid.tolist()])      # identity: pts_grid[in_hull] == pts_in_hull
        self.AB = self.pts_grid.shape[0]
        self.A = self.B = int(np.sqrt(self.AB))
        self.dist_entropy = np.zeros((self.Xd, self.Xd))

    def prep_net(self, gpu_id=0, prototxt_path='', caffemodel_path='', S=.2, state_dict=None, calibrate=None):
        ColorizeImageB200Caffe.prep_net(self, gpu_id, prototxt_path=prototxt_path, caffemodel_path=caffemodel_path,
                                        state_dict=state_dict, calibrate=calibrate)
        self.S = S

    def net_forward(self, input_ab, input_mask):
        if ColorizeImageBase.net_forward(self, input_ab, input_mask) == -1:
            return -1
        import torch
        from . import _lib
        A, B, M = self._engine_inputs()
        dev = "cuda:%d" % self._ctx.device
        dA, dB, dM = (torch.from_numpy(a).to(dev) for a in (A, B, M))
        self._ctx.forward_device(dA, dB, dM, 0.0)                      # trunk + hyper-column + pred_313 logits
        pred = self._ctx.caffe313_pred_ab(1, T=2.6)                    # annealed-mean `pred_ab` [1,2,X,X] (device)
        # lab2rgb_transpose(self.img_l, pred_ab) (data/colorize_image.py:20-28) on the float64 L plane the reference
        # converts, not on the FP32 L - 50 the network reads (an FP32 ulp of L can flip a truncating cast): an order-0
        # render at the net size samples pred_ab exactly
        Xd = self.Xd
        d_L = torch.from_numpy(np.ascontiguousarray(self.img_l, dtype=np.float64).reshape(Xd, Xd)).to(dev)
        d_ab = pred[0].double().contiguous()
        rgb = torch.empty((Xd, Xd, 3), dtype=torch.uint8, device=dev)
        st = torch.cuda.current_stream(self._ctx.device).cuda_stream
        rc = _lib.load().idc_render_planes_u8(self._ctx.device, Xd, Xd, d_ab.data_ptr(), 0, 0, None, 0,
                                              _lib.RENDER_L_PLANE, d_L.data_ptr(), Xd, Xd, rgb.data_ptr(), st)
        if rc != _lib.IDC_OK:
            raise _lib.IdcError(rc, "idc_render_planes_u8 failed")
        self.output_ab_raw = pred[0].cpu().numpy()
        self.output_rgb = rgb.cpu().numpy()
        self._set_out_ab_()
        self.dist_ab = _LazyDist313(self._ctx, self.Xd, self.S)
        self.dist_ab_set = True
        return self.output_rgb

    @property
    def dist_ab_full(self):
        return self.dist_ab.full(self.in_hull)

    @property
    def dist_ab_grid(self):
        return self.dist_ab_full.reshape((self.A, self.B, self.Xd, self.Xd))

    def get_ab_reccs(self, h, w, K=5, N=25000, return_conf=False, method='gpu'):
        """reference :515-547 on the 313 in-gamut bins.  method='gpu': weighted k-means on the device (the N -> infinity
        limit, as ColorizeImageB200Dist; idc_caffe313_reccs_batch on this one pixel); method='sampled': the reference's
        np.random + sklearn procedure."""
        if not self.dist_ab_set:
            print('Need to set prediction first')
            return 0
        if method == 'gpu':
            centers, conf, _ = self._ctx.caffe313_reccs_batch([(0, int(h), int(w))], K, S=self.S)
            centers, conf = centers[0].cpu().numpy().astype(np.float64), conf[0].cpu().numpy().astype(np.float64)
            return (centers, conf) if return_conf else centers
        if method != 'sampled':
            raise ValueError("method must be 'gpu' or 'sampled'")
        from sklearn.cluster import KMeans
        cmf = np.cumsum(np.asarray(self.dist_ab[:, int(h), int(w)], dtype=np.float64))
        cmf /= cmf[-1]
        samples = self.pts_in_hull[np.digitize(np.random.uniform(low=0, high=1.0, size=N), bins=cmf), :]
        km = KMeans(n_clusters=K).fit(samples)
        cnt = np.histogram(km.labels_, np.arange(0, K + 1))[0]
        order = np.argsort(cnt, axis=0)[::-1]
        centers, conf = km.cluster_centers_[order, :], 1. * cnt[order] / N
        return (centers, conf) if return_conf else centers

    def compute_entropy(self):
        self.dist_entropy = self.dist_ab.negentropy()
