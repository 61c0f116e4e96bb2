"""Thin Python handle on one `idc_ctx` (one device, one geometry).

Host-side plumbing only: pointer marshalling, torch tensors as device memory, streams.
All arithmetic of the forward happens in libidc_b200.so.
"""
import ctypes
import json
import math
import os

import numpy as np

from . import _lib


def _np_ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def as_hints(rects):
    """A hint list as the C ABI's idc_hint array: a structured array with the fields img, y0, x0, y1, x1, a, b (any
    numeric field types; a / b are rounded to float32 like the dense ab plane) or a sequence of such 7-tuples."""
    if isinstance(rects, np.ndarray) and rects.dtype.names:
        out = np.empty(rects.shape[0], _lib.HINT_DTYPE)
        for f in _lib.HINT_DTYPE.names:
            out[f] = rects[f]
        return out
    return np.array([tuple(r) for r in rects], dtype=_lib.HINT_DTYPE).reshape(-1)


# every activation buffer a context can store, in plan order (idc_act_name lists the ones a given context has:
# conv10_2 on the SIMT engine or with keep_conv10, hyper with caffe313)
ACT_BUFFERS = ("a1_1", "conv1_2", "a2_1", "conv2_2", "a3_1", "a3_2", "conv3_3", "a4_1", "a4_2", "conv4_3",
               "a5_1", "a5_2", "conv5_3", "a6_1", "a6_2", "conv6_3", "a7_1", "a7_2", "conv7_3",
               "a8_1", "a8_2", "conv8_3", "hyper", "a9_1", "conv9_3", "a10_1", "conv10_2")
CALIBRATION_MAX_N = 4        # images per forward of the temporary measuring context


def check_act_ranges(ranges):
    """-> {buffer: float} or ValueError naming the first entry that is not a known buffer with a finite range > 0."""
    if not isinstance(ranges, dict):
        raise ValueError("activation ranges: need a {buffer: max_abs} object, got %s" % type(ranges).__name__)
    out = {}
    for k, v in ranges.items():
        if k not in ACT_BUFFERS:
            raise ValueError("activation ranges: %r is not an activation buffer" % (k,))
        if isinstance(v, bool) or not isinstance(v, (int, float, np.floating, np.integer)) \
                or not math.isfinite(v) or not v > 0:
            raise ValueError("activation ranges: %s = %r must be a finite number > 0" % (k, v))
        out[k] = float(v)
    return out


def save_act_ranges(path, ranges):
    """Write measured ranges as a flat JSON object {buffer: max_abs}.  Ranges belong to a checkpoint (and its input
    scaling), not to a network size: a file measured at one Xd serves every Xd."""
    with open(path, "w") as f:
        json.dump(check_act_ranges(ranges), f, indent=1, sort_keys=True)
        f.write("\n")


def load_act_ranges(path):
    with open(path) as f:
        try:
            return check_act_ranges(json.load(f))
        except ValueError as e:
            raise ValueError("%s: %s" % (path, e))


def calibration_batch(images, X, hints=8, seed=0, device=0, global_hints=False):
    """Colour photos (paths or HxWx3 uint8 RGB arrays, at most 128) -> the network's own inputs (L_mc [n,1,X,X], ab
    [n,2,X,X], mask [n,1,X,X][, glob [n,316]]), device float32 tensors, through the same device steps as a photo batch
    (idc_photo_prep: cv2-exact resize, rgb2lab, L - 50).  A click session is what the network will see, so every
    second photo also carries `hints` hint rectangles, 1-9 pixels wide like the GUI's, at seeded places, painted with
    the photo's own ab at their centres; with global_hints every second photo carries its own global-statistics vector.
    More, and more varied, photos give safer ranges; the headroom of the exponent rule covers what they miss."""
    import torch
    from . import photos as P
    lib = _lib.load()
    imgs = [P.check_photo(P.read_photo(p) if not isinstance(p, np.ndarray) else np.ascontiguousarray(p), "photo %d" % i)
            for i, p in enumerate(images)]
    n = len(imgs)
    if not 1 <= n <= _lib.MAX_PHOTOS:
        raise ValueError("calibration needs 1 to %d photos, got %d" % (_lib.MAX_PHOTOS, n))
    dev = torch.device("cuda:%d" % device)
    st = torch.cuda.current_stream(dev).cuda_stream
    table, src = P.pack_photos(imgs)
    src = torch.from_numpy(src).to(dev)
    L_mc = torch.empty((n, 1, X, X), dtype=torch.float32, device=dev)
    rgb = torch.empty((n, X, X, 3), dtype=torch.uint8, device=dev)
    lab = torch.empty((n, 3, X, X), dtype=torch.float64, device=dev)
    _lib.check(None, lib.idc_photo_prep(device, n, table.ctypes.data, src.data_ptr(), X, L_mc.data_ptr(), rgb.data_ptr(), st))
    _lib.check(None, lib.idc_rgb2lab_f64(device, n, X, X, rgb.data_ptr(), lab.data_ptr(), st))
    own_ab = lab[:, 1:].cpu().numpy()
    rng = np.random.RandomState(seed)
    rects = [[] for _ in range(n)]
    for i in range(1, n, 2):
        for _ in range(hints):
            y, x, p = int(rng.randint(X)), int(rng.randint(X)), int(rng.randint(5))     # (2p+1)-pixel square, p = 0..4
            rects[i].append((i, max(y - p, 0), max(x - p, 0), min(y + p, X - 1), min(x + p, X - 1),
                             own_ab[i, 0, y, x], own_ab[i, 1, y, x]))
    count = sum(map(len, rects))
    if count > _lib.MAX_HINTS:
        raise ValueError("%d calibration hints, at most %d" % (count, _lib.MAX_HINTS))
    block = np.empty(P.HINT_BLOCK_BYTES, np.uint8)
    block = block[:P.pack_hints([as_hints(r) for r in rects], block)]
    d_block = torch.from_numpy(block).to(dev)
    ab = torch.empty((n, 2, X, X), dtype=torch.float32, device=dev)
    mask = torch.empty((n, 1, X, X), dtype=torch.float32, device=dev)
    _lib.check(None, lib.idc_hint_raster(device, n, X, X, count, d_block.data_ptr(), ab.data_ptr(), mask.data_ptr(), st))
    if not global_hints:
        return L_mc, ab, mask
    from . import prepost
    glob = torch.zeros((n, 316), dtype=torch.float32, device=dev)
    pts = torch.from_numpy(prepost.pts_in_hull()).to(dev)
    for i in range(1, n, 2):
        _lib.check(None, lib.idc_global_stats(device, X, X, rgb[i].data_ptr(), pts.data_ptr(), glob[i].data_ptr(), st))
    return L_mc, ab, mask, glob


def measure_act_ranges(sd, batches, H, W, device=0, maskcent=0., dist=False, global_hints=False, caffe313=False,
                       keep_conv10=False, options=None):
    """The largest |a| of every activation buffer of checkpoint `sd` over `batches` -> {buffer: max_abs}, for
    LhnContext.load_state_dict(sd, act_ranges=...).  batches: one (L_mc, ab, mask[, glob]) tuple or a list of them,
    float32 device tensors or host arrays ([n,1,H,W], [n,2,H,W], [n,1,H,W], [n,316]).
    The measurement runs on a temporary exact-FP32 context (engine="simt") of the same geometry and flags, not on the
    wgmma engine being calibrated: FP32 planes cannot saturate, so one pass gives every buffer's true range even where
    several buffers in a chain would saturate.  The context is closed before this returns, so its buffers are free
    again before the caller builds its own.  A buffer that stayed 0 is left out (it keeps the weight-derived
    exponent); a NaN or infinite range raises, naming the buffer."""
    import torch
    if isinstance(batches, tuple):
        batches = [batches]
    dev = torch.device("cuda:%d" % device)
    ctx = LhnContext(device=device, max_n=CALIBRATION_MAX_N, H=H, W=W, dist=dist, engine="simt", global_hints=global_hints,
                     caffe313=caffe313, keep_conv10=keep_conv10, options=options)
    try:
        ctx.load_state_dict(sd)
        names = ctx.act_names()
        top = dict.fromkeys(names, 0.0)
        for batch in batches:
            t = [torch.as_tensor(a, dtype=torch.float32).to(dev).contiguous() for a in batch]
            for i in range(0, t[0].shape[0], CALIBRATION_MAX_N):
                c = [a[i:i + CALIBRATION_MAX_N] for a in t]
                ctx.forward_device(c[0], c[1], c[2], maskcent, glob=c[3] if len(c) > 3 else None)
                for b in names:
                    v = ctx.act_absmax(b, c[0].shape[0])
                    top[b] = v if math.isnan(v) else max(top[b], v)
    finally:
        ctx.close()
    for b, v in top.items():
        if not math.isfinite(v):
            raise ValueError("activation %s reaches %r on the calibration images: the checkpoint does not compute "
                             "finite values" % (b, v))
    return {b: v for b, v in top.items() if v > 0}


def resolve_calibration(calibrate, measure):
    """The `calibrate=` argument of the wrappers -> {buffer: max_abs} or None: None; a dict; the path of a JSON file
    written by save_act_ranges; or a list of photos (paths / uint8 RGB arrays), measured now by measure(photos)."""
    if calibrate is None:
        return None
    if isinstance(calibrate, dict):
        return check_act_ranges(calibrate)
    if isinstance(calibrate, (str, bytes, os.PathLike)):
        return load_act_ranges(calibrate)
    return check_act_ranges(measure(list(calibrate)))


PHOTO_EXTS = (".jpg", ".jpeg", ".png", ".bmp", ".tif", ".tiff", ".webp")


def calibration_source(path, max_photos=16, seed=0):
    """The --calibrate argument of the command-line front ends -> a `calibrate=` value: a folder becomes a seeded
    sample of at most max_photos of its photos (sorted by name), a file is taken as a saved JSON of ranges."""
    if os.path.isdir(path):
        names = sorted(f for f in os.listdir(path) if os.path.splitext(f)[1].lower() in PHOTO_EXTS)
        if not names:
            raise ValueError("--calibrate %s: no photos in this folder" % path)
        if len(names) > max_photos:
            pick = np.random.RandomState(seed).choice(len(names), max_photos, replace=False)
            names = [names[i] for i in sorted(pick)]
        return [os.path.join(path, f) for f in names]
    if os.path.isfile(path):
        return path
    raise ValueError("--calibrate %s: neither a folder of photos nor a JSON file of ranges" % path)


class LhnContext(object):
    """Local Hints Network forward context (the H100 stand-in for
    `SIGGRAPHGenerator(...).cuda().eval()`, /root/reference/data/colorize_image.py:221-232)."""

    def __init__(self, device=0, max_n=1, H=256, W=256, dist=False, engine="wgmma", fast_fp16=False,
                 global_hints=False, use_graph=True, keep_conv10=False, caffe313=False, options=None):
        """engine: "wgmma" (tensor cores; "tcgen05" is accepted as the name earlier releases used) or "simt"
        (exact FP32 CUDA cores).  options: {name: int} plan-time switches, see include/idc_b200.h: idc_set_option
        (halo, pairs, mt, chunk_kb, split_k, host_pipe, pdl, side_dist, conv1_1_umma, tanh_scale, act_exp.<buffer>)."""
        self.lib = _lib.load()
        flags = 0
        if dist:
            flags |= _lib.FLAG_DIST
        if engine == "simt":
            flags |= _lib.FLAG_ENGINE_SIMT
        elif engine not in ("wgmma", "tcgen05"):
            raise ValueError("engine must be 'wgmma' or 'simt'")
        if fast_fp16:
            flags |= _lib.FLAG_FAST_FP16
        if global_hints:
            flags |= _lib.FLAG_GLOBAL_HINTS
        if not use_graph:
            flags |= _lib.FLAG_NO_GRAPH
        if keep_conv10:
            flags |= _lib.FLAG_KEEP_CONV10
        if caffe313:
            flags |= _lib.FLAG_CAFFE313
        self.device, self.max_n, self.H, self.W = int(device), int(max_n), int(H), int(W)
        self.dist, self.global_hints, self.flags = bool(dist), bool(global_hints), flags
        h = ctypes.c_void_p()
        rc = self.lib.idc_create(self.device, self.max_n, self.H, self.W, flags, ctypes.byref(h))
        if rc != _lib.IDC_OK:
            raise _lib.IdcError(rc, "idc_create(device=%d, max_n=%d, %dx%d) failed -- a CUDA sm_90 (H100) device is "
                                    "required; there is no CPU fallback" % (device, max_n, H, W))
        self.h = h
        self.ready = False
        self._pinned = []
        # bookkeeping of the reference-facing wrappers that share this context (colorize_image.py: _click)
        self._wrapper_click, self._wrapper_staged_l, self._wrapper_last, self._wrapper_shared = None, [], None, False
        self._dist_resident = False
        for k, v in (options or {}).items():
            self.set_option(k, v)

    def set_option(self, name, value):
        _lib.check(self.h, self.lib.idc_set_option(self.h, name.encode(), int(value)))

    # ---- weights ---------------------------------------------------------------------------
    def load_state_dict(self, sd, act_ranges=None):
        """sd: {reference state_dict key: torch.Tensor | ndarray}.  Packs + uploads.
        act_ranges: {buffer: max_abs} from measure_act_ranges: the wgmma engine then stores those buffers by their
        measured range instead of the estimate from the weights (idc_set_act_range); buffers this context does not
        store (conv10_2 with the fused head) are ignored.  Ranges stay with the context: loading another checkpoint
        into it later without act_ranges packs it with the ranges set here."""
        if act_ranges:
            mine = set(self.act_names())
            for b, v in check_act_ranges(act_ranges).items():
                if b in mine:
                    _lib.check(self.h, self.lib.idc_set_act_range(self.h, b.encode(), v))
        for k, v in sd.items():
            self._load_tensor(k, v)
        _lib.check(self.h, self.lib.idc_finalize_weights(self.h))
        self.ready = True

    def _load_tensor(self, k, v):
        a = v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)
        if a.dtype == np.float32:
            dt = _lib.F32
        elif a.dtype == np.float64:
            dt = _lib.F64
        elif a.dtype == np.int64:
            dt = _lib.I64
        else:
            a = a.astype(np.float32)
            dt = _lib.F32
        a = np.ascontiguousarray(a)
        dims = (ctypes.c_int64 * max(a.ndim, 1))(*a.shape)
        _lib.check(self.h, self.lib.idc_load_tensor(self.h, k.encode(), _np_ptr(a), dt, a.ndim, dims))

    def weights_arena(self):
        p, n = ctypes.c_void_p(), ctypes.c_size_t()
        _lib.check(self.h, self.lib.idc_weights_arena(self.h, ctypes.byref(p), ctypes.byref(n)))
        return p.value, n.value

    def reserve_weights(self):
        _lib.check(self.h, self.lib.idc_reserve_weights(self.h))

    def adopt_weights(self):
        """Take the arena as received (reserve_weights, then a copy into weights_arena()).  The Caffe 313-bin head's
        bin centres are not part of the arena: with caffe313 they are the package's pts_in_hull, the centres every
        loader of the Caffe distribution model adds (ColorizeImageB200Caffe.prep_net, PhotoColorizer)."""
        if self.flags & _lib.FLAG_CAFFE313:
            from .prepost import pts_in_hull
            self._load_tensor("caffe.pts_in_hull", pts_in_hull())
        _lib.check(self.h, self.lib.idc_adopt_weights(self.h))
        self.ready = True

    # ---- forward ---------------------------------------------------------------------------
    def forward_device(self, L_mc, ab, mask, maskcent=0.0, glob=None, want_dist=False, want_rgb=False,
                       out_ab=None, out_dist=None, out_rgb=None):
        """torch CUDA float32 tensors [n,1,H,W], [n,2,H,W], [n,1,H,W] -> dict of torch tensors.
        Asynchronous on torch's current stream."""
        import torch
        n = L_mc.shape[0]
        for t in (L_mc, ab, mask):
            assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
        dev = L_mc.device
        if out_ab is None:
            out_ab = torch.empty((n, 2, self.H, self.W), dtype=torch.float32, device=dev)
        if want_dist and out_dist is None:
            out_dist = torch.empty((n, 529, self.H // 4, self.W // 4), dtype=torch.float32, device=dev)
        if want_rgb and out_rgb is None:
            out_rgb = torch.empty((n, self.H, self.W, 3), dtype=torch.uint8, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        rc = self.lib.idc_forward(self.h, n, self.H, self.W, L_mc.data_ptr(), ab.data_ptr(), mask.data_ptr(),
                                  float(maskcent), glob.data_ptr() if glob is not None else None,
                                  out_ab.data_ptr(), out_dist.data_ptr() if want_dist else None,
                                  out_rgb.data_ptr() if want_rgb else None, st)
        _lib.check(self.h, rc)
        return {"ab": out_ab, "dist": out_dist if want_dist else None, "rgb": out_rgb if want_rgb else None}

    def set_image(self, L_mc):
        """Upload the mean-centred L planes [n,1,H,W] once (the reference's set_image / load_image half of a session);
        forward_host(None, ab, mask, ...) then reuses them.  None forgets the image."""
        if L_mc is None:
            _lib.check(self.h, self.lib.idc_set_image(self.h, 0, self.H, self.W, None))
            return
        assert L_mc.dtype == np.float32 and L_mc.flags["C_CONTIGUOUS"]
        _lib.check(self.h, self.lib.idc_set_image(self.h, int(L_mc.shape[0]), self.H, self.W, _np_ptr(L_mc)))

    def set_hints(self, rects):
        """The hint list the next forward_host(..., None, None, n=...) rasterises on the device (idc_set_hints):
        rectangles (img, y0, x0, y1, x1, a, b), inclusive and clipped to the image; later ones paint over earlier ones.
        See `as_hints` for the accepted forms."""
        h = as_hints(rects)
        if h.shape[0] > _lib.MAX_HINTS:
            raise ValueError("at most %d hints, got %d" % (_lib.MAX_HINTS, h.shape[0]))
        _lib.check(self.h, self.lib.idc_set_hints(self.h, int(h.shape[0]), _np_ptr(h) if h.shape[0] else None))

    def graph_captures(self):
        """Click-graph instantiations of this context so far."""
        return self.lib.idc_graph_captures(self.h)

    def forward_host(self, L_mc, ab, mask, maskcent=0.0, glob=None, want_dist=False, want_rgb=False,
                     out_ab=None, out_dist=None, out_rgb=None, want_abq=False, out_abq=None, n=None):
        """numpy float32 C-contiguous host arrays (pinned or pageable) -> dict of numpy arrays.
        Synchronous; includes H2D + D2H.  want_abq: also the reference's quantised output_ab
        (rgb2lab(rgb)[1:], float64; implies want_rgb).  L_mc None = the image uploaded by set_image.
        ab and mask None = the hint list of set_hints, rasterised on the device; pass the batch size as n."""
        want_rgb = want_rgb or want_abq
        if n is None:
            n = (ab if ab is not None else L_mc).shape[0]
        if L_mc is not None:                 # an explicit L replaces the resident image: wrappers must re-stage theirs
            self._wrapper_staged_l, self._wrapper_last = [], None
        for a in (ab, mask, L_mc):
            assert a is None or (a.dtype == np.float32 and a.flags["C_CONTIGUOUS"])
        if out_ab is None:
            out_ab = np.empty((n, 2, self.H, self.W), np.float32)
        if want_dist and out_dist is None:
            out_dist = np.empty((n, 529, self.H // 4, self.W // 4), np.float32)
        if want_rgb and out_rgb is None:
            out_rgb = np.empty((n, self.H, self.W, 3), np.uint8)
        if want_abq and out_abq is None:
            out_abq = np.empty((n, 2, self.H, self.W), np.float64)
        rc = self.lib.idc_forward_host_q(self.h, n, self.H, self.W, None if L_mc is None else _np_ptr(L_mc),
                                         None if ab is None else _np_ptr(ab), None if mask is None else _np_ptr(mask),
                                         float(maskcent), _np_ptr(glob) if glob is not None else None,
                                         _np_ptr(out_ab), _np_ptr(out_dist) if want_dist else None,
                                         _np_ptr(out_rgb) if want_rgb else None,
                                         _np_ptr(out_abq) if want_abq else None)
        _lib.check(self.h, rc)
        return {"ab": out_ab, "dist": out_dist if want_dist else None, "rgb": out_rgb if want_rgb else None,
                "abq": out_abq}

    # ---- zero-copy click path ---------------------------------------------------------------
    def click_buffers(self, n=1, glob=False, hints=False):
        """Page-locked I/O arrays for the interactive call (n <= 4), laid out back to back so that a click is one H2D and
        one D2H with NO copy by the CPU: pass them to forward_host (L_mc / ab / mask (/ glob) as inputs, out_ab / out_rgb /
        out_abq as outputs).  -> dict of numpy views; they stay valid until close().  hints=True: for hint-list clicks
        (set_hints); there is no ab / mask block ("ab" and "mask" are None)."""
        HW = self.H * self.W
        planes = 1 if hints else 4                   # [L | glob] or [L | ab | mask | glob]
        b_ab, b_rgb, b_q = n * 2 * HW * 4, n * 3 * HW, n * 2 * HW * 8
        blocks = [self._host_block(nbytes) for nbytes in ((n * planes * HW + (n * 316 if glob else 0)) * 4,
                                                          b_ab + b_rgb + b_q)]
        fin = blocks[0].view(np.float32)
        return {"L_mc": fin[:n * HW].reshape(n, 1, self.H, self.W),
                "ab": None if hints else fin[n * HW:3 * n * HW].reshape(n, 2, self.H, self.W),
                "mask": None if hints else fin[3 * n * HW:4 * n * HW].reshape(n, 1, self.H, self.W),
                "glob": fin[planes * n * HW:].reshape(n, 316) if glob else None,
                "out_ab": blocks[1][:b_ab].view(np.float32).reshape(n, 2, self.H, self.W),
                "out_rgb": blocks[1][b_ab:b_ab + b_rgb].reshape(n, self.H, self.W, 3),
                "out_abq": blocks[1][b_ab + b_rgb:].view(np.float64).reshape(n, 2, self.H, self.W)}

    def _host_block(self, nbytes):
        p = self.lib.idc_host_alloc(nbytes)
        if not p:
            raise _lib.IdcError(-2, "idc_host_alloc(%d) failed" % nbytes)
        self._pinned.append(p)
        return np.frombuffer((ctypes.c_char * nbytes).from_address(p), dtype=np.uint8)

    def set_dist_resident(self, on=True):
        """Interactive mode: the dist head runs on every forward_host but stays on the device."""
        _lib.check(self.h, self.lib.idc_set_dist_resident(self.h, 1 if on else 0))
        self._dist_resident = bool(on)

    def set_click(self, img=0, y4=-1, x4=0, K=0):
        """Announce the clicked pixel of the (H/4 x W/4) grid before forward_host: its pmf and K colour suggestions
        come back with the same graph launch (fetch_dist / ab_reccs for that pixel are then host-side reads).
        y4 < 0 switches the mode off."""
        _lib.check(self.h, self.lib.idc_set_click(self.h, int(img), int(y4), int(x4), int(K)))

    def fetch_dist(self, img=0, y4=None, x4=None):
        """dist[img, :, y4, x4] (529 floats), or the whole [529, H/4, W/4] plane when y4 is None."""
        if y4 is None:
            out = np.empty((529, self.H // 4, self.W // 4), np.float32)
            _lib.check(self.h, self.lib.idc_fetch_dist(self.h, img, -1, 0, _np_ptr(out)))
        else:
            out = np.empty((529,), np.float32)
            _lib.check(self.h, self.lib.idc_fetch_dist(self.h, img, int(y4), int(x4), _np_ptr(out)))
        return out

    def ab_reccs(self, img, y4, x4, K=5, max_iter=100, n_init=8, pts=None):
        """Colour suggestions at dist[img, :, y4, x4] (reference get_ab_reccs, data/colorize_image.py:322-354)
        computed on the device: (centres [K,2], mass [K], Lloyd iterations)."""
        centers, conf, iters = np.empty((K, 2), np.float32), np.empty((K,), np.float32), ctypes.c_int(0)
        p = None if pts is None else np.ascontiguousarray(pts, np.float32)
        assert p is None or p.shape == (529, 2)
        _lib.check(self.h, self.lib.idc_ab_reccs(self.h, int(img), int(y4), int(x4), int(K), int(max_iter), int(n_init),
                                                 None if p is None else _np_ptr(p), _np_ptr(centers), _np_ptr(conf),
                                                 ctypes.byref(iters)))
        return centers, conf, iters.value

    def ab_reccs_batch(self, queries, K=5, max_iter=100, n_init=8, pts=None, out=None, out_pmf=None):
        """Colour suggestions at many pixels of the last forward's images in one device pass (idc_ab_reccs_batch):
        queries int [Q,3] rows (img, y4, x4) -> (centres [Q,K,2] float32, mass [Q,K] float32, Lloyd iterations [Q]
        int32) torch CUDA tensors, asynchronous on torch's current stream.  Query i equals ab_reccs(*queries[i], ...) on
        the same forward bit for bit.  Needs dist=True; the forward may be any forward call.  out: optional
        (centres, mass, iterations) tensors of those shapes and dtypes to write into (mass / iterations may be None).
        out_pmf: optional float32 CUDA tensor [Q,529] that receives each query's pmf (dist[img, :, y4, x4])."""
        import torch
        q = np.ascontiguousarray(queries, np.int32).reshape(-1, 3)
        p = None if pts is None else np.ascontiguousarray(pts, np.float32)
        if p is not None and p.shape != (529, 2):
            raise ValueError("pts: need [529, 2] ab coordinates, got %s" % (p.shape,))
        dev = torch.device("cuda:%d" % self.device)
        if out is None:
            n, k = q.shape[0], max(int(K), 0)
            out = (torch.empty((n, k, 2), dtype=torch.float32, device=dev), torch.empty((n, k), dtype=torch.float32, device=dev),
                   torch.empty((n,), dtype=torch.int32, device=dev))
        centers, conf, iters = out
        st = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(self.h, self.lib.idc_ab_reccs_batch(self.h, int(q.shape[0]), _np_ptr(q), int(K), int(max_iter),
                                                       int(n_init), None if p is None else _np_ptr(p), centers.data_ptr(),
                                                       None if conf is None else conf.data_ptr(),
                                                       None if iters is None else iters.data_ptr(),
                                                       None if out_pmf is None else out_pmf.data_ptr(), st))
        return centers, conf, iters

    # ---- Caffe-spec 313-bin head (IDC_FLAG_CAFFE313) ----------------------------------------
    def caffe313_pred_ab(self, n, T=2.6):
        """Annealed-mean ab [n,2,H,W] (device tensor) from the 313-bin logits of the last forward."""
        import torch
        out = torch.empty((n, 2, self.H, self.W), dtype=torch.float32, device="cuda:%d" % self.device)
        st = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.h, self.lib.idc_caffe313_pred_ab(self.h, n, float(T), out.data_ptr(), st))
        return out

    def caffe313_dist_pixel(self, img, y, x, S=0.2):
        """dist_ab_S[:, y, x] (313 floats) at one full-resolution pixel."""
        out = np.empty((313,), np.float32)
        _lib.check(self.h, self.lib.idc_caffe313_dist_pixel(self.h, int(img), int(y), int(x), float(S), _np_ptr(out)))
        return out

    def caffe313_dist_map(self, n=1, S=0.2):
        """The whole dist_ab_S map [n,313,H,W] (device tensor, torch's current stream) from the 313-bin logits of the
        last forward; every pixel equals caffe313_dist_pixel bit for bit."""
        import torch
        out = torch.empty((n, 313, self.H, self.W), dtype=torch.float32, device="cuda:%d" % self.device)
        st = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.h, self.lib.idc_caffe313_dist_map(self.h, int(n), float(S), out.data_ptr(), st))
        return out

    def caffe313_reccs_batch(self, queries, K=5, S=0.2, max_iter=100, n_init=8, out=None, out_pmf=None):
        """Colour suggestions of the 313-bin head at many full-resolution pixels of the last forward's images in one
        device pass (idc_caffe313_reccs_batch): queries int [Q,3] rows (img, y, x) -> (centres [Q,K,2] float32, mass
        [Q,K] float32, Lloyd iterations [Q] int32) torch CUDA tensors, asynchronous on torch's current stream.  Query i
        equals ColorizeImageB200CaffeDist.get_ab_reccs(y, x, K)'s device k-means on the same forward bit for bit: the
        pmf caffe313_dist_pixel(img, y, x, S) and the bin centres, both zero-padded to 529.  Needs caffe313=True.  out:
        optional (centres, mass, iterations) tensors to write into (mass / iterations may be None).  out_pmf: optional
        float32 CUDA tensor [Q,529] that receives each query's padded pmf."""
        import torch
        q = np.ascontiguousarray(queries, np.int32).reshape(-1, 3)
        dev = torch.device("cuda:%d" % self.device)
        if out is None:
            n, k = q.shape[0], max(int(K), 0)
            out = (torch.empty((n, k, 2), dtype=torch.float32, device=dev), torch.empty((n, k), dtype=torch.float32, device=dev),
                   torch.empty((n,), dtype=torch.int32, device=dev))
        centers, conf, iters = out
        st = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(self.h, self.lib.idc_caffe313_reccs_batch(self.h, int(q.shape[0]), _np_ptr(q), float(S), int(K),
                                                             int(max_iter), int(n_init), centers.data_ptr(),
                                                             None if conf is None else conf.data_ptr(),
                                                             None if iters is None else iters.data_ptr(),
                                                             None if out_pmf is None else out_pmf.data_ptr(), st))
        return centers, conf, iters

    def dist_negentropy(self, img=0):
        """sum_k d * log(d) over the 529 bins of the resident distribution of image img -> [H/4, W/4] float32 (the
        reference's compute_entropy statement before its x4 upsample); only this plane leaves the device."""
        out = np.empty((self.H // 4, self.W // 4), np.float32)
        _lib.check(self.h, self.lib.idc_dist_negentropy(self.h, int(img), _np_ptr(out)))
        return out

    # ---- introspection (tests) -------------------------------------------------------------
    def op_names(self):
        return [self.lib.idc_op_name(self.h, i).decode() for i in range(self.lib.idc_num_ops(self.h))]

    def activation_shape(self, name):
        c, h, w = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        _lib.check(self.h, self.lib.idc_get_activation(self.h, name.encode(), None, 0, ctypes.byref(c),
                                                       ctypes.byref(h), ctypes.byref(w)))
        return c.value, h.value, w.value

    def act_exponent(self, name):
        """The exponent S with which the wgmma engine stores activation `name` (value * 2^S in FP16 hi/lo)."""
        e = ctypes.c_int()
        _lib.check(self.h, self.lib.idc_act_exponent(self.h, name.encode(), ctypes.byref(e)))
        return e.value

    def act_names(self):
        """The activation buffers this context stores, in plan order."""
        return [self.lib.idc_act_name(self.h, i).decode() for i in range(self.lib.idc_num_acts(self.h))]

    def act_exponents(self):
        return {b: self.act_exponent(b) for b in self.act_names()}

    def act_absmax(self, name, n):
        """max |a| over the first n images of activation `name` as the last forward left it (idc_act_absmax)."""
        v = ctypes.c_float()
        _lib.check(self.h, self.lib.idc_act_absmax(self.h, name.encode(), int(n), ctypes.byref(v)))
        return v.value

    def get_activation(self, name, n):
        import torch
        c, h, w = self.activation_shape(name)
        out = torch.empty((n, c, h, w), dtype=torch.float32, device="cuda:%d" % self.device)
        _lib.check(self.h, self.lib.idc_get_activation(self.h, name.encode(), out.data_ptr(), out.numel(), None, None, None))
        return out

    def set_activation(self, name, t):
        assert t.is_cuda and t.is_contiguous()
        _lib.check(self.h, self.lib.idc_set_activation(self.h, name.encode(), t.shape[0], t.data_ptr()))

    def run_op(self, op_name, n):
        import torch
        st = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.h, self.lib.idc_run_op(self.h, op_name.encode(), n, st))

    def set_profiling(self, on):
        _lib.check(self.h, self.lib.idc_set_profiling(self.h, 1 if on else 0))

    def get_profile(self):
        """-> list of (slot name, mean ms per forward, FLOPs per image) since profiling was enabled."""
        names = ["pack+conv1_1"] + self.op_names() + ["heads+post"]
        buf = (ctypes.c_float * len(names))()
        rc = self.lib.idc_get_profile(self.h, buf, len(names))
        if rc < 0:
            _lib.check(self.h, rc)
        flops = [2.0 * self.H * self.W * 64 * 36] + [self.lib.idc_op_flops(self.h, i) for i in range(len(names) - 2)] + [0.0]
        return [(names[i], float(buf[i]), flops[i]) for i in range(len(names))]

    def last_launch_count(self):
        return self.lib.idc_last_launch_count(self.h)

    def flops_per_image(self):
        return self.lib.idc_flops_per_image(self.h)

    def close(self):
        if getattr(self, "h", None):
            self.lib.idc_destroy(self.h)
            self.h = None
            for p in getattr(self, "_pinned", []):
                self.lib.idc_host_free(p)
            self._pinned = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
