"""Batched photo colorization: photos of any sizes in, full-resolution results out, one device pass per batch.

The per-photo loop of the reference wrapper (data/colorize_image.py) is

    load_image(path) -> net_forward(zeros, zeros) -> get_img_fullres()   (+ get_result_PSNR() when evaluating)

`PhotoColorizer.colorize` computes the same results for a list of photos.  A batch of photos is packed back to back
into one page-locked buffer and goes through the device as

    H2D (copy stream) -> idc_photo_prep -> idc_hint_raster -> idc_forward -> idc_rgb2lab_f64 -> idc_photo_render
    (-> idc_rgb_sse) -> D2H (copy stream)

with two sets of buffers, so that batch k+1 is read, packed and uploaded and batch k-1 is copied back while batch k
computes.  Every value equals the single-photo path on the same forward: prep is the cv2-exact resize + skimage Lab of
`load_image`, the render is `get_img_fullres`'s scipy zoom of the quantised output_ab, and the PSNR is numpy's.
"""
import collections
import concurrent.futures
import ctypes
import os

import numpy as np

from . import _lib, engine

PhotoResult = collections.namedtuple("PhotoResult", "fullres rgb ab psnr")
PhotoResult.__doc__ = """One colorized photo.
    fullres  uint8 [H,W,3]   get_img_fullres(): the photo's own L with the network's ab zoomed to full resolution
    rgb      uint8 [X,X,3]   output_rgb (the network-size result)
    ab       float32 [2,X,X] output_ab_raw (the raw network output)
    psnr     float or None   get_result_PSNR() against the network-size photo, when asked for"""

XFULLRES_MAX = 10000          # the wrapper's Xfullres_max (ColorizeImageBase): larger photos are resized on the host


def read_photo(path):
    """A photo as `load_image` reads it: cv2.imread(path, 1), BGR -> RGB."""
    import cv2
    bgr = cv2.imread(path, 1)
    if bgr is None:
        raise IOError("cannot read image %r" % (path,))
    return np.ascontiguousarray(cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB))


def check_photo(a, what="photo"):
    """Raise ValueError unless `a` is an HxWx3 uint8 array whose longest side is at most XFULLRES_MAX."""
    if not isinstance(a, np.ndarray) or a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or min(a.shape[:2]) < 1:
        raise ValueError("%s: need an HxWx3 uint8 RGB array, got %s" % (what, getattr(a, "shape", type(a).__name__)))
    if max(a.shape[:2]) > XFULLRES_MAX:
        raise ValueError("%s: %dx%d exceeds Xfullres_max = %d; the single-image wrapper resizes such photos on the host"
                         % (what, a.shape[0], a.shape[1], XFULLRES_MAX))
    return a


def cut_batches(items, batch, max_bytes, max_hints=_lib.MAX_HINTS):
    """items: iterable of (nbytes, nhints, payload) -> lists of payloads, in order.  A batch ends before the item that
    would take it past `batch` items, `max_bytes` source bytes or `max_hints` hints; an item over the byte budget on its
    own forms a batch by itself."""
    cur, nbytes, nhints = [], 0, 0
    for b, h, payload in items:
        if cur and (len(cur) == batch or nbytes + b > max_bytes or nhints + h > max_hints):
            yield cur
            cur, nbytes, nhints = [], 0, 0
        cur.append(payload)
        nbytes += b
        nhints += h
    if cur:
        yield cur


def read_ahead(sources, load, depth, workers):
    """load(source) for each source on a pool of `workers` threads, at most `depth` ahead of the consumer; results in
    input order."""
    pending = collections.deque()
    it = iter(sources)
    with concurrent.futures.ThreadPoolExecutor(max_workers=workers) as pool:
        for s in it:
            pending.append(pool.submit(load, s))
            if len(pending) >= depth:
                break
        while pending:
            r = pending.popleft().result()
            for s in it:
                pending.append(pool.submit(load, s))
                break
            yield r


class PhotoColorizer(object):
    """Automatic colorization of many photos on one GPU (see the module docstring).

    state_dict  weights of the reference PyTorch model (SIGGRAPHGenerator; plus the glob.* keys with global_hints)
    Xd          network size (a multiple of 8); batch: photos per device pass (at most IDC_MAX_PHOTOS)
    maskcent    centre the mask (siggraph_pretrained weights), as ColorizeImageTorch(maskcent=True)
    max_batch_bytes  source bytes per batch (a larger photo forms a batch by itself); two page-locked buffers of this
                size each way hold the batches in flight
    readahead   photos decoded ahead of the device (default 2 * batch); workers: decoding threads"""

    def __init__(self, state_dict, Xd=256, batch=32, device=0, maskcent=False, global_hints=False, engine="wgmma",
                 max_batch_bytes=96 << 20, readahead=None, workers=4):
        if Xd < 8 or Xd % 8:
            raise ValueError("Xd must be a multiple of 8, got %d" % Xd)
        if not 1 <= batch <= _lib.MAX_PHOTOS:
            raise ValueError("batch must be in [1, %d], got %d" % (_lib.MAX_PHOTOS, batch))
        self.Xd, self.batch, self.device = int(Xd), int(batch), int(device)
        self.maskcent, self.global_hints, self.engine = bool(maskcent), bool(global_hints), engine
        self.max_batch_bytes = int(max_batch_bytes)
        self.readahead = int(readahead) if readahead else 2 * self.batch
        self.workers = int(workers)
        self._backend = self._make_backend(state_dict)

    def _make_backend(self, state_dict):
        return _DeviceBatches(state_dict, self.Xd, self.batch, self.device, 0.5 if self.maskcent else 0.0,
                              self.global_hints, self.engine, self.max_batch_bytes)

    def colorize(self, photos, hints=None, glob=None, psnr=False):
        """photos: a sequence of paths (read as load_image reads them) or HxWx3 uint8 RGB arrays.
        hints: None or one hint list (colorize_image.HINT_LIST_DTYPE, network coordinates; `img` is ignored) per photo.
        glob: None or one [316] global-hints vector per photo (needs global_hints=True).
        -> iterator of PhotoResult, in input order.  Argument errors and in-memory photos that are not HxWx3 uint8 or
        exceed Xfullres_max raise ValueError here, before any device work; a path is checked when it is read, before
        its batch is submitted."""
        n = len(photos)
        for i, p in enumerate(photos):
            if isinstance(p, np.ndarray):
                check_photo(p, "photo %d" % i)
            elif not isinstance(p, (str, bytes, os.PathLike)):
                raise ValueError("photo %d: need a path or an HxWx3 uint8 array, got %s" % (i, type(p).__name__))
        if hints is not None:
            if len(hints) != n:
                raise ValueError("%d hint lists for %d photos" % (len(hints), n))
            hints = [self._hint_list(h, i) for i, h in enumerate(hints)]
        if glob is not None:
            if not self.global_hints:
                raise ValueError("glob vectors need PhotoColorizer(global_hints=True)")
            if len(glob) != n:
                raise ValueError("%d glob vectors for %d photos" % (len(glob), n))
            glob = [np.asarray(g, np.float32).reshape(-1) for g in glob]
            if any(g.shape != (316,) for g in glob):
                raise ValueError("every glob vector must have 316 values")
        return self._run(photos, hints, glob, bool(psnr))

    @staticmethod
    def _hint_list(h, i):
        if h is None:
            return None
        h = engine.as_hints(h)
        if h.shape[0] > _lib.MAX_HINTS:
            raise ValueError("photo %d: %d hints, at most %d" % (i, h.shape[0], _lib.MAX_HINTS))
        return h

    def _run(self, photos, hints, glob, psnr):
        def load(i):
            p = photos[i]
            if isinstance(p, np.ndarray):
                return i, np.ascontiguousarray(p)
            return i, check_photo(read_photo(p), "photo %d (%s)" % (i, p))

        def items():
            for i, a in read_ahead(range(len(photos)), load, self.readahead, self.workers):
                nh = 0 if hints is None or hints[i] is None else hints[i].shape[0]
                yield a.nbytes, nh, (i, a)

        # Batch k-1 is collected after batch k is submitted, so the device always has the next batch queued.  Whatever
        # ends the iteration early (a break, an abandoned iterator, a photo that fails to read) still collects the batch
        # in flight, so no batch is left behind in a buffer slot.
        pending = None
        try:
            for b in cut_batches(items(), self.batch, self.max_batch_bytes):
                idx = [i for i, _ in b]
                token = self._backend.submit([a for _, a in b], None if hints is None else [hints[i] for i in idx],
                                             None if glob is None else [glob[i] for i in idx], psnr)
                prev, pending = pending, token
                if prev is not None:
                    for r in self._backend.collect(prev):
                        yield r
            last, pending = pending, None
            if last is not None:
                for r in self._backend.collect(last):
                    yield r
        finally:
            if pending is not None:
                self._backend.discard(pending)

    def close(self):
        self._backend.close()


class _HostBuffer(object):
    """Page-locked host bytes from idc_host_alloc, seen as a numpy array and a torch tensor; free() returns them to the
    system (torch's own pinned allocator would keep them cached for the life of the process)."""

    def __init__(self, lib, nbytes):
        import torch
        self.lib, self.ptr = lib, lib.idc_host_alloc(nbytes)
        if not self.ptr:
            raise _lib.IdcError(-2, "idc_host_alloc(%d) failed" % nbytes)
        self.array = np.frombuffer((ctypes.c_char * nbytes).from_address(self.ptr), dtype=np.uint8)
        self.tensor = torch.from_numpy(self.array)

    def free(self):
        if self.ptr:
            self.array = self.tensor = None
            self.lib.idc_host_free(self.ptr)
            self.ptr = None


class _DeviceBatches(object):
    """Device side of PhotoColorizer: one LhnContext (max_n = batch) and two slots of batch buffers.  submit() packs and
    enqueues a batch on slot k % 2 and returns; collect() waits for that batch's copies and returns its results.
    submit() first waits until the slot's previous batch is off the device, so a slot is never overwritten while a
    kernel or a copy still uses it, whether or not that batch was collected; collecting a batch whose slot has been
    reused since raises instead of returning another batch's pixels.
    The source / result buffers of a slot hold max_bytes; a batch of one larger photo grows them for that batch, and
    the slot's next batch that fits, or close(), returns them to max_bytes (the page-locked host memory goes back to
    the system, the device memory to torch's caching allocator)."""

    def __init__(self, state_dict, X, batch, device, maskcent, global_hints, engine_name, max_bytes):
        import torch
        self.torch, self.lib = torch, _lib.load()
        self.X, self.batch, self.device, self.maskcent = X, batch, device, maskcent
        self.ctx = engine.LhnContext(device=device, max_n=batch, H=X, W=X, engine=engine_name, global_hints=global_hints)
        self.ctx.load_state_dict(state_dict)
        dev = self.dev = torch.device("cuda:%d" % device)
        f32 = torch.float32
        # used by the compute stream only: one copy
        self.L_mc = torch.empty((batch, 1, X, X), dtype=f32, device=dev)
        self.ab_in = torch.empty((batch, 2, X, X), dtype=f32, device=dev)
        self.mask = torch.empty((batch, 1, X, X), dtype=f32, device=dev)
        self.lab = torch.empty((batch, 3, X, X), dtype=torch.float64, device=dev)
        self.max_bytes = max_bytes
        self.slots = [self._slot() for _ in range(2)]
        self.s_in, self.s_comp, self.s_out = (torch.cuda.Stream(dev) for _ in range(3))
        self._after_alloc()
        self.k = 0

    def _after_alloc(self):
        """Buffers come from torch's allocator on the current stream; order the pipeline's streams after it, so that a
        block that stream freed is not written before the stream's own last use of it has run."""
        cur = self.torch.cuda.current_stream(self.dev)
        for st in (self.s_in, self.s_comp, self.s_out):
            st.wait_stream(cur)

    def _slot(self):
        torch, X, n, dev = self.torch, self.X, self.batch, self.dev
        pin = lambda shape, dt: torch.empty(shape, dtype=dt, pin_memory=True)
        hint_bytes = _lib.HINT_HDR_BYTES + _lib.MAX_HINTS * _lib.HINT_DTYPE.itemsize
        return {"cap": 0, "batch": 0,                                # batch: serial number of the batch the slot holds
                "src": None, "h_src": None, "h_full": None,      # sized by _reserve
                "hints": torch.empty((hint_bytes,), dtype=torch.uint8, device=dev), "h_hints": pin((hint_bytes,), torch.uint8),
                "glob": torch.empty((n, 316), dtype=torch.float32, device=dev), "h_glob": pin((n, 316), torch.float32),
                "img_rgb": torch.empty((n, X, X, 3), dtype=torch.uint8, device=dev),
                "ab": torch.empty((n, 2, X, X), dtype=torch.float32, device=dev), "h_ab": pin((n, 2, X, X), torch.float32),
                "rgb": torch.empty((n, X, X, 3), dtype=torch.uint8, device=dev), "h_rgb": pin((n, X, X, 3), torch.uint8),
                "sse": torch.empty((n,), dtype=torch.int64, device=dev), "h_sse": pin((n,), torch.int64),
                "ev_in": torch.cuda.Event(), "ev_comp": torch.cuda.Event(), "ev_out": torch.cuda.Event()}

    def _free_big(self, s):
        for k in ("h_src", "h_full"):
            if s[k] is not None:
                s[k].free()
        s["src"] = s["h_src"] = s["h_full"] = None
        s["cap"] = 0

    def _reserve(self, s, nbytes):
        """Source / result buffers of slot s for nbytes: max_bytes, or exactly nbytes for a larger batch.  The slot is
        idle (submit waited for it)."""
        if s["cap"] >= nbytes and (s["cap"] == self.max_bytes or nbytes > self.max_bytes):
            return
        cap = max(nbytes, self.max_bytes)
        self._free_big(s)
        s["src"] = self.torch.empty((cap,), dtype=self.torch.uint8, device=self.dev)
        s["h_src"], s["h_full"] = _HostBuffer(self.lib, cap), _HostBuffer(self.lib, cap)
        s["cap"] = cap
        self._after_alloc()

    def submit(self, photos, hints, glob, psnr):
        torch, lib, X = self.torch, self.lib, self.X
        n = len(photos)
        s = self.slots[self.k % 2]
        self.k += 1
        s["ev_out"].synchronize()          # the slot's previous batch (if any) is off the device: render, D2H, all
        s["batch"] = self.k
        table = np.zeros(n, _lib.PHOTO_DTYPE)
        off = 0
        for i, a in enumerate(photos):
            table[i] = (off, a.shape[0], a.shape[1])
            off += a.shape[0] * a.shape[1]
        nbytes = off * 3
        self._reserve(s, nbytes)
        h_src = s["h_src"].array
        for i, a in enumerate(photos):
            o = int(table[i]["off"]) * 3
            h_src[o:o + a.nbytes] = a.reshape(-1)
        count = 0
        if hints is not None:
            lists = []
            for i, h in enumerate(hints):
                if h is not None and h.shape[0]:
                    h = h.copy()
                    h["img"] = i
                    lists.append(h)
            block = np.concatenate(lists) if lists else np.zeros(0, _lib.HINT_DTYPE)
            count = block.shape[0]
        hb = s["h_hints"].numpy()
        hb[:_lib.HINT_HDR_BYTES].view(np.int32)[:] = (count, 0, 0, 0)
        if count:
            hb[_lib.HINT_HDR_BYTES:_lib.HINT_HDR_BYTES + block.nbytes] = block.view(np.uint8)
        if glob is not None:
            s["h_glob"].numpy()[:n] = np.stack(glob)
        hint_len = _lib.HINT_HDR_BYTES + count * _lib.HINT_DTYPE.itemsize

        with torch.cuda.stream(self.s_in):
            s["src"][:nbytes].copy_(s["h_src"].tensor[:nbytes], non_blocking=True)
            s["hints"][:hint_len].copy_(s["h_hints"][:hint_len], non_blocking=True)
            if glob is not None:
                s["glob"][:n].copy_(s["h_glob"][:n], non_blocking=True)
            s["ev_in"].record(self.s_in)

        st = self.s_comp
        st.wait_event(s["ev_in"])
        sh = st.cuda_stream
        tp = table.ctypes.data
        with torch.cuda.stream(st):
            _lib.check(None, lib.idc_photo_prep(self.device, n, tp, s["src"].data_ptr(), X, self.L_mc.data_ptr(),
                                                s["img_rgb"].data_ptr() if psnr else None, sh))
            _lib.check(None, lib.idc_hint_raster(self.device, n, X, X, count, s["hints"].data_ptr(), self.ab_in.data_ptr(),
                                                 self.mask.data_ptr(), sh))
            self.ctx.forward_device(self.L_mc[:n], self.ab_in[:n], self.mask[:n], self.maskcent,
                                    glob=None if glob is None else s["glob"][:n], want_rgb=True,
                                    out_ab=s["ab"][:n], out_rgb=s["rgb"][:n])
            _lib.check(None, lib.idc_rgb2lab_f64(self.device, n, X, X, s["rgb"].data_ptr(), self.lab.data_ptr(), sh))
            _lib.check(None, lib.idc_photo_render(self.device, n, tp, s["src"].data_ptr(), X, self.lab.data_ptr(),
                                                  s["src"].data_ptr(), sh))
            if psnr:
                _lib.check(None, lib.idc_rgb_sse(self.device, n, X, X, s["img_rgb"].data_ptr(), s["rgb"].data_ptr(),
                                                 s["sse"].data_ptr(), sh))
            s["ev_comp"].record(st)

        with torch.cuda.stream(self.s_out):
            self.s_out.wait_event(s["ev_comp"])
            s["h_full"].tensor[:nbytes].copy_(s["src"][:nbytes], non_blocking=True)
            s["h_ab"][:n].copy_(s["ab"][:n], non_blocking=True)
            s["h_rgb"][:n].copy_(s["rgb"][:n], non_blocking=True)
            if psnr:
                s["h_sse"][:n].copy_(s["sse"][:n], non_blocking=True)
            s["ev_out"].record(self.s_out)
        return s, s["batch"], table, psnr

    def collect(self, token):
        s, batch, table, psnr = token
        if s["batch"] != batch:
            raise RuntimeError("this batch's buffers were reused by a later batch: iterate one colorize() result at a "
                               "time per PhotoColorizer")
        s["ev_out"].synchronize()
        full, ab, rgb, sse = s["h_full"].array, s["h_ab"].numpy(), s["h_rgb"].numpy(), s["h_sse"].numpy()
        N = self.X * self.X * 3
        out = []
        for i, (off, h, w) in enumerate(table.tolist()):
            p = None
            if psnr:    # get_result_PSNR: 20 * log10(255 / sqrt(mean(err2))); the sum of err2 is exact, so is the mean
                p = float(20 * np.log10(255. / np.sqrt(np.float64(sse[i]) / N)))
            out.append(PhotoResult(full[off * 3:(off + h * w) * 3].reshape(h, w, 3).copy(), rgb[i].copy(), ab[i].copy(), p))
        return out

    def discard(self, token):
        """Wait for a batch nobody will collect (its results are dropped)."""
        s, batch = token[:2]
        if s["batch"] == batch:
            s["ev_out"].synchronize()

    def close(self):
        self.torch.cuda.synchronize(self.dev)
        for s in self.slots:
            self._free_big(s)
        self.ctx.close()
