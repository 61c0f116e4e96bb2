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

`PhotoColorizer.reveal_sweep` measures PSNR against the number of hint points revealed from each photo's own ground
truth (`reveal_points`), all levels of a photo in the same device pass:

    H2D -> idc_photo_prep -> idc_rgb2lab_f64 (ground truth) -> idc_hint_fill_mean -> idc_hint_raster per image
    -> L and img_rgb repeated once per level -> idc_forward -> idc_rgb_sse -> D2H of the network-size results

`PhotoColorizer.global_stats` gives each photo's global-hints statistics (313-bin ab histogram and mean saturation of
the network-size photo, global_stats.prototxt), and `PhotoColorizer.global_sweep` measures PSNR under the global-hints
conditions of GLOBAL_CONDITIONS, every condition of a photo in the same device pass:

    H2D -> idc_photo_prep -> idc_global_stats_batch -> glob rows per condition (exact 0/1 masks) -> L and img_rgb
    repeated once per condition -> zero ab / mask planes (idc_hint_raster) -> idc_forward -> idc_rgb_sse -> D2H

`PhotoColorizer.suggest` (a colorizer made with suggest=True, whose context carries the 529-bin distribution head)
colours every photo with its hints as `colorize(hints=...)` does and also answers the GUI palette's question, the K
colour suggestions get_ab_reccs(h, w, K) gives, at each photo's query points, on the distribution of that photo's own
forward: the colorize pass with idc_ab_reccs_batch right after idc_forward (every query of the batch in one pass).
"""
import collections
import concurrent.futures
import ctypes
import math
import os

import numpy as np

from . import _lib, engine

PhotoResult = collections.namedtuple("PhotoResult", "fullres rgb ab psnr")
PhotoResult.__doc__ = """One colorized photo.
    fullres  uint8 [H,W,3]   get_img_fullres(): the photo's own L with the network's ab zoomed to full resolution
    rgb      uint8 [X,X,3]   output_rgb (the network-size result)
    ab       float32 [2,X,X] output_ab_raw (the raw network output)
    psnr     float or None   get_result_PSNR() against the network-size photo, when asked for"""

RevealResult = collections.namedtuple("RevealResult", "psnr ab rgb points")
RevealResult.__doc__ = """One photo of a reveal sweep, over the L levels in the order given.
    psnr    float64 [L]          get_result_PSNR() of each level's output_rgb against the network-size photo
    ab      float32 [L,2,X,X]    output_ab_raw of each level
    rgb     uint8 [L,X,X,3]      output_rgb of each level
    points  int32 [max(levels),3] the revealed points (y0, x0, P) (reveal_points); level m used the first m"""

SuggestResult = collections.namedtuple("SuggestResult", "result centers conf")
SuggestResult.__doc__ = """One photo of PhotoColorizer.suggest, with P query points.
    result   PhotoResult   what colorize(hints=...) gives for the photo
    centers  float64 [P,K,2]  get_ab_reccs(h, w, K) at each point (ab centres, heaviest cluster first)
    conf     float64 [P,K]    the clusters' mass (get_ab_reccs(..., return_conf=True))"""

GlobalSweepResult = collections.namedtuple("GlobalSweepResult", "psnr ab rgb stats")
GlobalSweepResult.__doc__ = """One photo of a global-hints sweep, over the C conditions in the order given.
    psnr    float64 [C]          get_result_PSNR() of each condition's output_rgb against the network-size photo
    ab      float32 [C,2,X,X]    output_ab_raw of each condition
    rgb     uint8 [C,X,X,3]      output_rgb of each condition
    stats   float32 [316]        the photo's own statistics [313 histogram, 1, s_avg, 1] (idc_global_stats_batch)"""

XFULLRES_MAX = 10000          # the wrapper's Xfullres_max (ColorizeImageBase): larger photos are resized on the host
REVEAL_LEVELS = (0, 1, 2, 5, 10, 20, 50, 100, 200, 500)
# The paper's global-hints evaluation: no hints, the photo's own saturation, its own histogram, both.
GLOBAL_CONDITIONS = ("none", "sat", "hist", "hist+sat")
# Which entries of a [316] statistics row each condition keeps (the others are 0): the histogram with its indicator
# (313), the saturation (314) with its indicator (315).
_GLOB_KEEP = {"none": np.zeros(316, bool),
              "sat": np.r_[np.zeros(314, bool), True, True],
              "hist": np.r_[np.ones(314, bool), False, False],
              "hist+sat": np.ones(316, bool)}


def reveal_points(X, m, seed, index):
    """The first m points a simulated user reveals on the X x X network grid of photo number `index` -> int32 [m, 3],
    one row (y0, x0, P) per point: a P x P square with top-left corner (y0, x0), painted with the photo's mean
    ground-truth colour under it.  Following the paper's description of its simulated user (centred Gaussian
    locations, square patches of 1 to 9 pixels), with rng = np.random.default_rng([seed, index]), each point draws
        P = rng.integers(1, 10);  cy, cx = rng.normal(X / 2, X / 4, 2)
        y0 = clip(floor(cy) - (P - 1) // 2, 0, X - P),  x0 likewise from cx
    in that order.  A photo's points depend only on (seed, index), not on how photos are batched, and the first m points
    are a prefix of the first m + 1.  This is this package's rule, not the authors' evaluation sampling (which was not
    published with the code), so curves from it are not comparable with the paper's figures.  X must be at least 9."""
    if X < 9:
        raise ValueError("reveal_points: X = %d, need at least 9 for a 9 x 9 patch" % X)
    if m < 0:
        raise ValueError("reveal_points: m = %d < 0" % m)
    rng = np.random.default_rng([int(seed), int(index)])
    integers, normal = rng.integers, rng.normal
    out = []
    for _ in range(m):
        P = int(integers(1, 10))
        cy, cx = normal(X / 2, X / 4, 2).tolist()
        lo = (P - 1) // 2
        out.append((min(max(math.floor(cy) - lo, 0), X - P), min(max(math.floor(cx) - lo, 0), X - P), P))
    return np.array(out, np.int32).reshape(m, 3)


def check_levels(levels, batch):
    """levels of a reveal sweep -> tuple of int.  Raise ValueError unless they are distinct integers in
    [0, IDC_MAX_HINTS] and at most `batch` of them (one device pass carries every level of a photo)."""
    try:
        levels = list(levels)
    except TypeError:
        raise ValueError("levels: need a sequence of integers, got %r" % (levels,))
    if not levels:
        raise ValueError("levels: need at least one level")
    for v in levels:
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or not 0 <= v <= _lib.MAX_HINTS:
            raise ValueError("levels: %r is not an integer in [0, %d]" % (v, _lib.MAX_HINTS))
    levels = tuple(int(v) for v in levels)
    if len(set(levels)) != len(levels):
        raise ValueError("levels: %s repeats a level" % (levels,))
    if len(levels) > batch:
        raise ValueError("%d levels do not fit one device pass of batch = %d" % (len(levels), batch))
    return levels


def glob_vector(stats, condition):
    """A [316] statistics row [313 histogram, 1, s_avg, 1] -> the float32 glob vector of one condition of
    GLOBAL_CONDITIONS; every entry is copied or set to 0, so each vector is exact:
        none      all zeros (the reference's "run without this", data/colorize_image.py:454-456)
        sat       [0] * 313, 0, s_avg, 1
        hist      hist, 1, 0, 0   (what ColorizeImageB200GlobDist.net_forward(ab, mask, glob_dist=hist) feeds the engine)
        hist+sat  the row as it is
    colorize(photos, glob=[glob_vector(ref_stats, "hist")] * n) colours every photo like the reference photo whose
    statistics ref_stats are (DemoGlobalHistogramTransfer.ipynb)."""
    stats = np.asarray(stats, np.float32).reshape(-1)
    if stats.shape != (316,):
        raise ValueError("a statistics row has 316 values, got %d" % stats.size)
    if condition not in _GLOB_KEEP:
        raise ValueError("unknown global-hints condition %r, expected one of %s" % (condition, GLOBAL_CONDITIONS))
    return np.where(_GLOB_KEEP[condition], stats, np.float32(0))


def check_conditions(conditions, batch):
    """conditions of a global-hints sweep -> tuple of names.  Raise ValueError unless they are distinct names of
    GLOBAL_CONDITIONS, at least one and at most `batch` of them (one device pass carries every condition of a photo)."""
    if isinstance(conditions, str):
        raise ValueError("conditions: need a sequence of names, got the string %r" % conditions)
    try:
        conditions = tuple(conditions)
    except TypeError:
        raise ValueError("conditions: need a sequence of names, got %r" % (conditions,))
    if not conditions:
        raise ValueError("conditions: need at least one condition")
    for c in conditions:
        if not isinstance(c, str) or c not in GLOBAL_CONDITIONS:
            raise ValueError("conditions: %r is not one of %s" % (c, GLOBAL_CONDITIONS))
    if len(set(conditions)) != len(conditions):
        raise ValueError("conditions: %s repeats a condition" % (conditions,))
    if len(conditions) > batch:
        raise ValueError("%d conditions do not fit one device pass of batch = %d" % (len(conditions), batch))
    return conditions


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
    readahead   photos decoded ahead of the device (default 2 * batch); workers: decoding threads
    calibrate   None, or what sets the storage exponents of the wgmma engine's activations from measured ranges instead
                of the weights: a list of colour photos to measure on now, a {buffer: max_abs} dict, or the path of a
                JSON file of one (engine.save_act_ranges); the ranges used are kept in `act_ranges`
    caffe       the weights are a Caffe-scaled checkpoint (conv1_1 trained on raw L-50, ab and mask x 110, regression
                head tanh x 100), loaded as ColorizeImageB200Caffe.prep_net loads them (colorize_image.
                caffe_scaled_state_dict, option tanh_scale = 100); a hint's mask of 1 is then the reference's mask x 110.
                Not with maskcent.
    suggest     the context also carries the 529-bin distribution head, for `suggest` (the head runs beside the colour
                result and leaves it as it is).  Not with caffe or global_hints: their distribution models (313 bins,
                global hints) have no batched suggestions."""

    def __init__(self, state_dict, Xd=256, batch=32, device=0, maskcent=False, global_hints=False, engine="wgmma",
                 max_batch_bytes=96 << 20, readahead=None, workers=4, calibrate=None, caffe=False, suggest=False):
        if Xd < 8 or Xd % 8:
            raise ValueError("Xd must be a multiple of 8, got %d" % Xd)
        if not 1 <= batch <= _lib.MAX_PHOTOS:
            raise ValueError("batch must be in [1, %d], got %d" % (_lib.MAX_PHOTOS, batch))
        if caffe and maskcent:
            raise ValueError("caffe=True takes no maskcent: the Caffe models do not centre the mask")
        if suggest and (caffe or global_hints):
            raise ValueError("suggest=True works with the 529-bin distribution head only, not with %s"
                             % ("caffe=True" if caffe else "global_hints=True"))
        self.Xd, self.batch, self.device = int(Xd), int(batch), int(device)
        self.maskcent, self.global_hints, self.engine = bool(maskcent), bool(global_hints), engine
        self.caffe, self.dist = bool(caffe), bool(suggest)
        self.options = {"tanh_scale": 100} if self.caffe else None
        if self.caffe:
            from .colorize_image import caffe_scaled_state_dict
            state_dict = caffe_scaled_state_dict(state_dict)
        self.max_batch_bytes = int(max_batch_bytes)
        self.readahead = int(readahead) if readahead else 2 * self.batch
        self.workers = int(workers)
        self.act_ranges = self._calibrate(calibrate, state_dict)
        self._backend = self._make_backend(state_dict)

    def _calibrate(self, calibrate, state_dict):
        X, dev, glob = self.Xd, self.device, self.global_hints
        return engine.resolve_calibration(calibrate, lambda photos: engine.measure_act_ranges(
            state_dict, engine.calibration_batch(photos, X, device=dev, global_hints=glob), X, X, device=dev,
            maskcent=0.5 if self.maskcent else 0.0, global_hints=glob, options=self.options))

    def _make_backend(self, state_dict):
        return _DeviceBatches(state_dict, self.Xd, self.batch, self.device, 0.5 if self.maskcent else 0.0,
                              self.global_hints, self.engine, self.max_batch_bytes, self.act_ranges, self.options,
                              self.dist)

    def colorize(self, photos, hints=None, glob=None, psnr=False):
        """photos: a sequence of paths (read as load_image reads them) or HxWx3 uint8 RGB arrays.
        hints: None or one hint list (colorize_image.HINT_LIST_DTYPE, network coordinates; `img` is ignored) per photo.
        glob: None or one [316] global-hints vector per photo (needs global_hints=True).
        -> iterator of PhotoResult, in input order.  Argument errors and in-memory photos that are not HxWx3 uint8 or
        exceed Xfullres_max raise ValueError here, before any device work; a path is checked when it is read, before
        its batch is submitted."""
        n = len(photos)
        self._check_photos(photos)
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

    def suggest(self, photos, hints, points, K=9, psnr=False):
        """Colour suggestions at query points, with the colour result: for every photo, colorize(hints=..., psnr=...)'s
        PhotoResult and, at each of its points (h, w) (network coordinates, 0 <= h, w < Xd), the K suggestions
        get_ab_reccs(h, w, K, return_conf=True) of the single-image distribution model gives after net_forward with
        the photo's hints (8 restarts, 100 Lloyd iterations, the PyTorch wrapper's gamut grid), read from the
        distribution of the forward that used those hints.  Needs suggest=True.
        photos, hints: as colorize (hints may be None, or None per photo).  points: one int [P,2] array of (h, w) per
        photo (P may be 0).  K in [1, 32].
        -> iterator of SuggestResult, in input order.  Argument errors raise ValueError here, before any device work
        (paths as in colorize)."""
        if not self.dist:
            raise ValueError("suggest needs PhotoColorizer(suggest=True)")
        n = len(photos)
        if isinstance(K, (bool, np.bool_)) or not isinstance(K, (int, np.integer)) or not 1 <= K <= 32:
            raise ValueError("K must be an integer in [1, 32], got %r" % (K,))
        if len(points) != n:
            raise ValueError("%d point lists for %d photos" % (len(points), n))
        points = [self._point_list(p, i) for i, p in enumerate(points)]
        if hints is not None and len(hints) != n:
            raise ValueError("%d hint lists for %d photos" % (len(hints), n))
        self._check_photos(photos)
        if hints is not None:
            hints = [self._hint_list(h, i) for i, h in enumerate(hints)]
        return self._run(photos, hints, None, bool(psnr), points, int(K))

    def _point_list(self, p, i):
        p = np.asarray(p)
        if p.size == 0:
            return np.zeros((0, 2), np.int64)
        if p.ndim != 2 or p.shape[1] != 2 or not np.issubdtype(p.dtype, np.integer):
            raise ValueError("photo %d: points must be an integer [P,2] array of (h, w), got %s %s" % (i, p.dtype, p.shape))
        if p.min() < 0 or p.max() >= self.Xd:
            raise ValueError("photo %d: a point lies outside the %d x %d network grid" % (i, self.Xd, self.Xd))
        return p.astype(np.int64)

    def reveal_sweep(self, photos, levels=REVEAL_LEVELS, seed=0):
        """PSNR against the number of revealed hint points: for every photo and every level m, the network-size result
        with the first m points of reveal_points(Xd, max(levels), seed, i) (i = the photo's position in `photos`) as
        hints, each painted with the photo's mean ground-truth ab under it (idc_hint_fill_mean, the Lab of the
        network-size photo).  A device pass carries batch // len(levels) photos, each as len(levels) consecutive forward
        images; nothing is rendered at full resolution.
        photos: as colorize.  levels: distinct integers in [0, IDC_MAX_HINTS], at most `batch` of them.
        -> iterator of RevealResult, in input order.  Bad levels or photos raise ValueError here, before any device
        work (paths as in colorize)."""
        levels = check_levels(levels, self.batch)
        if self.Xd < 9:
            raise ValueError("reveal_sweep needs Xd >= 9 for a 9 x 9 patch, got %d" % self.Xd)
        self._check_photos(photos)
        seed = int(seed)
        M = max(levels)

        def items():
            for i, a in self._read(photos):
                yield a.nbytes, 0, (i, a, reveal_points(self.Xd, M, seed, i))

        per = self.batch // len(levels)
        return self._pipeline(cut_batches(items(), per, self.max_batch_bytes),
                              lambda b: self._backend.submit_reveal([a for _, a, _ in b], [p for _, _, p in b], levels),
                              self._backend.collect_reveal)

    def global_stats(self, photos):
        """The global-hints statistics of every photo: the float32 [316] row [313-bin ab histogram, 1, s_avg, 1] of the
        network-size photo, the cv2-exact INTER_LINEAR resize to Xd x Xd that get_global_histogram does on the host
        (idc_photo_prep, then idc_global_stats_batch; no forward).  photos: as colorize.  -> iterator of float32 [316],
        in input order.  glob_vector(row, "hist") of a reference photo's row is the histogram-transfer vector."""
        self._check_photos(photos)

        def items():
            for i, a in self._read(photos):
                yield a.nbytes, 0, a

        return self._pipeline(cut_batches(items(), self.batch, self.max_batch_bytes), self._backend.submit_stats,
                              self._backend.collect_stats)

    def global_sweep(self, photos, conditions=GLOBAL_CONDITIONS):
        """PSNR under global hints taken from each photo itself: for every photo and every condition of
        GLOBAL_CONDITIONS given, the network-size result with no local hints and glob_vector(stats, condition) as the
        global-hints input, stats being the photo's own statistics (global_stats).  A device pass carries
        batch // len(conditions) photos, each as len(conditions) consecutive forward images; nothing is rendered at full
        resolution.  Needs global_hints=True.
        photos: as colorize.  conditions: distinct names of GLOBAL_CONDITIONS, at most `batch` of them.
        -> iterator of GlobalSweepResult, in input order.  Bad conditions or photos raise ValueError here, before any
        device work (paths as in colorize)."""
        if not self.global_hints:
            raise ValueError("global_sweep needs PhotoColorizer(global_hints=True)")
        conditions = check_conditions(conditions, self.batch)
        self._check_photos(photos)

        def items():
            for i, a in self._read(photos):
                yield a.nbytes, 0, a

        per = self.batch // len(conditions)
        return self._pipeline(cut_batches(items(), per, self.max_batch_bytes),
                              lambda b: self._backend.submit_glob(b, conditions), self._backend.collect_glob)

    @staticmethod
    def _check_photos(photos):
        for i, p in enumerate(photos):
            if isinstance(p, np.ndarray):
                check_photo(p, "photo %d" % i)
            elif not isinstance(p, (str, bytes, os.PathLike)):
                raise ValueError("photo %d: need a path or an HxWx3 uint8 array, got %s" % (i, type(p).__name__))

    @staticmethod
    def _hint_list(h, i):
        if h is None:
            return None
        h = engine.as_hints(h)
        if h.shape[0] > _lib.MAX_HINTS:
            raise ValueError("photo %d: %d hints, at most %d" % (i, h.shape[0], _lib.MAX_HINTS))
        return h

    def _read(self, photos):
        """(index, photo array) in input order, decoded `readahead` ahead of the consumer."""
        def load(i):
            p = photos[i]
            if isinstance(p, np.ndarray):
                return i, np.ascontiguousarray(p)
            return i, check_photo(read_photo(p), "photo %d (%s)" % (i, p))
        return read_ahead(range(len(photos)), load, self.readahead, self.workers)

    def _run(self, photos, hints, glob, psnr, points=None, K=0):
        def items():
            for i, a in self._read(photos):
                nh = 0 if hints is None or hints[i] is None else hints[i].shape[0]
                yield a.nbytes, nh, (i, a)

        def submit(b):
            idx = [i for i, _ in b]
            args = ([a for _, a in b], None if hints is None else [hints[i] for i in idx],
                    None if glob is None else [glob[i] for i in idx], psnr)
            if points is None:
                return self._backend.submit(*args)
            return self._backend.submit(*args, points=[points[i] for i in idx], K=K)

        return self._pipeline(cut_batches(items(), self.batch, self.max_batch_bytes), submit, self._backend.collect)

    def _pipeline(self, batches, submit, collect):
        # Batch k-1 is collected after batch k is submitted, so the device always has the next batch queued.  Whatever
        # ends the iteration early (a break, an abandoned iterator, a photo that fails to read) still collects the batch
        # in flight, so no batch is left behind in a buffer slot.
        pending = None
        try:
            for b in batches:
                token = submit(b)
                prev, pending = pending, token
                if prev is not None:
                    for r in collect(prev):
                        yield r
            last, pending = pending, None
            if last is not None:
                for r in collect(last):
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

    def __init__(self, state_dict, X, batch, device, maskcent, global_hints, engine_name, max_bytes, act_ranges=None,
                 options=None, dist=False):
        import torch
        self.torch, self.lib = torch, _lib.load()
        self.X, self.batch, self.device, self.maskcent = X, batch, device, maskcent
        self.ctx = engine.LhnContext(device=device, max_n=batch, H=X, W=X, engine=engine_name, global_hints=global_hints,
                                     options=options, dist=dist)
        self.ctx.load_state_dict(state_dict, act_ranges=act_ranges)
        dev = self.dev = torch.device("cuda:%d" % device)
        f32 = torch.float32
        # used by the compute stream only: one copy
        self.L_mc = torch.empty((batch, 1, X, X), dtype=f32, device=dev)
        self.ab_in = torch.empty((batch, 2, X, X), dtype=f32, device=dev)
        self.mask = torch.empty((batch, 1, X, X), dtype=f32, device=dev)
        self.lab = torch.empty((batch, 3, X, X), dtype=torch.float64, device=dev)
        from . import prepost
        self.pts313 = torch.from_numpy(prepost.pts_in_hull()).to(dev)        # the 313 ab bin centres
        self._keep = {}                                                       # conditions -> _glob_keep's masks
        self.zero = torch.zeros((), dtype=f32, device=dev)
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
                "stats": torch.empty((n, 316), dtype=torch.float32, device=dev), "h_stats": pin((n, 316), torch.float32),
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

    def _next_slot(self):
        s = self.slots[self.k % 2]
        self.k += 1
        s["ev_out"].synchronize()          # the slot's previous batch (if any) is off the device: render, D2H, all
        s["batch"] = self.k
        return s

    def _pack(self, s, photos):
        """The batch's photo table; the photos packed back to back into slot s's page-locked source buffer."""
        table = np.zeros(len(photos), _lib.PHOTO_DTYPE)
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
        return table, nbytes

    def _reccs_buffers(self, s, size):
        """Slot s's suggestion outputs, room for `size` centres (queries x K): device and page-locked host.  The slot is
        idle (submit waited for it)."""
        if s.get("rc_cap", 0) < size:
            torch, dev = self.torch, self.dev
            s["cen"] = torch.empty((size, 2), dtype=torch.float32, device=dev)
            s["conf"] = torch.empty((size,), dtype=torch.float32, device=dev)
            s["h_cen"] = torch.empty((size, 2), dtype=torch.float32, pin_memory=True)
            s["h_conf"] = torch.empty((size,), dtype=torch.float32, pin_memory=True)
            s["rc_cap"] = size
            self._after_alloc()

    def submit(self, photos, hints, glob, psnr, points=None, K=0):
        torch, lib, X = self.torch, self.lib, self.X
        n = len(photos)
        s = self._next_slot()
        table, nbytes = self._pack(s, photos)
        queries = None
        if points is not None:   # one query (photo of the batch, y4, x4) per point, photo by photo
            queries = np.concatenate([np.zeros((0, 3), np.int32)] + [
                np.column_stack([np.full(len(p), i), p // 4]).astype(np.int32) for i, p in enumerate(points)])
            if len(queries):
                self._reccs_buffers(s, len(queries) * K)
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
            if queries is not None:        # on this forward's class logits, before the next forward replaces them
                Q, M = len(queries), _lib.MAX_RECCS_QUERIES
                for q0 in range(0, Q, M):
                    q1 = min(q0 + M, Q)
                    self.ctx.ab_reccs_batch(queries[q0:q1], K, out=(s["cen"][q0 * K:q1 * K].view(q1 - q0, K, 2),
                                                                    s["conf"][q0 * K:q1 * K].view(q1 - q0, K), None))
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
            if queries is not None and len(queries):
                s["h_cen"][:len(queries) * K].copy_(s["cen"][:len(queries) * K], non_blocking=True)
                s["h_conf"][:len(queries) * K].copy_(s["conf"][:len(queries) * K], non_blocking=True)
            s["ev_out"].record(self.s_out)
        return s, s["batch"], table, psnr, None if points is None else [len(p) for p in points], K

    def collect(self, token):
        s, batch, table, psnr, counts, K = token
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
        if counts is None:
            return out
        Q = sum(counts)
        cen = s["h_cen"].numpy()[:Q * K].reshape(Q, K, 2) if Q else np.zeros((0, K, 2), np.float32)
        conf = s["h_conf"].numpy()[:Q * K].reshape(Q, K) if Q else np.zeros((0, K), np.float32)
        ends = np.cumsum(counts)
        # float64 like get_ab_reccs (centers.astype(np.float64), conf.astype(np.float64))
        return [SuggestResult(r, cen[e - c:e].astype(np.float64), conf[e - c:e].astype(np.float64))
                for r, c, e in zip(out, counts, ends)]

    def _photo_buffers(self):
        """The prepared photos of a sweep before they are repeated per level or condition (compute stream only, one
        copy), made on the first sweep."""
        if getattr(self, "L_photo", None) is None:
            torch, X, n, dev = self.torch, self.X, self.batch, self.dev
            self.L_photo = torch.empty((n, 1, X, X), dtype=torch.float32, device=dev)
            self.rgb_photo = torch.empty((n, X, X, 3), dtype=torch.uint8, device=dev)
            self._after_alloc()

    def _reveal_buffers(self):
        """Buffers of reveal sweeps, made on the first one: _photo_buffers and, per slot, room for `batch` hint blocks
        of IDC_MAX_HINTS hints each."""
        self._photo_buffers()
        if "blocks" not in self.slots[0]:
            torch, n, dev = self.torch, self.batch, self.dev
            nb = n * (_lib.HINT_HDR_BYTES + _lib.MAX_HINTS * _lib.HINT_DTYPE.itemsize)
            for s in self.slots:
                s["blocks"] = torch.empty((nb,), dtype=torch.uint8, device=dev)
                s["h_blocks"] = torch.empty((nb,), dtype=torch.uint8, pin_memory=True)
            self._after_alloc()

    def submit_reveal(self, photos, points, levels):
        """One device pass of a reveal sweep: photo i of the batch is forward images i*L .. i*L+L-1 (L = len(levels)),
        image i*L+j with the first levels[j] rows of points[i] as hints."""
        torch, lib, X = self.torch, self.lib, self.X
        m, L = len(photos), len(levels)
        N = m * L
        self._reveal_buffers()
        s = self._next_slot()
        table, nbytes = self._pack(s, photos)
        # hint blocks, one per forward image, in idc_hint_raster's layout; the colours are filled on the device
        stride = _lib.HINT_HDR_BYTES + (max(levels) * _lib.HINT_DTYPE.itemsize + 15) // 16 * 16
        hb = s["h_blocks"].numpy()[:N * stride].reshape(N, stride)
        for i, pts in enumerate(points):
            rect = np.zeros(max(levels), _lib.HINT_DTYPE)
            rect["y0"], rect["x0"] = pts[:, 0], pts[:, 1]
            rect["y1"], rect["x1"] = pts[:, 0] + pts[:, 2] - 1, pts[:, 1] + pts[:, 2] - 1
            raw = rect.view(np.uint8)
            for j, c in enumerate(levels):
                row = hb[i * L + j]
                row[:_lib.HINT_HDR_BYTES].view(np.int32)[:] = (c, 0, 0, 0)
                row[_lib.HINT_HDR_BYTES:_lib.HINT_HDR_BYTES + c * _lib.HINT_DTYPE.itemsize] = raw[:c * _lib.HINT_DTYPE.itemsize]

        with torch.cuda.stream(self.s_in):
            s["src"][:nbytes].copy_(s["h_src"].tensor[:nbytes], non_blocking=True)
            s["blocks"][:N * stride].copy_(s["h_blocks"][:N * stride], non_blocking=True)
            s["ev_in"].record(self.s_in)

        st = self.s_comp
        st.wait_event(s["ev_in"])
        sh = st.cuda_stream
        blocks = s["blocks"].data_ptr()
        with torch.cuda.stream(st):
            _lib.check(None, lib.idc_photo_prep(self.device, m, table.ctypes.data, s["src"].data_ptr(), X,
                                                self.L_photo.data_ptr(), self.rgb_photo.data_ptr(), sh))
            _lib.check(None, lib.idc_rgb2lab_f64(self.device, m, X, X, self.rgb_photo.data_ptr(), self.lab.data_ptr(), sh))
            _lib.check(None, lib.idc_hint_fill_mean(self.device, N, L, X, self.lab.data_ptr(), blocks, stride, sh))
            for b in range(N):
                _lib.check(None, lib.idc_hint_raster(self.device, 1, X, X, levels[b % L], blocks + b * stride,
                                                     self.ab_in[b].data_ptr(), self.mask[b].data_ptr(), sh))
            self.L_mc[:N].view(m, L, 1, X, X).copy_(self.L_photo[:m, None].expand(m, L, 1, X, X))
            s["img_rgb"][:N].view(m, L, X, X, 3).copy_(self.rgb_photo[:m, None].expand(m, L, X, X, 3))
            self.ctx.forward_device(self.L_mc[:N], self.ab_in[:N], self.mask[:N], self.maskcent, want_rgb=True,
                                    out_ab=s["ab"][:N], out_rgb=s["rgb"][:N])
            _lib.check(None, lib.idc_rgb_sse(self.device, N, X, X, s["img_rgb"].data_ptr(), s["rgb"].data_ptr(),
                                             s["sse"].data_ptr(), sh))
            s["ev_comp"].record(st)

        with torch.cuda.stream(self.s_out):
            self.s_out.wait_event(s["ev_comp"])
            s["h_ab"][:N].copy_(s["ab"][:N], non_blocking=True)
            s["h_rgb"][:N].copy_(s["rgb"][:N], non_blocking=True)
            s["h_sse"][:N].copy_(s["sse"][:N], non_blocking=True)
            s["ev_out"].record(self.s_out)
        return s, s["batch"], points, L

    def collect_reveal(self, token):
        s, batch, points, L = token
        if s["batch"] != batch:
            raise RuntimeError("this batch's buffers were reused by a later batch: iterate one result iterator at a "
                               "time per PhotoColorizer")
        s["ev_out"].synchronize()
        ab, rgb, sse = s["h_ab"].numpy(), s["h_rgb"].numpy(), s["h_sse"].numpy()
        N = self.X * self.X * 3
        out = []
        for i, pts in enumerate(points):
            k = slice(i * L, (i + 1) * L)
            # the formula of collect(): get_result_PSNR with an exact sum of err2
            psnr = np.array([float(20 * np.log10(255. / np.sqrt(np.float64(e) / N))) for e in sse[k]], np.float64)
            out.append(RevealResult(psnr, ab[k].copy(), rgb[k].copy(), pts))
        return out

    def _upload_photos(self, s, nbytes, extra=()):
        """H2D of the packed photos (and the (device, host) pairs of `extra`) on the copy stream; the compute stream
        waits for it."""
        with self.torch.cuda.stream(self.s_in):
            s["src"][:nbytes].copy_(s["h_src"].tensor[:nbytes], non_blocking=True)
            for d, h in extra:
                d.copy_(h, non_blocking=True)
            s["ev_in"].record(self.s_in)
        self.s_comp.wait_event(s["ev_in"])

    def submit_stats(self, photos):
        """One device pass of global_stats: prep -> idc_global_stats_batch -> D2H of the [n,316] rows."""
        torch, lib, X = self.torch, self.lib, self.X
        n = len(photos)
        s = self._next_slot()
        table, nbytes = self._pack(s, photos)
        self._upload_photos(s, nbytes)
        st = self.s_comp
        sh = st.cuda_stream
        with torch.cuda.stream(st):
            _lib.check(None, lib.idc_photo_prep(self.device, n, table.ctypes.data, s["src"].data_ptr(), X,
                                                self.L_mc.data_ptr(), s["img_rgb"].data_ptr(), sh))
            _lib.check(None, lib.idc_global_stats_batch(self.device, n, X, X, s["img_rgb"].data_ptr(),
                                                        self.pts313.data_ptr(), s["stats"].data_ptr(), sh))
            s["ev_comp"].record(st)
        with torch.cuda.stream(self.s_out):
            self.s_out.wait_event(s["ev_comp"])
            s["h_stats"][:n].copy_(s["stats"][:n], non_blocking=True)
            s["ev_out"].record(self.s_out)
        return s, s["batch"], n

    def collect_stats(self, token):
        s, batch, n = token
        if s["batch"] != batch:
            raise RuntimeError("this batch's buffers were reused by a later batch: iterate one result iterator at a "
                               "time per PhotoColorizer")
        s["ev_out"].synchronize()
        return [r.copy() for r in s["h_stats"].numpy()[:n]]

    def _glob_keep(self, conditions):
        """[C,316] bool device tensor: the entries of a statistics row each condition keeps (_GLOB_KEEP)."""
        if conditions not in self._keep:
            self._keep[conditions] = self.torch.from_numpy(np.stack([_GLOB_KEEP[c] for c in conditions])).to(self.dev)
            self._after_alloc()
        return self._keep[conditions]

    def submit_glob(self, photos, conditions):
        """One device pass of a global-hints sweep: photo i of the batch is forward images i*C .. i*C+C-1 (C =
        len(conditions)), image i*C+j with glob_vector(stats_i, conditions[j]), no local hints."""
        torch, lib, X = self.torch, self.lib, self.X
        m, C = len(photos), len(conditions)
        N = m * C
        self._photo_buffers()
        keep = self._glob_keep(conditions)
        s = self._next_slot()
        table, nbytes = self._pack(s, photos)
        s["h_hints"].numpy()[:_lib.HINT_HDR_BYTES].view(np.int32)[:] = 0        # an empty hint block: zero planes
        self._upload_photos(s, nbytes, [(s["hints"][:_lib.HINT_HDR_BYTES], s["h_hints"][:_lib.HINT_HDR_BYTES])])
        st = self.s_comp
        sh = st.cuda_stream
        with torch.cuda.stream(st):
            _lib.check(None, lib.idc_photo_prep(self.device, m, table.ctypes.data, s["src"].data_ptr(), X,
                                                self.L_photo.data_ptr(), self.rgb_photo.data_ptr(), sh))
            _lib.check(None, lib.idc_global_stats_batch(self.device, m, X, X, self.rgb_photo.data_ptr(),
                                                        self.pts313.data_ptr(), s["stats"].data_ptr(), sh))
            # glob rows: each entry of the photo's row copied or 0 (exact, as glob_vector)
            torch.where(keep[None], s["stats"][:m, None], self.zero, out=s["glob"][:N].view(m, C, 316))
            self.L_mc[:N].view(m, C, 1, X, X).copy_(self.L_photo[:m, None].expand(m, C, 1, X, X))
            s["img_rgb"][:N].view(m, C, X, X, 3).copy_(self.rgb_photo[:m, None].expand(m, C, X, X, 3))
            _lib.check(None, lib.idc_hint_raster(self.device, N, X, X, 0, s["hints"].data_ptr(), self.ab_in.data_ptr(),
                                                 self.mask.data_ptr(), sh))
            self.ctx.forward_device(self.L_mc[:N], self.ab_in[:N], self.mask[:N], self.maskcent, glob=s["glob"][:N],
                                    want_rgb=True, out_ab=s["ab"][:N], out_rgb=s["rgb"][:N])
            _lib.check(None, lib.idc_rgb_sse(self.device, N, X, X, s["img_rgb"].data_ptr(), s["rgb"].data_ptr(),
                                             s["sse"].data_ptr(), sh))
            s["ev_comp"].record(st)
        with torch.cuda.stream(self.s_out):
            self.s_out.wait_event(s["ev_comp"])
            s["h_ab"][:N].copy_(s["ab"][:N], non_blocking=True)
            s["h_rgb"][:N].copy_(s["rgb"][:N], non_blocking=True)
            s["h_sse"][:N].copy_(s["sse"][:N], non_blocking=True)
            s["h_stats"][:m].copy_(s["stats"][:m], non_blocking=True)
            s["ev_out"].record(self.s_out)
        return s, s["batch"], m, C

    def collect_glob(self, token):
        s, batch, m, C = token
        if s["batch"] != batch:
            raise RuntimeError("this batch's buffers were reused by a later batch: iterate one result iterator at a "
                               "time per PhotoColorizer")
        s["ev_out"].synchronize()
        ab, rgb, sse, stats = s["h_ab"].numpy(), s["h_rgb"].numpy(), s["h_sse"].numpy(), s["h_stats"].numpy()
        N = self.X * self.X * 3
        out = []
        for i in range(m):
            k = slice(i * C, (i + 1) * C)
            # the formula of collect(): get_result_PSNR with an exact sum of err2
            psnr = np.array([float(20 * np.log10(255. / np.sqrt(np.float64(e) / N))) for e in sse[k]], np.float64)
            out.append(GlobalSweepResult(psnr, ab[k].copy(), rgb[k].copy(), stats[i].copy()))
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
