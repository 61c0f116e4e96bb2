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

    H2D -> idc_photo_prep -> idc_global_stats_batch -> glob rows per condition (exact 0/1 masks) -> zero ab / mask
    planes (idc_hint_raster) -> L and img_rgb repeated once per condition -> idc_forward -> idc_rgb_sse -> D2H

The two sweeps are one pass from the repeat of L and img_rgb on; they differ only in how they make the forward's ab /
mask planes and glob rows.

`PhotoColorizer.suggest` (a colorizer made with suggest=True, whose context carries the 529-bin distribution head)
colours every photo with its hints as `colorize(hints=...)` does and also answers the GUI palette's question, the K
colour suggestions get_ab_reccs(h, w, K) gives, at each photo's query points, on the distribution of that photo's own
forward: the colorize pass with idc_ab_reccs_batch right after idc_forward (every query of the batch in one pass).
A Caffe colorizer made with caffe_dist=True does the same with the checkpoint's 313-bin head, as the Caffe GUI pairs
ColorizeImageCaffe with ColorizeImageCaffeDist on one checkpoint: the regression head gives the colour result and the
313-bin logits of the same forward give each query's suggestions (idc_caffe313_reccs_batch, at full-resolution pixels).
"""
import collections
import concurrent.futures
import ctypes
import math
import os
import weakref

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


def _psnr(sse, X):
    """get_result_PSNR of an X x X result, 20 * log10(255 / sqrt(mean(err2))), from its exact sum of err2 (so the mean
    is exact too).  numpy's scalar log10, one result at a time, as get_result_PSNR computes it: the array log10 need
    not round the same way."""
    return float(20 * np.log10(255. / np.sqrt(np.float64(sse) / (X * X * 3))))


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
    for v in levels:
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or not 0 <= v <= _lib.MAX_HINTS:
            raise ValueError("levels: %r is not an integer in [0, %d]" % (v, _lib.MAX_HINTS))
    return _check_one_pass(tuple(int(v) for v in levels), "level", batch)


def _check_one_pass(values, noun, batch):
    """The variants of a sweep (a tuple) -> themselves.  Raise ValueError unless there is at least one, none repeats and
    at most `batch` of them fit one device pass.  noun: "level" or "condition", for the messages."""
    if not values:
        raise ValueError("%ss: need at least one %s" % (noun, noun))
    if len(set(values)) != len(values):
        raise ValueError("%ss: %s repeats a %s" % (noun, values, noun))
    if len(values) > batch:
        raise ValueError("%d %ss do not fit one device pass of batch = %d" % (len(values), noun, batch))
    return values


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
    for c in conditions:
        if not isinstance(c, str) or c not in GLOBAL_CONDITIONS:
            raise ValueError("conditions: %r is not one of %s" % (c, GLOBAL_CONDITIONS))
    return _check_one_pass(conditions, "condition", batch)


# The Caffe distribution head's weights (include/idc_b200.h, IDC_FLAG_CAFFE313); caffe.pts_in_hull comes with the package.
CAFFE313_KEYS = tuple("caffe.%s.%s" % (layer, p) for layer in ("conv3_pred", "conv4_pred", "conv5_pred", "conv6_pred",
                                                               "conv7_pred", "conv8_pred", "pred_313")
                      for p in ("weight", "bias"))
CAFFE_DIST_S = 0.2            # dist_ab_S's softening, the S every caller of the Caffe distribution model passes (prep_net)


def reccs_queries(points, caffe313):
    """Per photo of a batch an int [P,2] array of (h, w) network pixels -> int32 [sum P, 3] queries, photo by photo:
    (i, h, w) for the Caffe 313-bin head (its distribution is per pixel), (i, h // 4, w // 4) for the 529-bin head (one
    distribution per 4 x 4 cell)."""
    return np.concatenate([np.zeros((0, 3), np.int32)] + [
        np.column_stack([np.full(len(p), i), p if caffe313 else p // 4]).astype(np.int32) for i, p in enumerate(points)])


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


def pack_photos(imgs, out=None):
    """HxWx3 uint8 photos -> (table, out): the idc_photo table of the batch (PHOTO_DTYPE [n]; photo i's first pixel
    `off` comes right after photo i-1's last) and the photos packed back to back at those offsets into the uint8
    buffer `out` (one of exactly their size when None)."""
    if out is None:
        out = np.empty(sum(a.nbytes for a in imgs), np.uint8)
    table = np.zeros(len(imgs), _lib.PHOTO_DTYPE)
    off = 0
    for i, a in enumerate(imgs):
        h, w = a.shape[:2]
        table[i] = off, h, w
        out[off * 3:(off + h * w) * 3] = a.reshape(-1)
        off += h * w
    return table, out


HINT_BLOCK_BYTES = _lib.HINT_HDR_BYTES + _lib.MAX_HINTS * _lib.HINT_DTYPE.itemsize      # the largest hint block


def pack_hints(hints, out, levels=None, stride=None):
    """idc_hint_raster blocks, each a 16-byte header {count, 0, 0, 0} and then `count` idc_hint records (HINT_DTYPE),
    written into the uint8 buffer `out` -> the length of one block.
    Without levels, one block: hints holds one hint list (or None) per image of a batch, and each record gets its
    list's position as `img`; no lists, or only empty ones, make an empty block.
    With levels, len(hints) * len(levels) blocks `stride` bytes apart: block i * len(levels) + j holds the first
    levels[j] records of hints[i] as they are.  The default stride is the header plus max(levels) records, rounded up
    to 16 bytes; -> the stride."""
    hdr, rec = _lib.HINT_HDR_BYTES, _lib.HINT_DTYPE.itemsize
    if levels is None:
        lists = [np.zeros(0, _lib.HINT_DTYPE) if h is None else h for h in hints]
        block = np.concatenate([np.zeros(0, _lib.HINT_DTYPE)] + lists)
        block["img"] = np.repeat(np.arange(len(lists)), [len(h) for h in lists])
        out[:hdr].view(np.int32)[:] = len(block), 0, 0, 0
        out[hdr:hdr + block.nbytes] = block.view(np.uint8)
        return hdr + block.nbytes
    if stride is None:
        stride = hdr + (max(levels) * rec + 15) // 16 * 16
    raw = np.stack(hints).view(np.uint8)
    blocks = out[:len(raw) * len(levels) * stride].reshape(len(raw), len(levels), stride)
    blocks[:, :, :hdr].view(np.int32)[:] = [(c, 0, 0, 0) for c in levels]
    for j, c in enumerate(levels):
        blocks[:, j, hdr:hdr + c * rec] = raw[:, :c * rec]
    return stride


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
                result and leaves it as it is).  Not with caffe (use caffe_dist) or global_hints (the global model has
                no distribution head).
    caffe_dist  with caffe: the context also carries the checkpoint's Caffe 313-bin distribution head (the caffe.* keys
                of include/idc_b200.h), for `suggest`, as ColorizeImageB200CaffeDist loads it; the colour result still
                comes from the regression head and is what caffe=True alone gives.  Not with global_hints.

    One shard of a job.  When torch.distributed is initialised with world size > 1 (one process per GPU, under
    torchrun), every rank constructs a PhotoColorizer with the same arguments; state_dict and calibrate are needed on
    rank 0 only, where the checkpoint is checked, calibrated and loaded, and the other ranks receive the packed weights
    with one broadcast (parallel.share_weights; NCCL, or gloo for ranks that share a GPU).  Before that, every rank
    learns rank 0's outcome and compares its arguments (Xd, batch, the flags and options, the device's SM count) with
    rank 0's: if rank 0 failed, or any rank's arguments differ, every rank raises.  Every pass method then takes the
    whole job's lists (photos, hints, glob, points), checks them whole, and processes this rank's contiguous slice
    local_slice(len(photos)): its iterator yields result j for photo start + j.  The launch plan depends on batch and
    the SM count, never on a pass's photos, so every result equals the single-process one bit for bit, whatever the
    world size.  The process group belongs to the caller; close() releases this rank's buffers only."""

    def __init__(self, state_dict, Xd=256, batch=32, device=0, maskcent=False, global_hints=False, engine="wgmma",
                 max_batch_bytes=96 << 20, readahead=None, workers=4, calibrate=None, caffe=False, suggest=False,
                 caffe_dist=False):
        from . import parallel
        self.world, self.rank = parallel.world_rank()
        error = fingerprint = None
        try:
            fingerprint = self._setup(Xd, batch, device, maskcent, global_hints, engine, caffe, suggest, caffe_dist)
            if self.rank == 0:
                state_dict = self._load(state_dict, calibrate)
            else:
                self.act_ranges = None
        except Exception as e:
            if self.world == 1:
                raise
            error = e
        if self.world > 1:
            # no rank may go on to the weights' broadcast (or raise) alone
            self.act_ranges = parallel.agree(error, fingerprint, None if error else self.act_ranges, device=device)
        self.max_batch_bytes = int(max_batch_bytes)
        self.readahead = int(readahead) if readahead else 2 * self.batch
        self.workers = int(workers)
        self._backend = self._make_backend(state_dict)

    def _setup(self, Xd, batch, device, maskcent, global_hints, engine, caffe, suggest, caffe_dist):
        """The checks and settings of the arguments every rank is given -> what must be equal on every rank of a job
        (with the device's SM count, which the launch plan depends on)."""
        if Xd < 8 or Xd % 8:
            raise ValueError("Xd must be a multiple of 8, got %d" % Xd)
        if not 1 <= batch <= _lib.MAX_PHOTOS:
            raise ValueError("batch must be in [1, %d], got %d" % (_lib.MAX_PHOTOS, batch))
        if caffe and maskcent:
            raise ValueError("caffe=True takes no maskcent: the Caffe models do not centre the mask")
        if suggest and caffe:
            raise ValueError("suggest=True works with the 529-bin distribution head only; a Caffe checkpoint's "
                             "suggestions come from its 313-bin head: use caffe_dist=True")
        if suggest and global_hints:
            raise ValueError("suggest=True works with the 529-bin distribution head only, not with global_hints=True")
        if caffe_dist and not caffe:
            raise ValueError("caffe_dist=True needs caffe=True: the 313-bin head belongs to the Caffe checkpoint")
        if caffe_dist and global_hints:
            raise ValueError("caffe_dist=True excludes global_hints=True: the global model has no 313-bin head")
        self.Xd, self.batch, self.device = int(Xd), int(batch), int(device)
        self.maskcent, self.global_hints, self.engine = bool(maskcent), bool(global_hints), engine
        self.caffe, self.dist, self.caffe_dist = bool(caffe), bool(suggest), bool(caffe_dist)
        self.options = {"tanh_scale": 100} if self.caffe else None
        if self.world == 1:
            return None
        import torch
        # None without CUDA, where no device pass can run: only colorizers with a fake backend get that far
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count if torch.cuda.is_available() else None
        return dict(Xd=self.Xd, batch=self.batch, maskcent=self.maskcent, global_hints=self.global_hints,
                    engine=self.engine, caffe=self.caffe, suggest=self.dist, caffe_dist=self.caffe_dist,
                    options=self.options, sms=sms)

    def _load(self, state_dict, calibrate):
        """The checks of the checkpoint and the calibration, rank 0's alone in a job of many -> the state_dict as the
        context loads it; sets act_ranges."""
        if self.caffe_dist:
            missing = [k for k in CAFFE313_KEYS if k not in state_dict]
            if missing:
                raise ValueError("caffe_dist=True needs the checkpoint's 313-bin head: it has no %r" % missing[0])
        if self.caffe:
            from .colorize_image import caffe_scaled_state_dict
            state_dict = caffe_scaled_state_dict(state_dict)
        if self.caffe_dist:                      # the bin centres, as ColorizeImageB200Caffe.prep_net adds them
            import torch
            from .prepost import pts_in_hull
            state_dict["caffe.pts_in_hull"] = torch.from_numpy(pts_in_hull())
        self.act_ranges = self._calibrate(calibrate, state_dict)
        return state_dict

    def local_slice(self, n):
        """(start, count): the photos of an n-photo job this rank processes, photos[start:start + count]
        (parallel.shard_range; (0, n) on a single process)."""
        from .parallel import shard_range
        return shard_range(n, self.world, self.rank)

    def _calibrate(self, calibrate, state_dict):
        X, dev, glob = self.Xd, self.device, self.global_hints
        return engine.resolve_calibration(calibrate, lambda photos: engine.measure_act_ranges(
            state_dict, engine.calibration_batch(photos, X, device=dev, global_hints=glob), X, X, device=dev,
            maskcent=0.5 if self.maskcent else 0.0, global_hints=glob, caffe313=self.caffe_dist, options=self.options))

    def _make_backend(self, state_dict):
        return _DeviceBatches(state_dict, self.Xd, self.batch, self.device, 0.5 if self.maskcent else 0.0,
                              self.global_hints, self.engine, self.max_batch_bytes, self.act_ranges, self.options,
                              self.dist, self.caffe_dist)

    def colorize(self, photos, hints=None, glob=None, psnr=False):
        """photos: a sequence of paths (read as load_image reads them) or HxWx3 uint8 RGB arrays.
        hints: None or one hint list (colorize_image.HINT_LIST_DTYPE, network coordinates; `img` is ignored) per photo.
        glob: None or one [316] global-hints vector per photo (needs global_hints=True).
        -> iterator of PhotoResult, in input order.  Argument errors and in-memory photos that are not HxWx3 uint8 or
        exceed Xfullres_max raise ValueError here, before any device work; a path is checked when it is read, before
        its batch is submitted."""
        n = len(photos)
        self._check_photos(photos)
        hints = self._hint_lists(hints, n)
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
        distribution of the forward that used those hints.  Needs suggest=True, or caffe_dist=True: then the answers
        are ColorizeImageB200CaffeDist's (the 313-bin dist_ab_S at pixel (h, w) with S = 0.2, the 313 bin centres).
        photos, hints: as colorize (hints may be None, or None per photo).  points: one int [P,2] array of (h, w) per
        photo (P may be 0).  K in [1, 32].
        -> iterator of SuggestResult, in input order.  Argument errors raise ValueError here, before any device work
        (paths as in colorize)."""
        if not (self.dist or self.caffe_dist):
            raise ValueError("suggest needs PhotoColorizer(suggest=True), or caffe_dist=True with caffe=True")
        n = len(photos)
        if isinstance(K, (bool, np.bool_)) or not isinstance(K, (int, np.integer)) or not 1 <= K <= 32:
            raise ValueError("K must be an integer in [1, 32], got %r" % (K,))
        if len(points) != n:
            raise ValueError("%d point lists for %d photos" % (len(points), n))
        points = [self._point_list(p, i) for i, p in enumerate(points)]
        self._check_photos(photos)
        hints = self._hint_lists(hints, n)
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
        return self._pipeline(self._batches(photos, self.batch // len(levels)),
                              lambda idx, imgs: self._backend.submit_reveal(
                                  imgs, [reveal_points(self.Xd, M, seed, i) for i in idx], levels),
                              self._backend.collect_reveal)

    def global_stats(self, photos):
        """The global-hints statistics of every photo: the float32 [316] row [313-bin ab histogram, 1, s_avg, 1] of the
        network-size photo, the cv2-exact INTER_LINEAR resize to Xd x Xd that get_global_histogram does on the host
        (idc_photo_prep, then idc_global_stats_batch; no forward).  photos: as colorize.  -> iterator of float32 [316],
        in input order.  glob_vector(row, "hist") of a reference photo's row is the histogram-transfer vector."""
        self._check_photos(photos)
        return self._pipeline(self._batches(photos, self.batch), lambda idx, imgs: self._backend.submit_stats(imgs),
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
        return self._pipeline(self._batches(photos, self.batch // len(conditions)),
                              lambda idx, imgs: self._backend.submit_glob(imgs, conditions), self._backend.collect_glob)

    @staticmethod
    def _check_photos(photos):
        for i, p in enumerate(photos):
            if isinstance(p, np.ndarray):
                check_photo(p, "photo %d" % i)
            elif not isinstance(p, (str, bytes, os.PathLike)):
                raise ValueError("photo %d: need a path or an HxWx3 uint8 array, got %s" % (i, type(p).__name__))

    @staticmethod
    def _hint_lists(hints, n):
        """None, or one hint list (or None) per photo -> the same with each list as engine.as_hints gives it."""
        if hints is None:
            return None
        if len(hints) != n:
            raise ValueError("%d hint lists for %d photos" % (len(hints), n))
        out = []
        for i, h in enumerate(hints):
            if h is not None:
                h = engine.as_hints(h)
                if h.shape[0] > _lib.MAX_HINTS:
                    raise ValueError("photo %d: %d hints, at most %d" % (i, h.shape[0], _lib.MAX_HINTS))
            out.append(h)
        return out

    def _batches(self, photos, per_pass, hints=None):
        """This rank's photos (local_slice), decoded `readahead` ahead of the consumer, cut into device passes of at
        most per_pass photos, max_batch_bytes source bytes and IDC_MAX_HINTS hints -> (indices into photos, photo
        arrays) per pass, in input order."""
        start, count = self.local_slice(len(photos))
        def load(i):
            p = photos[i]
            if isinstance(p, np.ndarray):
                return i, np.ascontiguousarray(p)
            return i, check_photo(read_photo(p), "photo %d (%s)" % (i, p))

        def items():
            for i, a in read_ahead(range(start, start + count), load, self.readahead, self.workers):
                yield a.nbytes, 0 if hints is None or hints[i] is None else hints[i].shape[0], (i, a)

        for b in cut_batches(items(), per_pass, self.max_batch_bytes):
            yield [i for i, _ in b], [a for _, a in b]

    def _run(self, photos, hints, glob, psnr, points=None, K=0):
        def submit(idx, imgs):
            args = (imgs, None if hints is None else [hints[i] for i in idx],
                    None if glob is None else [glob[i] for i in idx], psnr)
            if points is None:
                return self._backend.submit(*args)
            return self._backend.submit(*args, points=[points[i] for i in idx], K=K)

        return self._pipeline(self._batches(photos, self.batch, hints), submit, self._backend.collect)

    def _pipeline(self, batches, submit, collect):
        # Batch k-1 is collected after batch k is submitted, so the device always has the next batch queued.  Whatever
        # ends the iteration early (a break, an abandoned iterator, a photo that fails to read) still collects the batch
        # in flight, so no batch is left behind in a buffer slot.
        pending = None
        try:
            for idx, imgs in batches:
                token = submit(idx, imgs)
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
    """Page-locked host bytes from idc_host_alloc, seen as a torch tensor; free() returns them to the system (torch's
    own pinned allocator would keep them cached for the life of the process)."""

    def __init__(self, lib, nbytes):
        import torch
        self.lib, self.ptr = lib, lib.idc_host_alloc(nbytes)
        if not self.ptr:
            raise _lib.IdcError(-2, "idc_host_alloc(%d) failed" % nbytes)
        self.tensor = torch.from_numpy(np.frombuffer((ctypes.c_char * nbytes).from_address(self.ptr), dtype=np.uint8))

    def free(self):
        if self.ptr:
            self.tensor = None
            self.lib.idc_host_free(self.ptr)
            self.ptr = None


class _Twin(object):
    """A buffer of _DeviceBatches: `rows` rows of shape `row` on the device and, as HostStaging pairs them on the C
    side, page-locked host copies of the same layout (_HostBuffer).  hosts=1: h_in and h_out are one copy; hosts=2:
    the device rows are uploaded from h_in and downloaded into h_out; hosts=0: device only."""

    def __init__(self, owner, row, dtype, rows=0, hosts=1, init=None):
        self.owner = weakref.proxy(owner)           # no cycle: the buffers go when their _DeviceBatches does
        self.row, self.dtype, self.hosts = tuple(row), dtype, hosts
        self.rows, self.dev, self.h_in, self.h_out, self._bufs = 0, None, None, None, ()
        self.grow(rows, init=init)

    def grow(self, rows, cap=None, init=None):
        """Room for `rows` rows, allocated again only while no enqueued work uses the buffer.  With cap the buffer
        holds exactly cap rows whenever rows fits in cap (so a buffer grown past cap shrinks back) and exactly `rows`
        otherwise.  Without cap it only grows: to exactly `rows` on the device, while its host copies, once they have
        to grow, at least double, so that a buffer that grows batch by batch seldom frees page-locked memory
        (idc_host_free waits for the whole device).  init: a host array the new device rows are copied from.  Every
        buffer of _DeviceBatches is allocated here, and the pipeline's streams are ordered after it."""
        if cap is not None and rows <= cap:
            if self.rows == cap:
                return
            rows = cap
        elif self.rows >= rows:
            return
        o, torch = self.owner, self.owner.torch
        self.dev = None
        if init is None:
            self.dev = torch.empty((rows,) + self.row, dtype=self.dtype, device=o.dev)
        else:
            self.dev = torch.from_numpy(init).to(o.dev)
        nbytes = self.dev.numel() * self.dev.element_size()
        have = self._bufs[0].tensor.numel() if self._bufs else 0
        if cap is not None or have < nbytes:
            for b in self._bufs:
                b.free()
            size = nbytes if cap is not None or not have else max(nbytes, 2 * have)
            self._bufs = tuple(_HostBuffer(o.lib, size) for _ in range(self.hosts))
        views = [b.tensor[:nbytes].view(self.dtype).view(self.dev.shape) for b in self._bufs]
        if views:
            self.h_in, self.h_out = views[0], views[-1]
        self.rows = rows
        o._after_alloc()

    def upload(self, n):
        self.dev[:n].copy_(self.h_in[:n], non_blocking=True)

    def download(self, n):
        self.h_out[:n].copy_(self.dev[:n], non_blocking=True)

    def free(self):
        """Return the host copies to the system and the device rows to torch's caching allocator."""
        for b in self._bufs:
            b.free()
        self.rows, self.dev, self.h_in, self.h_out, self._bufs = 0, None, None, None, ()


class _Slot(object):
    """One of the two buffer sets of _DeviceBatches, with the events of the batch in it.  The buffers of a pass kind
    that not every colorizer runs start empty and grow on the first batch that needs them."""

    def __init__(self, b):
        torch, X, n = b.torch, b.X, b.batch
        u8, f32 = torch.uint8, torch.float32
        self.serial = 0                                   # serial number of the batch the slot holds
        # the packed photos, uploaded from h_in, rendered over in place and downloaded into h_out: max_bytes, or more
        # for the one batch of a larger photo
        self.src = _Twin(b, (), u8, hosts=2)
        self.hints = _Twin(b, (), u8, HINT_BLOCK_BYTES)
        self.glob = _Twin(b, (316,), f32, n)
        self.img_rgb = _Twin(b, (X, X, 3), u8, n, hosts=0)
        self.ab = _Twin(b, (2, X, X), f32, n)
        self.rgb = _Twin(b, (X, X, 3), u8, n)
        self.sse = _Twin(b, (), torch.int64, n)
        self.stats = _Twin(b, (316,), f32, n)
        self.cen = _Twin(b, (2,), f32)                    # suggest: queries x K centres and their masses
        self.conf = _Twin(b, (), f32)
        self.blocks = _Twin(b, (), u8)                    # reveal sweeps: one hint block per forward image
        self.ev_in, self.ev_comp, self.ev_out = (torch.cuda.Event() for _ in range(3))

    def free(self):
        for t in vars(self).values():
            if isinstance(t, _Twin):
                t.free()


# What a _DeviceBatches submit returns and its collect takes: the slot, the serial number of the batch in it, the
# batch's n photos with V forward images each, and what the collect needs besides.
_Batch = collections.namedtuple("_Batch", "slot serial n V info")


class _DeviceBatches(object):
    """Device side of PhotoColorizer: one LhnContext (max_n = batch; its weights loaded, or received from rank 0 in a
    job of many ranks) and two _Slots of batch buffers.  submit() packs
    and enqueues a batch on slot k % 2 and returns; collect() waits for that batch's copies and returns its results.
    submit() first waits until the slot's previous batch is off the device, so a slot is never overwritten while a
    kernel or a copy still uses it, whether or not that batch was collected; collecting a batch whose slot has been
    reused since raises instead of returning another batch's pixels.
    The source / result buffers of a slot hold max_bytes; a batch of one larger photo grows them for that batch, and
    the slot's next batch that fits returns them to max_bytes.  close() returns every page-locked buffer to the system
    and the device memory to torch's caching allocator."""

    def __init__(self, state_dict, X, batch, device, maskcent, global_hints, engine_name, max_bytes, act_ranges=None,
                 options=None, dist=False, caffe313=False):
        import torch
        from . import prepost
        self.torch, self.lib = torch, _lib.load()
        self.X, self.batch, self.device, self.maskcent, self.caffe313 = X, batch, device, maskcent, caffe313
        from .parallel import share_weights
        self.ctx = share_weights(lambda: engine.LhnContext(device=device, max_n=batch, H=X, W=X, engine=engine_name,
                                                           global_hints=global_hints, options=options, dist=dist,
                                                           caffe313=caffe313), state_dict, act_ranges, device)
        self.dev = torch.device("cuda:%d" % device)
        self.s_in, self.s_comp, self.s_out = (torch.cuda.Stream(self.dev) for _ in range(3))
        f32 = torch.float32
        # used by the compute stream only: one copy
        self.L_mc, self.ab_in, self.mask = (_Twin(self, (c, X, X), f32, batch, hosts=0).dev for c in (1, 2, 1))
        self.lab = _Twin(self, (3, X, X), torch.float64, batch, hosts=0).dev
        # a sweep's prepared photos before they are repeated per level or condition, made on the first sweep
        self.L_photo = _Twin(self, (1, X, X), f32, hosts=0)
        self.rgb_photo = _Twin(self, (X, X, 3), torch.uint8, hosts=0)
        self.pts313 = _Twin(self, (2,), f32, 313, hosts=0, init=prepost.pts_in_hull()).dev    # the 313 ab bin centres
        self.zero = _Twin(self, (), f32, 1, hosts=0, init=np.zeros(1, np.float32)).dev[0]
        self.keep = {}                          # conditions -> [C,316] bool: the entries each keeps (_GLOB_KEEP)
        self.max_bytes = max_bytes
        self.slots = [_Slot(self) for _ in range(2)]
        self.k = 0

    def _after_alloc(self):
        """Buffers come from torch's allocator on the current stream; order the pipeline's streams after it, so that a
        block that stream freed is not written before the stream's own last use of it has run."""
        cur = self.torch.cuda.current_stream(self.dev)
        for st in (self.s_in, self.s_comp, self.s_out):
            st.wait_stream(cur)

    def _next_slot(self, photos):
        """The next slot, once its previous batch (if any) is off the device: render, D2H, all; the batch's photo table,
        and the photos packed back to back into the slot's page-locked source buffer -> (slot, table, nbytes)."""
        s = self.slots[self.k % 2]
        self.k += 1
        s.ev_out.synchronize()
        s.serial = self.k
        nbytes = sum(a.nbytes for a in photos)
        s.src.grow(nbytes, cap=self.max_bytes)
        return s, pack_photos(photos, s.src.h_in.numpy())[0], nbytes

    def _upload_photos(self, s, nbytes, *bufs):
        """H2D of the packed photos and of the first rows of each (buffer, rows) on the copy stream; the compute stream
        waits for it."""
        with self.torch.cuda.stream(self.s_in):
            for t, n in ((s.src, nbytes),) + bufs:
                t.upload(n)
            s.ev_in.record(self.s_in)
        self.s_comp.wait_event(s.ev_in)

    def _download(self, s, *bufs):
        """After the work enqueued on the compute stream so far: D2H of the first rows of each (buffer, rows) on the
        copy stream, then ev_out, which the slot's next batch and the collect wait for."""
        s.ev_comp.record(self.s_comp)
        with self.torch.cuda.stream(self.s_out):
            self.s_out.wait_event(s.ev_comp)
            for t, n in bufs:
                t.download(n)
            s.ev_out.record(self.s_out)

    def _finish(self, token):
        """Wait for a submitted batch's D2H -> its slot.  Raise if the slot has taken a later batch since."""
        s = token.slot
        if s.serial != token.serial:
            raise RuntimeError("this batch's buffers were reused by a later batch: iterate one result iterator at a "
                               "time per PhotoColorizer")
        s.ev_out.synchronize()
        return s

    def _prep(self, s, n, table, L, rgb):
        """idc_photo_prep of the slot's n photos into L [n,1,X,X] and, unless rgb is None, rgb [n,X,X,3]."""
        _lib.check(None, self.lib.idc_photo_prep(self.device, n, table.ctypes.data, s.src.dev.data_ptr(), self.X,
                                                 L.data_ptr(), None if rgb is None else rgb.data_ptr(),
                                                 self.s_comp.cuda_stream))

    def _prep_stats(self, s, n, table, L, rgb):
        """_prep, then each photo's [316] statistics row from rgb into the slot's stats (idc_global_stats_batch)."""
        self._prep(s, n, table, L, rgb)
        _lib.check(None, self.lib.idc_global_stats_batch(self.device, n, self.X, self.X, rgb.data_ptr(),
                                                         self.pts313.data_ptr(), s.stats.dev.data_ptr(),
                                                         self.s_comp.cuda_stream))

    def submit(self, photos, hints, glob, psnr, points=None, K=0):
        torch, lib, X = self.torch, self.lib, self.X
        n = len(photos)
        s, table, nbytes = self._next_slot(photos)
        queries = None if points is None else reccs_queries(points, self.caffe313)    # one per point, photo by photo
        QK = 0 if queries is None else len(queries) * K
        s.cen.grow(QK)
        s.conf.grow(QK)
        hints = hints or []
        count = sum(len(h) for h in hints if h is not None)
        up = [(s.hints, pack_hints(hints, s.hints.h_in.numpy()))]
        if glob is not None:
            s.glob.h_in.numpy()[:n] = np.stack(glob)
            up.append((s.glob, n))
        self._upload_photos(s, nbytes, *up)

        st = self.s_comp
        sh = st.cuda_stream
        with torch.cuda.stream(st):
            self._prep(s, n, table, self.L_mc, s.img_rgb.dev if psnr else None)
            _lib.check(None, lib.idc_hint_raster(self.device, n, X, X, count, s.hints.dev.data_ptr(),
                                                 self.ab_in.data_ptr(), self.mask.data_ptr(), sh))
            self.ctx.forward_device(self.L_mc[:n], self.ab_in[:n], self.mask[:n], self.maskcent,
                                    glob=None if glob is None else s.glob.dev[:n], want_rgb=True,
                                    out_ab=s.ab.dev[:n], out_rgb=s.rgb.dev[:n])
            if queries is not None:        # on this forward's logits, before the next forward replaces them
                Q, M = len(queries), _lib.MAX_RECCS_QUERIES
                for q0 in range(0, Q, M):
                    q1 = min(q0 + M, Q)
                    out = (s.cen.dev[q0 * K:q1 * K].view(q1 - q0, K, 2), s.conf.dev[q0 * K:q1 * K].view(q1 - q0, K),
                           None)
                    if self.caffe313:
                        self.ctx.caffe313_reccs_batch(queries[q0:q1], K, S=CAFFE_DIST_S, out=out)
                    else:
                        self.ctx.ab_reccs_batch(queries[q0:q1], K, out=out)
            _lib.check(None, lib.idc_rgb2lab_f64(self.device, n, X, X, s.rgb.dev.data_ptr(), self.lab.data_ptr(), sh))
            _lib.check(None, lib.idc_photo_render(self.device, n, table.ctypes.data, s.src.dev.data_ptr(), X,
                                                  self.lab.data_ptr(), s.src.dev.data_ptr(), sh))
            if psnr:
                _lib.check(None, lib.idc_rgb_sse(self.device, n, X, X, s.img_rgb.dev.data_ptr(), s.rgb.dev.data_ptr(),
                                                 s.sse.dev.data_ptr(), sh))

        down = [(s.src, nbytes), (s.ab, n), (s.rgb, n)]
        if psnr:
            down.append((s.sse, n))
        if QK:
            down += [(s.cen, QK), (s.conf, QK)]
        self._download(s, *down)
        return _Batch(s, s.serial, n, 1, (table, psnr, None if points is None else [len(p) for p in points], K))

    def collect(self, token):
        s = self._finish(token)
        table, psnr, counts, K = token.info
        full, ab, rgb, sse = (t.h_out.numpy() for t in (s.src, s.ab, s.rgb, s.sse))
        out = [PhotoResult(full[off * 3:(off + h * w) * 3].reshape(h, w, 3).copy(), rgb[i].copy(), ab[i].copy(),
                           _psnr(sse[i], self.X) if psnr else None)
               for i, (off, h, w) in enumerate(table.tolist())]
        if counts is None:
            return out
        Q = sum(counts)
        cen = s.cen.h_out.numpy()[:Q * K].reshape(Q, K, 2) if Q else np.zeros((0, K, 2), np.float32)
        conf = s.conf.h_out.numpy()[:Q * K].reshape(Q, K) if Q else np.zeros((0, K), np.float32)
        ends = np.cumsum(counts)
        # float64 like get_ab_reccs (centers.astype(np.float64), conf.astype(np.float64))
        return [SuggestResult(r, cen[e - c:e].astype(np.float64), conf[e - c:e].astype(np.float64))
                for r, c, e in zip(out, counts, ends)]

    def _submit_sweep(self, photos, V, fill):
        """One device pass of a sweep: photo i of the batch is forward images i*V .. i*V+V-1 (V variants: the levels or
        the conditions), each with the photo's prepared L and img_rgb.  fill(s, m, table, nbytes) uploads the batch,
        preps its m photos into L_photo / rgb_photo and makes the forward's ab / mask planes on the compute stream; it
        returns the forward's glob rows (or None) and the (buffer, rows) it adds to the D2H of ab, rgb and SSE."""
        torch, lib, X = self.torch, self.lib, self.X
        m = len(photos)
        N = m * V
        self.L_photo.grow(self.batch)
        self.rgb_photo.grow(self.batch)
        s, table, nbytes = self._next_slot(photos)
        glob, extra = fill(s, m, table, nbytes)
        with torch.cuda.stream(self.s_comp):
            self.L_mc[:N].view(m, V, 1, X, X).copy_(self.L_photo.dev[:m, None].expand(m, V, 1, X, X))
            s.img_rgb.dev[:N].view(m, V, X, X, 3).copy_(self.rgb_photo.dev[:m, None].expand(m, V, X, X, 3))
            self.ctx.forward_device(self.L_mc[:N], self.ab_in[:N], self.mask[:N], self.maskcent, glob=glob,
                                    want_rgb=True, out_ab=s.ab.dev[:N], out_rgb=s.rgb.dev[:N])
            _lib.check(None, lib.idc_rgb_sse(self.device, N, X, X, s.img_rgb.dev.data_ptr(), s.rgb.dev.data_ptr(),
                                             s.sse.dev.data_ptr(), self.s_comp.cuda_stream))
        self._download(s, (s.ab, N), (s.rgb, N), (s.sse, N), *extra)
        return _Batch(s, s.serial, m, V, None)

    def _collect_sweep(self, token):
        """A sweep's results -> per photo (psnr float64 [V], ab float32 [V,2,X,X], rgb uint8 [V,X,X,3])."""
        s, V = self._finish(token), token.V
        ab, rgb, sse = (t.h_out.numpy() for t in (s.ab, s.rgb, s.sse))
        out = []
        for i in range(token.n):
            k = slice(i * V, (i + 1) * V)
            out.append((np.array([_psnr(e, self.X) for e in sse[k]], np.float64), ab[k].copy(), rgb[k].copy()))
        return out

    def submit_reveal(self, photos, points, levels):
        """One device pass of a reveal sweep: image i*L+j of the sweep (L = len(levels)) has the first levels[j] rows of
        points[i] as hints, coloured with the mean ground-truth ab under each (idc_hint_fill_mean)."""
        lib, X, L = self.lib, self.X, len(levels)
        # the points as hint rectangles; their colours are filled on the device
        pts = np.stack(points)
        rects = np.zeros(pts.shape[:2], _lib.HINT_DTYPE)
        rects["y0"], rects["x0"] = pts[..., 0], pts[..., 1]
        rects["y1"], rects["x1"] = pts[..., 0] + pts[..., 2] - 1, pts[..., 1] + pts[..., 2] - 1

        def fill(s, m, table, nbytes):
            N = m * L
            s.blocks.grow(self.batch * HINT_BLOCK_BYTES)
            stride = pack_hints(rects, s.blocks.h_in.numpy(), levels)
            self._upload_photos(s, nbytes, (s.blocks, N * stride))
            sh, blocks, rgb = self.s_comp.cuda_stream, s.blocks.dev.data_ptr(), self.rgb_photo.dev
            self._prep(s, m, table, self.L_photo.dev, rgb)
            _lib.check(None, lib.idc_rgb2lab_f64(self.device, m, X, X, rgb.data_ptr(), self.lab.data_ptr(), sh))
            _lib.check(None, lib.idc_hint_fill_mean(self.device, N, L, X, self.lab.data_ptr(), blocks, stride, sh))
            for b in range(N):
                _lib.check(None, lib.idc_hint_raster(self.device, 1, X, X, levels[b % L], blocks + b * stride,
                                                     self.ab_in[b].data_ptr(), self.mask[b].data_ptr(), sh))
            return None, []

        return self._submit_sweep(photos, L, fill)._replace(info=points)

    def collect_reveal(self, token):
        return [RevealResult(p, ab, rgb, pts) for (p, ab, rgb), pts in zip(self._collect_sweep(token), token.info)]

    def submit_stats(self, photos):
        """One device pass of global_stats: prep -> idc_global_stats_batch -> D2H of the [n,316] rows."""
        n = len(photos)
        s, table, nbytes = self._next_slot(photos)
        self._upload_photos(s, nbytes)
        self._prep_stats(s, n, table, self.L_mc, s.img_rgb.dev)
        self._download(s, (s.stats, n))
        return _Batch(s, s.serial, n, 1, None)

    def collect_stats(self, token):
        return [r.copy() for r in self._finish(token).stats.h_out.numpy()[:token.n]]

    def submit_glob(self, photos, conditions):
        """One device pass of a global-hints sweep: image i*C+j of the sweep (C = len(conditions)) has no local hints
        and glob_vector(stats_i, conditions[j]), stats_i being photo i's own statistics."""
        torch, X, C = self.torch, self.X, len(conditions)
        if conditions not in self.keep:
            self.keep[conditions] = _Twin(self, (316,), torch.bool, C, hosts=0,
                                          init=np.stack([_GLOB_KEEP[c] for c in conditions])).dev
        keep = self.keep[conditions]

        def fill(s, m, table, nbytes):
            N = m * C
            self._upload_photos(s, nbytes, (s.hints, pack_hints([], s.hints.h_in.numpy())))    # empty: zero planes
            with torch.cuda.stream(self.s_comp):
                self._prep_stats(s, m, table, self.L_photo.dev, self.rgb_photo.dev)
                # glob rows: each entry of the photo's row copied or 0 (exact, as glob_vector)
                torch.where(keep[None], s.stats.dev[:m, None], self.zero, out=s.glob.dev[:N].view(m, C, 316))
                _lib.check(None, self.lib.idc_hint_raster(self.device, N, X, X, 0, s.hints.dev.data_ptr(),
                                                          self.ab_in.data_ptr(), self.mask.data_ptr(),
                                                          self.s_comp.cuda_stream))
            return s.glob.dev[:N], [(s.stats, m)]

        return self._submit_sweep(photos, C, fill)

    def collect_glob(self, token):
        out, stats = self._collect_sweep(token), token.slot.stats.h_out.numpy()
        return [GlobalSweepResult(p, ab, rgb, stats[i].copy()) for i, (p, ab, rgb) in enumerate(out)]

    def discard(self, token):
        """Wait for a batch nobody will collect (its results are dropped), unless its slot was reused since."""
        if token.slot.serial == token.serial:
            self._finish(token)

    def close(self):
        self.torch.cuda.synchronize(self.dev)
        for s in self.slots:
            s.free()
        self.ctx.close()
