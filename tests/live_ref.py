"""Drive the UNMODIFIED reference wrapper and network live, in FP32 or FP64 (test infrastructure; imports only oracle/
and tests/).

The golden vectors pin the port to one reference run on one photo.  The restatements the device paths are checked
against (oracle/lhn_ref.py, oracle/color_ref.py, tests/zoom_ref.py, oracle/hints_ref.py) could misread the reference
and agree with the port anyway.  These helpers run the reference's own `data/colorize_image.py` and
`models/pytorch/model.py` (oracle.ref_shims imports them as they are, from a checkout or from the copy
`__graft_entry__.build()` stages into oracle/_ref/) on the CPU, in the test process, so that the port is compared with
what the reference itself computes.

FP64 needs no change to the reference: its `forward` builds its inputs with `torch.Tensor(...)`, which follows
`torch.set_default_dtype`, so `net.double()` plus a float64 default dtype evaluates the whole session (network and
float64 post-processing) in double precision.  The default dtype is process-wide; every reference call restores it.
"""
import contextlib
import io
import os
import tempfile

import numpy as np
import torch

from oracle import ref_shims

THREADS = 8                  # fixed, so a run's CPU cost does not depend on the host's core count


def _require():
    if not ref_shims.reference_available():
        raise RuntimeError("the reference wrapper is not importable from %s: run `__graft_entry__.build()` (it stages "
                           "the reference's network and wrapper into oracle/_ref/) or set IDC_REFERENCE_ROOT"
                           % ref_shims.REF_ROOT)


def reference_wrapper():
    """-> the reference's data.colorize_image module.  Raises (never skips) when it cannot be imported."""
    _require()
    return ref_shims.import_reference_wrapper()


def reference_model():
    """-> the reference's models.pytorch.model module."""
    _require()
    return ref_shims.import_reference_model()


@contextlib.contextmanager
def precision(dtype):
    """Run reference code with `dtype` as torch's default dtype, a fixed thread count and its prints silenced; both
    settings are restored however the block ends."""
    old_dtype, old_threads = torch.get_default_dtype(), torch.get_num_threads()
    try:
        torch.set_default_dtype(dtype)
        torch.set_num_threads(THREADS)
        with contextlib.redirect_stdout(io.StringIO()), torch.no_grad():
            yield
    finally:
        torch.set_default_dtype(old_dtype)
        torch.set_num_threads(old_threads)


@contextlib.contextmanager
def one_thread():
    """sklearn's KMeans sums its clusters over OpenMP threads in no fixed order (centres move by ~1e-14 from run to
    run); with one thread two fits of the same samples from the same random state are bit-identical.  Enter it inside
    `precision`, whose torch.set_num_threads would otherwise raise the OpenMP thread count again."""
    from threadpoolctl import threadpool_limits
    with threadpool_limits(limits=1):
        yield


def reference_net(sd, dist, dtype):
    """The reference's SIGGRAPHGenerator with state_dict `sd`, in eval mode, in `dtype`."""
    M = reference_model()
    with precision(dtype):
        net = M.SIGGRAPHGenerator(dist=dist)
        net.load_state_dict({k: v for k, v in sd.items()})
        net.eval()
        if dtype == torch.float64:
            net.double()
    return net


def net_forward(net, dtype, L_mc, ab, mask, maskcent):
    """The reference network's own forward on one image ([1,H,W], [2,H,W], [1,H,W] arrays) -> numpy float64 output(s)
    as it returns them (dist=True: (regression x 110 x 110, upsampled distribution))."""
    with precision(dtype):
        out = net.forward(L_mc, ab, mask, maskcent)
    if isinstance(out, tuple):
        return tuple(o[0].cpu().numpy().astype(np.float64) for o in out)
    return out[0].cpu().numpy().astype(np.float64)


class RefSession(object):
    """One reference wrapper (ColorizeImageTorch, or ColorizeImageTorchDist with dist=True) prepared by its own
    `prep_net(path=...)` from a temporary .pth of `sd`.  `call(name, ...)` runs a wrapper method in the session's
    precision; `raw_ab()` is the regression map of the last net_forward (the wrapper does not keep it)."""

    def __init__(self, sd, Xd, maskcent, dist=False, dtype=torch.float32):
        CI = reference_wrapper()
        self.CI, self.dtype, self.dist = CI, dtype, dist
        with precision(dtype):
            self.cm = (CI.ColorizeImageTorchDist if dist else CI.ColorizeImageTorch)(Xd=Xd, maskcent=maskcent)
            with tempfile.TemporaryDirectory() as d:
                path = os.path.join(d, "weights.pth")
                torch.save({k: v for k, v in sd.items()}, path)
                self.cm.prep_net(path=path, dist=dist)
            if dtype == torch.float64:
                self.cm.net.double()

    def call(self, name, *args, **kwargs):
        with precision(self.dtype):
            return getattr(self.cm, name)(*args, **kwargs)

    def raw_ab(self):
        """float64 [2,Xd,Xd]: the reference network's own forward on the planes the last net_forward prepared.  The
        distribution model's regression output carries the x110 of models/pytorch/model.py twice; it is divided
        out once here."""
        cm = self.cm
        out = net_forward(cm.net, self.dtype, cm.img_l_mc, cm.input_ab_mc, cm.input_mask_mult, cm.mask_cent)
        return out[0] / 110.0 if self.dist else out

    def render(self, name, *args, **kwargs):
        """Call getter `name` and capture what the reference's lab2rgb_transpose computed before its truncating cast:
        -> (uint8 result, [(255 * clip(lab2rgb), 255 * lab2rgb)] per lab2rgb_transpose call, in call order)."""
        return capture_renders(self.CI, lambda: self.call(name, *args, **kwargs))


def capture_renders(CI, fn):
    """Run fn() with the reference module's lab2rgb_transpose wrapped so that each call also records its float64
    render before the cast: -> (fn(), [(clipped x 255, unclipped x 255)])."""
    orig, seen = CI.lab2rgb_transpose, []

    def lab2rgb_transpose(img_l, img_ab):
        lab = np.concatenate((img_l, img_ab), axis=0).transpose((1, 2, 0))
        rgb = CI.color.lab2rgb(lab)
        seen.append((np.clip(rgb, 0, 1) * 255, rgb * 255))
        return orig(img_l, img_ab)

    CI.lab2rgb_transpose = lab2rgb_transpose
    try:
        return fn(), seen
    finally:
        CI.lab2rgb_transpose = orig
