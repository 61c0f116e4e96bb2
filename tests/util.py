"""Shared helpers for the parity tests (test infrastructure; may import oracle/)."""
import os

import numpy as np
import torch

from oracle import lhn_ref, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

# op name -> (input activations, output activation) in engine / oracle naming
OP_IO = {
    "c1_2": (["a1_1"], "conv1_2"), "c2_1": (["conv1_2"], "a2_1"), "c2_2": (["a2_1"], "conv2_2"),
    "c3_1": (["conv2_2"], "a3_1"), "c3_2": (["a3_1"], "a3_2"), "c3_3": (["a3_2"], "conv3_3"),
    "c4_1": (["conv3_3"], "a4_1"), "c4_2": (["a4_1"], "a4_2"), "c4_3": (["a4_2"], "conv4_3"),
    "c5_1": (["conv4_3"], "a5_1"), "c5_2": (["a5_1"], "a5_2"), "c5_3": (["a5_2"], "conv5_3"),
    "c6_1": (["conv5_3"], "a6_1"), "c6_2": (["a6_1"], "a6_2"), "c6_3": (["a6_2"], "conv6_3"),
    "c7_1": (["conv6_3"], "a7_1"), "c7_2": (["a7_1"], "a7_2"), "c7_3": (["a7_2"], "conv7_3"),
    "up8": (["conv7_3", "conv3_3"], "a8_1"), "c8_2": (["a8_1"], "a8_2"), "c8_3": (["a8_2"], "conv8_3"),
    "up9": (["conv8_3", "conv2_2"], "a9_1"), "c9_2": (["a9_1"], "conv9_3"),
    "up10": (["conv9_3", "conv1_2"], "a10_1"), "c10_2": (["a10_1"], "conv10_2"),
}


def golden(name):
    return np.load(os.path.join(GOLDEN, name))


def at_pix(g, a):
    """[..., 256, 256] -> [..., K]: the pixels a golden file stores its 256x256 outputs at (g["pix_idx"])."""
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)
    return a.reshape(a.shape[:-2] + (-1,))[..., g["pix_idx"]]


def at_pix_hwc(g, a):
    """[256, 256, C] (an RGB image) -> [K, C] at the same pixels."""
    a = np.asarray(a)
    return a.reshape(-1, a.shape[-1])[g["pix_idx"]]


def oracle_forward(sd, L, ab, mask, maskcent=0.0, dist=False, glob_add=None, intermediates=False):
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    with torch.no_grad():
        return lhn_ref.lhn_forward(sd, L, ab, mask, maskcent, dist=dist, glob_add=glob_add, ref_quirks=False,
                                   return_intermediates=intermediates)


def make_ctx(sd, H, W, max_n=1, **kw):
    """kw may carry options={...} (plan-time switches, idc_set_option): applied before the weights are packed."""
    from interactive_deep_colorization_b200.engine import LhnContext
    ctx = LhnContext(device=0, max_n=max_n, H=H, W=W, **kw)
    ctx.load_state_dict(sd)
    return ctx


def caffe_scaled(sd):
    """A synthetic 'Caffe-scaled' weight set: conv1_1 expects raw L-50 / ab / mask*110 (SURVEY q4)."""
    out = dict(sd)
    s = torch.tensor([100.0, 110.0, 110.0, 110.0]).reshape(1, 4, 1, 1)
    out["model1.0.weight"] = (sd["model1.0.weight"].double() / s.double()).float()
    return out


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).float().cuda().contiguous()


def maxabs(a, b):
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)
    b = b.detach().cpu().numpy() if hasattr(b, "detach") else np.asarray(b)
    return float(np.max(np.abs(a.astype(np.float64) - b.astype(np.float64))))


def small_batch(n=2, X=64, seed=100):
    return synth.synthetic_batch(n, X, seed=seed, max_hints=4)


def render_edges(rgb255, margin=1e-9, unclipped=None):
    """Values of a float64 render before its truncating cast (255 * clip(lab2rgb(lab), 0, 1)) that lie within `margin`
    of an integer strictly inside (0, 255).  Only there can a last-ulp difference between CUDA's pow / cbrt and glibc's
    flip the cast; values clipped from well outside [0, 1] are exact on every path.  unclipped (optional): the same
    render before the clip, 255 * lab2rgb(lab); values it puts within `margin` of 255 are edges too (one path may
    clip 255.0000000001 to 255 where the other truncates 254.9999999999 to 254)."""
    frac = rgb255 - np.floor(rgb255)
    edge = ((frac < margin) | (frac > 1 - margin)) & (rgb255 > 0) & (rgb255 < 255)
    if unclipped is not None:
        edge |= np.abs(unclipped - 255) < margin
    return edge


def assert_render_exact(got, want, rgb255, what, unclipped=None):
    """The uint8 render `got` equals `want` in every value outside render_edges(rgb255, unclipped=unclipped).  Prints
    and returns how many values were excluded and how many of those differ."""
    assert got.shape == want.shape == rgb255.shape and got.dtype == want.dtype == np.uint8, (what, got.shape, want.shape)
    edge = render_edges(rgb255, unclipped=unclipped)
    diff = got != want
    bad = np.argwhere(diff & ~edge)
    assert len(bad) == 0, (what, len(bad), [(tuple(i), int(got[tuple(i)]), int(want[tuple(i)])) for i in bad[:5]])
    n_edge, n_flip = int(edge.sum()), int((diff & edge).sum())
    print("%s: %d of %d values excluded (within 1e-9 of a truncation edge), %d of them differ"
          % (what, n_edge, edge.size, n_flip))
    return n_edge, n_flip
