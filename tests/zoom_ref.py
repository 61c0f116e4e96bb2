"""numpy restatement of scipy.ndimage.zoom(order 0 / 1, mode='constant', cval=0, grid_mode=False) as scipy 1.18
evaluates it, the rule render_planes_kernel follows (include/idc_b200.h: idc_render_planes_u8).  Test infrastructure.

Per axis, output o samples c = o * ratio with ratio = (n_in-1)/(n_out-1) rounded to float64 first (1 for n_out == 1).
When the ratio rounds up, the last output lands just past the input (c > n_in-1) and reads cval = 0.  Order 0 takes
floor(c + 0.5); order 1 blends floor(c) and the next sample with w0 = 1 - t, w1 = 1 - w0, and adds the four taps of a
2-D plane in scipy's order, each as (v * wy) * wx."""
import numpy as np


def ratio(n_in, n_out):
    return (n_in - 1) / (n_out - 1) if n_out > 1 else 1.0


def coords(n_in, n_out):
    return np.arange(n_out, dtype=np.float64) * ratio(n_in, n_out)


def overshoot(n_in, n_out):
    """Boolean [n_out]: the outputs scipy fills with cval."""
    return coords(n_in, n_out) > n_in - 1


def taps(n_in, n_out, order):
    """-> (inside, i0, i1, w0, w1), each [n_out]."""
    c = coords(n_in, n_out)
    inside = c <= n_in - 1
    if order == 0:
        i0 = np.minimum(np.floor(c + 0.5).astype(np.int64), n_in - 1)
        return inside, i0, i0, np.ones(n_out), np.zeros(n_out)
    f = np.floor(c)
    w0 = 1.0 - (c - f)
    w1 = 1.0 - w0
    i0 = np.minimum(f.astype(np.int64), n_in - 1)
    return inside, i0, np.minimum(i0 + 1, n_in - 1), w0, w1


def zoom_1d(v, n_out, order):
    inside, i0, i1, w0, w1 = taps(v.shape[0], n_out, order)
    out = v[i0].astype(np.float64) if order == 0 else v[i0] * w0 + v[i1] * w1
    out[~inside] = 0.0
    return out


def zoom_plane(v, h, w, order):
    """[h_in, w_in] -> [h, w] float64."""
    iy, y0, y1, wy0, wy1 = taps(v.shape[0], h, order)
    ix, x0, x1, wx0, wx1 = taps(v.shape[1], w, order)
    v = np.asarray(v, dtype=np.float64)
    if order == 0:
        out = v[y0][:, x0]
    else:
        out = (v[y0][:, x0] * wy0[:, None]) * wx0[None]
        out = out + (v[y0][:, x1] * wy0[:, None]) * wx1[None]
        out = out + (v[y1][:, x0] * wy1[:, None]) * wx0[None]
        out = out + (v[y1][:, x1] * wy1[:, None]) * wx1[None]
    out[~iy] = 0.0
    out[:, ~ix] = 0.0
    return out


def out_len(n_in, full, like):
    """Output length of `_to_fullres` along one axis: scipy's int(round(n_in * factor)), factor = full / like."""
    return int(round(n_in * (1. * full / like)))
