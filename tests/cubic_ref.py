"""numpy restatement of cv2.resize(img, (W, H), interpolation=cv2.INTER_CUBIC) on float64 planes as OpenCV 4 evaluates
it, the rule cubic_lab2rgb_kernel follows (include/idc_b200.h: idc_cubic_lab2rgb_u8).  Test infrastructure.

Per axis, output d samples f = float32((d + 0.5) * scale - 0.5) with scale = 1 / (n_out / n_in) in float64; s = floor(f)
and x = f - s in float32.  The four float32 weights of taps s-1 ... s+2 (indices clamped to the image) are OpenCV's
interpolateCubic with A = -0.75, the last one 1 - w0 - w1 - w2.  The horizontal pass sums the four products left to
right in float64, then the vertical pass does the same over four horizontal results; every product and sum is rounded
on its own (no fused multiply-add)."""
import numpy as np

_F = np.float32
A = _F(-0.75)


def weights(x):
    """float32 x in [0, 1) -> float32 [4, n] weights, in OpenCV's order of operations."""
    x = np.asarray(x, dtype=_F)
    x1, one = x + _F(1), _F(1)
    w0 = ((A * x1 - _F(5) * A) * x1 + _F(8) * A) * x1 - _F(4) * A
    w1 = ((A + _F(2)) * x - (A + _F(3))) * x * x + one
    w2 = ((A + _F(2)) * (one - x) - (A + _F(3))) * (one - x) * (one - x) + one
    w3 = one - w0 - w1 - w2
    return np.stack([w0, w1, w2, w3])


def taps(n_in, n_out):
    """-> (idx int64 [4, n_out] clamped to 0 ... n_in-1, w float32 [4, n_out])."""
    scale = 1.0 / (n_out / n_in)
    f = ((np.arange(n_out, dtype=np.float64) + 0.5) * scale - 0.5).astype(_F)
    s = np.floor(f)
    x = f - s
    idx = s.astype(np.int64)[None] + np.arange(-1, 3)[:, None]
    return np.clip(idx, 0, n_in - 1), weights(x)


def resize(img, W, H):
    """[h_in, w_in] or [h_in, w_in, C] float64 -> [H, W] / [H, W, C] float64, == cv2.resize(img, (W, H), INTER_CUBIC)."""
    v = np.asarray(img, dtype=np.float64)
    if (v.shape[0], v.shape[1]) == (H, W):
        return v.copy()                                    # cv2.resize copies when the size does not change
    v = v.reshape(v.shape[:2] + (-1,))
    iy, wy = taps(v.shape[0], H)
    ix, wx = taps(v.shape[1], W)
    wx, wy = wx.astype(np.float64)[:, :, None], wy.astype(np.float64)[:, :, None, None]
    h = v[:, ix[0]] * wx[0]
    for k in range(1, 4):
        h = h + v[:, ix[k]] * wx[k]
    out = h[iy[0]] * wy[0]
    for j in range(1, 4):
        out = out + h[iy[j]] * wy[j]
    return out.reshape((H, W) + np.asarray(img).shape[2:])
