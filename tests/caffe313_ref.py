"""float64 numpy restatement of the x4 up-sample of the Caffe 313-bin head: the two grouped x2 "bilinear" deconvolutions
pred_313_us / pred_313_rs (oracle/caffe_spec.py: US_KERNEL, stride 2, pad 1, groups 313) in the closed form that
decode313_kernel, dist313_pixel_kernel and dist313_map_kernel implement.  Test infrastructure.

Per axis, output 4i + r is w0[r] * a[i] + w1[r] * a[i + 1] with w0 = {1, .75, .5, .25}, w1 = {0, .25, .5, .75} and
a[len] = 0: past the last cell the deconvolutions read their zero padding, so the last three outputs of each axis fade
towards zero instead of holding the last cell's value.  The plane is up-sampled in y, then in x."""
import numpy as np

W0 = np.array([1.0, 0.75, 0.5, 0.25])
W1 = np.array([0.0, 0.25, 0.5, 0.75])


def up4_axis(a, axis):
    """x4 along `axis` of a float64 array."""
    a = np.moveaxis(np.asarray(a, dtype=np.float64), axis, -1)
    nxt = np.concatenate([a[..., 1:], np.zeros(a.shape[:-1] + (1,))], axis=-1)          # a[i + 1], a[len] = 0
    out = W0 * a[..., :, None] + W1 * nxt[..., :, None]                                  # [..., len, 4]
    return np.moveaxis(out.reshape(a.shape[:-1] + (4 * a.shape[-1],)), -1, axis)


def up4(logits):
    """[..., H4, W4] -> [..., 4 H4, 4 W4] float64."""
    return up4_axis(up4_axis(logits, -2), -1)


def softmax(v, axis):
    v = np.asarray(v, dtype=np.float64)
    e = np.exp(v - v.max(axis=axis, keepdims=True))
    return e / e.sum(axis=axis, keepdims=True)


def dist_ab_S(logits, S=0.2):
    """[N, 313, H4, W4] logits -> softmax(S * up4) [N, 313, 4 H4, 4 W4] float64 (dist_ab_S)."""
    return softmax(S * up4(logits), axis=1)


def pred_ab(logits, pts, T=2.6):
    """[N, 313, H4, W4] logits, [313, 2] bin centres -> annealed mean [N, 2, 4 H4, 4 W4] float64."""
    return np.einsum("nbhw,bc->nchw", softmax(T * up4(logits), axis=1), np.asarray(pts, dtype=np.float64))


def negentropy(d):
    """sum_k d log d over axis 0 (data/colorize_image.py:358, :547); 0 * log 0 = NaN as in numpy."""
    d = np.asarray(d)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.sum(d * np.log(d), axis=0)
