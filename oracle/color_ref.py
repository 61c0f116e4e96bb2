"""numpy float64 restatement of scikit-image 0.13 ``color.rgb2lab`` / ``color.lab2rgb``
(sRGB, D65, 2-degree observer) -- the third-party arithmetic behind
/root/reference/data/colorize_image.py:20-36 (lab2rgb_transpose / rgb2lab_transpose).
scikit-image is pinned by the reference README (scikit-image=0.13.0) but is neither
vendored nor installed here, so this follows its published algorithm
(skimage/color/colorconv.py: rgb2xyz, xyz2lab, lab2xyz, xyz2rgb).

PARITY UNPINNED by any reference test; see oracle/__init__.py.
Test infrastructure only.
"""
import numpy as np

XYZ_FROM_RGB = np.array([[0.412453, 0.357580, 0.180423],
                         [0.212671, 0.715160, 0.072169],
                         [0.019334, 0.119193, 0.950227]])
RGB_FROM_XYZ = np.linalg.inv(XYZ_FROM_RGB)
WHITE_D65_2 = np.array([0.95047, 1.0, 1.08883])


def _as_float(img):
    img = np.asarray(img)
    if img.dtype == np.uint8:
        return img.astype(np.float64) / 255.0      # skimage img_as_float
    return img.astype(np.float64)


def rgb2xyz_white(rgb):
    """rgb2lab's intermediate: XYZ / the D65 white point, the values lab_f's 0.008856 branch tests."""
    arr = _as_float(rgb).copy()
    m = arr > 0.04045
    arr[m] = np.power((arr[m] + 0.055) / 1.055, 2.4)
    arr[~m] /= 12.92
    xyz = arr @ XYZ_FROM_RGB.T
    return xyz / WHITE_D65_2


def rgb2lab(rgb):
    xyz = rgb2xyz_white(rgb)
    m = xyz > 0.008856
    xyz[m] = np.cbrt(xyz[m])
    xyz[~m] = 7.787 * xyz[~m] + 16.0 / 116.0
    x, y, z = xyz[..., 0], xyz[..., 1], xyz[..., 2]
    L = 116.0 * y - 16.0
    a = 500.0 * (x - y)
    b = 200.0 * (y - z)
    return np.concatenate([v[..., np.newaxis] for v in (L, a, b)], axis=-1)


def lab2linear(lab):
    """lab2rgb's intermediate: linear RGB, the values the 0.0031308 gamma branch tests."""
    lab = np.asarray(lab, dtype=np.float64)
    L, a, b = lab[..., 0], lab[..., 1], lab[..., 2]
    y = (L + 16.0) / 116.0
    x = (a / 500.0) + y
    z = y - (b / 200.0)
    z = np.where(z < 0, 0.0, z)                      # skimage: invalid z clamped to 0
    out = np.stack([x, y, z], axis=-1)
    m = out > 0.2068966
    out[m] = np.power(out[m], 3.0)
    out[~m] = (out[~m] - 16.0 / 116.0) / 7.787
    out *= WHITE_D65_2
    return out @ RGB_FROM_XYZ.T


def lab2rgb(lab):
    arr = lab2linear(lab)
    m = arr > 0.0031308
    arr[m] = 1.055 * np.power(arr[m], 1.0 / 2.4) - 0.055
    arr[~m] *= 12.92
    return arr                                        # 0.13 does not clip; the caller does (:27)


def lab2rgb_transpose(img_l, img_ab):
    """data/colorize_image.py:20-28: 1xXxX, 2xXxX -> XxXx3 uint8 (truncating cast)."""
    pred_lab = np.concatenate((img_l, img_ab), axis=0).transpose((1, 2, 0))
    return (np.clip(lab2rgb(pred_lab), 0, 1) * 255).astype("uint8")


def rgb2lab_transpose(img_rgb):
    """data/colorize_image.py:31-36: XxXx3 -> 3xXxX."""
    return rgb2lab(img_rgb).transpose((2, 0, 1))
