"""numpy restatement of the GUI's gamut map, `abGrid(gamut_size, D).update_gamut(L)` (data/lab_gamut.py:55-78), on the
package's colour module (interactive_deep_colorization_b200/color.py).  Besides the reference's two outputs it returns
the float64 quantities the two decisions hang on, so a test can tell a genuine difference from one that sits on a
truncation edge or on the threshold.

Test infrastructure only.
"""
import numpy as np

from interactive_deep_colorization_b200 import color


def grid(gamut_size=110, D=1):
    """(vals_a, vals_b) of abGrid: row <-> a, column <-> b (np.meshgrid, lab_gamut.py:58-59)."""
    vals_b, vals_a = np.meshgrid(np.arange(-gamut_size, gamut_size + D, D), np.arange(-gamut_size, gamut_size + D, D))
    return vals_a, vals_b


def update_gamut(L, gamut_size=110, D=1, details=False):
    """-> (masked_rgb uint8 [A,B,3], mask bool [A,B]) [+ (rgb255 float64 [A,B,3] before truncation, norm [A,B])]."""
    vals_a, vals_b = grid(gamut_size, D)
    pts = np.concatenate((L + np.zeros(vals_a.shape + (1,)), vals_a[..., None], vals_b[..., None]), axis=2)
    rgb255 = 255 * np.clip(color.lab2rgb(pts), 0, 1)
    rgb = rgb255.astype(np.uint8)
    norm = np.linalg.norm(pts - color.rgb2lab(rgb), axis=2)
    mask = norm < 1.0
    masked = rgb.copy()
    masked[~mask] = 255
    return (masked, mask, rgb255, norm) if details else (masked, mask)


def edge_cells(rgb255, norm, margin=1e-9):
    """Cells whose float64 decision is within `margin` of a truncation edge (any unclipped channel) or of the threshold.
    Clipped channels (exactly 0 or 255) are exact on every path and are no edge."""
    frac = rgb255 - np.floor(rgb255)
    near_int = np.any(((frac < margin) | (frac > 1 - margin)) & (rgb255 > 0) & (rgb255 < 255), axis=2)
    return near_int | (np.abs(norm - 1.0) < margin)
