"""numpy raster of a hint list -- the semantics of idc_set_hints (include/idc_b200.h).

A hint is a rectangle painted with one ab colour, as the GUI's PointEdit.updateInput (ui/ui_control.py:52-63, a filled
cv2.rectangle) and the notebook's put_point (DemoInteractiveColorization.ipynb) paint it.  Pixel (y, x) of image i takes
the last hint in list order with img == i that covers it; rectangles are inclusive, clipped to the image, and empty when
y1 < y0 or x1 < x0.

Test infrastructure only.
"""
import numpy as np


def raster(hints, n, H, W, dtype=np.float32):
    """hints: structured array / sequence with fields (img, y0, x0, y1, x1, a, b) -> (ab [n,2,H,W], mask [n,1,H,W])."""
    ab = np.zeros((n, 2, H, W), dtype)
    mask = np.zeros((n, 1, H, W), dtype)
    for h in hints:
        img, y0, x0, y1, x1, a, b = (h[k] for k in ("img", "y0", "x0", "y1", "x1", "a", "b")) \
            if getattr(h, "dtype", None) is not None and h.dtype.names else h
        y0, x0, y1, x1 = max(int(y0), 0), max(int(x0), 0), min(int(y1), H - 1), min(int(x1), W - 1)
        if y1 < y0 or x1 < x0:
            continue
        ab[int(img), 0, y0:y1 + 1, x0:x1 + 1] = a
        ab[int(img), 1, y0:y1 + 1, x0:x1 + 1] = b
        mask[int(img), 0, y0:y1 + 1, x0:x1 + 1] = 1
    return ab, mask
