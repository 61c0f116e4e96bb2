"""Writes tests/golden/gamut_ref.npz: the gamut map of the UNMODIFIED reference `data/lab_gamut.abGrid().update_gamut(L)`
for a handful of L values, imported behind oracle/ref_shims (scikit-image's rgb2lab / lab2rgb restated in
oracle/color_ref.py).  Needs a reference checkout (IDC_REFERENCE_ROOT); the tests read only the .npz.

    python tests/golden/make_gamut_golden.py
"""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

L_VALUES = (0.0, 12.5, 33.0, 50.0, 71.25, 88.0, 100.0)


def main():
    from oracle import ref_shims
    if not ref_shims.reference_available():
        raise SystemExit("no reference checkout (set IDC_REFERENCE_ROOT)")
    ref_shims._install_shims()
    sys.path.insert(0, ref_shims.REF_ROOT)
    lab_gamut = importlib.import_module("data.lab_gamut")
    grid = lab_gamut.abGrid(gamut_size=110, D=1)
    rgb, mask = [], []
    for L in L_VALUES:
        r, m = grid.update_gamut(L)
        rgb.append(r.copy())
        mask.append(m.copy())
    out = os.path.join(ROOT, "tests", "golden", "gamut_ref.npz")
    np.savez_compressed(out, L=np.array(L_VALUES), gamut_size=110, D=1, masked_rgb=np.stack(rgb),
                        mask=np.packbits(np.stack(mask), axis=-1), mask_shape=np.array(np.stack(mask).shape))
    print("wrote %s (%d bytes)" % (out, os.path.getsize(out)))


if __name__ == "__main__":
    main()
