"""CPU: the C-ABI library loads, exports every symbol include/idc_b200.h declares, and fails
loudly (no fallback) without a GPU.  No compute calls here."""
import ctypes
import os
import re

import numpy as np
import pytest

from interactive_deep_colorization_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "idc_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(idc_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    names = _header_functions()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), "libidc_b200.so does not export %s" % n
    assert sorted(s[0] for s in _lib.SYMBOLS) == names, "ctypes table and header disagree"
    assert b"sm_90a" in lib.idc_version()


def test_error_codes_match_header():
    """Every IDC_ERR_* of the header, IDC_ERR_RANGE included, has the same value in _lib."""
    src = open(os.path.join(ROOT, "include", "idc_b200.h")).read()
    codes = {m.group(1): int(m.group(2)) for m in re.finditer(r"\bIDC_ERR_([A-Z]+)\s*=\s*(-?\d+)", src)}
    assert codes["RANGE"] == -7
    assert codes == {k[4:]: v for k, v in vars(_lib).items() if k.startswith("ERR_")}


def test_argument_validation_without_gpu():
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.idc_create(0, 1, 250, 256, 0, ctypes.byref(h)) == -1      # H not a multiple of 8
    assert lib.idc_create(0, 0, 256, 256, 0, ctypes.byref(h)) == -1      # max_n < 1
    assert lib.idc_destroy(None) == -1
    assert lib.idc_last_error(None) == b"null ctx"


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from interactive_deep_colorization_b200.engine import LhnContext
    with pytest.raises(_lib.IdcError):
        LhnContext(device=0, max_n=1, H=64, W=64)
    from interactive_deep_colorization_b200.colorize_image import ColorizeImageB200
    from oracle import synth
    cm = ColorizeImageB200(Xd=64)
    cm.prep_net(state_dict=synth.torch_state_dict())
    with pytest.raises(_lib.IdcError):                  # image prep runs on the GPU once a net is set (row f1)
        cm.set_image(np.zeros((64, 64, 3), np.uint8))
    cm = ColorizeImageB200(Xd=64, gpu_prepost=False)    # explicit host pre/post: the network itself still has no fallback
    cm.prep_net(state_dict=synth.torch_state_dict())
    cm.set_image(np.zeros((64, 64, 3), np.uint8))
    with pytest.raises(_lib.IdcError):
        cm.net_forward(np.zeros((2, 64, 64)), np.zeros((1, 64, 64)))


def test_sass_is_hopper_native():
    """The shipped cubin must contain warpgroup MMA (wgmma) and TMA instructions."""
    import shutil
    import subprocess
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not on PATH")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for mnem in ("HGMMA", "UTMALDG"):
        assert mnem in sass, mnem
    assert "sm_90a" in subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
