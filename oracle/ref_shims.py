"""Import the UNMODIFIED reference (a checkout named by IDC_REFERENCE_ROOT, or the staged copy).

The reference wrapper needs matplotlib and scikit-image, both absent here
(data/colorize_image.py:3-4).  We inject a stub ``matplotlib`` and a ``skimage.color``
backed by oracle/color_ref.py into sys.modules, then import the reference modules as
they are.  Where no checkout exists, callers must check
``reference_available()`` and skip.

Test infrastructure only -- see oracle/__init__.py.
"""
import os
import sys
import types

_HERE = os.path.dirname(os.path.abspath(__file__))
STAGED_ROOT = os.path.join(_HERE, "_ref")        # git-ignored; filled by stage_reference() from __graft_entry__.build()
# files of the reference that the timed CPU arm needs (the network, the wrapper, their package markers)
STAGED_FILES = ["models/__init__.py", "models/pytorch/__init__.py", "models/pytorch/model.py",
                "data/__init__.py", "data/colorize_image.py"]


def _pick_root():
    for r in (os.environ.get("IDC_REFERENCE_ROOT"), "/root/reference", STAGED_ROOT):
        if r and os.path.isfile(os.path.join(r, "models", "pytorch", "model.py")):
            return r
    return "/root/reference"


REF_ROOT = _pick_root()


def reference_available():
    return os.path.isfile(os.path.join(REF_ROOT, "models", "pytorch", "model.py"))


def full_reference_available():
    """The whole tree (test images, colour-bin fixtures) -- not the staged subset."""
    return os.path.isfile(os.path.join(REF_ROOT, "test_imgs", "mortar_pestle.jpg"))


def stage_reference(src="/root/reference"):
    """Build step (called by __graft_entry__.build()): copy the reference's own network + wrapper files,
    byte for byte, into the git-ignored oracle/_ref/ so that a machine without the checkout can
    time the UNMODIFIED reference CPU path in `bench.py --impl reference`.  Nothing staged is product or test source:
    oracle/_ref/ is listed in .gitignore (never committed) and only bench.py's CPU arm reads it."""
    import shutil
    if not os.path.isfile(os.path.join(src, "models", "pytorch", "model.py")):
        return False
    for rel in STAGED_FILES:
        dst = os.path.join(STAGED_ROOT, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(os.path.join(src, rel), dst)
    return True


def _install_shims():
    from . import color_ref
    if "matplotlib" not in sys.modules:
        try:
            import matplotlib  # noqa: F401
        except ImportError:
            mpl = types.ModuleType("matplotlib")
            plt = types.ModuleType("matplotlib.pyplot")
            mpl.pyplot = plt
            sys.modules["matplotlib"] = mpl
            sys.modules["matplotlib.pyplot"] = plt
    if "skimage" not in sys.modules:
        try:
            import skimage  # noqa: F401
        except ImportError:
            sk = types.ModuleType("skimage")
            col = types.ModuleType("skimage.color")
            col.rgb2lab = color_ref.rgb2lab
            col.lab2rgb = color_ref.lab2rgb
            sk.color = col
            sys.modules["skimage"] = sk
            sys.modules["skimage.color"] = col


def import_reference_model():
    """-> module /root/reference/models/pytorch/model.py (SIGGRAPHGenerator)."""
    if not reference_available():
        raise RuntimeError("reference tree not present at %s" % REF_ROOT)
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    import importlib
    return importlib.import_module("models.pytorch.model")


def import_reference_wrapper():
    """-> module /root/reference/data/colorize_image.py (ColorizeImageTorch...)."""
    if not reference_available():
        raise RuntimeError("reference tree not present at %s" % REF_ROOT)
    _install_shims()
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    import importlib
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return importlib.import_module("data.colorize_image")
