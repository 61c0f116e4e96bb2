"""ctypes binding of libidc_b200.so (include/idc_b200.h).

No fallback: if the shared library is missing or fails to load this raises, and every
public entry point of the package raises with it.  PyTorch is used by callers for device
memory / streams only; nothing in here touches torch.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libidc_b200.so")
if os.environ.get("IDC_B200_LIB"):            # tools only: a build elsewhere (make OUT=...)
    LIB_PATH = os.environ["IDC_B200_LIB"]

IDC_OK = 0
# error codes (include/idc_b200.h)
ERR_ARG, ERR_CUDA, ERR_STATE, ERR_KEY, ERR_UNSUPPORTED, ERR_WATCHDOG, ERR_RANGE = -1, -2, -3, -4, -5, -6, -7
FLAG_DIST = 1 << 0
FLAG_ENGINE_SIMT = 1 << 1
FLAG_FAST_FP16 = 1 << 2
FLAG_GLOBAL_HINTS = 1 << 3
FLAG_NO_GRAPH = 1 << 4
FLAG_KEEP_CONV10 = 1 << 5
FLAG_CAFFE313 = 1 << 6
F32, F64, I64 = 0, 1, 2
MAX_HINTS = 1024                      # IDC_MAX_HINTS
MAX_PHOTOS = 128                      # IDC_MAX_PHOTOS
MAX_PHOTO_SIDE = 1 << 24               # IDC_MAX_PHOTO_SIDE
MAX_PHOTO_X = 16384                   # IDC_MAX_PHOTO_X
MAX_RECCS_QUERIES = 65535             # IDC_MAX_RECCS_QUERIES
HINT_HDR_BYTES = 16                   # header {count, 0, 0, 0} of an idc_hint_raster block
# idc_photo: a photo of a packed batch, its first pixel and its size
PHOTO_DTYPE = np.dtype([("off", "<i8"), ("h", "<i4"), ("w", "<i4")])
RENDER_L_PLANE, RENDER_L_MASK, RENDER_L_SUP = 0, 1, 2     # idc_render_planes_u8 l_mode
# idc_hint: inclusive pixel rectangle of image `img` painted with one ab colour (28 bytes, no padding)
HINT_DTYPE = np.dtype([("img", "<i4"), ("y0", "<i4"), ("x0", "<i4"), ("y1", "<i4"), ("x1", "<i4"),
                       ("a", "<f4"), ("b", "<f4")])

# every symbol include/idc_b200.h declares: (name, restype, argtypes)
_c = ctypes
_P = _c.c_void_p
SYMBOLS = [
    ("idc_version", _c.c_char_p, []),
    ("idc_create", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _c.c_int, _c.c_uint, _c.POINTER(_P)]),
    ("idc_load_tensor", _c.c_int, [_P, _c.c_char_p, _P, _c.c_int, _c.c_int, _c.POINTER(_c.c_int64)]),
    ("idc_finalize_weights", _c.c_int, [_P]),
    ("idc_weights_arena", _c.c_int, [_P, _c.POINTER(_P), _c.POINTER(_c.c_size_t)]),
    ("idc_reserve_weights", _c.c_int, [_P]),
    ("idc_adopt_weights", _c.c_int, [_P]),
    ("idc_forward", _c.c_int, [_P, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P, _c.c_float, _P, _P, _P, _P, _P]),
    ("idc_forward_host", _c.c_int, [_P, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P, _c.c_float, _P, _P, _P, _P]),
    ("idc_forward_host_q", _c.c_int, [_P, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P, _c.c_float, _P, _P, _P, _P, _P]),
    ("idc_set_option", _c.c_int, [_P, _c.c_char_p, _c.c_int]),
    ("idc_set_image", _c.c_int, [_P, _c.c_int, _c.c_int, _c.c_int, _P]),
    ("idc_set_hints", _c.c_int, [_P, _c.c_int, _P]),
    ("idc_gamut_ab", _c.c_int, [_c.c_int, _c.c_double, _c.c_int, _c.c_int, _P, _P, _P]),
    ("idc_graph_captures", _c.c_int, [_P]),
    ("idc_host_alloc", _P, [_c.c_size_t]),
    ("idc_host_free", _c.c_int, [_P]),
    ("idc_set_dist_resident", _c.c_int, [_P, _c.c_int]),
    ("idc_fetch_dist", _c.c_int, [_P, _c.c_int, _c.c_int, _c.c_int, _P]),
    ("idc_set_click", _c.c_int, [_P, _c.c_int, _c.c_int, _c.c_int, _c.c_int]),
    ("idc_ab_reccs", _c.c_int, [_P, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P, _P]),
    ("idc_ab_reccs_pmf", _c.c_int, [_c.c_int, _P, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P, _P]),
    ("idc_ab_reccs_batch", _c.c_int, [_P, _c.c_int, _P, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P, _P, _P, _P]),
    ("idc_ab_reccs_batch_check", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _P, _c.c_int, _c.c_int,
                                            _c.c_int, _P, _c.c_size_t]),
    ("idc_caffe313_pred_ab", _c.c_int, [_P, _c.c_int, _c.c_float, _P, _P]),
    ("idc_caffe313_dist_pixel", _c.c_int, [_P, _c.c_int, _c.c_int, _c.c_int, _c.c_float, _P]),
    ("idc_caffe313_dist_map", _c.c_int, [_P, _c.c_int, _c.c_float, _P, _P]),
    ("idc_negentropy", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P]),
    ("idc_dist_negentropy", _c.c_int, [_P, _c.c_int, _P]),
    ("idc_lab2rgb_u8", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P, _P]),
    ("idc_rgb2lab_f64", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P]),
    ("idc_global_stats", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _P, _P, _P, _P]),
    ("idc_zoom_lab2rgb_u8", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _P, _c.c_int, _c.c_int, _P, _P, _P]),
    ("idc_render_planes_u8", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _P, _c.c_int, _c.c_int, _P, _c.c_int, _c.c_int,
                                        _P, _c.c_int, _c.c_int, _P, _P]),
    ("idc_resize_u8_linear", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _P, _c.c_int, _c.c_int, _P, _P]),
    ("idc_cubic_lab2rgb_u8", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _P, _c.c_int, _c.c_int, _P, _P, _P]),
    ("idc_photo_prep", _c.c_int, [_c.c_int, _c.c_int, _P, _P, _c.c_int, _P, _P, _P]),
    ("idc_photo_render", _c.c_int, [_c.c_int, _c.c_int, _P, _P, _c.c_int, _P, _P, _P]),
    ("idc_hint_raster", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P, _P]),
    ("idc_rgb_sse", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P, _P]),
    ("idc_hint_fill_mean", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _c.c_int, _P, _P, _c.c_size_t, _P]),
    ("idc_global_stats_batch", _c.c_int, [_c.c_int, _c.c_int, _c.c_int, _c.c_int, _P, _P, _P, _P]),
    ("idc_get_activation", _c.c_int, [_P, _c.c_char_p, _P, _c.c_size_t, _c.POINTER(_c.c_int),
                                      _c.POINTER(_c.c_int), _c.POINTER(_c.c_int)]),
    ("idc_set_activation", _c.c_int, [_P, _c.c_char_p, _c.c_int, _P]),
    ("idc_act_exponent", _c.c_int, [_P, _c.c_char_p, _c.POINTER(_c.c_int)]),
    ("idc_num_acts", _c.c_int, [_P]),
    ("idc_act_name", _c.c_char_p, [_P, _c.c_int]),
    ("idc_act_absmax", _c.c_int, [_P, _c.c_char_p, _c.c_int, _c.POINTER(_c.c_float)]),
    ("idc_set_act_range", _c.c_int, [_P, _c.c_char_p, _c.c_double]),
    ("idc_run_op", _c.c_int, [_P, _c.c_char_p, _c.c_int, _P]),
    ("idc_num_ops", _c.c_int, [_P]),
    ("idc_op_name", _c.c_char_p, [_P, _c.c_int]),
    ("idc_set_profiling", _c.c_int, [_P, _c.c_int]),
    ("idc_get_profile", _c.c_int, [_P, _c.POINTER(_c.c_float), _c.c_int]),
    ("idc_op_flops", _c.c_double, [_P, _c.c_int]),
    ("idc_last_launch_count", _c.c_int, [_P]),
    ("idc_flops_per_image", _c.c_double, [_P]),
    ("idc_last_error", _c.c_char_p, [_P]),
    ("idc_destroy", _c.c_int, [_P]),
]

_lib = None


class IdcError(RuntimeError):
    def __init__(self, code, msg):
        RuntimeError.__init__(self, "idc_b200 error %d: %s" % (code, msg))
        self.code = code


def load():
    """Load the shared library (once) and declare the prototypes.  Raises if it is absent:
    there is deliberately no CPU / PyTorch fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise ImportError("libidc_b200.so not built (%s missing); run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "or `make -C interactive_deep_colorization_b200/csrc`" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, res, args in SYMBOLS:
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(ctx, rc):
    if rc != IDC_OK:
        msg = load().idc_last_error(ctx) if ctx else b""
        raise IdcError(rc, (msg or b"").decode("utf-8", "replace"))
