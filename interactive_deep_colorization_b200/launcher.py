"""`ideepcolor.py` with an H100 backend (SURVEY row f4).

    python -m interactive_deep_colorization_b200.launcher --backend b200 --reference_root /path/to/ideepcolor \\
        --color_model caffemodel.pth [--pytorch_maskcent] [--image_file ...] [--win_size 512] [--gpu 0]

Mirrors the reference entry point (ideepcolor.py:13-46 arguments, :60-74 backend selection, :76-86 window set-up):
the SAME Qt window classes (`ui.gui_design.GUIDesign`, imported from the reference tree, PyQt4 or the docker tree's
PyQt5 port) receive `ColorizeImageB200` / `ColorizeImageB200Dist` objects instead of the Torch / Caffe ones.  Nothing
of the GUI is re-implemented here.

Per-click colour suggestions: the reference commented out `self.predict_color()` after a new / erased point
(ui/gui_draw.py:134,142) because a distribution forward cost ~1.5 s on its CPU path; here it costs < 1 ms, so
`enable_per_click_suggestions()` re-enables exactly those two calls by wrapping `GUIDraw.update_ui` (its return value
`is_predict` is true precisely where the commented-out lines sit).  `use_gpu_display()` swaps the per-click display
step of `compute_result` (:280-283: cv2 cubic resize + lab2rgb, ~10 ms of numpy) for the fused GPU kernel.
`use_device_hints()` hands the user edits to the models as a rectangle list (rasterised on the device) instead of
painting and converting a whole image per call, and `use_gpu_gamut()` computes the gamut map on the device.
"""
from __future__ import print_function

import argparse
import sys

import numpy as np

BACKENDS = ("b200", "b200-caffe")


def parse_args(argv=None):
    p = argparse.ArgumentParser(description='iDeepColor: deep interactive colorization (H100 backend)')
    # same names / defaults as ideepcolor.py:13-46
    p.add_argument('--win_size', dest='win_size', help='the size of the main window', type=int, default=512)
    p.add_argument('--image_file', dest='image_file', help='input image', type=str, default='test_imgs/mortar_pestle.jpg')
    p.add_argument('--gpu', dest='gpu', help='gpu id', type=int, default=0)
    p.add_argument('--color_model', dest='color_model', help='colorization model (state_dict .pth)', type=str,
                   default='./models/pytorch/caffemodel.pth')
    p.add_argument('--dist_model', dest='color_model', help='distribution prediction model (same file, ideepcolor.py:36-37)', type=str)
    p.add_argument('--color_caffemodel', dest='color_caffemodel', type=str, default='',
                   help='b200-caffe: Caffe-scaled state_dict of the regression net (see ColorizeImageB200Caffe)')
    p.add_argument('--dist_caffemodel', dest='dist_caffemodel', type=str, default='',
                   help='b200-caffe: Caffe-scaled state_dict of the 313-bin distribution net')
    p.add_argument('--backend', dest='backend', type=str, help='|'.join(BACKENDS), default='b200')
    p.add_argument('--pytorch_maskcent', dest='pytorch_maskcent', action='store_true',
                   help='need to center mask (activate for siggraph_pretrained but not for converted caffemodel)')
    p.add_argument('--load_size', dest='load_size', help='image size', type=int, default=256)
    # additions
    p.add_argument('--reference_root', type=str, default='.', help='checkout of the reference repo (for its ui/ package)')
    p.add_argument('--no_click_suggestions', action='store_true', help='keep the reference behaviour: suggestions only on load / reset')
    p.add_argument('--host_display', action='store_true', help='keep the numpy display step of compute_result')
    p.add_argument('--separate_models', action='store_true',
                   help='b200: two contexts (two forwards per click) like the reference, instead of one shared trunk')
    p.add_argument('--calibrate', type=str, default='', metavar='DIR_OR_JSON',
                   help='set the activation storage exponents from measured ranges: a folder of colour photos to measure '
                        'on at start-up, or a JSON file saved by ideepcolor_b200.py --save_act_ranges (no measurement)')
    args = p.parse_args(argv)
    args.calibrate_source = None
    if args.calibrate:
        from . import engine
        try:
            args.calibrate_source = engine.calibration_source(args.calibrate)
        except ValueError as e:
            p.error(str(e))
        if args.backend == 'b200-caffe' and isinstance(args.calibrate_source, str):
            p.error("--calibrate %s: ranges belong to one checkpoint and b200-caffe loads two (--color_caffemodel, "
                    "--dist_caffemodel); give a folder of photos, each checkpoint is then measured on it" % args.calibrate)
    return args


def build_models(args):
    """ideepcolor.py:60-74 for the H100 backends -> (colorModel, distModel)."""
    from . import colorize_image as CI
    if args.backend == 'b200':
        # "PyTorch (same model used for both)" (ideepcolor.py:34-38): one checkpoint, so one trunk -- the distribution
        # model shares the colour model's context and a click is ONE forward (ColorizeImageB200Dist.share_trunk)
        share = not getattr(args, 'separate_models', False)
        colorModel = CI.ColorizeImageB200(Xd=args.load_size, maskcent=args.pytorch_maskcent)
        cal = getattr(args, 'calibrate_source', None)
        colorModel.prep_net(gpu_id=args.gpu, path=args.color_model, dist=share, calibrate=cal)
        distModel = CI.ColorizeImageB200Dist(Xd=args.load_size, maskcent=args.pytorch_maskcent)
        if share:
            distModel.share_trunk(colorModel)
        else:
            distModel.prep_net(gpu_id=args.gpu, path=args.color_model, dist=True, calibrate=colorModel.act_ranges)
    elif args.backend == 'b200-caffe':
        colorModel = CI.ColorizeImageB200Caffe(Xd=args.load_size)
        cal = getattr(args, 'calibrate_source', None)      # a photo folder is measured once per checkpoint
        colorModel.prep_net(args.gpu, caffemodel_path=args.color_caffemodel, calibrate=cal)
        distModel = CI.ColorizeImageB200CaffeDist(Xd=args.load_size)
        distModel.prep_net(args.gpu, caffemodel_path=args.dist_caffemodel, calibrate=cal)
    else:
        raise SystemExit('backend type [%s] not found! (choose from %s)' % (args.backend, ', '.join(BACKENDS)))
    return colorModel, distModel


def enable_per_click_suggestions(gui_draw_cls):
    """Re-enable the two `self.predict_color()` calls the reference commented out (ui/gui_draw.py:134,142).
    `update_ui` returns is_predict == True exactly on those two paths (new point / removed point)."""
    if getattr(gui_draw_cls, "_b200_click_suggestions", False):
        return gui_draw_cls
    inner = gui_draw_cls.update_ui

    def update_ui(self, *a, **kw):
        is_predict = inner(self, *a, **kw)
        if is_predict:
            self.predict_color()
        return is_predict
    gui_draw_cls.update_ui = update_ui
    gui_draw_cls._b200_click_suggestions = True
    return gui_draw_cls


def use_gpu_display(gui_draw_cls, update_signal=None):
    """Replace the display step of `compute_result` (ui/gui_draw.py:272-286) by the fused GPU kernel: the network call
    and the hint preparation stay byte-for-byte the reference's statements; only :280-283 (cv2 cubic resize of
    output_ab to the window + lab2rgb + uint8) moves to `prepost.display_rgb_gpu`.  `update_signal(self, result)` emits
    the toolkit's `update_result` signal (PyQt4 old-style emit vs the PyQt5 port's bound signal)."""
    import numpy as np
    from . import color, prepost

    def compute_result(self):
        im, mask = self.uiControl.get_input()
        im_mask0 = mask > 0.0
        self.im_mask0 = im_mask0.transpose((2, 0, 1))
        im_lab = color.rgb2lab(im).transpose((2, 0, 1))
        self.im_ab0 = im_lab[1:3, :, :]
        self.model.net_forward(self.im_ab0, self.im_mask0)
        self.result = prepost.display_rgb_gpu(np.asarray(self.model.output_ab), self.l_win, self.model._device())
        if update_signal is not None:
            update_signal(self, self.result)
        self.update()
    gui_draw_cls.compute_result = compute_result
    return gui_draw_cls


def gui_hint_list(ui_control):
    """The hint list `ui_control.get_input()` would paint (ui/ui_control.py:177-187): one rectangle per user edit, in
    paint order, each from that edit's own scale_point / width / scale exactly as PointEdit.updateInput places its
    filled cv2.rectangle (:52-63), with the ab of its colour.  Each distinct colour is converted once, all in one
    color.rgb2lab batch, instead of the whole painted image."""
    from . import color
    from .colorize_image import HINT_LIST_DTYPE
    edits = list(ui_control.userEdits)
    rects = np.zeros(len(edits), HINT_LIST_DTYPE)
    rgb = np.zeros((len(edits), 3), np.uint8)
    for i, ue in enumerate(edits):
        w = int(ue.width / ue.scale)
        xa, ya = ue.scale_point(ue.pnt.x(), ue.pnt.y(), -w)
        xb, yb = ue.scale_point(ue.pnt.x(), ue.pnt.y(), w)
        rects[i] = (0, min(ya, yb), min(xa, xb), max(ya, yb), max(xa, xb), 0.0, 0.0)   # cv2 orders the corners
        rgb[i] = (ue.color.red(), ue.color.green(), ue.color.blue())
    if len(edits):
        uniq, inv = np.unique(rgb, axis=0, return_inverse=True)
        lab = color.rgb2lab(uniq[np.newaxis])[0]
        rects["a"], rects["b"] = lab[inv.reshape(-1), 1], lab[inv.reshape(-1), 2]
    return rects


class _LazyGuiPlanes(object):
    """`im_ab0` / `im_mask0` of GUIDraw after a hint-list forward: what the dense statements would have stored (ab of
    the painted image, mask > 0), read from the model's lazily rasterised input planes when save_result asks."""

    def __init__(self, name):
        self.name = name

    def __get__(self, obj, cls=None):
        if obj is None:
            return self
        d = obj.__dict__
        if self.name not in d:
            model = d.get("_b200_hint_model")
            if model is None:
                raise AttributeError(self.name)
            d[self.name] = model.input_ab if self.name == "im_ab0" else model.input_mask > 0
        return d[self.name]

    def __set__(self, obj, value):
        obj.__dict__[self.name] = value


def use_device_hints(gui_draw_cls, update_signal=None, gpu_display=True):
    """Replace the `get_input()` + `rgb2lab` statements of `compute_result` / `predict_color` (ui/gui_draw.py:250-258,
    :272-279): the models get the user edits as a hint list (net_forward_hints), which the click graph rasterises on the
    device.  The display step is `prepost.display_rgb_gpu` (gpu_display) or the reference's host statements
    (:280-283).  `self.im_ab0` / `self.im_mask0` stay readable for save_result; they are computed when read."""
    from . import color, prepost

    def _hint_forward(self, model):
        for k in ("im_ab0", "im_mask0"):
            self.__dict__.pop(k, None)
        model.net_forward_hints(gui_hint_list(self.uiControl))
        self.__dict__["_b200_hint_model"] = model

    def compute_result(self):
        _hint_forward(self, self.model)
        if gpu_display:
            self.result = prepost.display_rgb_gpu(np.asarray(self.model.output_ab), self.l_win, self.model._device())
        else:
            import cv2
            ab_win = cv2.resize(self.model.output_ab.transpose((1, 2, 0)), (self.win_w, self.win_h),
                                interpolation=cv2.INTER_CUBIC)
            pred_lab = np.concatenate((self.l_win[..., np.newaxis], ab_win), axis=2)
            self.result = (np.clip(color.lab2rgb(pred_lab), 0, 1) * 255).astype('uint8')
        if update_signal is not None:
            update_signal(self, self.result)
        self.update()

    def predict_color(self):
        if self.dist_model is not None and self.image_loaded:
            _hint_forward(self, self.dist_model)

    gui_draw_cls.compute_result = compute_result
    gui_draw_cls.predict_color = predict_color
    gui_draw_cls.im_ab0 = _LazyGuiPlanes("im_ab0")
    gui_draw_cls.im_mask0 = _LazyGuiPlanes("im_mask0")
    return gui_draw_cls


def use_gpu_gamut(lab_gamut_module, device=0):
    """Patch `abGrid.update_gamut` (data/lab_gamut.py:66-78, run on every colour change by ui/gui_gamut.py:17-20) with
    the device kernel (prepost.gamut_gpu): same (masked_rgb, mask), also stored on the grid object."""
    from . import prepost

    def update_gamut(self, l_in):
        self.masked_rgb, self.mask = prepost.gamut_gpu(l_in, self.gamut_size, self.D, device)
        return self.masked_rgb, self.mask
    lab_gamut_module.abGrid.update_gamut = update_gamut
    return lab_gamut_module


def main(argv=None):
    args = parse_args(argv)
    for arg in vars(args):
        print('[%s] =' % arg, getattr(args, arg))
    args.win_size = int(args.win_size / 4.0) * 4          # ideepcolor.py:57
    colorModel, distModel = build_models(args)
    sys.path.insert(0, args.reference_root)
    try:                                                  # the reference's own window (PyQt4) or its docker PyQt5 port
        from PyQt4.QtGui import QApplication
        from PyQt4.QtCore import SIGNAL
        from ui import gui_design, gui_draw
        emit = lambda self, result: self.emit(SIGNAL('update_result'), result)
    except ImportError:
        try:
            from PyQt5.QtWidgets import QApplication
            sys.path.insert(0, args.reference_root + '/docker')
            from ui_PyQt5 import gui_design, gui_draw
            emit = lambda self, result: self.update_result.emit(result)
        except ImportError as e:
            raise SystemExit("the Qt window is the reference's own (ui/*.py + PyQt4, or docker/ui_PyQt5 + PyQt5); neither is "
                             "importable here (%s).  The headless front end is ideepcolor_b200.py." % (e,))
    if not args.no_click_suggestions:
        enable_per_click_suggestions(gui_draw.GUIDraw)
    if not args.host_display:
        use_gpu_display(gui_draw.GUIDraw, emit)
    # hints as rectangle lists rasterised on the device, and the gamut map on the device (both replace per-click numpy)
    use_device_hints(gui_draw.GUIDraw, emit, gpu_display=not args.host_display)
    from data import lab_gamut
    use_gpu_gamut(lab_gamut, args.gpu)
    app = QApplication(sys.argv)
    window = gui_design.GUIDesign(color_model=colorModel, dist_model=distModel, img_file=args.image_file,
                                  load_size=args.load_size, win_size=args.win_size)
    window.setWindowTitle('iColor (H100)')
    window.show()
    app.exec_()


if __name__ == '__main__':
    main()
