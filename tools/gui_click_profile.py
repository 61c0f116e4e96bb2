"""Per-click cost of the GUI path, dense planes vs hint lists (prints one JSON object).

Replays a fixed 20-click script (add / move / erase, config-5 style) through a Qt-free fake GUIDraw, alternating the
reference statements (`get_input()` + `rgb2lab` + net_forward of the dense planes, then the host gamut map) and the
device hooks of launcher.py (`use_device_hints`, `use_gpu_gamut`), and reports
  * host wall time per press (compute_result + predict_color + update_gamut) and per drag move (compute_result),
  * device time of the click graph, batch 1 at 256^2, dense vs hint mode (CUDA events around the graph launch),
  * the n = 64 end-to-end idc_forward_host, dense vs hint mode,
  * the card name and its power limit.

    python tools/gui_click_profile.py [--reps 5]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from interactive_deep_colorization_b200 import _lib, color, launcher  # noqa: E402
from interactive_deep_colorization_b200 import colorize_image as CI  # noqa: E402
from oracle import gamut_ref, hints_ref, synth  # noqa: E402
from tests.test_hints_cpu import FakePointEdit, FakeUIControl  # noqa: E402


class FakeGUI(object):
    def __init__(self, model, dist_model, ui, l_win):
        self.model, self.dist_model, self.uiControl, self.l_win = model, dist_model, ui, l_win
        self.image_loaded = True
        self.win_w = self.win_h = l_win.shape[0]

    def update(self):
        pass

    # the reference's statements (ui/gui_draw.py:250-258, :272-279), display on the device as launcher.use_gpu_display
    def compute_result_dense(self):
        from interactive_deep_colorization_b200 import prepost
        im, mask = self.uiControl.get_input()
        self.im_mask0 = (mask > 0.0).transpose((2, 0, 1))
        self.im_ab0 = color.rgb2lab(im).transpose((2, 0, 1))[1:3]
        self.model.net_forward(self.im_ab0, self.im_mask0)
        self.result = prepost.display_rgb_gpu(np.asarray(self.model.output_ab), self.l_win, self.model._device())

    def predict_color_dense(self):
        im, mask = self.uiControl.get_input()
        self.im_mask0 = (mask > 0.0).transpose((2, 0, 1))
        self.im_ab0 = color.rgb2lab(im).transpose((2, 0, 1))[1:3]
        self.dist_model.net_forward(self.im_ab0, self.im_mask0)


def script(rs):
    """20 clicks: ('press', edits) adds / erases / recolours a point, ('move', edits) drags the last one."""
    edits, out = [], []
    for step in range(20):
        kind = ("add", "move", "add", "move", "erase")[step % 5]
        if kind == "add" or not edits:
            edits.append(FakePointEdit((int(rs.randint(40, 470)), int(rs.randint(80, 430))),
                                       tuple(int(v) for v in rs.randint(0, 256, 3)), 6))
            out.append(("press", list(edits)))
        elif kind == "move":
            e = edits[-1]
            edits[-1] = FakePointEdit((e.pnt.x() + 7, e.pnt.y() + 3), e.color.rgb, e.width)
            out.append(("move", list(edits)))
        else:
            edits.pop(0)
            out.append(("press", list(edits)))
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = [s.strip() for s in q.split(",")]
        return name, plim
    except Exception as e:                                     # the numbers stay valid; the label is then unknown
        return "unknown (%s)" % e, "unknown"


def gui_replay(sd, reps):
    X = 256
    img = (np.random.RandomState(0).rand(X, X, 3) * 255).astype(np.uint8)
    cm = CI.ColorizeImageB200(Xd=X)
    cm.prep_net(0, state_dict=sd, dist=True)
    cm.set_image(img)
    dm = CI.ColorizeImageB200Dist(Xd=X).share_trunk(cm)
    dm.set_image(img)
    hinted = type("FakeGUIHinted", (FakeGUI,), {})
    launcher.use_device_hints(hinted)
    grid = type("G", (), {"gamut_size": 110, "D": 1})()
    gpu_gamut = type("M", (), {"abGrid": type("abGrid", (), {})})
    launcher.use_gpu_gamut(gpu_gamut)
    clicks = script(np.random.RandomState(1))
    t = {"dense": {"press": [], "move": []}, "hints": {"press": [], "move": []}}
    for _ in range(reps):
        for mode in ("dense", "hints"):                           # alternate the two arms
            for kind, edits in clicks:
                ui = FakeUIControl(edits)
                g = (FakeGUI if mode == "dense" else hinted)(cm, dm, ui, np.full((512, 512), 50.0))
                L = float(50 + 20 * np.sin(len(edits)))
                t0 = time.perf_counter()
                if mode == "dense":
                    g.compute_result_dense()
                    if kind == "press":
                        g.predict_color_dense()
                        gamut_ref.update_gamut(L)
                else:
                    g.compute_result()
                    if kind == "press":
                        g.predict_color()
                        gpu_gamut.abGrid.update_gamut(grid, L)
                t[mode][kind].append((time.perf_counter() - t0) * 1e3)
    return {m: {k: float(np.median(v)) for k, v in d.items()} for m, d in t.items()}


def device_click(sd, reps):
    X = 256
    from tests import util
    ctx = util.make_ctx(sd, X, X, max_n=1, dist=True)
    lib = _lib.load()
    lib.idc_debug_graph_timing.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
    lib.idc_debug_graph_timing(ctx.h, 1, None)
    ctx.set_dist_resident(True)
    L, _, _ = synth.synthetic_batch(1, X, seed=2, max_hints=0)
    rects = CI.hints_from_points([((int(y), int(x)), 3, (20.0, -40.0)) for y, x in np.random.RandomState(3).randint(0, X, (20, 2))], X)
    out = {}
    for mode in ("dense", "hints"):
        buf = ctx.click_buffers(1, hints=mode == "hints")
        buf["L_mc"][...] = L
        ctx.set_image(buf["L_mc"])
        if mode == "dense":
            ab, m = hints_ref.raster(rects, 1, X, X)
            buf["ab"][...] = ab
            buf["mask"][...] = m
        else:
            ctx.set_hints(rects)
        ms = []
        for i in range(20 + reps * 20):
            ctx.forward_host(None, buf["ab"], buf["mask"], 0.5, n=1, want_rgb=True, want_abq=True, out_ab=buf["out_ab"],
                             out_rgb=buf["out_rgb"], out_abq=buf["out_abq"])
            v = ctypes.c_float()
            lib.idc_debug_graph_timing(ctx.h, 1, ctypes.byref(v))
            if i >= 20:
                ms.append(v.value)
        out[mode] = {"p50_ms": float(np.median(ms)), "p90_ms": float(np.percentile(ms, 90))}
    ctx.close()
    return out


def batch64(sd, reps):
    X, n = 256, 64
    from tests import util
    ctx = util.make_ctx(sd, X, X, max_n=n)
    L, _, _ = synth.synthetic_batch(n, X, seed=4, max_hints=0)
    rs = np.random.RandomState(5)
    rects = np.zeros(n * 10, _lib.HINT_DTYPE)
    for i in range(rects.shape[0]):
        y, x = rs.randint(0, X - 7, 2)
        rects[i] = (i // 10, y, x, y + 6, x + 6, rs.uniform(-90, 90), rs.uniform(-90, 90))
    ab, m = hints_ref.raster(rects, n, X, X)
    ab, m = np.ascontiguousarray(ab), np.ascontiguousarray(m)
    ctx.set_hints(rects)
    out_ab = np.empty((n, 2, X, X), np.float32)
    t = {"dense": [], "hints": []}
    for i in range(3 + reps * 4):
        for mode in ("dense", "hints"):
            t0 = time.perf_counter()
            if mode == "dense":
                ctx.forward_host(L, ab, m, 0.5, out_ab=out_ab)
            else:
                ctx.forward_host(L, None, None, 0.5, out_ab=out_ab, n=n)
            if i >= 3:
                t[mode].append((time.perf_counter() - t0) * 1e3)
    ctx.close()
    return {k: {"p50_ms": float(np.median(v))} for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    sd = synth.torch_state_dict(1234)
    name, plim = card()
    res = {"card": name, "power_limit": plim, "gui_host_ms": gui_replay(sd, args.reps),
           "click_graph_device_ms": device_click(sd, args.reps), "forward_host_n64_ms": batch64(sd, args.reps)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
