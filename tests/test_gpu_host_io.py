"""GPU: the copies of the host-pointer forward (idc_forward_host_q).

Every call is compared bit for bit with the device-pointer forward (idc_forward) on the same inputs: ab, rgb and dist.
The quantised ab has no device-pointer counterpart; it is compared with the same call made on a context that takes
the other host path (no click graph at n <= 4, no chunked overlap at n >= 8).  The cases cover the click graph
(n <= 4) and the eager path (n >= 5, chunked from n = 8) on contexts whose max_n is larger than n; caller memory that
is page-locked, pageable, mixed, or the context's click buffers; dense planes and hint lists; explicit and resident L;
global hints; and the dist, rgb and quantised-ab outputs on and off.  The last test pins how often the click graph is
captured when the caller's memory changes."""
import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import _lib
from oracle import caffe_spec, hints_ref, synth
from tests import util

pytestmark = pytest.mark.gpu

X, MAX_N = 64, 16
MEMORY = ["pinned", "pageable", "pinned_in", "pinned_out", "click"]
# (hint list, resident L, want_dist, want_rgb, want_abq)
VARIANTS = [(False, False, True, True, True), (False, True, False, False, False),
            (True, False, True, True, False), (True, True, False, True, True)]


def _glob_sd():
    sd = dict(synth.torch_state_dict(1234))
    sd.update({k: torch.from_numpy(v) for k, v in caffe_spec.synthetic_glob_state_dict().items()})
    return sd


@pytest.fixture(scope="module")
def contexts():
    """glob -> (context under test, reference context on the other host path)"""
    out = {}
    for glob in (False, True):
        sd = _glob_sd() if glob else synth.torch_state_dict(1234)
        kw = dict(max_n=MAX_N, dist=True, global_hints=glob)
        out[glob] = (util.make_ctx(sd, X, X, **kw),
                     util.make_ctx(sd, X, X, use_graph=False, options={"host_pipe": 0}, **kw))
    yield out
    for pair in out.values():
        for ctx in pair:
            ctx.close()


def _host(a, pinned):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a).pin_memory().numpy() if pinned else a.copy()


def _empty(shape, dtype, pinned):
    return _host(np.empty(shape, dtype), pinned)


def _rects(rs, n):
    out = np.zeros(12, _lib.HINT_DTYPE)
    for i in range(len(out)):
        y0, x0 = rs.randint(-2, X, 2)
        h, w = rs.randint(0, 7, 2)
        out[i] = (rs.randint(n), y0, x0, y0 + h, x0 + w, rs.uniform(-90, 90), rs.uniform(-90, 90))
    return out


def _device_ref(ctx, L, ab, m, glob):
    r = ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5, glob=None if glob is None else util.dev(glob),
                           want_dist=True, want_rgb=True)
    return {k: r[k].cpu().numpy() for k in ("ab", "dist", "rgb")}, ctx.last_launch_count()


@pytest.mark.parametrize("glob_on", [False, True])
@pytest.mark.parametrize("mem", MEMORY)
@pytest.mark.parametrize("n", [1, 3, 4, 5, 8, 12])
def test_forward_host_equals_forward_device(contexts, n, mem, glob_on):
    ctx, other = contexts[glob_on]
    rs = np.random.RandomState(100 * n + MEMORY.index(mem) + 7 * glob_on)
    L, ab_planes, m_planes = synth.synthetic_batch(n, X, seed=int(rs.randint(1 << 20)), max_hints=4)
    glob = rs.rand(n, 316).astype(np.float32) if glob_on else None
    for hints, resident, want_dist, want_rgb, want_abq in VARIANTS:
        if hints:
            rects = _rects(rs, n)
            ab, m = (np.ascontiguousarray(a) for a in hints_ref.raster(rects, n, X, X))
            ctx.set_hints(rects)
            other.set_hints(rects)
        else:
            ab, m = ab_planes, m_planes
        want, launches = _device_ref(ctx, L, ab, m, glob)
        pin_in, pin_out = mem in ("pinned", "pinned_in"), mem in ("pinned", "pinned_out")
        if mem == "click":
            buf = ctx.click_buffers(n, glob=glob_on, hints=hints)
            hL, hg = buf["L_mc"], buf["glob"]
            hL[...] = L
            if glob_on:
                hg[...] = glob
            if not hints:
                buf["ab"][...] = ab
                buf["mask"][...] = m
            hab, hm = buf["ab"], buf["mask"]
            outs = dict(out_ab=buf["out_ab"], out_rgb=buf["out_rgb"] if want_rgb or want_abq else None,
                        out_abq=buf["out_abq"] if want_abq else None, out_dist=None)
        else:
            hL, hg = _host(L, pin_in), None if glob is None else _host(glob, pin_in)
            hab, hm = (None, None) if hints else (_host(ab, pin_in), _host(m, pin_in))
            outs = dict(out_ab=_empty((n, 2, X, X), np.float32, pin_out),
                        out_rgb=_empty((n, X, X, 3), np.uint8, pin_out) if want_rgb or want_abq else None,
                        out_abq=_empty((n, 2, X, X), np.float64, pin_out) if want_abq else None,
                        out_dist=_empty((n, 529, X // 4, X // 4), np.float32, pin_out) if want_dist else None)
        if resident:
            ctx.set_image(hL)
        got = ctx.forward_host(None if resident else hL, hab, hm, 0.5, glob=hg, want_dist=want_dist, want_rgb=want_rgb,
                               want_abq=want_abq, n=n, **outs)
        what = (hints, resident, want_dist, want_rgb, want_abq)
        assert np.array_equal(got["ab"], want["ab"]), what
        if want_dist:
            assert np.array_equal(got["dist"], want["dist"]), what
        if want_rgb or want_abq:
            assert np.array_equal(got["rgb"], want["rgb"]), what
        if want_abq:
            ref = other.forward_host(L, None if hints else ab, None if hints else m, 0.5, glob=glob, want_abq=True, n=n)
            assert np.array_equal(ref["ab"], want["ab"]) and np.array_equal(ref["rgb"], want["rgb"]), what
            assert np.array_equal(got["abq"], ref["abq"]), what
        if n >= 8 and want_dist and want_rgb:    # chunked: conv1_1 and the last op ran once per chunk
            assert ctx.last_launch_count() > launches, what


def test_click_graph_captures(synth_sd):
    """Identical calls through the click buffers replay one graph; a change between page-locked and pageable memory,
    or to the dist copy, re-captures it (the counts of the parent implementation)."""
    ctx = util.make_ctx(synth_sd, X, X, max_n=4, dist=True)
    L, ab, m = synth.synthetic_batch(1, X, seed=5, max_hints=4)
    buf = ctx.click_buffers(1)
    buf["L_mc"][...], buf["ab"][...], buf["mask"][...] = L, ab, m
    want = ctx.forward_device(util.dev(L), util.dev(ab), util.dev(m), 0.5, want_rgb=True)["ab"].cpu().numpy()
    pinned = dict(out_ab=buf["out_ab"], out_rgb=buf["out_rgb"])
    calls = [("click", {}), ("click", {}), ("pageable", {}), ("pageable", {}), ("click", {}),
             ("click", dict(want_dist=True)), ("click", dict(want_dist=True)), ("click", {}),
             ("pinned_in", {}), ("pageable", {})]
    counts = []
    for mem, kw in calls:
        if mem == "pageable":
            r = ctx.forward_host(L.copy(), ab.copy(), m.copy(), 0.5, want_rgb=True, **kw)
        elif mem == "pinned_in":
            r = ctx.forward_host(buf["L_mc"], buf["ab"], buf["mask"], 0.5, want_rgb=True, **kw)
        else:
            r = ctx.forward_host(buf["L_mc"], buf["ab"], buf["mask"], 0.5, want_rgb=True, **pinned, **kw)
        assert np.array_equal(r["ab"], want), (mem, kw)
        counts.append(ctx.graph_captures())
    assert counts == [1, 1, 2, 2, 3, 4, 4, 5, 6, 6]
    ctx.close()
