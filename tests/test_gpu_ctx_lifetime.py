"""GPU: what a context owns.  Closing a context returns every device buffer it made, the lazily built ones included,
and a plan-time option changed after the weights are final re-plans the context as if it had been created with it."""
import numpy as np
import pytest
import torch

from oracle import caffe_spec, synth
from tests import util

pytestmark = pytest.mark.gpu

X = 256
MIB = 1 << 20


def _hint_rects(n):
    return [(0, 40 + 9 * i, 50, 46 + 9 * i, 57, 20.0 - 7 * i, -30.0 + 5 * i) for i in range(n)]


def _cycle_lhn(sd, engine, L, ab, m):
    """Builds every lazy group and scratch buffer of an LHN context, then closes it."""
    ctx = util.make_ctx(sd, X, X, max_n=8, dist=True, engine=engine)
    ctx.set_image(np.ascontiguousarray(L[:1]))                          # host staging
    ctx.set_hints(_hint_rects(3))                                       # hint block
    ctx.forward_host(None, None, None, 0.5, n=1)
    ctx.set_dist_resident(True)
    ctx.set_click(0, 20, 30, K=5)                                       # click block
    ctx.forward_host(None, ab[:1], m[:1], 0.5)                          # side branch + click branch (wgmma)
    ctx.fetch_dist(0, 20, 30)
    ctx.fetch_dist(0)
    ctx.ab_reccs(0, 10, 12, K=3)                                        # reccs scratch
    ctx.dist_negentropy(0)                                              # negentropy scratch
    ctx.set_click(0, -1)
    ctx.forward_host(L, ab, m, 0.5, want_abq=True)                      # host pipe + quantised-ab staging (n = 8)
    ctx.set_profiling(True)                                             # profiling events
    ctx.forward_device(util.dev(L[:2]), util.dev(ab[:2]), util.dev(m[:2]), 0.5, want_dist=True)
    torch.cuda.synchronize()
    assert len(ctx.get_profile()) == len(ctx.op_names()) + 2
    ctx.close()


def _cycle_caffe313(sd, L, ab, m):
    ctx = util.make_ctx(sd, X, X, max_n=1, caffe313=True)
    ctx.forward_device(util.dev(L[:1]), util.dev(ab[:1]), util.dev(m[:1]), 0.5)
    ctx.caffe313_dist_pixel(0, 100, 60)                                 # dist313 scratch
    ctx.caffe313_dist_map(1)
    torch.cuda.synchronize()
    ctx.close()


def _free_after_cleanup():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def test_teardown_returns_device_memory(synth_sd):
    """Three cycles of wgmma, SIMT and Caffe 313-bin contexts that build every lazy resource: after cycles 2 and 3 the
    device has as much free memory as after cycle 1 (which absorbs module loading), within 2 MiB."""
    L, ab, m = synth.synthetic_batch(8, X, seed=21, max_hints=4)
    csd = caffe_spec.synthetic_caffe313_state_dict(pts_in_hull=util.golden("pts_in_hull.npy"))
    sd313 = dict(synth_sd)
    sd313.update({k: torch.from_numpy(v) for k, v in csd.items()})
    free = []
    for _ in range(3):
        _cycle_lhn(synth_sd, "wgmma", L, ab, m)
        _cycle_lhn(synth_sd, "simt", L, ab, m)
        _cycle_caffe313(sd313, L, ab, m)
        free.append(_free_after_cleanup())
    print("free device memory after each cycle (MiB):", [f / MIB for f in free])
    for f in free[1:]:
        assert abs(f - free[0]) <= 2 * MIB, [f / MIB for f in free]


def _click(ctx, L, ab, m, y4, x4, K):
    ctx.set_click(0, y4, x4, K=K)
    out = ctx.forward_host(L, ab, m, 0.5, want_rgb=True)
    centers, conf, iters = ctx.ab_reccs(0, y4, x4, K=K)
    return {"ab": out["ab"].copy(), "rgb": out["rgb"].copy(), "pmf": ctx.fetch_dist(0, y4, x4),
            "centers": centers, "conf": conf, "iters": np.array(iters)}


def _same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in a)


def test_replan_after_weights_final(synth_sd):
    """set_option after load_state_dict re-plans: the next click re-captures the click graph once and equals, bit for
    bit, a context created with those options; setting the defaults back reproduces the first click."""
    L, ab, m = synth.synthetic_batch(1, X, seed=33, max_hints=4)
    changed = {"halo": 0, "split_k": 1, "mt": 1}
    defaults = {"halo": 1, "split_k": -1, "mt": -1}
    ctx = util.make_ctx(synth_sd, X, X, max_n=1, dist=True)
    ctx.set_dist_resident(True)
    first = _click(ctx, L, ab, m, 30, 25, 5)
    captures = ctx.graph_captures()
    for k, v in changed.items():
        ctx.set_option(k, v)
    replanned = _click(ctx, L, ab, m, 30, 25, 5)
    assert ctx.graph_captures() == captures + 1

    fresh = util.make_ctx(synth_sd, X, X, max_n=1, dist=True, options=changed)
    fresh.set_dist_resident(True)
    assert _same(_click(fresh, L, ab, m, 30, 25, 5), replanned)
    fresh.close()

    for k, v in defaults.items():
        ctx.set_option(k, v)
    assert _same(_click(ctx, L, ab, m, 30, 25, 5), first)
    ctx.close()
