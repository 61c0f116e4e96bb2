#!/usr/bin/env python
"""GPU tool: the batch-1 interactive path (max_n=1 ctx, dist head on) under different plan-time options:
per-op device time (CUDA events between the launches, PDL off by construction), the wall-clock p50 of the
graph-replayed idc_forward_host_q (the click), and the same through the ColorizeImageB200 wrapper.

    python tools/latency_profile.py [name=opt:val,opt:val ...]      e.g.  base=pdl:0 new=
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import synth  # noqa: E402
from tests import util  # noqa: E402


def run(tag, options, per_op=True):
    sd = synth.torch_state_dict(1234)
    L, ab, m = synth.synthetic_batch(1, 256, seed=0)
    if per_op:
        ctx = util.make_ctx(sd, 256, 256, max_n=1, dist=True, use_graph=False, options=options)
        dL, dab, dm = util.dev(L), util.dev(ab), util.dev(m)
        for _ in range(5):
            ctx.forward_device(dL, dab, dm, 0.5, want_dist=True, want_rgb=True)
        torch.cuda.synchronize()
        ctx.set_profiling(True)
        for _ in range(20):
            ctx.forward_device(dL, dab, dm, 0.5, want_dist=True, want_rgb=True)
        prof = ctx.get_profile()
        ctx.set_profiling(False)
        tot = sum(ms for _, ms, _ in prof)
        print("[%s] per-op us (sum %.1f us): " % (tag, tot * 1e3) + " ".join("%s=%.1f" % (n, ms * 1e3) for n, ms, _ in prof))
        # device time of whole forwards back to back (no events in between: PDL active if enabled)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(50):
            ctx.forward_device(dL, dab, dm, 0.5, want_dist=True, want_rgb=True)
        e1.record()
        torch.cuda.synchronize()
        print("[%s] stream-launched forward (dist+rgb): %.1f us each" % (tag, e0.elapsed_time(e1) * 1e3 / 50))
        ctx.close()
    if os.environ.get("IDC_PER_OP_ONLY"):
        return
    for want_dist in (True, False):
        for pinned in (False, True):
            ctx = util.make_ctx(sd, 256, 256, max_n=1, dist=True, use_graph=True, options=options)
            if want_dist:
                ctx.set_dist_resident(True)
            kw = {}
            a, b, c = L, ab, m
            if pinned:
                buf = ctx.click_buffers(1)
                buf["L_mc"][...] = L; buf["ab"][...] = ab; buf["mask"][...] = m
                a, b, c = buf["L_mc"], buf["ab"], buf["mask"]
                kw = dict(out_ab=buf["out_ab"], out_rgb=buf["out_rgb"], out_abq=buf["out_abq"])
            ts = []
            for i in range(40):
                t = time.perf_counter()
                ctx.forward_host(a, b, c, 0.5, want_rgb=True, want_abq=True, **kw)
                ts.append((time.perf_counter() - t) * 1e3)
            print("[%s] forward_host_q graph resident_dist=%s %s buffers p50 %.3f ms  min %.3f ms"
                  % (tag, want_dist, "page-locked" if pinned else "pageable", np.percentile(ts[5:], 50), min(ts)))
            ctx.close()


if __name__ == "__main__":
    specs = sys.argv[1:] or ["no_pdl=pdl:0", "no_split_k=split_k:1", "new="]
    for spec in specs:
        name, _, body = spec.partition("=")
        opts = {kv.split(":")[0]: int(kv.split(":")[1]) for kv in body.split(",") if kv}
        run(name, opts)
