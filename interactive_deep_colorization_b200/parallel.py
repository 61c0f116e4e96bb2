"""Multi-GPU: one process per GPU, images sharded across ranks, ONE broadcast of the packed
weight arena at init, no per-step collective (SURVEY.md 8e -- images are independent: the
network has no cross-image state, BatchNorm runs in eval mode,
/root/reference/data/colorize_image.py:232).

Host logic here is backend-agnostic (`gloo` on CPU in the tests, `nccl` over NVLink on the box).
"""
import numpy as np
import torch
import torch.distributed as dist


def shard_range(n_total, world, rank):
    """Contiguous, balanced slice [start, start+count) of n_total images for `rank`."""
    base, rem = divmod(int(n_total), int(world))
    count = base + (1 if rank < rem else 0)
    start = rank * base + min(rank, rem)
    return start, count


class _DevBlob(object):
    """Exposes a raw device pointer to torch through __cuda_array_interface__ (no copy)."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False),
                                         "version": 2, "strides": None}


def broadcast_blob(t, src=0):
    """Broadcast a byte tensor in place (NCCL: device tensor; gloo: CPU tensor)."""
    dist.broadcast(t, src=src)
    return t


def max_over_ranks(value, device=None):
    """Device-timed durations are reduced with MAX so a step is as slow as its slowest rank."""
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


class ShardedColorizer(object):
    """Per-rank Local-Hints-Network context with weights received from rank 0.

    `state_dict` is only needed on rank 0; the other ranks allocate the (deterministically laid
    out) arena, receive it with a single NCCL broadcast over NVLink/NVSwitch and adopt it.

    calibrate (rank 0 only; see PhotoColorizer): photos to measure the activation ranges on (H == W only: photos are
    prepared square; calibrate_maskcent is the mask centring the forwards will use), or a saved measurement.
    The measured storage exponents are part of the arena, so the other ranks receive them with the weights."""

    def __init__(self, H, W, per_rank_batch, state_dict=None, device=None, dist_head=False, calibrate=None,
                 calibrate_maskcent=0.0, **ctx_kw):
        from . import engine
        from .engine import LhnContext
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.rank = dist.get_rank() if dist.is_initialized() else 0
        self.device = torch.cuda.current_device() if device is None else device
        ranges = None
        if self.rank == 0 and calibrate is not None:
            if H != W and not isinstance(calibrate, (dict, str, bytes)):
                raise ValueError("calibrate=[photos] needs a square geometry, got %dx%d: measure at a square size with "
                                 "engine.measure_act_ranges and pass the ranges (they do not depend on the size)" % (H, W))
            flags = {k: v for k, v in ctx_kw.items() if k in ("global_hints", "caffe313", "keep_conv10", "options")}
            ranges = engine.resolve_calibration(calibrate, lambda photos: engine.measure_act_ranges(
                state_dict, engine.calibration_batch(photos, H, device=self.device,
                                                     global_hints=flags.get("global_hints", False)),
                H, W, device=self.device, maskcent=float(calibrate_maskcent), **flags))
        self.ctx = LhnContext(device=self.device, max_n=per_rank_batch, H=H, W=W, dist=dist_head, **ctx_kw)
        if self.world == 1:
            self.ctx.load_state_dict(state_dict, act_ranges=ranges)
            return
        if self.rank == 0:
            if state_dict is None:
                raise ValueError("rank 0 needs the state_dict")
            self.ctx.load_state_dict(state_dict, act_ranges=ranges)
        else:
            self.ctx.reserve_weights()
        ptr, nbytes = self.ctx.weights_arena()
        blob = torch.as_tensor(_DevBlob(ptr, nbytes), device="cuda:%d" % self.device)
        broadcast_blob(blob, src=0)                     # the only collective of the whole job
        torch.cuda.synchronize(self.device)
        if self.rank != 0:
            self.ctx.adopt_weights()
        self.arena_bytes = nbytes

    def local_slice(self, n_total):
        return shard_range(n_total, self.world, self.rank)

    def forward(self, L_mc, ab, mask, maskcent=0.0, **kw):
        """Rank-local images only (device tensors)."""
        return self.ctx.forward_device(L_mc, ab, mask, maskcent, **kw)
