"""Multi-GPU: one process per GPU, images sharded across ranks, ONE broadcast of the packed
weight arena at init, no per-step collective (SURVEY.md 8e -- images are independent: the
network has no cross-image state, BatchNorm runs in eval mode,
/root/reference/data/colorize_image.py:232).  Before the broadcast the ranks agree (agree) that
every one of them is ready for it, so a rank that fails makes all of them raise instead of wait.
ShardedColorizer (device tensors) and photos.PhotoColorizer (photo batches and sweeps) both
get their context from share_weights.

Host logic here is backend-agnostic (`gloo` on CPU in the tests, `nccl` over NVLink on the box).
"""
import contextlib

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


def world_rank():
    """(world size, rank) of the default process group; (1, 0) when there is none."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(), dist.get_rank()
    return 1, 0


def _object_device(device):
    """NCCL's object collectives stage through the current CUDA device: make it this rank's for their duration."""
    if dist.get_backend() == "nccl":
        return torch.cuda.device(device)
    return contextlib.nullcontext()


def agree(error, fingerprint=None, payload=None, device=0):
    """One all_gather_object of every rank's outcome so far, so that all ranks leave a set-up step together: either
    every rank goes on, or every rank raises.  error: the exception this rank met (None if none); fingerprint: what must
    be equal on every rank; payload: what rank 0 hands to every rank (-> the return value).
    Raises on every rank: the lowest failing rank's error (that rank re-raises its own exception, the others a
    ValueError with its text), else, when a rank's fingerprint differs from rank 0's, a ValueError naming both."""
    world, rank = world_rank()
    got = [None] * world
    with _object_device(device):
        dist.all_gather_object(got, (None if error is None else "%s: %s" % (type(error).__name__, error),
                                     fingerprint, payload))
    for r, (msg, _, _) in enumerate(got):
        if msg is not None:
            if r == rank:
                raise error
            raise ValueError("rank %d failed: %s" % (r, msg))
    for r, (_, fp, _) in enumerate(got):
        if fp != got[0][1]:
            raise ValueError("rank %d was given %r, rank 0 %r: every rank of a job needs the same arguments"
                             % (r, fp, got[0][1]))
    return got[0][2]


def share_weights(make_ctx, state_dict, act_ranges=None, device=0):
    """A context with the job's weights on every rank.  Without a process group (or world size 1) make_ctx() loads
    state_dict.  Otherwise rank 0 loads state_dict (act_ranges set its storage exponents, which the arena carries), the
    other ranks reserve_weights(), receive the packed arena with ONE broadcast and adopt_weights(); state_dict is needed
    on rank 0 only.  Whether every rank built its context is agreed first, so a rank that fails there makes every rank
    raise instead of leaving the others in the broadcast.  Over gloo the arena goes through a host byte tensor, which
    lets ranks share one GPU (NCCL refuses two ranks on one device)."""
    world, rank = world_rank()
    if world == 1:
        ctx = make_ctx()
        try:
            ctx.load_state_dict(state_dict, act_ranges=act_ranges)
        except BaseException:
            ctx.close()
            raise
        return ctx
    ctx, error = None, None
    try:
        ctx = make_ctx()
        if rank == 0:
            if state_dict is None:
                raise ValueError("rank 0 needs the state_dict")
            ctx.load_state_dict(state_dict, act_ranges=act_ranges)
        else:
            ctx.reserve_weights()
    except Exception as e:
        error = e
    try:
        agree(error, device=device)
        ptr, nbytes = ctx.weights_arena()
        blob = torch.as_tensor(_DevBlob(ptr, nbytes), device="cuda:%d" % device)
        if dist.get_backend() == "gloo":
            host = blob.cpu() if rank == 0 else torch.empty(nbytes, dtype=torch.uint8)
            broadcast_blob(host, src=0)
            if rank != 0:
                blob.copy_(host)
        else:
            broadcast_blob(blob, src=0)
        torch.cuda.synchronize(device)
        if rank != 0:
            ctx.adopt_weights()
    except BaseException:
        if ctx is not None:
            ctx.close()
        raise
    return ctx


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
        self.world, self.rank = world_rank()
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
        self.ctx = share_weights(lambda: LhnContext(device=self.device, max_n=per_rank_batch, H=H, W=W,
                                                    dist=dist_head, **ctx_kw), state_dict, ranges, self.device)
        if self.world > 1:
            self.arena_bytes = self.ctx.weights_arena()[1]

    def local_slice(self, n_total):
        return shard_range(n_total, self.world, self.rank)

    def forward(self, L_mc, ab, mask, maskcent=0.0, **kw):
        """Rank-local images only (device tensors)."""
        return self.ctx.forward_device(L_mc, ab, mask, maskcent, **kw)
