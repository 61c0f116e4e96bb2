"""Photos/s of PhotoColorizer sharded over a job of ranks against one process: the colorize leg on in-memory arrays and
on PNG files, and the reveal-sweep leg, at world 1 and world N.

    python tools/photo_shard_profile.py --out DIR [--world 2] [--photos 256] [--Xd 256] [--batch 32]

The tool starts its ranks itself (spawned processes, a fresh process group per world size) and joins them all before
it returns.  On a node with fewer GPUs than --world every rank shares device 0 over gloo (ranks time-slice the GPU);
otherwise each rank has its own GPU and the group is NCCL.  Each leg follows one untimed warm-up pass of the same
photos on every rank; a rank's time is host wall time from a barrier to its last result, and a leg's rate is the job's
photos over the slowest rank's time.  Every rank's time is reported, since static shards of ragged work can leave ranks
uneven.  The card's name, power limit and maximum SM clock are read in the same run and written with the numbers to
DIR/photo_shard_profile.json.
"""
import argparse
import json
import os
import socket
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.reveal_sweep_profile import card, photo  # noqa: E402

LEVELS = (0, 1, 2, 5, 10, 20, 50)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _rank(rank, world, port, backend, a, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch
    import torch.distributed as dist
    from interactive_deep_colorization_b200 import photos
    from oracle import synth
    device = rank if backend == "nccl" else 0
    torch.cuda.set_device(device)
    dist.init_process_group(backend, rank=rank, world_size=world)
    try:
        imgs = [photo(100 + i) for i in range(a.photos)]
        paths = [os.path.join(a.png_dir, "p%04d.png" % i) for i in range(a.photos)]
        pc = photos.PhotoColorizer(synth.torch_state_dict(1234) if rank == 0 else None, Xd=a.Xd, batch=a.batch,
                                   device=device)
        legs = {"colorize_arrays": lambda: sum(1 for _ in pc.colorize(imgs)),
                "colorize_png": lambda: sum(1 for _ in pc.colorize(paths)),
                "reveal_sweep": lambda: sum(1 for _ in pc.reveal_sweep(imgs, levels=LEVELS))}
        out = {}
        for name, leg in legs.items():
            leg()                                      # warm-up
            dist.barrier()
            t0 = time.perf_counter()
            count = leg()
            torch.cuda.synchronize(device)
            out[name] = (count, time.perf_counter() - t0)
        pc.close()
        q.put((rank, out))
    except BaseException as e:
        q.put((rank, "%s: %s" % (type(e).__name__, e)))
        raise
    finally:
        dist.destroy_process_group()


def run_world(world, a):
    """Every leg at one world size -> {leg: {"photos_per_s", "rank_seconds", "rank_photos"}}, backend."""
    import torch
    import torch.multiprocessing as mp
    backend = "nccl" if world > 1 and torch.cuda.device_count() >= world else "gloo"
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank, args=(r, world, port, backend, a, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    try:
        for _ in procs:
            r, v = q.get(timeout=3600)
            got[r] = v
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    bad = {r: v for r, v in got.items() if isinstance(v, str)}
    if bad or len(got) != world:
        raise RuntimeError("world %d failed: %s" % (world, bad or "a rank never reported"))
    res = {}
    for leg in got[0]:
        secs = [got[r][leg][1] for r in range(world)]
        res[leg] = {"photos_per_s": a.photos / max(secs), "rank_seconds": secs,
                    "rank_photos": [got[r][leg][0] for r in range(world)]}
    return res, backend


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--photos", type=int, default=256)
    ap.add_argument("--Xd", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    a = ap.parse_args()
    import cv2
    os.makedirs(a.out, exist_ok=True)
    a.png_dir = os.path.join(a.out, "png")
    os.makedirs(a.png_dir, exist_ok=True)
    for i in range(a.photos):
        cv2.imwrite(os.path.join(a.png_dir, "p%04d.png" % i), photo(100 + i)[:, :, ::-1])
    name, limits = card()
    report = {"card": name, "power.limit,clocks.max.sm": limits, "photos": a.photos, "photo": "375x500",
              "Xd": a.Xd, "batch": a.batch, "reveal_levels": LEVELS, "worlds": {}}
    for world in (1, a.world):
        res, backend = run_world(world, a)
        report["worlds"][str(world)] = {"backend": backend, "legs": res}
        for leg, r in res.items():
            print("world %d (%s) %-16s %8.1f photos/s  rank seconds %s" % (
                world, backend, leg, r["photos_per_s"], ", ".join("%.3f" % s for s in r["rank_seconds"])))
    for f in os.listdir(a.png_dir):
        os.remove(os.path.join(a.png_dir, f))
    os.rmdir(a.png_dir)
    with open(os.path.join(a.out, "photo_shard_profile.json"), "w") as f:
        json.dump(report, f, indent=1)
    print("%s, %s" % (name, limits))


if __name__ == "__main__":
    main()
