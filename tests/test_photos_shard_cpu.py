"""CPU: PhotoColorizer and the folder mode of ideepcolor_b200.py as shards of a job, on fake devices (the
_make_backend seam) in spawned gloo process groups of world size 2 and 3.  Every rank takes its contiguous slice, the
hints, glob vectors and query points follow their photos, the reveal points keep their global index, rank 0's merged
CSVs are byte-identical to one process's, and a failure on any rank (rank 0's checks, arguments that differ, a photo
that fails to read) makes every rank raise instead of waiting.  Every process is joined with a timeout."""
import os
import queue
import socket
import traceback

import numpy as np
import pytest

from interactive_deep_colorization_b200 import photos
from interactive_deep_colorization_b200.colorize_image import HINT_LIST_DTYPE
from interactive_deep_colorization_b200.parallel import shard_range

N, X = 11, 64


class FakeDevice(object):
    """Each result carries what the device was given for its photo: the tag of the photo (its first pixel), its hint
    count, its glob vector's first value and its points."""

    def __init__(self):
        self.pending = 0

    def _take(self, token):
        self.pending -= 1
        return token

    def submit(self, imgs, hints, glob, psnr, points=None, K=0):
        self.pending += 1
        return imgs, hints, glob, psnr, points

    def collect(self, token):
        imgs, hints, glob, psnr, points = self._take(token)
        out = []
        for k, a in enumerate(imgs):
            tag = int(a[0, 0, 0])
            r = photos.PhotoResult(a, tag, None if hints is None or hints[k] is None else len(hints[k]),
                                   tag + 0.1 if glob is None else float(glob[k][0]))
            out.append(r if points is None else photos.SuggestResult(r, points[k], None))
        return out

    def submit_reveal(self, imgs, points, levels):
        self.pending += 1
        return imgs, points, levels

    def collect_reveal(self, token):
        imgs, points, levels = self._take(token)
        return [photos.RevealResult(int(a[0, 0, 0]) + np.arange(len(levels)) / 7., None, int(a[0, 0, 0]), p)
                for a, p in zip(imgs, points)]

    def submit_glob(self, imgs, conditions):
        self.pending += 1
        return imgs, conditions

    def collect_glob(self, token):
        imgs, conds = self._take(token)
        return [photos.GlobalSweepResult(int(a[0, 0, 0]) + np.arange(len(conds)) / 3., None, None, None) for a in imgs]

    def discard(self, token):
        self.pending -= 1

    def close(self):
        assert self.pending == 0


class FakeColorizer(photos.PhotoColorizer):
    def _make_backend(self, state_dict):
        return FakeDevice()


def _img(tag, h=6, w=9):
    a = np.zeros((h, w, 3), np.uint8)
    a[0, 0, 0] = tag
    a[1:, 1:] = (37 * tag) % 251
    return a


def _job_lists():
    imgs = [_img(i) for i in range(N)]
    hints = [None if i % 4 == 0 else np.zeros(i, HINT_LIST_DTYPE) for i in range(N)]
    glob = [np.full(316, i + 0.5, np.float32) for i in range(N)]
    points = [np.full((i % 3, 2), i, np.int64) for i in range(N)]
    return imgs, hints, glob, points


# ---- what the ranks run ----------------------------------------------------------------------------------------------

def _shard_passes(rank, world, arg):
    imgs, hints, glob, points = _job_lists()
    pc = FakeColorizer(None, Xd=X, batch=3, global_hints=True)
    out = {"slice": pc.local_slice(N),
           "colorize": [(r.rgb, r.ab, r.psnr) for r in pc.colorize(imgs, hints=hints, glob=glob)],
           "reveal": [(r.rgb, r.points) for r in pc.reveal_sweep(imgs, levels=(0, 2, 4), seed=5)]}
    pc.close()
    pc = FakeColorizer(None, Xd=X, batch=3, suggest=True)
    out["suggest"] = [(r.result.rgb, r.result.ab, r.centers) for r in pc.suggest(imgs, hints, points)]
    pc.close()
    return out


def _rank0_error(rank, world, arg):
    # rank 0's checkpoint lacks the 313-bin head; the other ranks have no checkpoint to check
    FakeColorizer({} if rank == 0 else None, Xd=X, batch=4, caffe=True, caffe_dist=True)


def _argument_mismatch(rank, world, arg):
    FakeColorizer({}, Xd=X, batch=5 if rank == 1 else 4)


def _cli(rank, world, arg):
    import ideepcolor_b200
    photos.PhotoColorizer = FakeColorizer
    return ideepcolor_b200.main(arg)


JOBS = {"passes": _shard_passes, "rank0_error": _rank0_error, "mismatch": _argument_mismatch, "cli": _cli}


def _worker(rank, world, port, job, arg, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch.distributed as dist
    own_group = job != "cli"                  # the folder mode makes its own process group
    if own_group:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        q.put((rank, "ok", JOBS[job](rank, world, arg)))
    except BaseException as e:
        q.put((rank, "raised", "%s: %s" % (type(e).__name__, e)))
        traceback.print_exc()
    finally:
        if own_group:
            dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _run(world, job, arg=None, timeout=120):
    """Spawn `world` ranks running JOBS[job] -> [(status, value)] by rank; every process is joined (and killed if it
    outlives the timeout, which fails the test)."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, job, arg, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    try:
        for _ in procs:
            rank, status, value = q.get(timeout=timeout)
            got[rank] = (status, value)
    except queue.Empty:
        pass
    finally:
        for p in procs:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
                p.join()
    assert sorted(got) == list(range(world)), "ranks %s never finished" % sorted(set(range(world)) - set(got))
    return [got[r] for r in range(world)]


# ---- tests ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("world", [2, 3])
def test_shards_cover_every_photo_once_with_their_inputs(world):
    res = _run(world, "passes")
    assert all(s == "ok" for s, _ in res), res
    outs = [v for _, v in res]
    assert [o["slice"] for o in outs] == [shard_range(N, world, r) for r in range(world)]
    imgs, hints, glob, points = _job_lists()
    tags = sum(([t for t, _, _ in o["colorize"]] for o in outs), [])
    assert tags == list(range(N))                                  # every photo once, in order, rank after rank
    for o in outs:
        start, count = o["slice"]
        assert [t for t, _, _ in o["colorize"]] == list(range(start, start + count))
    # the hints and glob vectors of photo i travel with photo i
    assert [h for o in outs for _, h, _ in o["colorize"]] == [None if h is None else len(h) for h in hints]
    assert [g for o in outs for _, _, g in o["colorize"]] == [float(g[0]) for g in glob]
    sug = [r for o in outs for r in o["suggest"]]
    assert [t for t, _, _ in sug] == list(range(N))
    assert all(np.array_equal(c, points[i]) for i, (_, _, c) in enumerate(sug))
    # reveal points use the photo's index in the whole job, so the sweep does not depend on the world size
    rev = [r for o in outs for r in o["reveal"]]
    assert [t for t, _ in rev] == list(range(N))
    for i, (_, p) in enumerate(rev):
        assert np.array_equal(p, photos.reveal_points(X, 4, 5, i)), i


def _folder(tmp_path, bad=None):
    cv2 = pytest.importorskip("cv2")
    import torch
    d = tmp_path / "in"
    d.mkdir()
    for i in range(N):
        p = d / ("img%02d.png" % i)
        if i == bad:
            p.write_bytes(b"not a png")
        else:
            cv2.imwrite(str(p), _img(i)[:, :, ::-1])
    torch.save({}, str(tmp_path / "m.pth"))
    return d


def _cli_args(tmp_path, d, out, *extra):
    return ["--color_model", str(tmp_path / "m.pth"), "--image_dir", str(d), "--out", str(out), "--load_size", str(X),
            "--batch", "4", "--dist_backend", "gloo"] + list(extra)


def _files(d):
    return {f: (d / f).read_bytes() for f in sorted(os.listdir(str(d)))}


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("extra", [["--psnr"], ["--reveal_sweep", "0,1,5"], ["--global_hints", "--glob_sweep"]],
                         ids=["psnr", "reveal", "glob"])
def test_merged_csvs_equal_one_process(tmp_path, monkeypatch, capsys, world, extra):
    import ideepcolor_b200
    d = _folder(tmp_path)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setattr(photos, "PhotoColorizer", FakeColorizer)
    assert ideepcolor_b200.main(_cli_args(tmp_path, d, tmp_path / "one", *extra)) == 0
    one = capsys.readouterr().out
    res = _run(world, "cli", _cli_args(tmp_path, d, tmp_path / "many", *extra))
    assert res == [("ok", 0)] * world
    a, b = _files(tmp_path / "one"), _files(tmp_path / "many")
    assert sorted(a) == sorted(b) and any(f.endswith(".csv") for f in a)
    for f in a:
        assert a[f] == b[f], f
    assert one                                          # what one process prints, rank 0 prints (GPU test)


def test_rank0_check_fails_every_rank():
    res = _run(3, "rank0_error")
    assert [s for s, _ in res] == ["raised"] * 3
    msgs = [v for _, v in res]
    assert msgs[0].startswith("ValueError: caffe_dist=True needs the checkpoint's 313-bin head")
    assert msgs[1] == msgs[2] == "ValueError: rank 0 failed: " + msgs[0]


@pytest.mark.parametrize("world", [2, 3])
def test_argument_mismatch_fails_every_rank(world):
    res = _run(world, "mismatch")
    assert [s for s, _ in res] == ["raised"] * world
    for _, msg in res:
        assert msg.startswith("ValueError: rank 1 was given") and "'batch': 5" in msg and "'batch': 4" in msg


def test_photo_that_fails_to_read_on_rank1_fails_every_rank(tmp_path):
    d = _folder(tmp_path, bad=8)                       # rank 1 of 2 colours photos 6 .. 10
    res = _run(2, "cli", _cli_args(tmp_path, d, tmp_path / "out", "--psnr"))
    assert res == [("ok", 1), ("ok", 1)]
    assert not (tmp_path / "out" / "psnr.csv").exists()


def test_image_file_refused_under_torchrun(monkeypatch, capsys):
    import ideepcolor_b200
    monkeypatch.setenv("WORLD_SIZE", "2")
    assert ideepcolor_b200.main(["--color_model", "m.pth", "--image_file", "x.png"]) == 2
    assert "--image_dir" in capsys.readouterr().out


def test_no_process_group_is_one_shard():
    pc = FakeColorizer(None, Xd=X, batch=3)
    assert (pc.world, pc.rank) == (1, 0) and pc.local_slice(N) == (0, N)
    assert [r.rgb for r in pc.colorize([_img(i) for i in range(5)])] == list(range(5))
    pc.close()
