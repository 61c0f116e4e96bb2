"""GPU: PhotoColorizer and the folder mode of ideepcolor_b200.py sharded across two ranks (gloo, both on device 0),
against one process with the same arguments.  19 seeded ragged photos, part arrays and part PNG files, at batch = 4:
the shard boundary (photo 10) falls inside a batch of the single process and both ranks end on a partial batch.  The
ranks' results, concatenated in rank order, must equal the single process's bit for bit for every pass method, and
the folder mode must write byte-identical files."""
import json
import os
import pickle
import socket
import subprocess
import sys
import traceback

import cv2
import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import photos, prepost
from interactive_deep_colorization_b200 import colorize_image as CI
from oracle import caffe_spec, synth
from tests import util
from tests.test_gpu_photos import _photo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, BATCH, X, WORLD = 19, 4, 64, 2


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _inputs(folder):
    """The 19 photos (every third one a PNG file in `folder`), a hint list and query points per photo."""
    rs = np.random.RandomState(7)
    imgs, hints, points = [], [], []
    for i in range(N):
        a = _photo(int(rs.randint(24, 300)), int(rs.randint(24, 300)), 300 + i)
        if i % 3 == 1:
            p = os.path.join(folder, "p%02d.png" % i)
            cv2.imwrite(p, a[:, :, ::-1])
            a = p
        imgs.append(a)
        k = int(rs.randint(0, 6))
        locs = rs.randint(0, X, (k, 2))
        hints.append(None if k == 0 else CI.hints_from_points([(l, int(rs.randint(0, 3)), rs.uniform(-80, 80, 2))
                                                               for l in locs], X))
        points.append(np.concatenate([locs, rs.randint(0, X, (2, 2))]).astype(np.int64))
    return imgs, hints, points


def _state_dicts():
    """The checkpoints of the cases: the synthetic network, its Caffe-scaled global-hints model, and a Caffe checkpoint
    with the 313-bin head."""
    sd = synth.torch_state_dict(1234)
    glob = dict(sd)
    glob.update({k: torch.from_numpy(v) for k, v in caffe_spec.synthetic_glob_state_dict().items()})
    csd = util.caffe_scaled(sd)
    csd.update({k: torch.from_numpy(v) for k, v in caffe_spec.synthetic_caffe313_state_dict(
        pts_in_hull=prepost.pts_in_hull()).items()})
    return {"plain": sd, "glob": util.caffe_scaled(glob), "caffe": csd}


def _run_cases(sds, imgs, hints, points, rank):
    """Every pass method on this process's share -> {case: list of results} (and the calibrated context's exponents).
    sds: the checkpoints on rank 0, None elsewhere."""
    def pc(which, **kw):
        return photos.PhotoColorizer(sds[which] if sds else None, Xd=X, batch=BATCH, **kw)

    out = {}
    p = pc("plain")
    out["colorize"] = list(p.colorize(imgs, hints=hints, psnr=True))
    out["reveal"] = list(p.reveal_sweep(imgs, levels=(0, 1, 5), seed=3))
    p.close()
    p = pc("plain", suggest=True)
    out["suggest"] = list(p.suggest(imgs, hints, points, K=5, psnr=True))
    p.close()
    p = pc("glob", global_hints=True, caffe=True)
    out["stats"] = list(p.global_stats(imgs))
    out["glob_sweep"] = list(p.global_sweep(imgs))
    p.close()
    p = pc("caffe", caffe=True, caffe_dist=True)
    out["caffe_suggest"] = list(p.suggest(imgs, hints, points, K=5))
    p.close()
    p = pc("plain", calibrate=[a for a in imgs[:3]] if rank == 0 else None)
    out["calibrated"] = list(p.colorize(imgs, psnr=True))
    out["act_exponents"] = p._backend.ctx.act_exponents()
    p.close()
    return out


def _rank_main(rank, port, folder, result):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    try:
        imgs, hints, points = _inputs(folder)
        out = _run_cases(_state_dicts() if rank == 0 else None, imgs, hints, points, rank)
        with open(result, "wb") as f:
            pickle.dump(out, f)
    except BaseException:
        with open(result + ".err", "w") as f:
            f.write(traceback.format_exc())
        raise
    finally:
        dist.destroy_process_group()


def _spawn(target, args_of_rank, timeout=900):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=target, args=args_of_rank(r)) for r in range(WORLD)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(timeout=timeout)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    return [p.exitcode for p in procs]


def _equal(a, b):
    if isinstance(a, tuple):
        return type(a) is type(b) and len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    if a is None or isinstance(a, float):
        return a == b
    return isinstance(b, np.ndarray) and a.dtype == b.dtype and np.array_equal(a, b)


def test_two_ranks_equal_one_process(tmp_path):
    folder = str(tmp_path)
    port = _free_port()
    res = [os.path.join(folder, "rank%d.pkl" % r) for r in range(WORLD)]
    codes = _spawn(_rank_main, lambda r: (r, port, folder, res[r]))
    for r in range(WORLD):
        if os.path.exists(res[r] + ".err"):
            print(open(res[r] + ".err").read())
    assert codes == [0] * WORLD
    ranks = []
    for r in res:
        with open(r, "rb") as f:
            ranks.append(pickle.load(f))
    imgs, hints, points = _inputs(folder)
    one = _run_cases(_state_dicts(), imgs, hints, points, 0)
    assert [len(o["colorize"]) for o in ranks] == [10, 9]
    for case, want in one.items():
        if case == "act_exponents":
            assert ranks[1][case] == ranks[0][case] == want
            continue
        got = ranks[0][case] + ranks[1][case]
        assert len(got) == len(want) == N, case
        for i, (g, w) in enumerate(zip(got, want)):
            assert _equal(g, w), (case, i)


def _cli(folder, out, extra, env):
    return subprocess.run([sys.executable, os.path.join(ROOT, "ideepcolor_b200.py"), "--color_model",
                           os.path.join(folder, "m.pth"), "--image_dir", os.path.join(folder, "photos"), "--out", out,
                           "--load_size", str(X), "--batch", str(BATCH)] + extra,
                          cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)


def _files(d):
    return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}


@pytest.mark.parametrize("extra", [["--psnr"], ["--reveal_sweep", "0,1,5"], ["--hints_dir", "HDIR", "--suggest", "9"]],
                         ids=["psnr", "reveal", "suggest"])
def test_command_line_two_ranks_write_what_one_process_writes(tmp_path, extra):
    folder = str(tmp_path)
    torch.save(synth.torch_state_dict(1234), os.path.join(folder, "m.pth"))
    os.mkdir(os.path.join(folder, "photos"))
    os.mkdir(os.path.join(folder, "hints"))
    rs = np.random.RandomState(11)
    for i in range(N):
        cv2.imwrite(os.path.join(folder, "photos", "img%02d.png" % i),
                    _photo(int(rs.randint(24, 200)), int(rs.randint(24, 200)), 500 + i)[:, :, ::-1])
        if i % 2:
            hl = [{"loc": [int(v) for v in rs.randint(0, X, 2)], "size": int(rs.randint(0, 3)),
                   "ab": [float(v) for v in rs.uniform(-80, 80, 2)]} for _ in range(int(rs.randint(1, 5)))]
            with open(os.path.join(folder, "hints", "img%02d.json" % i), "w") as f:
                json.dump(hl, f)
    extra = [os.path.join(folder, "hints") if e == "HDIR" else e for e in extra]
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    one = _cli(folder, os.path.join(folder, "one"), extra, env)
    assert one.returncode == 0, one.stdout + one.stderr
    port = str(_free_port())
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "ideepcolor_b200.py"), "--color_model",
                               os.path.join(folder, "m.pth"), "--image_dir", os.path.join(folder, "photos"), "--out",
                               os.path.join(folder, "two"), "--load_size", str(X), "--batch", str(BATCH),
                               "--dist_backend", "gloo"] + extra, cwd=ROOT,
                              env=dict(env, RANK=str(r), LOCAL_RANK="0", WORLD_SIZE=str(WORLD), LOCAL_WORLD_SIZE="2",
                                       MASTER_ADDR="127.0.0.1", MASTER_PORT=port),
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(WORLD)]
    logs = []
    try:
        for p in procs:
            logs.append(p.communicate(timeout=900))
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    assert [p.returncode for p in procs] == [0, 0], "\n".join(o + e for o, e in logs)
    a, b = _files(os.path.join(folder, "one")), _files(os.path.join(folder, "two"))
    assert sorted(a) == sorted(b)
    for f in a:
        assert a[f] == b[f], f
    # what one process prints (the mean rows of a sweep) comes from rank 0 alone
    assert logs[0][0] == one.stdout.replace(os.path.join(folder, "one"), os.path.join(folder, "two"))
    assert logs[1][0] == ""
