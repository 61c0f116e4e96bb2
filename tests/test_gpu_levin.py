"""GPU: the Levin baseline of reveal sweeps (idc_levin_weights, idc_levin_solve, idc_lab2rgb_u8_mc and
PhotoColorizer.reveal_sweep(method="levin")) against the float64 oracle of tests/levin_ref.py, against direct calls on
numpy-painted planes, and across runs, batch sizes, positions and ranks."""
import os
import pickle
import sys
import traceback

import cv2
import numpy as np
import pytest
import torch

from interactive_deep_colorization_b200 import _lib, photos
from oracle import synth
from tests import levin_ref
from tests.test_gpu_photos_shard import _equal, _files, _free_port, _spawn
from tests.test_gpu_reveal import _paint, _photo, _single, SIZES

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL_AB = 1e-4
# test_gpu_reveal's photo sizes without the one-pixel-wide ones: stretched to X x X, every row (or column) of those is
# the same, the weights across them can fall to ~1e-200 without reaching 0, and the system is too close to singular for
# BiCGSTAB in FP64 to converge (DESIGN.md §11); the sweep raises for them, as test_non_convergence shows with max_iter
SOLVE_SIZES = [s for s in SIZES if min(s) > 1]


def _st():
    return torch.cuda.current_stream().cuda_stream


def _edges_photo(H, W=None):
    """Flat regions with hard edges between them, and one ramp: H x W (H x H by default)."""
    W = H if W is None else W
    a = np.zeros((H, W, 3), np.uint8)
    a[:, :W // 2] = (20, 40, 200)
    a[:, W // 2:] = (240, 230, 30)
    a[H // 2:, :W // 3] = (128, 128, 128)
    a[:H // 3, W // 2:, 0] = np.linspace(120, 250, W - W // 2).astype(np.uint8)
    return a


def _labs(X):
    """The Lab of the network-size photos: four of test_gpu_reveal's ragged photos and the hard-edge image."""
    imgs = [_photo(h, w, 30 + i) for i, (h, w) in enumerate(SIZES[:4])] + [_edges_photo(300)]
    return [_single(a, X) for a in imgs]


def _solve_labs(X):
    imgs = [_photo(h, w, 30 + i) for i, (h, w) in enumerate(SOLVE_SIZES[:4])] + [_edges_photo(300)]
    return [_single(a, X) for a in imgs]


def _weights(labs):
    """idc_levin_weights of Lab planes [n,3,X,X] float64 (host) -> [n,8,X,X] float64 (host)."""
    lab = torch.from_numpy(np.ascontiguousarray(np.stack(labs))).cuda()
    n, _, h, w = lab.shape
    wts = torch.empty((n, 8, h, w), dtype=torch.float64, device="cuda")
    assert _lib.load().idc_levin_weights(0, n, h, w, lab.data_ptr(), wts.data_ptr(), _st()) == 0
    return wts


def _solve(wts, ab, mask, levels, tol=photos.LEVIN_TOL, max_iter=photos.LEVIN_MAX_ITER):
    """idc_levin_solve on device weights and host planes ab [n,2,h,w], mask [n,1,h,w] -> (ab float32, iters, relres)."""
    lib = _lib.load()
    n, _, h, w = ab.shape
    d_ab, d_mask = (torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in (ab, mask))
    out = torch.empty((n, 2, h, w), device="cuda")
    iters = torch.empty((n, 2), dtype=torch.int32, device="cuda")
    relres = torch.empty((n, 2), dtype=torch.float64, device="cuda")
    nbytes = lib.idc_levin_workspace_bytes(n, h, w)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    assert lib.idc_levin_solve(0, n, levels, h, w, wts.data_ptr(), d_ab.data_ptr(), d_mask.data_ptr(), tol, max_iter,
                               out.data_ptr(), iters.data_ptr(), relres.data_ptr(), ws.data_ptr(), nbytes, _st()) == 0
    return out.cpu().numpy(), iters.cpu().numpy(), relres.cpu().numpy()


def _render(L_mc, ab):
    """idc_lab2rgb_u8_mc of host L_mc [n,1,X,X] and ab [n,2,X,X] -> uint8 [n,X,X,3]."""
    n, _, h, w = ab.shape
    dL, dab = (torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in (L_mc, ab))
    rgb = torch.empty((n, h, w, 3), dtype=torch.uint8, device="cuda")
    assert _lib.load().idc_lab2rgb_u8_mc(0, n, h, w, dL.data_ptr(), dab.data_ptr(), rgb.data_ptr(), _st()) == 0
    return rgb.cpu().numpy()


@pytest.mark.parametrize("X", [64, 256])
def test_weights_equal_the_oracle(X):
    labs = [lab for _, _, lab in _labs(X)]
    got = _weights(labs).cpu().numpy()
    for i, lab in enumerate(labs):
        want = levin_ref.weights(lab[0])
        tiny = (np.abs(want) < 1e-290) & (np.abs(got[i]) < 1e-290)        # at the edge of float64's range
        bad = ~tiny & (np.abs(got[i] - want) > 1e-13 * np.abs(want))
        assert not bad.any(), (i, np.argwhere(bad)[:5])
        assert ((got[i] == 0) == (want == 0)).mean() > 0.999
    assert (got[-1] == 0).any()                          # neighbours outside the image weigh 0


REPORT = []


@pytest.mark.parametrize("X", [32, 64, 256])
def test_solve_equals_the_direct_solve(X):
    """1, 5, 50 and 500 revealed points on every photo, against spsolve on the pixels that reach a hint."""
    labs = [lab for _, _, lab in _solve_labs(X)]
    wts = _weights(labs)
    w_host = wts.cpu().numpy()
    counts = (1, 5, 50, 500)
    ab, mask = [], []
    for i, lab in enumerate(labs):
        pts = photos.reveal_points(X, max(counts), 11, i)
        for m in counts:
            a, k, _ = _paint(lab, pts[:m])
            ab.append(a)
            mask.append(k)
    ab, mask = np.stack(ab), np.stack(mask)
    got, iters, relres = _solve(wts, ab, mask, len(counts))
    bad = ~(relres <= photos.LEVIN_TOL)
    assert not bad.any(), (np.argwhere(bad).tolist(), iters[bad].tolist(), relres[bad].tolist())
    worst = 0.0
    for j in range(len(ab)):
        want = levin_ref.solve(w_host[j // len(counts)], ab[j], mask[j, 0])
        worst = max(worst, float(np.abs(got[j] - want).max()))
        assert np.abs(got[j] - want).max() <= TOL_AB, (j, np.abs(got[j] - want).max())
        assert np.array_equal(got[j][:, mask[j, 0] > 0], ab[j][:, mask[j, 0] > 0])
    it = iters.reshape(len(labs), len(counts), 2)
    REPORT.append((X, worst, {m: (int(np.median(it[:, k])), int(it[:, k].max())) for k, m in enumerate(counts)}))
    print("levin solve X=%d: max |d ab| = %.3g, iterations (median, max) per hint count %s"
          % (X, worst, REPORT[-1][2]))


def test_closed_set_and_level_zero_are_exact_zeros():
    w = np.zeros((8, 4, 4))
    k = {o: i for i, o in enumerate(levin_ref.OFFSETS)}
    w[k[(0, 1)], 0, 0] = w[k[(0, -1)], 0, 1] = 1.0                # (0, 0) and (0, 1) point only at each other
    for y in range(4):
        for x in range(4):
            if y == 0 and x < 2:
                continue
            nbs = [o for o in ((0, -1), (0, 1), (1, 0), (-1, 0)) if 0 <= y + o[0] < 4 and 0 <= x + o[1] < 4
                   and not (y + o[0] == 0 and x + o[1] < 2)]
            for o in nbs:
                w[k[o], y, x] = 1.0 / len(nbs)
    wts = torch.from_numpy(np.stack([w, w])).cuda()
    ab = np.zeros((2, 2, 4, 4), np.float32)
    mask = np.zeros((2, 1, 4, 4), np.float32)
    ab[0, :, 3, 3], mask[0, 0, 3, 3] = (12.0, -7.0), 1
    ab[1] = 5.0                                           # level 0: colours without a mask are not hints
    got, iters, relres = _solve(wts, ab, mask, 1)
    assert (got[0, :, 0, :2] == 0).all() and (got[1] == 0).all()
    assert iters[1].tolist() == [0, 0] and relres[1].tolist() == [0.0, 0.0]
    want = levin_ref.solve(w, ab[0], mask[0, 0])
    assert np.abs(got[0] - want).max() <= TOL_AB


@pytest.fixture(scope="module")
def sd():
    return synth.torch_state_dict(1234)


@pytest.mark.parametrize("X", [64, 256])
def test_sweep_equals_direct_calls_and_render_matches_the_network(sd, X):
    imgs = [_photo(h, w, 30 + i) for i, (h, w) in enumerate(SOLVE_SIZES[:4])] + [_edges_photo(300)]
    levels = (0, 1, 5, 50)
    pc = photos.PhotoColorizer(sd, Xd=X, batch=8)
    lev = list(pc.reveal_sweep(imgs, levels=levels, seed=4, method="levin"))
    net = list(pc.reveal_sweep(imgs, levels=levels, seed=4))
    pc.close()
    for i, (a, r, n) in enumerate(zip(imgs, lev, net)):
        L_mc, small, lab = _single(a, X)
        assert np.array_equal(r.points, n.points)
        planes = [_paint(lab, r.points[:m]) for m in levels]
        ab = np.stack([p[0] for p in planes])
        mask = np.stack([p[1] for p in planes])
        want_ab, _, _ = _solve(_weights([lab]), ab, mask, len(levels))
        assert np.array_equal(r.ab, want_ab), i
        want_rgb = _render(np.repeat(L_mc[None], len(levels), 0), want_ab)
        assert np.array_equal(r.rgb, want_rgb), i
        sse = ((small[None].astype(np.int64) - want_rgb) ** 2).reshape(len(levels), -1).sum(1)
        assert r.psnr.tolist() == [photos._psnr(e, X) for e in sse]
        # the network's own ab through the baseline's render is its output_rgb
        assert np.array_equal(_render(np.repeat(L_mc[None], len(levels), 0), n.ab), n.rgb), i
        assert (r.ab[0] == 0).all()                       # level 0
        assert r.psnr[-1] > r.psnr[0]


def test_sweep_is_deterministic_across_runs_batches_and_positions(sd):
    imgs = [_photo(h, w, 60 + i) for i, (h, w) in enumerate(SOLVE_SIZES)] + [_edges_photo(200), _photo(300, 200, 9)]
    levels = (0, 2, 20)
    runs = []
    for batch, order in ((3, range(7)), (21, range(7)), (12, range(6, -1, -1)), (3, range(7))):
        pc = photos.PhotoColorizer(sd, Xd=64, batch=batch)
        got = list(pc.reveal_sweep([imgs[i] for i in order], levels=levels, seed=0, method="levin"))
        pc.close()
        # the points depend on the position in `photos`: keep the photo's own by giving each its own run below
        runs.append({i: r for i, r in zip(order, got)})
    for i in range(7):
        assert _equal(tuple(runs[0][i]), tuple(runs[1][i])) and _equal(tuple(runs[0][i]), tuple(runs[3][i]))
    # reversed order: photo i sits at position 6 - i and so gets other points; equal to a run with those points
    pc = photos.PhotoColorizer(sd, Xd=64, batch=3)
    single = [list(pc.reveal_sweep([imgs[6 - j] for j in range(k + 1)], levels=levels, seed=0, method="levin"))[-1]
              for k in (0, 3, 6)]
    pc.close()
    for k, r in zip((0, 3, 6), single):
        assert _equal(tuple(runs[2][6 - k]), tuple(r))


def test_non_convergence_names_photo_and_level(sd):
    imgs = [_photo(h, w, 80 + i) for i, (h, w) in enumerate(SOLVE_SIZES[:3])]
    pc = photos.PhotoColorizer(sd, Xd=64, batch=6)
    with pytest.raises(RuntimeError, match=r"photo 0, level 5 did not converge"):
        list(pc.reveal_sweep(imgs, levels=(0, 5), seed=1, method="levin", levin_max_iter=1))
    # the colorizer stays usable
    assert len(list(pc.reveal_sweep(imgs, levels=(0, 5), seed=1, method="levin"))) == 3
    pc.close()


N, BATCH, X_SHARD, WORLD = 7, 4, 64, 2


def _shard_inputs():
    rs = np.random.RandomState(9)
    return [_photo(int(rs.randint(24, 300)), int(rs.randint(24, 300)), 700 + i) for i in range(N)]


def _rank_main(rank, port, result):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    try:
        pc = photos.PhotoColorizer(synth.torch_state_dict(1234) if rank == 0 else None, Xd=X_SHARD, batch=BATCH)
        out = list(pc.reveal_sweep(_shard_inputs(), levels=(0, 1, 5), seed=3, method="levin"))
        pc.close()
        with open(result, "wb") as f:
            pickle.dump(out, f)
    except BaseException:
        with open(result + ".err", "w") as f:
            f.write(traceback.format_exc())
        raise
    finally:
        dist.destroy_process_group()


def test_two_ranks_equal_one_process(tmp_path, sd):
    res = [str(tmp_path / ("rank%d.pkl" % r)) for r in range(WORLD)]
    port = _free_port()
    codes = _spawn(_rank_main, lambda r: (r, port, res[r]))
    for r in res:
        if os.path.exists(r + ".err"):
            print(open(r + ".err").read())
    assert codes == [0] * WORLD
    got = []
    for r in res:
        with open(r, "rb") as f:
            got += pickle.load(f)
    pc = photos.PhotoColorizer(sd, Xd=X_SHARD, batch=BATCH)
    want = list(pc.reveal_sweep(_shard_inputs(), levels=(0, 1, 5), seed=3, method="levin"))
    pc.close()
    assert len(got) == len(want) == N
    for g, w in zip(got, want):
        assert _equal(tuple(g), tuple(w))


def test_command_line_two_ranks_write_the_same_csvs(tmp_path):
    import subprocess
    folder = str(tmp_path)
    torch.save(synth.torch_state_dict(1234), os.path.join(folder, "m.pth"))
    os.mkdir(os.path.join(folder, "photos"))
    for i, a in enumerate(_shard_inputs()):
        cv2.imwrite(os.path.join(folder, "photos", "img%02d.png" % i), a[:, :, ::-1])
    base = [sys.executable, os.path.join(ROOT, "ideepcolor_b200.py"), "--color_model", os.path.join(folder, "m.pth"),
            "--image_dir", os.path.join(folder, "photos"), "--load_size", str(X_SHARD), "--batch", str(BATCH),
            "--reveal_sweep", "0,1,5", "--reveal_levin"]
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    one = subprocess.run(base + ["--out", os.path.join(folder, "one")], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=900)
    assert one.returncode == 0, one.stdout + one.stderr
    port = str(_free_port())
    procs = [subprocess.Popen(base + ["--out", os.path.join(folder, "two"), "--dist_backend", "gloo"], cwd=ROOT,
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
    assert sorted(a) == ["reveal_psnr.csv", "reveal_psnr_levin.csv"] and a == b
