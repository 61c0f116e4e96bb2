#!/usr/bin/env python
"""Generate the golden vectors in tests/golden/ by running the UNMODIFIED reference
(a checkout imported read-only through oracle/ref_shims.py) with the seeded
synthetic state_dict of oracle/synth.py.  Run where the reference checkout is available:

    python tests/golden/make_golden.py

Outputs (committed):
    lhn_256.npz     configs 1-2 + notebook KAT on test_imgs/mortar_pestle.jpg @256
    lhn_dist_256.npz  ColorizeImageTorchDist sample (config 5 semantics)
    lhn_64.npz      small synthetic case incl. per-layer checksums (fast CPU check)

Every file stays below 1 MB: the 256x256 outputs of lhn_256.npz are stored at a fixed, seeded sample of
PIX_COUNT pixels (flat indices in `pix_idx`; inputs img_rgb / img_l_mc stay whole), and the 529-bin distributions of
lhn_64.npz at a seeded sample of DIST_BINS bins (`dist16_bins`).
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import synth, ref_shims  # noqa: E402

SEED = 1234
PIX_COUNT = 16384                # of the 65536 pixels of a 256x256 output: every output-parity class is represented
DIST_BINS = 64                   # of the 529 distribution bins


def pix_idx():
    return np.sort(np.random.RandomState(256).choice(256 * 256, PIX_COUNT, replace=False)).astype(np.int32)


def dist_bins():
    return np.sort(np.random.RandomState(529).choice(529, DIST_BINS, replace=False)).astype(np.int32)


def sample_256(key, a, idx):
    """[C, 256, 256] -> [C, PIX_COUNT]; [256, 256, 3] (RGB) -> [PIX_COUNT, 3]; anything else unchanged."""
    if key in ("img_rgb", "img_l_mc") or a.ndim != 3:
        return a
    if a.shape[:2] == (256, 256):
        return a.reshape(256 * 256, a.shape[2])[idx]
    if a.shape[1:] == (256, 256):
        return a.reshape(a.shape[0], 256 * 256)[:, idx]
    return a


def sample_64(key, a, bins):
    return a[bins] if key.startswith("dist16_") and key != "dist16_bins" else a


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    CI = ref_shims.import_reference_wrapper()
    model = ref_shims.import_reference_model()
    tmp = tempfile.mkdtemp()
    wpath = os.path.join(tmp, "synthetic_%d.pth" % SEED)
    torch.save(synth.torch_state_dict(SEED), wpath)
    img_path = os.path.join(ref_shims.REF_ROOT, "test_imgs", "mortar_pestle.jpg")

    # ---------------- 256x256, ColorizeImageTorch (configs 1, 2, notebook KAT) -------------
    out = {}
    for maskcent in (False, True):
        tag = "mc1" if maskcent else "mc0"
        cm = CI.ColorizeImageTorch(Xd=256, maskcent=maskcent)
        cm.prep_net(path=wpath)
        cm.load_image(img_path)
        if not maskcent:
            out["img_rgb"] = cm.img_rgb.copy()                        # uint8 256x256x3 (cv2 resize)
            out["img_l_mc"] = cm.img_l_mc.astype(np.float64)
        cases = {}
        cases["zero"] = (np.zeros((2, 256, 256)), np.zeros((1, 256, 256)))
        cases["rand5"] = synth.synthetic_hints(256, 5, 0)
        ab, m = np.zeros((2, 256, 256)), np.zeros((1, 256, 256))
        synth.put_point(ab, m, [135, 160], 3, [23, -69])
        synth.put_point(ab, m, [100, 160], 3, [0, 0])
        cases["kat"] = (ab, m)
        for name, (ab, m) in cases.items():
            rgb = cm.net_forward(ab.copy(), m.copy())
            # raw net output (SURVEY q2): re-run the net exactly as data/colorize_image.py:263 does
            raw = cm.net.forward(cm.img_l_mc, cm.input_ab_mc, cm.input_mask_mult, cm.mask_cent)[0].cpu().data.numpy()
            if maskcent and name != "rand5":
                continue                                              # keep the fixture small
            out["%s_%s_ab_raw" % (tag, name)] = raw.astype(np.float32)
            if not maskcent:
                out["%s_%s_rgb" % (tag, name)] = rgb.copy()
            if tag == "mc0" and name == "kat":
                out["%s_%s_output_ab" % (tag, name)] = cm.output_ab.astype(np.float32)
            if tag == "mc0" and name == "kat":
                out["kat_fullres_rgb_small"] = cm.get_img_fullres()[::8, ::8].copy()
    idx = pix_idx()
    out = {k: sample_256(k, v, idx) for k, v in out.items()}
    out["pix_idx"] = idx
    np.savez_compressed(os.path.join(HERE, "lhn_256.npz"), **out)
    print("lhn_256.npz", {k: v.shape for k, v in out.items()})

    # ---------------- dist model ------------------------------------------------------------
    cd = CI.ColorizeImageTorchDist(Xd=256, maskcent=True)
    cd.prep_net(path=wpath, dist=True)
    cd.load_image(img_path)
    ab, m = synth.synthetic_hints(256, 5, 0)
    ret = cd.net_forward(ab.copy(), m.copy())
    d = cd.dist_ab                                                     # [529,256,256] float32
    dd = {"ret_quirk": ret.astype(np.float32),
          "dist_rows": d[:, ::4, ::4][:, ::8, ::8].astype(np.float32),   # [529,8,8] of the 64x64 grid
          "dist_upsample_ok": np.array(np.all(d == np.repeat(np.repeat(d[:, ::4, ::4], 4, 1), 4, 2))),
          "dist_sum64": d[:, ::4, ::4].sum(0).astype(np.float32),
          "dist_argmax64": d[:, ::4, ::4].argmax(0).astype(np.int32),
          "dist_max64": d[:, ::4, ::4].max(0).astype(np.float32)}
    np.random.seed(0)
    dd["reccs_128_128_K9"] = cd.get_ab_reccs(128, 128, K=9, N=25000)
    np.savez_compressed(os.path.join(HERE, "lhn_dist_256.npz"), **dd)
    print("lhn_dist_256.npz", {k: v.shape for k, v in dd.items()})

    # ---------------- 64x64 synthetic with per-layer statistics ------------------------------
    L, ab, m = synth.synthetic_batch(2, 64, seed=100, max_hints=4)
    net = model.SIGGRAPHGenerator(dist=True)
    net.load_state_dict(torch.load(wpath))
    net.eval()
    inter = {}
    names = ["model1", "model2", "model3", "model4", "model5", "model6", "model7", "model8", "model9", "model10"]
    hooks = [getattr(net, n).register_forward_hook(lambda mod, i, o, n=n: inter.__setitem__(n, o.detach().numpy().copy()))
             for n in names]
    small = {"L": L, "ab": ab, "mask": m}
    for i in range(2):
        reg, dist = net.forward(L[i], ab[i], m[i], 0.5)
        small["reg_quirk_%d" % i] = reg[0].detach().numpy().astype(np.float32)
        small["dist16_%d" % i] = dist[0, :, ::4, ::4].detach().numpy().astype(np.float32)
        for n in names:
            t = inter[n][0].astype(np.float32)
            small["%s_%d_c8" % (n, i)] = t[:8].copy()                  # first 8 channels, full plane
            small["%s_%d_chmean" % (n, i)] = t.mean(axis=(1, 2))       # every channel, spatial mean
            small["%s_%d_absmax" % (n, i)] = np.abs(t).max(axis=(1, 2))
    for h in hooks:
        h.remove()
    bins = dist_bins()
    small = {k: sample_64(k, v, bins) for k, v in small.items()}
    small["dist16_bins"] = bins
    np.savez_compressed(os.path.join(HERE, "lhn_64.npz"), **small)
    print("lhn_64.npz", {k: v.shape for k, v in small.items()})


if __name__ == "__main__":
    main()
