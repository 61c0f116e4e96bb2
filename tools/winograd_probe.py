#!/usr/bin/env python
"""CPU probe (VERDICT r1 item 4): would Winograd F(2x2,3x3) on the stride-1 3x3 layers stay inside the 1e-3 ab budget
with the engine's 22-bit (FP16 hi + lo) operand representation?

The whole Local Hints Network is evaluated in float64 with every conv operand (activations AND weights, in the domain
in which the tensor core would see them) rounded to 22 significant bits -- the hi/lo FP16 split -- and exact
accumulation, once with direct convolutions (what the engine does) and once with Winograd F(2x2,3x3) on every eligible
layer (stride-1 3x3, incl. the dilation-2 ones via their 4 parity sub-grids): input tiles transformed B^T d B in FP32
then rounded to 22 bits, weights transformed G g G^T in FP64 then rounded, 16 element-wise GEMMs, output transform
A^T m A in FP32.  Both are compared with the plain FP32 oracle (the parity target) and an FP64 evaluation.

    python tools/winograd_probe.py            -> prints the table
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import lhn_ref, synth  # noqa: E402

BT = torch.tensor([[1, 0, -1, 0], [0, 1, 1, 0], [0, -1, 1, 0], [0, 1, 0, -1]], dtype=torch.float64)
G = torch.tensor([[1, 0, 0], [.5, .5, .5], [.5, -.5, .5], [0, 0, 1]], dtype=torch.float64)
AT = torch.tensor([[1, 1, 1, 0], [0, 1, -1, -1]], dtype=torch.float64)


def r22(x):
    """round to 22 significant bits (FP16 hi + FP16 lo of a pre-scaled value), float64 in/out"""
    m, e = torch.frexp(x)
    return torch.ldexp(torch.round(m * (1 << 22)) / (1 << 22), e)


def r24(x):
    return x.float().double()


def wino_conv(x, w, b, bits_fn):
    """3x3 stride-1 pad-1 conv via F(2x2,3x3).  x [N,C,H,W] float64 (H, W even), w [Co,Ci,3,3]."""
    N, C, H, W = x.shape
    xp = F.pad(x, (1, 1, 1, 1))
    d = xp.unfold(2, 4, 2).unfold(3, 4, 2)                     # [N,C,H/2,W/2,4,4]
    V = r24(torch.einsum("ij,ncabjk,lk->ncabil", BT, d, BT))    # FP32 transform (adds only), then ...
    V = bits_fn(V)                                              # ... the operand representation of the MMA
    U = bits_fn(torch.einsum("ij,ocjk,lk->ocil", G, w, G))      # weights: FP64 offline, then the representation
    M = torch.einsum("ncabil,ocil->noabil", V, U)               # 16 GEMMs, exact accumulation
    Y = r24(torch.einsum("ij,noabjk,lk->noabil", AT, r24(M), AT))   # FP32 output transform
    return Y.permute(0, 1, 2, 4, 3, 5).reshape(N, -1, H, W) + b.view(1, -1, 1, 1)


def conv(sd, key, x, mode, dilation=1):
    w, b = sd[key + ".weight"].double(), sd[key + ".bias"].double()
    if mode == "fp64":
        return F.conv2d(x, w, b, padding=dilation, dilation=dilation)
    if mode == "direct22" or w.shape[-1] != 3:
        return F.conv2d(r22(x), r22(w), b, padding=dilation * (w.shape[-1] // 2), dilation=dilation)
    if dilation == 1:
        return wino_conv(r22(x), w, b, r22)
    out = torch.empty(x.shape[0], w.shape[0], x.shape[2], x.shape[3], dtype=torch.float64)
    for py in range(2):                                         # dilation 2 = 4 independent parity sub-grids
        for px in range(2):
            out[:, :, py::2, px::2] = wino_conv(r22(x[:, :, py::2, px::2]), w, b, r22)
    return out


def deconv(sd, key, x, mode):
    w, b = sd[key + ".weight"].double(), sd[key + ".bias"].double()
    if mode == "fp64":
        return F.conv_transpose2d(x, w, b, stride=2, padding=1)
    return F.conv_transpose2d(r22(x), r22(w), b, stride=2, padding=1)


def bn(sd, key, x):
    g, b = sd[key + ".weight"].double(), sd[key + ".bias"].double()
    m, v = sd[key + ".running_mean"].double(), sd[key + ".running_var"].double()
    s = g / torch.sqrt(v + 1e-5)
    return x * s.view(1, -1, 1, 1) + (b - m * s).view(1, -1, 1, 1)


def forward(sd, L, ab, mask, mc, mode):
    x = torch.cat((L.double() / 100.0, ab.double() / 110.0, mask.double() - mc), 1)
    dmode = "fp64" if mode == "fp64" else "direct22"
    wm = mode if mode != "wino22_mid" else "wino22"
    mid = lambda name: wm if (mode != "wino22_mid" or name) else dmode
    h = F.relu(conv(sd, "model1.0", x, dmode))                  # Cin = 4: CUDA cores either way
    h = F.relu(conv(sd, "model1.2", h, wm if mode == "wino22" else dmode)); c1 = bn(sd, "model1.4", h)
    h = F.relu(conv(sd, "model2.0", c1[:, :, ::2, ::2], dmode))  # stride-2 input: direct
    h = F.relu(conv(sd, "model2.2", h, wm if mode == "wino22" else dmode)); c2 = bn(sd, "model2.4", h)
    h = F.relu(conv(sd, "model3.0", c2[:, :, ::2, ::2], dmode))
    h = F.relu(conv(sd, "model3.2", h, wm)); h = F.relu(conv(sd, "model3.4", h, wm)); c3 = bn(sd, "model3.6", h)
    h = F.relu(conv(sd, "model4.0", c3[:, :, ::2, ::2], dmode))
    h = F.relu(conv(sd, "model4.2", h, wm)); h = F.relu(conv(sd, "model4.4", h, wm)); h = bn(sd, "model4.6", h)
    for blk, dil in (("model5", 2), ("model6", 2), ("model7", 1)):
        for i in (0, 2, 4):
            h = F.relu(conv(sd, "%s.%d" % (blk, i), h, wm, dil))
        h = bn(sd, blk + ".6", h)
    h = F.relu(deconv(sd, "model8up.0", h, dmode) + conv(sd, "model3short8.0", c3, dmode))
    h = F.relu(conv(sd, "model8.1", h, wm)); h = F.relu(conv(sd, "model8.3", h, wm)); c8 = bn(sd, "model8.5", h)
    h = F.relu(deconv(sd, "model9up.0", c8, dmode) + conv(sd, "model2short9.0", c2, dmode))
    h = F.relu(conv(sd, "model9.1", h, wm if mode == "wino22" else dmode)); c9 = bn(sd, "model9.3", h)
    h = F.relu(deconv(sd, "model10up.0", c9, dmode) + conv(sd, "model1short10.0", c1, dmode))
    h = F.leaky_relu(conv(sd, "model10.1", h, wm if mode == "wino22" else dmode), 0.2)
    w, b = sd["model_out.0.weight"].double(), sd["model_out.0.bias"].double()
    return torch.tanh(F.conv2d(h, w, b)) * 110.0


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    X = int(sys.argv[1]) if len(sys.argv) > 1 else 128
    sd = synth.torch_state_dict(1234)
    L, ab, m = synth.synthetic_batch(1, X, seed=3, max_hints=6)
    L, ab, m = torch.from_numpy(L), torch.from_numpy(ab), torch.from_numpy(m)
    with torch.no_grad():
        ref32 = lhn_ref.lhn_forward(sd, L, ab, m, 0.5).double()
        out = {k: forward(sd, L, ab, m, 0.5, k) for k in ("fp64", "direct22", "wino22_mid", "wino22")}
    print("Local Hints Network %dx%d, synthetic weights, 22-bit operands (FP16 hi+lo), exact accumulation" % (X, X))
    print("%-44s %12s %12s" % ("variant", "vs FP32 ref", "vs FP64"))
    names = {"direct22": "direct conv, 22-bit operands (the engine)",
             "wino22_mid": "Winograd F(2x2,3x3) on the 17 layers <= 64^2",
             "wino22": "Winograd F(2x2,3x3) on all 21 eligible layers"}
    print("%-44s %12s %12.3e" % ("FP32 reference oracle", "-", float((ref32 - out["fp64"]).abs().max())))
    for k in ("direct22", "wino22_mid", "wino22"):
        print("%-44s %12.3e %12.3e" % (names[k], float((out[k] - ref32).abs().max()), float((out[k] - out["fp64"]).abs().max())))


if __name__ == "__main__":
    main()
