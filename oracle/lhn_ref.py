"""CPU restatement (plain torch fp32 functional ops) of the reference Local Hints
Network forward, /root/reference/models/pytorch/model.py:134-175, batched.

Test infrastructure only -- see oracle/__init__.py.  Pinned against the unmodified
reference module through golden vectors generated from it (tests/golden/make_golden.py,
tests/golden/make_ref_forward_golden.py) and checked by tests/test_oracle.py.
"""
import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-5  # torch BatchNorm2d default (SURVEY q7)


def _t(x, dtype=torch.float32):
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(x)).to(dtype)
    return x.to(dtype)


def _conv(sd, key, x, dilation=1):
    # nn.Conv2d(k=3, stride 1, padding=dilation) model.py:13-101 ; 1x1 heads :105,:108
    w = _t(sd[key + ".weight"], x.dtype)
    pad = dilation * (w.shape[-1] // 2)
    return F.conv2d(x, w, _t(sd[key + ".bias"], x.dtype), stride=1, padding=pad, dilation=dilation)


def _deconv(sd, key, x):
    # nn.ConvTranspose2d(k=4, stride 2, padding 1) model.py:75,86,96
    return F.conv_transpose2d(x, _t(sd[key + ".weight"], x.dtype), _t(sd[key + ".bias"], x.dtype), stride=2, padding=1)


def _bn(sd, key, x, batch_stats=None):
    # eval-mode BatchNorm2d (data/colorize_image.py:232 net.eval()) model.py:17...93
    t = lambda s: _t(sd[key + s], x.dtype)
    if batch_stats is not None:
        # normalise with the batch's own per-channel mean and (biased) variance instead, and record them
        mean, var = x.mean(dim=(0, 2, 3)), x.var(dim=(0, 2, 3), unbiased=False)
        batch_stats[key] = (mean, var)
        return F.batch_norm(x, mean, var, t(".weight"), t(".bias"), False, 0.0, BN_EPS)
    return F.batch_norm(x, t(".running_mean"), t(".running_var"), t(".weight"), t(".bias"), False, 0.0, BN_EPS)


def lhn_forward(sd, L_mc, ab, mask, maskcent=0.0, dist=False, glob_add=None, ref_quirks=True,
                return_intermediates=False, dtype=torch.float32, batch_stats=None):
    """L_mc [N,1,H,W] in [-50,50]; ab [N,2,H,W] in [-110,110]; mask [N,1,H,W] in [0,1].
    Returns out_reg [N,2,H,W] (dist=False) or (out_reg_quirk, dist[N,529,H/4,W/4]) -- the
    nearest x4 upsample (model.py:160 upsample4) is NOT materialised here; use
    `upsample4()` below.  glob_add [N,512] is broadcast-added to conv4_3 (row a15).
    With ref_quirks the dist=True regression output is tanh*110*110 (model.py:166-168, q1).
    dtype=torch.float64 evaluates the same network in double precision (inputs and weights converted).
    batch_stats={} runs every BatchNorm on the statistics of its input batch (training-mode normalisation, in network
    order) and fills the dict with {BN key: (mean, biased var)}."""
    inter = {}
    bs = batch_stats
    A = _t(L_mc, dtype)
    B = _t(ab, dtype)
    M = _t(mask, dtype) - maskcent                                              # model.py:142
    x = torch.cat((A / 100.0, B / 110.0, M), dim=1)                      # model.py:148
    # model1 (:13-17)
    h = F.relu(_conv(sd, "model1.0", x)); inter["a1_1"] = h
    h = F.relu(_conv(sd, "model1.2", h))
    conv1_2 = _bn(sd, "model1.4", h, bs); inter["conv1_2"] = conv1_2
    # model2 on [:, :, ::2, ::2] (:149, :21-25)
    h = F.relu(_conv(sd, "model2.0", conv1_2[:, :, ::2, ::2])); inter["a2_1"] = h
    h = F.relu(_conv(sd, "model2.2", h))
    conv2_2 = _bn(sd, "model2.4", h, bs); inter["conv2_2"] = conv2_2
    # model3 (:150, :29-35)
    h = F.relu(_conv(sd, "model3.0", conv2_2[:, :, ::2, ::2])); inter["a3_1"] = h
    h = F.relu(_conv(sd, "model3.2", h)); inter["a3_2"] = h
    h = F.relu(_conv(sd, "model3.4", h))
    conv3_3 = _bn(sd, "model3.6", h, bs); inter["conv3_3"] = conv3_3
    # model4 (:151, :39-45)
    h = F.relu(_conv(sd, "model4.0", conv3_3[:, :, ::2, ::2])); inter["a4_1"] = h
    h = F.relu(_conv(sd, "model4.2", h)); inter["a4_2"] = h
    h = F.relu(_conv(sd, "model4.4", h))
    conv4_3 = _bn(sd, "model4.6", h, bs)
    if glob_add is not None:
        # models/global_model/deploy_nodist.prototxt:501-527: SpatialRep + Eltwise SUM on conv4_3norm
        conv4_3 = conv4_3 + _t(glob_add, dtype)[:, :, None, None]
    inter["conv4_3"] = conv4_3
    # model5, model6 dilation 2 (:48-63), model7 (:66-72)
    h = conv4_3
    for blk, dil in (("model5", 2), ("model6", 2), ("model7", 1)):
        for i in (0, 2, 4):
            h = F.relu(_conv(sd, "%s.%d" % (blk, i), h, dilation=dil))
            inter["a%s_%d" % (blk[-1], i // 2 + 1)] = h
        h = _bn(sd, blk + ".6", h, bs)
        inter["conv%s_3" % blk[-1]] = h
    conv7_3 = h
    # decoder level 8 (:156-157, :75-83)
    conv8_up = _deconv(sd, "model8up.0", conv7_3) + _conv(sd, "model3short8.0", conv3_3)
    h = F.relu(conv8_up); inter["a8_1"] = h
    h = F.relu(_conv(sd, "model8.1", h)); inter["a8_2"] = h
    h = F.relu(_conv(sd, "model8.3", h))
    conv8_3 = _bn(sd, "model8.5", h, bs); inter["conv8_3"] = conv8_3
    # level 9 (:162-163, :86-93)
    conv9_up = _deconv(sd, "model9up.0", conv8_3) + _conv(sd, "model2short9.0", conv2_2)
    h = F.relu(conv9_up); inter["a9_1"] = h
    h = F.relu(_conv(sd, "model9.1", h))
    conv9_3 = _bn(sd, "model9.3", h, bs); inter["conv9_3"] = conv9_3
    # level 10 (:164-165, :96-102)
    conv10_up = _deconv(sd, "model10up.0", conv9_3) + _conv(sd, "model1short10.0", conv1_2)
    h = F.relu(conv10_up); inter["a10_1"] = h
    conv10_2 = F.leaky_relu(_conv(sd, "model10.1", h), 0.2); inter["conv10_2"] = conv10_2
    # regression head (:108-109, :174-175)
    out_reg = torch.tanh(_conv(sd, "model_out.0", conv10_2)) * 110.0
    inter["out_reg"] = out_reg
    if not dist:
        return (out_reg, inter) if return_intermediates else out_reg
    # dist head (:105, :131-132, :160) -- kept at H/4 x W/4
    logits = _conv(sd, "model_class.0", conv8_3)
    dist64 = F.softmax(logits * 0.2, dim=1)
    inter["dist64"] = dist64
    reg = out_reg * 110.0 if ref_quirks else out_reg                      # q1, model.py:166-168
    return ((reg, dist64), inter) if return_intermediates else (reg, dist64)


def upsample4(dist64):
    """nn.Upsample(scale_factor=4, mode='nearest') model.py:131,160."""
    return dist64.repeat_interleave(4, dim=2).repeat_interleave(4, dim=3)
