"""CPU restatement of the Caffe-only pieces of the hot path (no Caffe runtime exists here and
the reference holds no test vectors for them: PARITY UNPINNED -- see oracle/__init__.py).

  global_hints_vector   models/global_model/deploy_nodist.prototxt:38-172
                        glob_conv1(glob_ab_313_mask[314]) + s_conv1(s_avg_mask[2]) -> ReLU -> BatchNorm,
                        then 3 x (1x1 conv 512->512, ReLU, BatchNorm); the result is broadcast over
                        space (SpatialRepLayer, caffe_files/caffe_traininglayers.py:14-50) and added to
                        conv4_3norm (:501-527) -- that add is `glob_add` in oracle/lhn_ref.py.
                        Input driver: data/colorize_image.py:452-463.

Test infrastructure only.
"""
import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-5


def synthetic_glob_state_dict(seed=4321):
    """Keys glob.{0..3}.weight [512, 316|512], .bias, .bn.{weight,bias,running_mean,running_var}.
    Layer 0's weight is [glob_conv1 (314 cols) | s_conv1 (2 cols)], bias = sum of both biases."""
    rng = np.random.RandomState(seed)
    sd = {}
    for l in range(4):
        cin = 316 if l == 0 else 512
        std = np.sqrt(2.0 / (8.0 if l == 0 else cin))     # layer-0 inputs are a pmf + indicators: small fan-in
        sd["glob.%d.weight" % l] = (rng.standard_normal((512, cin)) * std).astype(np.float32)
        sd["glob.%d.bias" % l] = rng.uniform(-0.1, 0.1, 512).astype(np.float32)
        sd["glob.%d.bn.weight" % l] = rng.uniform(0.6, 1.4, 512).astype(np.float32)
        sd["glob.%d.bn.bias" % l] = (rng.standard_normal(512) * 0.1).astype(np.float32)
        sd["glob.%d.bn.running_mean" % l] = rng.uniform(0.1, 0.6, 512).astype(np.float32)
        sd["glob.%d.bn.running_var" % l] = rng.uniform(0.3, 1.2, 512).astype(np.float32)
    return sd


def global_hints_vector(gsd, glob316, dtype=torch.float32):
    """glob316 [N,316] = [313 histogram, indicator, mean saturation, indicator] -> [N,512]."""
    x = torch.as_tensor(np.asarray(glob316), dtype=dtype)
    for l in range(4):
        t = lambda k: torch.as_tensor(np.asarray(gsd["glob.%d.%s" % (l, k)]), dtype=dtype)
        x = F.relu(F.linear(x, t("weight"), t("bias")))
        x = F.batch_norm(x, t("bn.running_mean"), t("bn.running_var"), t("bn.weight"), t("bn.bias"), False, 0.0, BN_EPS)
    return x


# ---------------------------------------------------------------------------------------------
# 313-bin hyper-column head + annealed-mean decode (row a14)
#   models/reference_model/deploy_nopred.prototxt:651-850; kernel / centre injection
#   data/colorize_image.py:405-413.  PARITY UNPINNED (no Caffe runtime, no vectors).
# ---------------------------------------------------------------------------------------------
US_KERNEL = np.array(((.25, .5, .25, 0), (.5, 1., .5, 0), (.25, .5, .25, 0), (0, 0, 0, 0)), dtype=np.float32)


def synthetic_caffe313_state_dict(seed=777, pts_in_hull=None):
    rng = np.random.RandomState(seed)
    sd = {}
    for name, cin in (("conv3_pred", 256), ("conv8_pred", 256)):
        sd["caffe.%s.weight" % name] = (rng.standard_normal((384, cin, 3, 3)) * np.sqrt(2.0 / (6 * cin * 9))).astype(np.float32)
        sd["caffe.%s.bias" % name] = rng.uniform(-0.05, 0.05, 384).astype(np.float32)
    for l in (4, 5, 6, 7):     # Caffe Deconvolution blobs are [Cin, Cout, kh, kw]
        sd["caffe.conv%d_pred.weight" % l] = (rng.standard_normal((512, 384, 4, 4)) * np.sqrt(2.0 / (6 * 512 * 4))).astype(np.float32)
        sd["caffe.conv%d_pred.bias" % l] = rng.uniform(-0.05, 0.05, 384).astype(np.float32)
    sd["caffe.pred_313.weight"] = (rng.standard_normal((313, 384, 1, 1)) * (3.0 / np.sqrt(384))).astype(np.float32)
    sd["caffe.pred_313.bias"] = rng.uniform(-0.1, 0.1, 313).astype(np.float32)
    if pts_in_hull is not None:
        sd["caffe.pts_in_hull"] = np.asarray(pts_in_hull, dtype=np.float32)
    return sd


def caffe313_head(csd, inter, T=2.6, S=0.2, return_logits=False, dtype=torch.float32):
    """inter: intermediates of oracle/lhn_ref.lhn_forward (conv3_3 ... conv8_3 are the *norm blobs).
    -> (pred_ab [N,2,H,W], dist_ab_S [N,313,H,W]).  dtype=torch.float64 evaluates the same head in double
    precision from the same FP32 trunk activations: the T = 2.6 softmax amplifies FP32 summation-order noise of
    the logits, so two FP32 evaluations of this head differ from each other by ~1e-3 in ab; the FP64 run is the
    arithmetic-exact statement of the spec that both are measured against."""
    t = lambda k: torch.as_tensor(np.asarray(csd[k]), dtype=dtype)
    inter = {k: v.to(dtype) for k, v in inter.items() if k in ("conv3_3", "conv4_3", "conv5_3", "conv6_3", "conv7_3", "conv8_3")}
    h = F.conv2d(inter["conv3_3"], t("caffe.conv3_pred.weight"), t("caffe.conv3_pred.bias"), padding=1)
    for l in (4, 5, 6, 7):
        h = h + F.conv_transpose2d(inter["conv%d_3" % l], t("caffe.conv%d_pred.weight" % l), t("caffe.conv%d_pred.bias" % l),
                                   stride=2, padding=1)
    h = h + F.conv2d(inter["conv8_3"], t("caffe.conv8_pred.weight"), t("caffe.conv8_pred.bias"), padding=1)
    h = F.relu(h)                                                          # relu345678_pred
    logits = F.conv2d(h, t("caffe.pred_313.weight"), t("caffe.pred_313.bias"))
    k = torch.from_numpy(US_KERNEL).to(dtype)[None, None].repeat(313, 1, 1, 1)       # data/colorize_image.py:409-413
    up = F.conv_transpose2d(logits, k, None, stride=2, padding=1, groups=313)        # pred_313_us
    up = F.conv_transpose2d(up, k, None, stride=2, padding=1, groups=313)            # pred_313_rs
    dist_S = F.softmax(up * S, dim=1)                                      # scale_S + dist_ab_S
    dist_T = F.softmax(up * T, dim=1)                                      # scale_T + dist_ab (T)
    pts = t("caffe.pts_in_hull")                                           # pred_ab weights = pts_in_hull.T (:405-407)
    pred_ab = torch.einsum("nbhw,bc->nchw", dist_T, pts)
    if return_logits:
        return pred_ab, dist_S, logits, h
    return pred_ab, dist_S


def global_stats(rgb_u8, pts_in_hull):
    """numpy restatement of models/global_model/global_stats.prototxt for one uint8 RGB image:
    Lab (skimage, oracle/color_ref.py) -> 4x4 average pool of ab -> NNEncLayer (NN=1: nearest bin) ->
    global average; mean HSV saturation.  -> [313 hist, 1, s_avg, 1].  PARITY UNPINNED."""
    from . import color_ref
    lab = color_ref.rgb2lab(rgb_u8)
    H, W = lab.shape[:2]
    ab = lab[..., 1:].reshape(H // 4, 4, W // 4, 4, 2).mean(axis=(1, 3)).reshape(-1, 2).astype(np.float32)
    pts = np.asarray(pts_in_hull, dtype=np.float32)
    d = ((ab[:, None, :] - pts[None, :, :]) ** 2).sum(-1)
    hist = np.bincount(d.argmin(1), minlength=313).astype(np.float64) / ab.shape[0]
    c = rgb_u8.astype(np.float64) / 255.0
    mx, mn = c.max(-1), c.min(-1)
    s = np.where(mx > 0, (mx - mn) / np.where(mx > 0, mx, 1.0), 0.0)
    return np.concatenate([hist, [1.0], [s.mean()], [1.0]]).astype(np.float32)
