"""Power-of-two rescaled twins of a state_dict (test infrastructure).

For a gain g = 2^k on one activation buffer the twin stores g times that buffer and computes the same function:

  * inner buffer (a ReLU output between two convs, e.g. a3_1): the producer conv's weight and bias times g, every
    consumer conv's weight times 1/g (its bias stays).  a8_1 / a9_1 / a10_1 have two producers, the up-sampling
    deconv and the shortcut conv.
  * BN output (conv1_2 ... conv9_3): the BN's weight and bias times g (its running statistics stay), every consumer
    times 1/g.  With global hints the last BN of the global MLP is scaled with conv4_3, so the vector added to it
    scales too.
  * conv10_2 (the fused head's input): model10.1 weight and bias times g, model_out times 1/g.
  * hyper (Caffe 313-bin head): the six caffe.conv*_pred sources times g, caffe.pred_313's weight times 1/g.

ReLU and LeakyReLU are positively homogeneous and powers of two are exact in floating point, so the twin's output
equals the original's up to summation noise, and every intermediate is exactly g times the original's in exact
arithmetic.  Keys that are absent from the state_dict (no global hints, no Caffe head) are skipped.
"""
import torch

# buffer -> (producer parameter keys scaled by g (weight and bias), consumer weight keys scaled by 1/g)
_BN = {"conv1_2": "model1.4", "conv2_2": "model2.4", "conv3_3": "model3.6", "conv4_3": "model4.6", "conv5_3": "model5.6",
       "conv6_3": "model6.6", "conv7_3": "model7.6", "conv8_3": "model8.5", "conv9_3": "model9.3"}
_CONSUMERS = {
    "a1_1": ["model1.2"], "conv1_2": ["model2.0", "model1short10.0"],
    "a2_1": ["model2.2"], "conv2_2": ["model3.0", "model2short9.0"],
    "a3_1": ["model3.2"], "a3_2": ["model3.4"], "conv3_3": ["model4.0", "model3short8.0", "caffe.conv3_pred"],
    "a4_1": ["model4.2"], "a4_2": ["model4.4"], "conv4_3": ["model5.0", "caffe.conv4_pred"],
    "a5_1": ["model5.2"], "a5_2": ["model5.4"], "conv5_3": ["model6.0", "caffe.conv5_pred"],
    "a6_1": ["model6.2"], "a6_2": ["model6.4"], "conv6_3": ["model7.0", "caffe.conv6_pred"],
    "a7_1": ["model7.2"], "a7_2": ["model7.4"], "conv7_3": ["model8up.0", "caffe.conv7_pred"],
    "a8_1": ["model8.1"], "a8_2": ["model8.3"], "conv8_3": ["model9up.0", "model_class.0", "caffe.conv8_pred"],
    "a9_1": ["model9.1"], "conv9_3": ["model10up.0"],
    "a10_1": ["model10.1"], "conv10_2": ["model_out.0"],
    "hyper": ["caffe.pred_313"],
}
_PRODUCERS = {
    "a1_1": ["model1.0"], "a2_1": ["model2.0"], "a3_1": ["model3.0"], "a3_2": ["model3.2"],
    "a4_1": ["model4.0"], "a4_2": ["model4.2"], "a5_1": ["model5.0"], "a5_2": ["model5.2"],
    "a6_1": ["model6.0"], "a6_2": ["model6.2"], "a7_1": ["model7.0"], "a7_2": ["model7.2"],
    "a8_1": ["model8up.0", "model3short8.0"], "a8_2": ["model8.1"],
    "a9_1": ["model9up.0", "model2short9.0"], "a10_1": ["model10up.0", "model1short10.0"],
    "conv10_2": ["model10.1"],
    "hyper": ["caffe.conv%d_pred" % l for l in range(3, 9)],
}
_PRODUCERS.update({b: [k] for b, k in _BN.items()})
_PRODUCERS["conv4_3"] = ["model4.6", "glob.3.bn"]

# every buffer the engines store (a1_1 and each op output except conv10_2), in network order, then the two extras
STORED = ["a1_1", "conv1_2", "a2_1", "conv2_2", "a3_1", "a3_2", "conv3_3", "a4_1", "a4_2", "conv4_3",
          "a5_1", "a5_2", "conv5_3", "a6_1", "a6_2", "conv6_3", "a7_1", "a7_2", "conv7_3",
          "a8_1", "a8_2", "conv8_3", "a9_1", "conv9_3", "a10_1"]
BUFFERS = STORED + ["conv10_2", "hyper"]


def _scaled(sd, key, k):
    v = sd[key]
    t = v if torch.is_tensor(v) else torch.as_tensor(v)
    return t * (2.0 ** k)        # a power of two: exact in the tensor's own dtype


def rescale(sd, gains):
    """sd: {state_dict key: tensor | ndarray}; gains: {buffer name: integer k} (gain 2^k).  -> a new dict (torch
    tensors for the keys it changed, the original objects for the others)."""
    out = dict(sd)
    for buf, k in gains.items():
        if buf not in _PRODUCERS:
            raise KeyError("no rescaling rule for buffer %r" % buf)
        if int(k) != k:
            raise ValueError("gain exponent of %s must be an integer, got %r" % (buf, k))
        k = int(k)
        if k == 0:
            continue
        for p in _PRODUCERS[buf]:
            for suffix in (".weight", ".bias"):
                if p + suffix in out:
                    out[p + suffix] = _scaled(out, p + suffix, k)
        for c in _CONSUMERS[buf]:
            if c + ".weight" in out:
                out[c + ".weight"] = _scaled(out, c + ".weight", -k)
    return out


def random_gains(seed, lo, hi, buffers=BUFFERS):
    """One integer exponent in [lo, hi] per buffer, seeded."""
    g = torch.Generator().manual_seed(seed)
    return {b: int(v) for b, v in zip(buffers, torch.randint(lo, hi + 1, (len(buffers),), generator=g).tolist())}
