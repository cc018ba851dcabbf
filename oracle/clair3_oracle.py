"""ORACLE — test infrastructure only (never imported by the product path).

Plain-numpy CPU restatement of the Clair3 inference forward pass, used by ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` leg to check the sm_90a kernels.
Each function cites the reference lines it restates (paths relative to the HKU-BAL/Clair3 repo):

* ``pileup_forward``  -> ``clair3/model.py:130-161``  (``Clair3_P.forward``)
* ``lstm_bidir``      -> torch ``nn.LSTM`` semantics used at ``clair3/model.py:96-107,132-133``
                         (gate row order i,f,g,o; h0=c0=0; reverse direction runs t=T-1..0;
                         output = concat[fwd, bwd] per time step)
* ``fa_forward``      -> ``clair3/model.py:377-416``  (``Clair3_F.forward``)
* ``conv_bn``         -> ``clair3/model.py:183-197``  (Conv2d 3x3 pad 1 + BatchNorm2d(eps=1e-3, eval) [+ReLU])
* ``basic_block``     -> ``clair3/model.py:200-235``
* ``pyramid_pool``    -> ``clair3/model.py:250-279``  (TF-'SAME' zero pad, max pool, NHWC flatten)
* ``heads``           -> ``clair3/model.py:136-159 / 391-411``  (SELU dense stack, softmax, concat)

The arithmetic itself lives in a third-party dependency that the reference does not vendor or
pin (PyTorch ATen / oneDNN; ``Dockerfile:36-38`` installs an unpinned ``torch``).  The restated
definitions are the published ones: LSTM cell, ``nn.SELU`` (alpha=1.6732632423543772,
scale=1.0507009873554805), eval-mode BatchNorm, softmax.

Pinning: the reference holds no golden vectors for this path (SURVEY.md §4), so the oracle is pinned
against outputs of the reference itself: ``tests/golden/make_golden.py`` imports
the reference's ``clair3/model.py`` (a checkout named by ``CLAIR3_REFERENCE``), runs it in fp32 on seeded inputs and
commits outputs + taps under ``tests/golden/``; ``tests/test_oracle.py`` checks this file against them.

Computation dtype defaults to float64 so the oracle is "the math"; the fp32 reference differs from
it by ~1e-6 on output probabilities.
"""
from __future__ import annotations

import numpy as np

SELU_ALPHA = 1.6732632423543772
SELU_SCALE = 1.0507009873554805
BN_EPS = 1e-3
NORMALIZE_NUM = 100.0   # shared/param_f.py:36


def selu(x):
    return SELU_SCALE * np.where(x > 0, x, SELU_ALPHA * np.expm1(np.minimum(x, 0)))


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def softmax(x):
    e = np.exp(x - x.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)


def lstm_dir(x, w_ih, w_hh, b_ih, b_hh, reverse):
    """One direction of a batch_first LSTM layer.  x: [B,T,I] -> [B,T,H]."""
    B, T, _ = x.shape
    H = w_hh.shape[1]
    h = np.zeros((B, H), dtype=x.dtype)
    c = np.zeros((B, H), dtype=x.dtype)
    out = np.zeros((B, T, H), dtype=x.dtype)
    xw = x @ w_ih.T + (b_ih + b_hh)            # [B,T,4H]
    steps = range(T - 1, -1, -1) if reverse else range(T)
    for t in steps:
        g = xw[:, t] + h @ w_hh.T
        i = sigmoid(g[:, 0 * H:1 * H])
        f = sigmoid(g[:, 1 * H:2 * H])
        gg = np.tanh(g[:, 2 * H:3 * H])
        o = sigmoid(g[:, 3 * H:4 * H])
        c = f * c + i * gg
        h = o * np.tanh(c)
        out[:, t] = h
    return out


def lstm_bidir(x, sd, name):
    fwd = lstm_dir(x, sd[f"{name}.weight_ih_l0"], sd[f"{name}.weight_hh_l0"],
                   sd[f"{name}.bias_ih_l0"], sd[f"{name}.bias_hh_l0"], False)
    bwd = lstm_dir(x, sd[f"{name}.weight_ih_l0_reverse"], sd[f"{name}.weight_hh_l0_reverse"],
                   sd[f"{name}.bias_ih_l0_reverse"], sd[f"{name}.bias_hh_l0_reverse"], True)
    return np.concatenate([fwd, bwd], axis=-1)


def dense(x, sd, name):
    return x @ sd[f"{name}.weight"].T + sd[f"{name}.bias"]


def heads(x, sd, add_indel_length, taps=None):
    names = [("L5_1", "Y_gt21_logits"), ("L5_2", "Y_genotype_logits")]
    if add_indel_length:
        names += [("L5_3", "Y_indel_length_logits_1"), ("L5_4", "Y_indel_length_logits_2")]
    outs = []
    for l5, y in names:
        z = selu(dense(selu(dense(x, sd, l5)), sd, y))
        if taps is not None:
            taps[f"pre_softmax.{y}"] = z
        outs.append(softmax(z))
    return np.concatenate(outs, axis=1)


def _cast_sd(sd, dtype):
    return {k: (np.asarray(v).astype(dtype) if np.asarray(v).dtype.kind == "f" else np.asarray(v))
            for k, v in sd.items()}


def pileup_forward(sd, x, add_indel_length=False, dtype=np.float64, taps=None):
    """Clair3_P.forward (clair3/model.py:130-161).  x: [B,33,C] any int/float dtype -> [B,24|90]."""
    sd = _cast_sd(sd, dtype)
    h = np.asarray(x).astype(dtype)                      # x.float()            :131
    h = lstm_bidir(h, sd, "LSTM1")                       #                      :132
    if taps is not None:
        taps["lstm1"] = h
    h = lstm_bidir(h, sd, "LSTM2")                       #                      :133
    if taps is not None:
        taps["lstm2"] = h
    h = h.reshape(h.shape[0], -1)                        # flatten t*320+dir*160+j :135
    z = dense(h, sd, "L4")
    if taps is not None:
        taps["l4_pre"] = z
    h = selu(z)                                          #                      :136
    return heads(h, sd, add_indel_length, taps)


def _im2col3x3(x, stride):
    """x: [B,C,H,W] -> cols [B,Ho,Wo,C*9] (k index = c*9 + kh*3 + kw), pad=1."""
    B, C, H, W = x.shape
    Ho = (H + 2 - 3) // stride + 1
    Wo = (W + 2 - 3) // stride + 1
    xp = np.zeros((B, C, H + 2, W + 2), dtype=x.dtype)
    xp[:, :, 1:H + 1, 1:W + 1] = x
    cols = np.zeros((B, Ho, Wo, C, 3, 3), dtype=x.dtype)
    for kh in range(3):
        for kw in range(3):
            cols[:, :, :, :, kh, kw] = xp[:, :, kh:kh + stride * Ho:stride, kw:kw + stride * Wo:stride] \
                .transpose(0, 2, 3, 1)
    return cols.reshape(B, Ho, Wo, C * 9), Ho, Wo


def conv_bn(x, sd, conv, bn, stride, relu):
    """Conv2d(3x3, pad 1, bias) -> BatchNorm2d(eval, eps=1e-3) [-> ReLU]; NCHW."""
    w = sd[f"{conv}.weight"]
    cols, Ho, Wo = _im2col3x3(x, stride)
    y = cols @ w.reshape(w.shape[0], -1).T + sd[f"{conv}.bias"]      # [B,Ho,Wo,Cout]
    y = (y - sd[f"{bn}.running_mean"]) / np.sqrt(sd[f"{bn}.running_var"] + BN_EPS) \
        * sd[f"{bn}.weight"] + sd[f"{bn}.bias"]
    if relu:
        y = np.maximum(y, 0)
    return y.transpose(0, 3, 1, 2)


def basic_block(x, sd, prefix):
    y = conv_bn(x, sd, f"{prefix}.conv1", f"{prefix}.bn1", 1, True)
    y = conv_bn(y, sd, f"{prefix}.conv2", f"{prefix}.bn2", 1, False)
    return np.maximum(x + y, 0)                          # identity downsample (:215-221)


def pyramid_pool(x, pool_sizes=(3, 2, 1)):
    """PyramidPolling.forward (clair3/model.py:250-279). x: [B,C,H,W] -> [B, sum(p*p)*C]."""
    B, C, H, W = x.shape
    pooled = []
    for p in pool_sizes:
        wh, ww = int(np.ceil(H / p)), int(np.ceil(W / p))
        oh, ow = int(np.ceil(H / wh)), int(np.ceil(W / ww))
        ph = max((oh - 1) * wh + wh - H, 0)
        pw = max((ow - 1) * ww + ww - W, 0)
        pt, pl = ph // 2, pw // 2
        xp = np.zeros((B, C, H + ph, W + pw), dtype=x.dtype)
        xp[:, :, pt:pt + H, pl:pl + W] = x
        # F.max_pool2d floor mode: out = floor((Hp - wh)/wh) + 1
        oh2 = (H + ph - wh) // wh + 1
        ow2 = (W + pw - ww) // ww + 1
        out = np.zeros((B, oh2, ow2, C), dtype=x.dtype)
        for i in range(oh2):
            for j in range(ow2):
                out[:, i, j] = xp[:, :, i * wh:(i + 1) * wh, j * ww:(j + 1) * ww].max(axis=(2, 3))
        pooled.append(out.reshape(B, -1))                # NHWC flatten
    return np.concatenate(pooled, axis=1)


def fa_forward(sd, x, add_indel_length=True, dtype=np.float64, taps=None):
    """Clair3_F.forward (clair3/model.py:377-416).  x: [B,D,33,C] int8 NHWC -> [B,24|90]."""
    sd = _cast_sd(sd, dtype)
    h = np.asarray(x).astype(dtype) / dtype(NORMALIZE_NUM)   # :378
    cin = sd["conv1.conv.weight"].shape[1]
    if h.ndim == 4 and h.shape[-1] == cin:
        h = h.transpose(0, 3, 1, 2)                          # :379-380
    h = conv_bn(h, sd, "conv1.conv", "conv1.bn", 2, True)
    if taps is not None:
        taps["conv1"] = h
    h = basic_block(h, sd, "res_block1.0")
    if taps is not None:
        taps["res_block1"] = h
    h = conv_bn(h, sd, "conv3.conv", "conv3.bn", 2, True)
    if taps is not None:
        taps["conv3"] = h
    h = basic_block(h, sd, "res_block2.0")
    if taps is not None:
        taps["res_block2"] = h
    h = conv_bn(h, sd, "conv5.conv", "conv5.bn", 2, True)
    if taps is not None:
        taps["conv5"] = h
    h = basic_block(h, sd, "res_block3.0")
    if taps is not None:
        taps["res_block3"] = h
    h = pyramid_pool(h)
    if taps is not None:
        taps["spp"] = h
    z = dense(h, sd, "L4")
    if taps is not None:
        taps["l4_pre"] = z
    return heads(selu(z), sd, add_indel_length, taps)


def depth_rescale_with(x, depths, max_depth=144):
    """CPU-branch pileup depth rescale (clair3/CallVariantsFromCffi.py:278-285): for sites deeper than
    1.5*max_depth the [33,18] tensor is divided by depth/max_depth and assigned back into the int32
    array, i.e. truncated toward zero.  ``depths`` is the per-site depth the caller reads from alt_info."""
    x = np.array(x, copy=True)
    for i, d in enumerate(depths):
        if d > 1.5 * max_depth:
            scale = d / max_depth
            x[i] = (x[i] / scale).astype(x.dtype)            # numpy cast = trunc toward zero
    return x
