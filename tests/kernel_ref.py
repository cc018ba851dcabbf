"""Operand-precision float64 references of the tensor-core kernels, one layer at a time.

Every function here computes ONE kernel's output from that kernel's own inputs as the GPU saw them (its input tap), with the
weights rebuilt from the state dict exactly as ``finalize`` in ``c3b_api.cu`` packs them (fp32 folding, then the fp16 cast).
The only difference left between the kernel and the reference is then the kernel's own arithmetic: fp32 accumulation, the
fp16 rounding of its output and, in the recurrences, ``tanh.approx``.  The bounds below cover exactly that, per element, so a
one-term mistake (a dropped k-group, a swapped tap, a bias on the wrong gate, a border slot read from the neighbouring site)
exceeds them.

* GEMM-type layers (proj2, the convolutions, L4):
  ``|gpu - ref| <= EPS * S + 2^-11 * |ref| + 2^-24`` with ``S = sum |a||w| + |bias| + |residual|``; the middle term is the
  fp16 rounding of the output and is dropped for fp32 outputs (L4).  ReLU is 1-Lipschitz, so the bound holds through it.
* Recurrences (LSTM1, LSTM2), teacher-forced: step t uses the GPU's own ``h_{t-1}`` (``h_{t+1}`` in the reverse direction), the
  cell state is chained in float64, and ``|gpu - ref| <= tau + 2 * EPS * S_gates`` per (site, t, direction, unit), where
  ``S_gates`` is the four gates' ``S``.  Teacher forcing keeps h differences from compounding, so tau can be tight.
* Exact: LSTM1's input operand (the hi/lo split of the raw counts) and the pyramid pooling (a max of fp16 values).
* Heads: float64 heads on the GPU's own L4 pre-activation; absolute tolerance on the probabilities.

EPS stays at least 8x below 1 / K_max (K_max = 10 560, the pileup L4) so that one wrong product term of typical size exceeds
the bound.
"""
from __future__ import annotations

import numpy as np

from oracle.clair3_oracle import pyramid_pool

EPS = 2.0 ** -18            # fp32 accumulation error relative to S
TAU_F32 = 2.0 ** -10        # recurrences with fp32 tanh.approx gate activations
TAU_MUFU16 = 2.0 ** -5      # recurrences with packed tanh.approx.f16x2 gate activations (option lstm_mufu16)
HEADS_TOL = 2e-5            # heads: absolute, on the probabilities
F16_ULP = 2.0 ** -11        # half an fp16 ulp, relative
TINY = 2.0 ** -24
K_MAX = 10560

T = 33
H1, H2 = 128, 160
X1_COLS = 48
BN_EPS = np.float32(1e-3)
CONV_KEYS = [("conv1.conv", "conv1.bn"), ("res_block1.0.conv1", "res_block1.0.bn1"), ("res_block1.0.conv2", "res_block1.0.bn2"),
             ("conv3.conv", "conv3.bn"), ("res_block2.0.conv1", "res_block2.0.bn1"), ("res_block2.0.conv2", "res_block2.0.bn2"),
             ("conv5.conv", "conv5.bn"), ("res_block3.0.conv1", "res_block3.0.bn1"), ("res_block3.0.conv2", "res_block3.0.bn2")]
# the GPU tap holding each convolution's output (level l = i // 3)
CONV_TAPS = ["conv1", "res_block1_mid", "res_block1", "conv3", "res_block2_mid", "res_block2", "conv5", "res_block3_mid",
             "res_block3"]
HEAD_NAMES = [("L5_1", "Y_gt21_logits"), ("L5_2", "Y_genotype_logits"), ("L5_3", "Y_indel_length_logits_1"),
              ("L5_4", "Y_indel_length_logits_2")]
SELU_ALPHA = 1.6732632423543772
SELU_SCALE = 1.0507009873554805


# ------------------------------------------------------------------------------------------------ fp16 operands
def f16(x):
    """fp32 -> fp16 round-to-nearest-even, saturating at +-65504 (``cvt.rn.satfinite.f16.f32`` / host ``c3b_f2op``); returned
    as float64."""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(over="ignore"):
        h = x.astype(np.float16)
    h = np.where(np.isinf(h), np.copysign(np.float16(65504.0), x).astype(np.float16), h)
    return h.astype(np.float64)


def hi_lo(x):
    """The ingest kernel's split of a raw count: hi = fp16(x), lo = fp16(x - hi), both saturating; x is first converted to
    fp32 like the kernel's ``(float)v``."""
    xf = np.asarray(x).astype(np.float32)
    hi = f16(xf)
    lo = f16(xf - hi.astype(np.float32))
    return hi, lo


def lstm1_x(x):
    """LSTM1's input operand [B,33,48] of a dense [B,33,C] count tensor: columns [hi (C) | 1 | lo (C) | 0..]."""
    x = np.asarray(x)
    C = x.shape[-1]
    hi, lo = hi_lo(x)
    out = np.zeros(x.shape[:-1] + (X1_COLS,))
    out[..., :C] = hi
    out[..., C] = 1.0
    out[..., C + 1:2 * C + 1] = lo
    return out


def windows(cols, starts):
    """The dense [B,33,C] tensor ``forward_windows`` reads: rows starts[b] .. +32 of the column matrix, zero outside it."""
    cols = np.asarray(cols)
    rows = np.asarray(starts, dtype=np.int64)[:, None] + np.arange(T)[None, :]
    ok = (rows >= 0) & (rows < cols.shape[0])
    out = cols[np.clip(rows, 0, cols.shape[0] - 1)]
    out[~ok] = 0
    return out


# ------------------------------------------------------------------------------------------------ layouts (c3b_internal.h)
def lstm_row(R, H):
    """``c3b_lstm_row``: torch gate row of row R of the recurrent kernels' permuted gate order."""
    pp, blk, r = R // 128, (R // 64) & 1, R % 64
    w, q = r // 16, r % 16
    return (2 * blk + (q >= 8)) * H + 32 * pp + 8 * w + (q & 7)


def lstm2_pg_row(C):
    """``c3b_lstm2_pg_row``: torch gate row of LSTM2 pre-gate column C in [0, 640) of one direction (gate-quad order)."""
    return (C & 3) * H2 + 32 * (C >> 7) + ((C & 127) >> 2)


PG_ROWS = np.array([lstm2_pg_row(C) for C in range(640)])


def pregates_torch_order(pg):
    """The "lstm2_pregates" tap [B,33,1280] (kernel column order) -> [2][B,33,640] in torch gate-row order per direction."""
    out = np.empty((2,) + pg.shape[:-1] + (640,))
    for d in range(2):
        out[d][..., PG_ROWS] = pg[..., d * 640:(d + 1) * 640]
    return out


# ------------------------------------------------------------------------------------------------ weights as finalize packs them
def _f32(sd, k):
    return np.asarray(sd[k], dtype=np.float32)


def gate_scale(H):
    """Per torch gate row: 0.5 for the sigmoid gates i, f, o (pre-halved), 1 for g."""
    s = np.full(4 * H, 0.5, dtype=np.float32)
    s[2 * H:3 * H] = 1.0
    return s


def _sfx(d):
    return "_l0_reverse" if d else "_l0"


def lstm1_weights(sd, d):
    """LSTM1's operand image of direction d in torch row order: [512][48 + 128] fp16 values; x columns [W_ih | b | W_ih | 0]."""
    wih, whh = _f32(sd, "LSTM1.weight_ih" + _sfx(d)), _f32(sd, "LSTM1.weight_hh" + _sfx(d))
    b = _f32(sd, "LSTM1.bias_ih" + _sfx(d)) + _f32(sd, "LSTM1.bias_hh" + _sfx(d))
    C = wih.shape[1]
    gs = gate_scale(H1)[:, None]
    w = np.zeros((4 * H1, X1_COLS + H1), dtype=np.float32)
    w[:, :C] = wih * gs
    w[:, C] = b * gs[:, 0]
    w[:, C + 1:2 * C + 1] = wih * gs
    w[:, X1_COLS:] = whh * gs
    return f16(w)


def lstm2_weights(sd, d):
    """LSTM2 of direction d in torch row order: (W_hh [640][160] fp16, proj2 weights [640][256] fp16, proj2 bias [640] fp32)."""
    gs = gate_scale(H2)
    whh = f16(_f32(sd, "LSTM2.weight_hh" + _sfx(d)) * gs[:, None])
    wp = f16(_f32(sd, "LSTM2.weight_ih" + _sfx(d)) * gs[:, None])
    bp = ((_f32(sd, "LSTM2.bias_ih" + _sfx(d)) + _f32(sd, "LSTM2.bias_hh" + _sfx(d))) * gs).astype(np.float64)
    return whh, wp, bp


def conv_weights(sd, i):
    """Convolution i (CONV_KEYS order) with BatchNorm folded in fp32 as finalize does: ([9 taps][cin][cout] fp16, bias fp32)."""
    conv, bn = CONV_KEYS[i]
    w, cb = _f32(sd, conv + ".weight"), _f32(sd, conv + ".bias")
    g, be = _f32(sd, bn + ".weight"), _f32(sd, bn + ".bias")
    mu, var = _f32(sd, bn + ".running_mean"), _f32(sd, bn + ".running_var")
    s = g / np.sqrt(var + BN_EPS)
    bias = (cb - mu) * s + be
    wf = w * s[:, None, None, None]
    if i == 0:
        wf = wf * (np.float32(1.0) / np.float32(100.0))
    cout, cin = w.shape[:2]
    return f16(wf).transpose(2, 3, 1, 0).reshape(9, cin, cout), bias.astype(np.float64)


def l4_weights(sd):
    return f16(_f32(sd, "L4.weight"))


# ------------------------------------------------------------------------------------------------ checks (max err / bound)
def bound_ratio(gpu, ref, S, fp16_out):
    """(max err / bound, max share of the accumulation allowance EPS*S + 2^-24 used once the fp16 output rounding's own
    allowance is taken off).  The first is what the checks assert; for fp16 outputs it can approach 1 by the rounding alone,
    so the second is what shows how much room EPS leaves."""
    if not np.size(ref):
        return 0.0, 0.0
    err = np.abs(np.asarray(gpu, dtype=np.float64) - ref)
    rnd = F16_ULP * np.abs(ref) if fp16_out else 0.0
    acc = EPS * S + TINY
    return float(np.max(err / (acc + rnd))), float(np.max(np.maximum(err - rnd, 0.0) / acc))


def _worst(a, b):
    return max(a[0], b[0]), max(a[1], b[1])


def gemm(a, w, bias=None, residual=None, relu=False):
    """(ref, S) of relu?(a @ w.T + bias + residual) in float64: a [M,K], w [N,K]."""
    a = np.asarray(a, dtype=np.float64)
    ref = a @ w.T
    S = np.abs(a) @ np.abs(w).T
    if bias is not None:
        ref = ref + bias
        S = S + np.abs(bias)
    if residual is not None:
        ref = ref + residual
        S = S + np.abs(residual)
    if relu:
        ref = np.maximum(ref, 0.0)
    return ref, S


def proj2_ratio(h1, pg, sd):
    """proj2: pre-gates [B,33,1280] (kernel order, fp16) from LSTM1's output h1 [B,33,256].  Returns bound_ratio's pair."""
    got = pregates_torch_order(pg)
    r = (0.0, 0.0)
    for d in range(2):
        _, wp, bp = lstm2_weights(sd, d)
        ref, S = gemm(h1.reshape(-1, 256), wp, bias=bp)
        r = _worst(r, bound_ratio(got[d].reshape(-1, 640), ref, S, True))
    return r


def lstm_ratio(u, su, whh, h, reverse, tau):
    """Teacher-forced check of one direction of a recurrence.

    u, su [B,33,4H]: the input part of the (pre-halved) gate pre-activations in torch row order and its S; whh [4H][H] the
    recurrent operand; h [B,33,H] the GPU's output of this direction.  Returns max |h - ref| / (tau + 2 EPS S_gates)."""
    B, _, G = u.shape
    H = G // 4
    hp = np.zeros_like(h, dtype=np.float64)
    if reverse:
        hp[:, :-1] = h[:, 1:]
    else:
        hp[:, 1:] = h[:, :-1]
    z = u + hp @ whh.T
    S = su + np.abs(hp) @ np.abs(whh).T
    sg = S[..., :H] + S[..., H:2 * H] + S[..., 2 * H:3 * H] + S[..., 3 * H:]
    c = np.zeros((B, H))
    r = 0.0
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        zt = z[:, t]
        i = 0.5 * np.tanh(zt[:, :H]) + 0.5
        f = 0.5 * np.tanh(zt[:, H:2 * H]) + 0.5
        g = np.tanh(zt[:, 2 * H:3 * H])
        o = 0.5 * np.tanh(zt[:, 3 * H:]) + 0.5
        c = f * c + i * g
        ref = o * np.tanh(c)
        r = max(r, float(np.max(np.abs(h[:, t] - ref) / (tau + 2 * EPS * sg[:, t]))))
    return r


def lstm1_ratio(xop, h1, sd, tau):
    """LSTM1 from its input operand xop [B,33,48] (the "lstm1_x" tap) to h1 [B,33,256]."""
    r = 0.0
    for d in range(2):
        w = lstm1_weights(sd, d)
        wx = w[:, :X1_COLS]
        u, su = xop @ wx.T, np.abs(xop) @ np.abs(wx).T
        r = max(r, lstm_ratio(u, su, w[:, X1_COLS:], h1[..., d * H1:(d + 1) * H1], d == 1, tau))
    return r


def lstm2_ratio(pg, h2, sd, tau):
    """LSTM2 from the GPU's pre-gates [B,33,1280] (the "lstm2_pregates" tap) to h2 [B,33,320]."""
    got = pregates_torch_order(pg)
    r = 0.0
    for d in range(2):
        whh, _, _ = lstm2_weights(sd, d)
        r = max(r, lstm_ratio(got[d], np.abs(got[d]), whh, h2[..., d * H2:(d + 1) * H2], d == 1, tau))
    return r


def conv_out(v):
    return (v - 1) // 2 + 1


def im2col(x, stride):
    """NHWC [B,h,w,c] -> [B,ho,wo,9*c] with k = tap*c + ci, tap = dh*3 + dw (pad 1): the kernel's k order."""
    B, h, w, c = x.shape
    ho, wo = (conv_out(h), conv_out(w)) if stride == 2 else (h, w)
    xp = np.zeros((B, h + 2, w + 2, c))
    xp[:, 1:h + 1, 1:w + 1] = x
    cols = np.empty((B, ho, wo, 9, c))
    for dh in range(3):
        for dw in range(3):
            cols[:, :, :, dh * 3 + dw] = xp[:, dh:dh + stride * ho:stride, dw:dw + stride * wo:stride]
    return cols.reshape(B, ho, wo, 9 * c)


def conv_ratio(x, out, wb, stride, residual=None):
    """One convolution (+bias, +residual, ReLU) from its NHWC input x to the GPU's NHWC output; wb = conv_weights(...).
    Returns bound_ratio's pair."""
    w, bias = wb
    cols = im2col(np.asarray(x, dtype=np.float64), stride)
    B, ho, wo, K = cols.shape
    res = None if residual is None else np.asarray(residual, dtype=np.float64).reshape(-1, w.shape[2])
    ref, S = gemm(cols.reshape(-1, K), w.reshape(K, -1).T, bias=bias, residual=res, relu=True)
    return bound_ratio(np.asarray(out).reshape(-1, w.shape[2]), ref, S, True)


def l4_ratio(act, z4, sd):
    """L4 (fp32 output, split-K partials summed, no bias) from its [B, l4_in] fp16 input.  Returns bound_ratio's pair."""
    ref, S = gemm(act, l4_weights(sd))
    return bound_ratio(z4, ref, S, False)


def selu(x):
    return SELU_SCALE * np.where(x > 0, x, SELU_ALPHA * np.expm1(np.minimum(x, 0)))


def heads(z4, sd, nheads):
    """float64 heads on the L4 pre-activation z4 (no bias): SELU(z4 + b4) -> per head SELU(L5) -> softmax(SELU(Y))."""
    a4 = selu(np.asarray(z4, dtype=np.float64) + _f32(sd, "L4.bias"))
    outs = []
    for l5, y in HEAD_NAMES[:nheads]:
        a5 = selu(a4 @ _f32(sd, l5 + ".weight").T.astype(np.float64) + _f32(sd, l5 + ".bias"))
        v = selu(a5 @ _f32(sd, y + ".weight").T.astype(np.float64) + _f32(sd, y + ".bias"))
        e = np.exp(v - v.max(axis=1, keepdims=True))
        outs.append(e / e.sum(axis=1, keepdims=True))
    return np.concatenate(outs, axis=1)


def spp(x):
    """Pyramid pooling (3x3, 2x2, 1x1; TF-'SAME' zero padding, NHWC flatten) of an NHWC map: exact on fp16 values."""
    return pyramid_pool(np.asarray(x, dtype=np.float64).transpose(0, 3, 1, 2))
