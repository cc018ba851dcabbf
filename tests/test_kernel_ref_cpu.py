"""The per-layer checker of ``kernel_ref.py`` on the CPU: it must accept an fp32 emulation of each kernel that carries the
kernel's own rounding (fp32 accumulation noise, ``tanh.approx`` error, fp16 outputs), and it must reject each of a set of
one-line kernel mistakes.  Also pins the hi/lo split of LSTM1's raw counts."""
import numpy as np
import pytest

import kernel_ref as kr
from clair3_b200 import synth

ACC_NOISE = 2.0 ** -20          # emulated fp32 accumulation error, relative to S (a quarter of kr.EPS)
TANH_F32 = 2.0 ** -11           # tanh.approx.f32: about 2^-11 relative
TANH_F16 = 2.0 ** -10           # tanh.approx.f16x2 before the fp16 rounding of its result


# ---------------------------------------------------------------------------------------------- hi/lo split of the raw counts
def test_hi_lo_split_exact_up_to_67552():
    x = np.arange(-67552, 67553)
    hi, lo = kr.hi_lo(x)
    assert np.array_equal(hi + lo, x)
    assert np.abs(hi).max() <= 65504 and np.abs(lo).max() <= 2048


def test_hi_lo_split_rounds_past_67552_and_saturates_past_131008():
    for s in (1, -1):
        hi, lo = kr.hi_lo(s * np.array([67553]))
        assert hi + lo != s * 67553 and abs(hi + lo - s * 67553) == 1
        x = s * np.arange(0, 131009)
        hi, lo = kr.hi_lo(x)
        err = np.abs(hi + lo - x)
        assert err.max() == 16
        assert np.flatnonzero(err)[0] == 67553
        assert err.max() / 131008 <= 2.0 ** -12
        big = s * np.array([131008, 131009, 131023, 131024, 200000, 1 << 24])
        hi, lo = kr.hi_lo(big)
        assert np.array_equal(hi + lo, s * np.full(len(big), 131008.0))


def test_f16_matches_numpy_and_saturates():
    v = np.array([0.0, 1e-8, 2.0 ** -25, 2.0 ** -24, 1.0 + 2.0 ** -11, 65504, 65519.99, 65520, 1e9, -65520, np.float32(np.inf)])
    got = kr.f16(v)
    assert list(got[:6]) == [0.0, 0.0, 0.0, 2.0 ** -24, 1.0, 65504]
    assert list(got[6:]) == [65504, 65504, 65504, -65504, 65504]


def test_gate_layouts_restated():
    """c3b_lstm_row is a permutation whose 64-row block 2p holds gates i, f and block 2p+1 gates g, o of units 32p .. 32p+31;
    c3b_lstm2_pg_row puts the four gates of one unit in four adjacent columns."""
    for H in (kr.H1, kr.H2):
        rows = [kr.lstm_row(R, H) for R in range(4 * H)]
        assert sorted(rows) == list(range(4 * H))
        for R, row in enumerate(rows):
            gate, unit = divmod(row, H)
            assert unit // 32 == R // 128 and gate // 2 == (R // 64) % 2
    assert sorted(kr.PG_ROWS.tolist()) == list(range(640))
    for C in range(0, 640, 4):
        units = {kr.PG_ROWS[C + g] % kr.H2 for g in range(4)}
        assert len(units) == 1 and [kr.PG_ROWS[C + g] // kr.H2 for g in range(4)] == [0, 1, 2, 3]


# ---------------------------------------------------------------------------------------------- fp32 emulations
def _rng(seed):
    return np.random.default_rng(seed)


def emu_gemm(a, w, r, bias=None, residual=None, relu=False, fp16_out=True):
    """fp32 GEMM with accumulation noise of ACC_NOISE * S, then the kernel's epilogue and output rounding."""
    a = np.asarray(a, dtype=np.float64)
    acc = (a.astype(np.float32) @ w.astype(np.float32).T).astype(np.float64)
    S = np.abs(a) @ np.abs(w).T
    acc += r.uniform(-1, 1, acc.shape) * ACC_NOISE * S
    if bias is not None:
        acc = acc + bias.astype(np.float32)
    if residual is not None:
        acc = acc + residual
    if relu:
        acc = np.maximum(acc, 0)
    return kr.f16(acc) if fp16_out else acc.astype(np.float32).astype(np.float64)


def _tanh(x, r, mufu16):
    if mufu16:
        x = kr.f16(x)
        return kr.f16(np.tanh(x) * (1 + r.uniform(-1, 1, np.shape(x)) * TANH_F16))
    return np.tanh(x) * (1 + r.uniform(-1, 1, np.shape(x)) * TANH_F32)


def emu_lstm(u, su, whh, r, reverse, mufu16=False, mutation=None):
    """One direction of the recurrent kernel: gates = u + W_hh h_prev in fp32 with accumulation noise, approximate gate
    activations, fp32 cell state, fp16 h.  mutation 'reverse_reads_prev': the reverse direction reads h_{t-1}."""
    B, _, G = u.shape
    H = G // 4
    hs = np.zeros((B, kr.T, H))
    c = np.zeros((B, H), dtype=np.float32)
    for t in (range(kr.T - 1, -1, -1) if reverse else range(kr.T)):
        tp = t + 1 if reverse else t - 1
        if mutation == "reverse_reads_prev" and reverse:
            tp = t - 1
        hp = hs[:, tp] if 0 <= tp < kr.T else np.zeros((B, H))
        z = u[:, t] + hp @ whh.T
        z += r.uniform(-1, 1, z.shape) * ACC_NOISE * (su[:, t] + np.abs(hp) @ np.abs(whh).T)
        sg = lambda v: (kr.f16(0.5 * _tanh(v, r, True) + 0.5) if mufu16 else 0.5 * _tanh(v, r, False) + 0.5)  # noqa: E731
        i, f, o = sg(z[:, :H]), sg(z[:, H:2 * H]), sg(z[:, 3 * H:])
        g = _tanh(z[:, 2 * H:3 * H], r, mufu16)
        ig = kr.f16(i * g) if mufu16 else i * g
        c = (f * c + ig).astype(np.float32)
        hs[:, t] = kr.f16(o * _tanh(c.astype(np.float64), r, mufu16))
    return hs


def _pileup_case(seed=5, batch=6):
    sd = synth.pileup_state_dict(False, seed=seed)
    x = synth.pileup_inputs(batch, seed=seed)
    x[0, 3, :4] = [70000, -90000, 3000, 131008]
    return sd, x


def emu_lstm1(sd, xop, r, mufu16=False, mutation=None):
    out = []
    for d in range(2):
        w = kr.lstm1_weights(sd, d)
        if mutation == "bias_on_wrong_gate" and d == 0:
            C = 18
            w = w.copy()
            w[[5, kr.H1 + 5], C] = w[[kr.H1 + 5, 5], C]     # unit 5: the i and f gate biases trade places
        wx = w[:, :kr.X1_COLS]
        out.append(emu_lstm(xop @ wx.T, np.abs(xop) @ np.abs(wx).T, w[:, kr.X1_COLS:], r, d == 1, mufu16,
                            mutation if d == 1 else None))
    return np.concatenate(out, axis=-1)


def emu_proj2(sd, h1, r, mutation=None):
    """-> the "lstm2_pregates" tap, kernel column order.  mutation 'dropped_kgroup': k-group 3 missing from one row tile."""
    B = h1.shape[0]
    a = h1.reshape(-1, 256).copy()
    if mutation == "dropped_kgroup":
        a[:128 if B * kr.T > 128 else B * kr.T, 24:32] = 0
    pg = np.empty((B, kr.T, 1280))
    for d in range(2):
        _, wp, bp = kr.lstm2_weights(sd, d)
        pgt = emu_gemm(a, wp, r, bias=bp).reshape(B, kr.T, 640)
        pg[..., d * 640:(d + 1) * 640] = pgt[..., kr.PG_ROWS]
    return pg


def emu_lstm2(sd, pg, r, mufu16=False):
    got = kr.pregates_torch_order(pg)
    return np.concatenate([emu_lstm(got[d], np.abs(got[d]), kr.lstm2_weights(sd, d)[0], r, d == 1, mufu16) for d in range(2)],
                          axis=-1)


def emu_l4(act, sd, r, nsplit=5, mutation=None):
    """Split-K L4: fp32 partial sums over 64-wide k-chunks, summed in order.  mutation 'missing_partial': the last is lost."""
    w = kr.l4_weights(sd)
    K = act.shape[1]
    per = -(-K // 64 // nsplit) * 64
    parts = [emu_gemm(act[:, k0:k0 + per], w[:, k0:k0 + per], r, fp16_out=False) for k0 in range(0, K, per)]
    if mutation == "missing_partial":
        parts = parts[:-1]
    return np.sum(parts, axis=0, dtype=np.float32).astype(np.float64)


def emu_conv(x, wb, stride, r, residual=None, mutation=None):
    """mutations: 'swapped_tap' (taps (0,1) and (1,0) trade weights); 'border_from_neighbour' (site b's top border row holds
    the last real row of site b-1)."""
    w, bias = wb
    if mutation == "swapped_tap":
        w = w.copy()
        w[[1, 3]] = w[[3, 1]]
    cols = kr.im2col(x, stride)
    if mutation == "border_from_neighbour":
        B, h, wd, c = x.shape
        xp = np.zeros((B, h + 2, wd + 2, c))
        xp[:, 1:h + 1, 1:wd + 1] = x
        xp[1:, 0, 1:wd + 1] = x[:-1, -1]
        ho, wo = cols.shape[1:3]
        cols = np.stack([xp[:, dh:dh + stride * ho:stride, dw:dw + stride * wo:stride] for dh in range(3) for dw in range(3)],
                        axis=3).reshape(cols.shape)
    B, ho, wo, K = cols.shape
    res = None if residual is None else residual.reshape(-1, w.shape[2])
    return emu_gemm(cols.reshape(-1, K), w.reshape(K, -1).T, r, bias=bias, residual=res, relu=True).reshape(B, ho, wo, -1)


@pytest.mark.parametrize("mufu16", [False, True])
def test_pileup_emulation_passes_the_checker(mufu16):
    sd, x = _pileup_case()
    r = _rng(1)
    tau = kr.TAU_MUFU16 if mufu16 else kr.TAU_F32
    xop = kr.lstm1_x(x)
    h1 = emu_lstm1(sd, xop, r, mufu16)
    pg = emu_proj2(sd, h1, r)
    h2 = emu_lstm2(sd, pg, r, mufu16)
    z4 = emu_l4(h2.reshape(len(x), -1), sd, r)
    assert kr.lstm1_ratio(xop, h1, sd, tau) <= 1.0
    assert kr.proj2_ratio(h1, pg, sd)[0] <= 1.0
    assert kr.lstm2_ratio(pg, h2, sd, tau) <= 1.0
    assert kr.l4_ratio(h2.reshape(len(x), -1), z4, sd)[0] <= 1.0
    y = kr.heads(z4.astype(np.float32), sd, 2).astype(np.float32)
    assert np.abs(y - kr.heads(z4, sd, 2)).max() <= kr.HEADS_TOL


def _fa_case(batch=3, depth=17, seed=6):
    sd = synth.fa_state_dict(True, channels=8, seed=seed)
    x = kr.f16(synth.fa_inputs(batch, depth=depth, channels=8, seed=seed).astype(np.float32))
    return sd, x


def test_conv_emulation_passes_the_checker():
    sd, x = _fa_case()
    r = _rng(2)
    cur = x
    for lvl in range(3):
        i = 3 * lvl
        a0 = emu_conv(cur, kr.conv_weights(sd, i), 2, r)
        a1 = emu_conv(a0, kr.conv_weights(sd, i + 1), 1, r)
        a2 = emu_conv(a1, kr.conv_weights(sd, i + 2), 1, r, residual=a0)
        assert kr.conv_ratio(cur, a0, kr.conv_weights(sd, i), 2)[0] <= 1.0
        assert kr.conv_ratio(a0, a1, kr.conv_weights(sd, i + 1), 1)[0] <= 1.0
        assert kr.conv_ratio(a1, a2, kr.conv_weights(sd, i + 2), 1, residual=a0)[0] <= 1.0
        cur = a2
    sp = kr.spp(cur)
    z4 = emu_l4(sp, sd, r, nsplit=3)
    assert kr.l4_ratio(sp, z4, sd)[0] <= 1.0


@pytest.mark.parametrize("mutation", ["dropped_kgroup", "swapped_tap", "bias_on_wrong_gate", "reverse_reads_prev",
                                      "border_from_neighbour", "missing_partial"])
def test_checker_rejects_one_line_mistakes(mutation):
    r = _rng(3)
    if mutation in ("swapped_tap", "border_from_neighbour"):
        sd, x = _fa_case()
        a0 = emu_conv(x, kr.conv_weights(sd, 0), 2, r)
        a1 = emu_conv(a0, kr.conv_weights(sd, 1), 1, r, mutation=mutation)
        assert kr.conv_ratio(a0, a1, kr.conv_weights(sd, 1), 1)[0] > 1.0
        return
    sd, x = _pileup_case()
    xop = kr.lstm1_x(x)
    if mutation in ("bias_on_wrong_gate", "reverse_reads_prev"):
        h1 = emu_lstm1(sd, xop, r, mutation=mutation)
        assert kr.lstm1_ratio(xop, h1, sd, kr.TAU_F32) > 1.0
        return
    h1 = emu_lstm1(sd, xop, r)
    if mutation == "dropped_kgroup":
        assert kr.proj2_ratio(h1, emu_proj2(sd, h1, r, mutation), sd)[0] > 1.0
        return
    pg = emu_proj2(sd, h1, r)
    act = emu_lstm2(sd, pg, r).reshape(len(x), -1)
    assert kr.l4_ratio(act, emu_l4(act, sd, r, mutation=mutation), sd)[0] > 1.0
