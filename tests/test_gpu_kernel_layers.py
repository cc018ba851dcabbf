"""Every tensor-core layer of both networks checked on its own, per element, against the float64 operand-precision reference
of ``kernel_ref.py`` (``pytest -m gpu`` on an H100).

Each kernel's reference is computed from the GPU's own input tap, so errors do not carry over from earlier layers, and each
element must satisfy the bound of its layer (see ``kernel_ref``): ingest and pyramid pooling bit-exact; proj2, the nine
convolutions and L4 within ``EPS*S + 2^-11|ref| + 2^-24``; the recurrences, teacher-forced, within ``tau + 2*EPS*S_gates``;
the heads within 2e-5 on the probabilities.

Edges covered: pileup batches 1, 127, 128, 129, 600 (uneven proj2 tile ranges), 1024 and 2200 (heads' 4-head ``pairs == 1``
path with chunk_sites=4096); channels 1, 18, 23; LSTM tiles 16/32/64 x lstm_wg 1/2 x lstm_mufu16 0/1 at 129 sites; realistic,
uniform, int8-wrapped, fractional float32, overhanging ``forward_windows`` inputs and counts around every edge of the hi/lo
split; full-alignment depths 17, 55, 89, 512, channels 1, 8, 9, 16, batches 1, 3, 129, 256, int8 extremes, a 3-site call
reusing a 256-site planar layout; add_indel on and off, batches 511 / 512 on both sides of the heads' site-group switch;
synthetic weights, LSTM weights x4 (saturated gates) and BN gammas near 1e-4 (fp16-subnormal folded conv weights).

Observed maxima of err/bound over this whole file on an H100 80GB HBM3 (SXM) at a 400 W power limit:
    lstm1_x, spp                      bit-exact
    lstm1 / lstm2, fp32 tanh.approx   0.245 / 0.247      (tau = 2^-10)
    lstm1 / lstm2, lstm_mufu16        0.336 / 0.229      (tau = 2^-5)
    proj2                             0.978, accumulation share 0.028
    conv0 .. conv8                    0.93 .. 0.985, accumulation share 0.0018 .. 0.057
    L4 pileup / full-alignment        0.020 / 0.011      (fp32 output: accumulation only)
    heads                             0.143              (2.9e-6 on the probabilities)
For the fp16 outputs (proj2, the convolutions) err/bound approaches 1 by the output rounding alone, which its 2^-11|ref| term
covers exactly; the "accumulation share" is what is left of the error once that term is taken off, over EPS*S + 2^-24, and
shows EPS = 2^-18 is more than 2x above what the fp32 accumulation needs.  tau and the heads tolerance are also 2x or more above
the observed maxima.
"""
import json
import os

import numpy as np
import pytest
import torch

import kernel_ref as kr

pytestmark = pytest.mark.gpu

OBSERVED = {}


def _record(case, ratios):
    for k, v in ratios.items():
        OBSERVED[k] = max(OBSERVED.get(k, 0.0), v)
    print("KERNEL_LAYERS", case, json.dumps(ratios, sort_keys=True))
    out = os.environ.get("C3B_REPORT_DIR")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "kernel_layers.json"), "w") as f:
            json.dump(OBSERVED, f, indent=1, sort_keys=True)
    bad = {k: v for k, v in ratios.items() if not v <= 1.0}
    assert not bad, (case, bad)


def _sd_t(sd):
    return {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}


def _model(cls, sd, channels, add_indel, **opts):
    m = cls(add_indel_length=add_indel, predict=True, input_channels=channels)
    m.set_option("taps", 1)
    for k, v in opts.items():
        m.set_option(k, v)
    m.to(torch.device("cuda"))
    m.load_state_dict(_sd_t(sd))
    return m


def _sites(n, extra=8, seed=0):
    """Sites the per-element references run on: all of a small batch; otherwise the first and last site of every 128-site tile
    (so every row tile of every GEMM is visited, including the last, partial one) plus a few random ones."""
    if n <= 160:
        return np.arange(n)
    s = {0, 1, n - 2, n - 1}
    for b0 in range(0, n, 128):
        s.update((b0, min(b0 + 127, n - 1)))
    s.update(np.random.default_rng(seed).integers(0, n, extra).tolist())
    return np.array(sorted(s))


def _tap(m, name, n, *shape):
    return m.tap(name).reshape(n, *shape).astype(np.float64)


# ---------------------------------------------------------------------------------------------- pileup
def check_pileup(case, m, x_dense, sd, y, nheads, tau=kr.TAU_F32, rnn=True):
    n = len(y)
    idx = _sites(n)
    h2 = _tap(m, "lstm2", n, kr.T, 320)
    z4 = _tap(m, "l4_pre", n, 128)
    r = {}
    r["l4"], r["l4_acc"] = kr.l4_ratio(h2[idx].reshape(len(idx), -1), z4[idx], sd)
    hd = float(np.abs(y.astype(np.float64) - kr.heads(z4, sd, nheads)).max())
    r["heads"] = hd / kr.HEADS_TOL
    if rnn:
        xop = _tap(m, "lstm1_x", n, kr.T, kr.X1_COLS)
        want = kr.lstm1_x(x_dense)
        assert np.array_equal(xop, want), (case, "lstm1_x", np.argwhere(xop != want)[:5])
        h1 = _tap(m, "lstm1", n, kr.T, 256)
        pg = _tap(m, "lstm2_pregates", n, kr.T, 1280)
        mu = "_mufu16" if tau == kr.TAU_MUFU16 else ""
        r["lstm1" + mu] = kr.lstm1_ratio(xop[idx], h1[idx], sd, tau)
        r["proj2"], r["proj2_acc"] = kr.proj2_ratio(h1[idx], pg[idx], sd)
        r["lstm2" + mu] = kr.lstm2_ratio(pg[idx], h2[idx], sd, tau)
    _record(case, r)


def _run_p(sd, x, channels=18, add_indel=False, **opts):
    from clair3_b200.model import Clair3_P
    m = _model(Clair3_P, sd, channels, add_indel, **opts)
    y = m(torch.from_numpy(x).cuda()).cpu().numpy()
    return m, y


@pytest.mark.parametrize("batch", [1, 127, 128, 129, 600, 1024])
def test_pileup_layers_across_batch_sizes(batch):
    from clair3_b200 import synth
    sd = synth.pileup_state_dict(False, seed=41)
    x = synth.pileup_inputs(batch, seed=41)
    m, y = _run_p(sd, x)
    check_pileup("pileup_b%d" % batch, m, x, sd, y, 2)


@pytest.mark.parametrize("channels", [1, 23])
def test_pileup_layers_other_channel_counts(channels):
    """The generic ingest branch (channels != 18) and LSTM1 operands with 1 and 23 real x columns."""
    from clair3_b200 import synth
    sd = synth.pileup_state_dict(False, channels=channels, seed=42)
    r = np.random.default_rng(42)
    x = r.integers(-60, 61, size=(129, kr.T, channels)).astype(np.int32)
    x[r.random(x.shape) < 0.01] = 70000
    m, y = _run_p(sd, x, channels)
    check_pileup("pileup_c%d" % channels, m, x, sd, y, 2)


@pytest.mark.parametrize("tile", [16, 32, 64])
@pytest.mark.parametrize("wg", [1, 2])
@pytest.mark.parametrize("mufu16", [0, 1])
def test_pileup_recurrence_variants(tile, wg, mufu16):
    """Every LSTM kernel variant at 129 sites (two 128-site tiles, the second with one real site); lstm2 runs min(tile, 32)."""
    from clair3_b200 import synth
    sd = synth.pileup_state_dict(False, seed=43)
    x = synth.pileup_inputs(129, seed=43)
    m, y = _run_p(sd, x, lstm_tile=tile, lstm_wg=wg, lstm_mufu16=mufu16)
    check_pileup("pileup_t%d_wg%d_mufu%d" % (tile, wg, mufu16), m, x, sd, y, 2, kr.TAU_MUFU16 if mufu16 else kr.TAU_F32)


def _special_counts(batch, seed):
    vals = np.array([2047, 2048, 2049, 65504, 65519, 65520, 67552, 67553, 131008, 131009, 200000, 1000000])
    vals = np.concatenate([vals, -vals])
    r = np.random.default_rng(seed)
    x = r.integers(0, 50, size=(batch, kr.T, 18))
    mask = r.random(x.shape) < 0.05
    x[mask] = r.choice(vals, size=int(mask.sum()))
    x[0, :, :] = np.resize(vals, (kr.T, 18))          # every special count at least once
    return x.astype(np.int32)


@pytest.mark.parametrize("kind", ["uniform", "int8_wrap", "float_fraction", "special_counts"])
def test_pileup_layers_input_kinds(kind):
    from clair3_b200 import synth
    sd = synth.pileup_state_dict(True, seed=44)
    if kind == "uniform":
        x = synth.pileup_inputs(129, seed=44, realistic=False)
    elif kind == "int8_wrap":
        x = synth.pileup_inputs(129, seed=44, dtype=np.int8)
    elif kind == "float_fraction":
        x = (np.random.default_rng(44).uniform(-80, 80, size=(129, kr.T, 18))).astype(np.float32)
    else:
        x = _special_counts(129, 44)
    m, y = _run_p(sd, x, add_indel=True)
    check_pileup("pileup_" + kind, m, x, sd, y, 4)


def test_pileup_layers_overhanging_windows():
    """forward_windows: windows that start before the column matrix and run past its end read zero rows."""
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_P
    sd = synth.pileup_state_dict(False, seed=45)
    cols = synth.pileup_inputs(20, seed=45).reshape(-1, 18)[:600].astype(np.int64)
    starts = np.concatenate([np.arange(-40, 640, 7), [-32, 599, 0, 567]]).astype(np.int64)
    m = _model(Clair3_P, sd, 18, False)
    y = m.forward_windows(torch.from_numpy(cols), torch.from_numpy(starts)).numpy()
    check_pileup("pileup_windows", m, kr.windows(cols, starts), sd, y, 2)


def test_pileup_layers_saturated_gates():
    """LSTM weights x4: most gates saturate, the cell state runs to its extremes."""
    from clair3_b200 import synth
    sd = synth.pileup_state_dict(False, seed=46)
    for k in sd:
        if k.startswith("LSTM"):
            sd[k] = (np.asarray(sd[k]) * 4).astype(np.float32)
    x = synth.pileup_inputs(129, seed=46)
    for mufu16 in (0, 1):
        m, y = _run_p(sd, x, lstm_mufu16=mufu16)
        check_pileup("pileup_lstm_x4_mufu%d" % mufu16, m, x, sd, y, 2, kr.TAU_MUFU16 if mufu16 else kr.TAU_F32)


@pytest.mark.parametrize("batch,add_indel,chunk", [(511, False, 0), (512, True, 0), (2200, True, 4096)])
def test_tail_layers(batch, add_indel, chunk):
    """L4 and the heads on both sides of the heads' 8/16-site group switch, and one 2200-site chunk (more than 132 site
    groups: the 4-head kernel walks both head pairs in one block, with a different split-K count)."""
    from clair3_b200 import synth
    sd = synth.pileup_state_dict(add_indel, seed=47)
    x = synth.pileup_inputs(batch, seed=47)
    m, y = _run_p(sd, x, add_indel=add_indel, chunk_sites=chunk)
    check_pileup("tail_b%d_indel%d" % (batch, add_indel), m, x, sd, y, 4 if add_indel else 2, rnn=False)


# ---------------------------------------------------------------------------------------------- full alignment
def check_fa(case, m, x, sd, y, nheads):
    n, depth = x.shape[:2]
    hh, ww = [depth], [33]
    for _ in range(3):
        hh.append(kr.conv_out(hh[-1]))
        ww.append(kr.conv_out(ww[-1]))
    idx = np.unique([0, 1, n // 2, n - 2, n - 1]) if n > 4 else np.arange(n)     # every pixel of these sites: borders included
    taps = {}
    for i, name in enumerate(kr.CONV_TAPS):
        lv = i // 3 + 1
        taps[name] = _tap(m, name, n, hh[lv], ww[lv], 64 << (i // 3))[idx]
    r = {}
    prev = kr.f16(np.asarray(x, dtype=np.float32)[idx])
    for i, name in enumerate(kr.CONV_TAPS):
        l, j = divmod(i, 3)
        stem, mid = kr.CONV_TAPS[3 * l], kr.CONV_TAPS[3 * l + 1]
        inp = prev if j == 0 else taps[stem] if j == 1 else taps[mid]
        res = taps[stem] if j == 2 else None
        r["conv%d" % i], r["conv%d_acc" % i] = kr.conv_ratio(inp, taps[name], kr.conv_weights(sd, i), 2 if j == 0 else 1, res)
        if j == 2:
            prev = taps[name]
    rb3 = _tap(m, "res_block3", n, hh[3], ww[3], 256)
    sp = _tap(m, "spp", n, 3584)
    assert np.array_equal(sp, kr.spp(rb3)), (case, "spp")
    z4 = _tap(m, "l4_pre", n, 256)
    r["l4_fa"], r["l4_fa_acc"] = kr.l4_ratio(sp[idx], z4[idx], sd)
    r["heads"] = float(np.abs(y.astype(np.float64) - kr.heads(z4, sd, nheads)).max()) / kr.HEADS_TOL
    _record(case, r)


def _run_f(sd, x, channels, add_indel=True, m=None):
    from clair3_b200.model import Clair3_F
    if m is None:
        m = _model(Clair3_F, sd, channels, add_indel)
    y = m(torch.from_numpy(x).cuda()).cpu().numpy()
    return m, y


@pytest.mark.parametrize("depth,channels,batch", [(89, 8, 1), (17, 1, 129), (55, 9, 3), (512, 16, 3), (89, 8, 256)])
def test_full_alignment_layers(depth, channels, batch):
    from clair3_b200 import synth
    sd = synth.fa_state_dict(True, channels=channels, seed=51)
    x = synth.fa_inputs(batch, depth=depth, channels=channels, seed=51, realistic=channels >= 5)
    m, y = _run_f(sd, x, channels)
    check_fa("fa_d%d_c%d_b%d" % (depth, channels, batch), m, x, sd, y, 4)


def test_full_alignment_layers_int8_extremes_and_layout_reuse():
    """Inputs at -128 / 127 on a 256-site call, then a 3-site call on the same model that reuses the 256-site planar layout."""
    from clair3_b200 import synth
    sd = synth.fa_state_dict(False, channels=8, seed=52)
    r = np.random.default_rng(52)
    x = r.choice(np.array([-128, 127, 0], dtype=np.int8), size=(256, 55, 33, 8))
    m, y = _run_f(sd, x, 8, add_indel=False)
    check_fa("fa_int8_extremes", m, x, sd, y, 2)
    x3 = synth.fa_inputs(3, depth=55, channels=8, seed=53)
    m, y3 = _run_f(sd, x3, 8, m=m)
    check_fa("fa_reuse_3_after_256", m, x3, sd, y3, 2)


def test_full_alignment_layers_tiny_bn_gammas():
    """BN gammas near 1e-4: the folded conv weights land in fp16's subnormal range (conv1's, with the 1/100 scale, partly
    flush to zero); the reference packs them the same way."""
    from clair3_b200 import synth
    sd = synth.fa_state_dict(True, channels=8, seed=54)
    r = np.random.default_rng(54)
    for conv, bn in kr.CONV_KEYS:
        sd[bn + ".weight"] = (r.uniform(0.5, 1.5, sd[bn + ".weight"].shape) * 1e-4).astype(np.float32)
    x = synth.fa_inputs(3, depth=55, channels=8, seed=54)
    m, y = _run_f(sd, x, 8)
    check_fa("fa_tiny_gamma", m, x, sd, y, 4)
