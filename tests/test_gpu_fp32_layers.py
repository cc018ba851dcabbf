"""Every layer of the fp32 CUDA-core debug path (option ``precision = 1``, ``kernels_fp32.cu``) checked on its own, per element,
against the float64 references of ``kernel_ref.py``'s fp32 section (``pytest -m gpu`` on an H100); and the bitwise properties
that let the per-layer guarantees of both paths carry over to the calls production makes.

Each layer's reference is computed from the GPU's own input tap: the ingest / window gather and the pyramid pooling must be
bit-exact; the nine convolutions and L4 within ``EPS32*S + 2^-24``; the recurrences, teacher-forced from the GPU's own h,
within ``TAU32 + 2*EPS32*S_gates``; the heads within 2e-5 on the probabilities.

Edges covered: pileup batches 1, 7, 8, 9 (dense_f32's 8-site groups), 129, 1024 and 2200 (chunk_sites=4096); channels 1, 18, 23
(LSTM1 stages its inputs one per thread; LSTM2 stages 256 inputs with 160 threads, twice for the first 96); L4's K = 10 560
ending in a 64-wide partial chunk; add_indel on and off; realistic, uniform, int8-wrapped, fractional float32 and int32 counts
above 2^24; ``forward_windows`` overhanging and bounded on int8 / int32 / int64 / float32 matrices; LSTM
weights x4 (saturated gates); full-alignment depths 17 (153 pixels per site at level 1: 4-pixel conv blocks straddle two sites),
55, 89, 512 (padded pyramid windows at 17 and 512), channels 1, 8, 9, 16, batches 1, 3, 129, 256, int8 extremes.  L4, the heads,
the ingest and the pooling are checked at every site, so both sides of every 8-site group boundary; the recurrences at every
site of batches up to 160 and a sample of larger ones (one block per site: no work is split across sites); the convolutions at
every pixel of a few sites and at every 4-pixel block that straddles two sites.

Observed maxima of err/bound over this whole file on an H100 80GB HBM3 (SXM) at a 700 W power limit:
    lstm1_in, spp                 bit-exact
    lstm1 / lstm2                 0.0584 / 0.00727   (TAU32 = 2^-16)
    conv0 .. conv8                0.152 .. 0.250     (EPS32 = 2^-19)
    L4 pileup / full-alignment    0.1717 / 0.1720
    heads                         0.1722             (3.44e-6 on the probabilities)
(as ``_record`` writes them to fp32_layers.json under C3B_REPORT_DIR; the three near 0.172 are independent maxima that happen
to agree to three digits.)  Every bound is 4x or more above what the kernels need.  EPS32 = 2^-20 left the convolutions at
0.50, so it is 2^-19; K_max * EPS32 = 0.02 stays far below 1/8.  One-line mistakes made in kernels_fp32.cu (gate f reading gate
i's bias, dense_f32 skipping L4's partial last k-chunk, conv3x3_f32 taking a straddling block's site from its first pixel)
exceeded these bounds 900 times or more, and without the fp32 branch's ``w->fa_zeroed = false`` in c3b_api.cu
test_precision_switching_full_alignment fails.  The whole file runs in about 30 s.

The bitwise properties (``torch.equal``):
* fp32 batch invariance: every fp32 kernel computes a site in a fixed order, independent of its neighbours (dense_f32 and
  conv3x3_f32 accumulate sequentially; the heads get one split-K partial, and their 8/16-site grouping does not change the
  arithmetic), so a site's output row is the same across batch sizes, chunk_sites, its position in the batch, concurrent
  streams and input dtypes that hold its values exactly.
* Precision switching on one model and stream: tensor-core, fp32, tensor-core again gives what models that never switched give.
  The fp32 full-alignment path overwrites the planar region the tensor-core path keeps zero-bordered; the next tensor-core call
  must clear it again.
* Debug options: ``taps``, ``profile`` and ``lstm_trace`` leave every output unchanged on both paths, so the per-layer guarantees
  (measured with ``taps = 1``) hold for production calls (``taps = 0``).
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
    print("FP32_LAYERS", case, json.dumps(ratios, sort_keys=True))
    out = os.environ.get("C3B_REPORT_DIR")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "fp32_layers.json"), "w") as f:
            json.dump(OBSERVED, f, indent=1, sort_keys=True)
    bad = {k: v for k, v in ratios.items() if not v <= 1.0}
    assert not bad, (case, bad)


def _sd_t(sd):
    return {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}


def _model(cls, sd, channels, add_indel, precision=1, **opts):
    m = cls(add_indel_length=add_indel, predict=True, input_channels=channels)
    m.set_option("precision", precision)
    for k, v in opts.items():
        m.set_option(k, v)
    m.to(torch.device("cuda"))
    m.load_state_dict(_sd_t(sd))
    return m


def _sites(n, extra=8, seed=0):
    """Sites the recurrences' references run on: all of a batch up to 160; otherwise the first and last site of every
    128-site stretch plus a few random ones."""
    if n <= 160:
        return np.arange(n)
    s = {0, 1, n - 2, n - 1}
    for b0 in range(0, n, 128):
        s.update((b0, min(b0 + 127, n - 1)))
    s.update(np.random.default_rng(seed).integers(0, n, extra).tolist())
    return np.array(sorted(s))


def _tap(m, name, n, *shape):
    return m.tap(name).reshape(n, *shape)


def _l4_ratio(act, z4, sd):
    return max(kr.l4_32_ratio(act[b0:b0 + 256].astype(np.float64), z4[b0:b0 + 256], sd) for b0 in range(0, len(act), 256))


# ---------------------------------------------------------------------------------------------- pileup
def check_pileup(case, m, x_dense, sd, y, nheads, tau=kr.TAU32):
    n = len(y)
    C = x_dense.shape[-1]
    xin = _tap(m, "lstm1_in", n, kr.T, C)
    want = kr.fp32_input(x_dense)
    assert np.array_equal(xin, want), (case, "lstm1_in", np.argwhere(xin != want)[:5])
    h1 = _tap(m, "lstm1", n, kr.T, 256)
    h2 = _tap(m, "lstm2", n, kr.T, 320)
    z4 = _tap(m, "l4_pre", n, 128)
    idx = _sites(n)
    r = {"lstm1": kr.lstm32_ratio(xin[idx], h1[idx], sd, 0, tau),
         "lstm2": kr.lstm32_ratio(h1[idx], h2[idx], sd, 1, tau),
         "l4": _l4_ratio(h2.reshape(n, -1), z4, sd),
         "heads": float(np.abs(y.astype(np.float64) - kr.heads(z4, sd, nheads)).max()) / kr.HEADS_TOL}
    _record(case, r)


def _run_p(sd, x, channels=18, add_indel=False, **opts):
    from clair3_b200.model import Clair3_P
    m = _model(Clair3_P, sd, channels, add_indel, taps=1, **opts)
    y = m(torch.from_numpy(x).cuda()).cpu().numpy()
    return m, y


@pytest.mark.parametrize("batch,chunk", [(1, 0), (7, 0), (8, 0), (9, 0), (129, 0), (1024, 0), (2200, 4096)])
def test_fp32_pileup_layers_across_batch_sizes(batch, chunk):
    from clair3_b200 import synth
    add_indel = batch in (9, 2200)
    sd = synth.pileup_state_dict(add_indel, seed=61)
    x = synth.pileup_inputs(batch, seed=61)
    m, y = _run_p(sd, x, add_indel=add_indel, chunk_sites=chunk)
    check_pileup("fp32_pileup_b%d" % batch, m, x, sd, y, 4 if add_indel else 2)


@pytest.mark.parametrize("channels", [1, 23])
def test_fp32_pileup_layers_other_channel_counts(channels):
    from clair3_b200 import synth
    sd = synth.pileup_state_dict(False, channels=channels, seed=62)
    r = np.random.default_rng(62)
    x = r.integers(-60, 61, size=(129, kr.T, channels)).astype(np.int32)
    x[r.random(x.shape) < 0.01] = 70000
    m, y = _run_p(sd, x, channels)
    check_pileup("fp32_pileup_c%d" % channels, m, x, sd, y, 2)


@pytest.mark.parametrize("kind", ["uniform", "int8_wrap", "float_fraction", "counts_above_2p24"])
def test_fp32_pileup_layers_input_kinds(kind):
    from clair3_b200 import synth
    sd = synth.pileup_state_dict(True, seed=63)
    r = np.random.default_rng(63)
    if kind == "uniform":
        x = synth.pileup_inputs(129, seed=63, realistic=False)
    elif kind == "int8_wrap":
        x = synth.pileup_inputs(129, seed=63, dtype=np.int8)
    elif kind == "float_fraction":
        x = r.uniform(-80, 80, size=(129, kr.T, 18)).astype(np.float32)
    else:       # the (float) cast rounds these; every site's input tap must still match the cast exactly
        x = synth.pileup_inputs(129, seed=63).astype(np.int32)
        big = np.array([(1 << 24) + 1, (1 << 24) + 3, 33554435, 123456789, 2 ** 31 - 1])
        mask = r.random(x.shape) < 0.02
        x[mask] = r.choice(np.concatenate([big, -big]), size=int(mask.sum()))
    m, y = _run_p(sd, x, add_indel=True)
    check_pileup("fp32_pileup_" + kind, m, x, sd, y, 4)


@pytest.mark.parametrize("dtype", [np.int8, np.int32, np.int64, np.float32])
def test_fp32_pileup_layers_windows(dtype):
    """forward_windows: windows that start before the column matrix and run past its end, then the same windows with bounds
    that cut them at either end (rows outside the bounds read as zero)."""
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_P
    sd = synth.pileup_state_dict(False, seed=64)
    r = np.random.default_rng(64)
    cols = synth.pileup_inputs(20, seed=64).reshape(-1, 18)[:600]
    if dtype == np.float32:
        cols = cols + r.uniform(-0.5, 0.5, cols.shape)
    elif dtype != np.int8:
        cols[r.random(cols.shape) < 0.01] = 40000000          # rounded by the (float) cast
    cols = cols.astype(dtype)
    starts = np.concatenate([np.arange(-40, 640, 7), [-32, 599, 0, 567]]).astype(np.int64)
    lo = starts + r.integers(-3, 20, len(starts))
    bounds = np.stack([lo, lo + r.integers(0, 40, len(starts))], axis=1).astype(np.int64)
    m = _model(Clair3_P, sd, 18, False, taps=1)
    name = np.dtype(dtype).name
    for bd in (None, bounds):
        y = m.forward_windows(torch.from_numpy(cols), torch.from_numpy(starts), bounds=None if bd is None else
                              torch.from_numpy(bd)).numpy()
        check_pileup("fp32_windows_%s_%s" % (name, "unbounded" if bd is None else "bounded"), m, kr.windows(cols, starts, bd),
                     sd, y, 2)


def test_fp32_pileup_layers_saturated_gates():
    """LSTM weights x4: most gates saturate, the fp32 cell state runs to its extremes."""
    from clair3_b200 import synth
    sd = synth.pileup_state_dict(False, seed=65)
    for k in sd:
        if k.startswith("LSTM"):
            sd[k] = (np.asarray(sd[k]) * 4).astype(np.float32)
    x = synth.pileup_inputs(129, seed=65)
    m, y = _run_p(sd, x)
    check_pileup("fp32_pileup_lstm_x4", m, x, sd, y, 2)


# ---------------------------------------------------------------------------------------------- full alignment
def _fa_levels(depth):
    hh, ww = [depth], [33]
    for _ in range(3):
        hh.append(kr.conv_out(hh[-1]))
        ww.append(kr.conv_out(ww[-1]))
    return hh, ww


def _fa_pixels(n, P, sites):
    """Flat output pixels checked at a level of P pixels per site: every pixel of `sites`, and every 4-pixel block of the
    conv kernel that straddles two sites."""
    pix = [np.arange(b * P, (b + 1) * P) for b in sites]
    for b in range(1, n):
        p = b * P
        if p % 4:
            pix.append(np.arange(p // 4 * 4, min(p // 4 * 4 + 4, n * P)))
    return np.unique(np.concatenate(pix))


def check_fa(case, m, x, sd, y, nheads):
    n, depth = x.shape[:2]
    hh, ww = _fa_levels(depth)
    sites = np.arange(n) if n <= 8 else np.unique([0, 1, n // 2, n - 2, n - 1])
    taps = {name: _tap(m, name, n, hh[i // 3 + 1], ww[i // 3 + 1], 64 << (i // 3)) for i, name in enumerate(kr.CONV_TAPS)}
    r = {}
    prev = kr.fp32_input(x)
    for i, name in enumerate(kr.CONV_TAPS):
        l, j = divmod(i, 3)
        stem, mid = kr.CONV_TAPS[3 * l], kr.CONV_TAPS[3 * l + 1]
        inp = prev if j == 0 else taps[stem] if j == 1 else taps[mid]
        res = taps[stem] if j == 2 else None
        pix = _fa_pixels(n, hh[l + 1] * ww[l + 1], sites)
        r["conv%d" % i] = kr.conv32_ratio(inp, taps[name], kr.conv32_weights(sd, i), 2 if j == 0 else 1, res, pix)
        if j == 2:
            prev = taps[name]
    sp = _tap(m, "spp", n, 3584)
    z4 = _tap(m, "l4_pre", n, 256)
    r["l4_fa"] = _l4_ratio(sp, z4, sd)
    r["heads"] = float(np.abs(y.astype(np.float64) - kr.heads(z4, sd, nheads)).max()) / kr.HEADS_TOL
    _record(case, r)
    assert np.array_equal(sp, kr.spp(taps["res_block3"])), (case, "spp")


def _run_f(sd, x, channels, add_indel=True):
    from clair3_b200.model import Clair3_F
    m = _model(Clair3_F, sd, channels, add_indel, taps=1)
    y = m(torch.from_numpy(x).cuda()).cpu().numpy()
    return m, y


@pytest.mark.parametrize("depth,channels,batch", [(89, 8, 1), (17, 1, 129), (55, 9, 3), (512, 16, 3), (89, 8, 256),
                                                  (17, 8, 256)])
def test_fp32_full_alignment_layers(depth, channels, batch):
    from clair3_b200 import synth
    sd = synth.fa_state_dict(True, channels=channels, seed=71)
    x = synth.fa_inputs(batch, depth=depth, channels=channels, seed=71, realistic=channels >= 5)
    m, y = _run_f(sd, x, channels)
    check_fa("fp32_fa_d%d_c%d_b%d" % (depth, channels, batch), m, x, sd, y, 4)


def test_fp32_full_alignment_layers_int8_extremes():
    from clair3_b200 import synth
    sd = synth.fa_state_dict(False, channels=8, seed=72)
    x = np.random.default_rng(72).choice(np.array([-128, 127, 0], dtype=np.int8), size=(129, 55, 33, 8))
    m, y = _run_f(sd, x, 8, add_indel=False)
    check_fa("fp32_fa_int8_extremes", m, x, sd, y, 2)


# ---------------------------------------------------------------------------------------------- bitwise properties
def _fwd(m, x, stream=None):
    """m(x) on device tensors, on `stream` (default: the current one); returns the device output."""
    xd = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x)).cuda()
    y = torch.empty((xd.shape[0], m.out_dim), dtype=torch.float32, device="cuda")
    with torch.cuda.stream(stream or torch.cuda.current_stream()):
        m.forward_into(xd, y)
    return y


def _batch_invariance(m, x, big):
    """Every output row of the fp32 path depends on its own site only: x [B, ...] small integers (exact in int8 / int32 /
    float32), big: a larger batch made of x's sites."""
    want = _fwd(m, x)
    B = len(x)
    for n in (1, 2, 9):
        assert torch.equal(_fwd(m, x[:n]), want[:n]), n
    reps = -(-big // B)
    xb = np.concatenate([x] * reps)[:big]
    assert torch.equal(_fwd(m, xb), want.repeat(reps, 1)[:big]), big
    perm = np.random.default_rng(3).permutation(B)
    assert torch.equal(_fwd(m, x[perm]), want[torch.from_numpy(perm).cuda()])
    for dt in (np.int8, np.float32):
        assert torch.equal(_fwd(m, x.astype(dt)), want), dt
    for chunk in (1, 7):
        m.set_option("chunk_sites", chunk)
        assert torch.equal(_fwd(m, x), want), chunk
    m.set_option("chunk_sites", 0)
    streams = [torch.cuda.Stream() for _ in range(3)]
    xs = [torch.from_numpy(np.ascontiguousarray(x[perm] if i % 2 else x)).cuda() for i in range(3)]
    torch.cuda.synchronize()
    ys = [_fwd(m, xs[i], streams[i]) for i in range(3)]
    torch.cuda.synchronize()
    for i, yi in enumerate(ys):
        assert torch.equal(yi, want[torch.from_numpy(perm).cuda()] if i % 2 else want), i


def test_fp32_pileup_batch_invariance():
    """Batch sizes up to 1100 (two 1024-site chunks, the heads' 16-site groups), chunk_sites 1 / 7 / default, a permutation,
    three concurrent streams, int8 / int32 / float32 input."""
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_P
    sd = synth.pileup_state_dict(True, seed=66)
    x = synth.pileup_inputs(37, seed=66, realistic=False)
    _batch_invariance(_model(Clair3_P, sd, 18, True), x, 1100)


def test_fp32_full_alignment_batch_invariance():
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_F
    sd = synth.fa_state_dict(True, channels=8, seed=73)
    x = synth.fa_inputs(37, depth=17, channels=8, seed=73).astype(np.int32)
    _batch_invariance(_model(Clair3_F, sd, 8, True), x, 300)


def test_precision_switching_pileup():
    """Tensor-core, fp32, tensor-core again on one model and stream equal fresh models of each precision."""
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_P
    sd = synth.pileup_state_dict(True, seed=67)
    xa, xb = synth.pileup_inputs(300, seed=67), synth.pileup_inputs(129, seed=68)
    m = _model(Clair3_P, sd, 18, True, precision=0)
    got = []
    for prec, x in ((0, xa), (1, xb), (0, xa), (1, xa)):
        m.set_option("precision", prec)
        got.append(_fwd(m, x))
    for (prec, x), y in zip(((0, xa), (1, xb), (0, xa), (1, xa)), got):
        assert torch.equal(y, _fwd(_model(Clair3_P, sd, 18, True, precision=prec), x)), (prec, len(x))


def test_precision_switching_full_alignment():
    """Tensor-core and fp32 calls interleaved on one model and stream, with depth changes and ragged sizes 256 / 44 / 300 (a
    300-site call runs a 256-site and a 44-site chunk).  The fp32 path overwrites the planar region the tensor-core path keeps
    zero-bordered, so the next tensor-core call must clear it again.  The workspace also forgets its zeros when it grows or
    when the depth or site capacity changes; so the first call is an fp32 one, which sizes the workspace for both paths, and
    the fp32 calls of the pairs (1, 55, 256) -> (0, 55, 256) and (1, 55, 44) -> (0, 55, 44) neither grow it nor change depth
    or capacity (256 sites at depth 55): those tensor-core calls are right only if the fp32 call itself marks the region as
    dirty.  Each tensor-core output equals that of a twin model making the same tensor-core calls without the fp32 ones in
    between (the same workspace layout history), each fp32 output that of a fresh fp32 model."""
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_F
    sd = synth.fa_state_dict(True, channels=8, seed=74)
    xs = {(d, n): synth.fa_inputs(n, depth=d, channels=8, seed=d + n) for d, n in ((55, 256), (55, 44), (89, 300))}
    calls = [(1, 55, 256), (0, 55, 256), (1, 55, 256), (0, 55, 256), (1, 55, 44), (0, 55, 44), (1, 89, 300), (0, 89, 300),
             (1, 55, 256), (0, 55, 256)]
    m = _model(Clair3_F, sd, 8, True, precision=1)
    twin = _model(Clair3_F, sd, 8, True, precision=0)
    for prec, d, n in calls:
        m.set_option("precision", prec)
        x = xs[(d, n)]
        y = _fwd(m, x)
        want = _fwd(twin, x) if prec == 0 else _fwd(_model(Clair3_F, sd, 8, True, precision=1), x)
        assert torch.equal(y, want), (prec, d, n)


@pytest.mark.parametrize("precision", [0, 1])
def test_debug_options_leave_outputs_unchanged(precision):
    """taps, profile and lstm_trace on vs off: the same outputs, both networks."""
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_F, Clair3_P
    sd = synth.pileup_state_dict(True, seed=69)
    x = synth.pileup_inputs(129, seed=69)
    sdf = synth.fa_state_dict(True, channels=8, seed=75)
    xf = synth.fa_inputs(44, depth=55, channels=8, seed=75)
    for cls, s, c, inp in ((Clair3_P, sd, 18, x), (Clair3_F, sdf, 8, xf)):
        plain = _model(cls, s, c, True, precision=precision)
        dbg = _model(cls, s, c, True, precision=precision, taps=1, profile=1, lstm_trace=1)
        want = _fwd(plain, inp)
        for _ in range(2):
            assert torch.equal(_fwd(dbg, inp), want), (cls.__name__, precision)
