"""LSTM2 split by block pair at 48 sites per CTA (option ``lstm2_split`` = 2: one h operand buffer, the chain accumulating onto
the pre-gates) against the same kernel at 32 sites (``lstm2_split`` = 1), on an H100 (``pytest -m gpu``).

Every LSTM2 kernel starts each gate's wgmma chain from the site's pre-gate and adds W_hh h_{t-1} in the same k order; a site is
one N column whatever N is, so the probabilities and the ``lstm2`` tap must be equal bit for bit between the two settings: at
batches around the 48-site CTA (the last one runs past the padded batch), the 128-site padding and the 1024-site chunk, through
``forward_windows``, and with the packed-fp16 gate math.  ``lstm2_pregates`` (the proj2 output both read) must be equal too, and
option 2 must really run 48-site CTAs.  Taps describe one chunk, so they are compared for one-chunk calls (<= 1024 sites).
"""
import numpy as np
import pytest
import torch

import kernel_ref as kr

pytestmark = pytest.mark.gpu

BATCHES = [1, 47, 48, 49, 600, 1024, 2200]


def _model(**opts):
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_P
    sd = synth.pileup_state_dict(False, seed=73)
    m = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    m.set_option("taps", 1)
    for k, v in opts.items():
        m.set_option(k, v)
    m.to(torch.device("cuda"))
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    return m


def _runs(m, call, taps):
    """call() under lstm2_split 1 and 2 -> [(probabilities, lstm2 tap, pre-gate tap)] (taps None unless `taps`)."""
    out = []
    for split in (1, 2):
        m.set_option("lstm2_split", split)
        y = call()
        torch.cuda.synchronize()
        out.append((y.cpu(), m.tap("lstm2") if taps else None, m.tap("lstm2_pregates") if taps else None))
    return out


def _same(runs, what):
    (y0, t0, p0), (y1, t1, p1) = runs
    if t0 is not None:
        assert np.array_equal(p0, p1), (what, "pre-gates")
        assert np.array_equal(t0, t1), (what, "lstm2 tap", np.argwhere(t0 != t1)[:5])
    assert torch.equal(y0, y1), (what, "probabilities")


def _counts(batch, seed):
    from clair3_b200 import synth
    x = synth.pileup_inputs(batch, seed=seed).astype(np.int32)
    r = np.random.default_rng(seed)
    n_cols = batch + 40
    cols = r.integers(0, 128, size=(n_cols, 18)).astype(np.int32)
    starts = r.integers(-40, n_cols + 8, size=batch).astype(np.int64)
    lo = starts + r.integers(0, 12, size=batch)
    hi = starts + kr.T - r.integers(0, 12, size=batch)
    return x, cols, starts, np.stack([lo, hi], axis=1).astype(np.int64)


@pytest.mark.parametrize("batch", BATCHES)
def test_lstm2_split48_bit_identical(batch):
    m = _model()
    x, cols, starts, bounds = _counts(batch, 500 + batch)
    xd = torch.from_numpy(x).cuda()
    _same(_runs(m, lambda: m(xd), batch <= 1024), "dense, batch %d" % batch)
    c, s, b = (torch.from_numpy(a).cuda() for a in (cols, starts, bounds))
    _same(_runs(m, lambda: m.forward_windows(c, s, bounds=b), batch <= 1024), "windows, batch %d" % batch)


@pytest.mark.parametrize("batch", [49, 1024])
def test_lstm2_split48_mufu16(batch):
    m = _model(lstm_mufu16=1)
    x, _, _, _ = _counts(batch, 600 + batch)
    xd = torch.from_numpy(x).cuda()
    _same(_runs(m, lambda: m(xd), True), "lstm_mufu16, batch %d" % batch)


def test_lstm2_split48_runs_48_site_ctas():
    """A device-resident 1024-site call (stream-ordered: LSTM1 runs 64-site tiles) launches 2 x ceil(1024 / 48) LSTM2 CTAs under
    lstm2_split 2, and 2 x 1024 / 32 under the default (1)."""
    from clair3_b200._ffi import check, ffi, lib
    m = _model()
    xd = torch.from_numpy(_counts(1024, 7)[0]).cuda()

    def ctas():
        m.set_option("profile", 1)
        m(xd)
        torch.cuda.synchronize()
        pc = ffi.new("double *")
        check(lib().c3b_get_profile_ctas(m._handle, b"lstm2", pc))
        m.set_option("profile", 0)
        return pc[0]

    assert ctas() == 2 * 32
    m.set_option("lstm2_split", 2)
    assert ctas() == 2 * 22


def test_lstm2_split_option_range():
    m = _model()
    with pytest.raises(Exception):
        m.set_option("lstm2_split", 3)
