"""LSTM1 builds its x operand itself from the caller's counts (``pytest -m gpu`` on an H100).

The same sites go through every input dtype, through a dense tensor and through ``forward_windows`` (with and without bounds,
windows overhanging both ends of the column matrix), and through inputs whose base is only element-aligned (the one-load-per-count
path).  The outputs must be equal bit for bit, and the operand LSTM1 built (tap ``lstm1_x``) must equal ``kernel_ref.lstm1_x`` of
the dense tensor bit for bit, at every LSTM1 sub-tile width.
"""
import numpy as np
import pytest
import torch

import kernel_ref as kr

pytestmark = pytest.mark.gpu

DENSE_DTYPES = (torch.int8, torch.int32, torch.float32)
WINDOW_DTYPES = (torch.int64, torch.int32, torch.int8, torch.float32)


def _model(tile):
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_P
    sd = synth.pileup_state_dict(False, seed=61)
    m = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    m.set_option("taps", 1)
    m.set_option("lstm_tile", tile)
    m.to(torch.device("cuda"))
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    return m


def _unaligned(x):
    """x's values in a contiguous device tensor whose base is one element past an aligned address."""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device="cuda")
    out = buf[1:].view(x.shape)
    out.copy_(x)
    return out


def _case(batch, seed):
    """A column matrix of int8-safe counts and windows into it: some start before row 0, some run past the last row."""
    r = np.random.default_rng(seed)
    n_cols = batch + 40
    cols = r.integers(0, 128, size=(n_cols, 18)).astype(np.int64)
    starts = r.integers(-40, n_cols + 8, size=batch).astype(np.int64)
    starts[:2] = [-32, n_cols - 1][:batch]
    lo = starts + r.integers(0, 12, size=batch)
    hi = starts + kr.T - r.integers(0, 12, size=batch)
    return cols, starts, np.stack([lo, hi], axis=1).astype(np.int64)


def _check(m, y, want_x, base, what):
    xop = m.tap("lstm1_x").reshape(len(want_x), kr.T, kr.X1_COLS).astype(np.float64)
    assert np.array_equal(xop, want_x), (what, "lstm1_x", np.argwhere(xop != want_x)[:5])
    assert torch.equal(y, base), (what, "outputs")


@pytest.mark.parametrize("tile", [16, 32, 64])
@pytest.mark.parametrize("batch", [1, 129, 1024])
def test_lstm1_input_sources_agree(batch, tile):
    m = _model(tile)
    cols, starts, bounds = _case(batch, 60 + batch)
    for bnd in (None, bounds):
        dense = kr.windows(cols, starts, bnd)
        want_x = kr.lstm1_x(dense)
        base = m(torch.from_numpy(dense.astype(np.int32)).cuda())
        _check(m, base, want_x, base, "dense int32")
        for dt in DENSE_DTYPES:
            x = torch.from_numpy(dense).to(dt).cuda()
            _check(m, m(x), want_x, base, "dense %s" % dt)
            _check(m, m(_unaligned(x)), want_x, base, "dense %s, element-aligned base" % dt)
        s = torch.from_numpy(starts).cuda()
        b = None if bnd is None else torch.from_numpy(bnd).cuda()
        for dt in WINDOW_DTYPES:
            c = torch.from_numpy(cols).to(dt).cuda()
            what = "windows %s%s" % (dt, "" if bnd is None else ", bounded")
            _check(m, m.forward_windows(c, s, bounds=b), want_x, base, what)
            _check(m, m.forward_windows(_unaligned(c), s, bounds=b), want_x, base, what + ", element-aligned base")
