"""LSTM2 split by block pair (option ``lstm2_split`` = 1: five warpgroups per CTA, one block pair each) against the sub-tile
kernel (``lstm2_split`` = 0), on an H100 (``pytest -m gpu``).

Each gate pre-activation is the same wgmma chain in both kernels (the same A block, B columns, k order and N) and the cell math
is the same, so the probabilities and the ``lstm2`` tap must be equal bit for bit: at LSTM2 tiles 16 and 32, at batches around
the 32-site CTA and the 1024-site chunk, through ``forward_windows``, for int8 / int32 / int64 input, with the packed-fp16 gate
math, and with the library's own tile choice for device-resident and host-buffer calls.
"""
import numpy as np
import pytest
import torch

import kernel_ref as kr

pytestmark = pytest.mark.gpu

BATCHES = [1, 31, 32, 33, 1023, 1024, 1025, 2600]
DTYPES = (torch.int8, torch.int32, torch.int64)


def _model(**opts):
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_P
    sd = synth.pileup_state_dict(False, seed=71)
    m = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    m.set_option("taps", 1)
    for k, v in opts.items():
        m.set_option(k, v)
    m.to(torch.device("cuda"))
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    return m


def _runs(m, call, settings=(0, 1)):
    """call() with each lstm2_split setting -> [(probabilities, lstm2 tap)] in that order."""
    out = []
    for split in settings:
        m.set_option("lstm2_split", split)
        y = call()
        torch.cuda.synchronize()
        out.append((y.cpu(), m.tap("lstm2")))
    return out


def _same(runs, what):
    y0, t0 = runs[0]
    for y1, t1 in runs[1:]:
        assert torch.equal(y0, y1), (what, "probabilities")
        assert np.array_equal(t0, t1), (what, "lstm2 tap", np.argwhere(t0 != t1)[:5])


def _counts(batch, seed):
    """int8-safe counts of realistic sites, and a column matrix with windows into it (overhanging both ends, bounded)."""
    from clair3_b200 import synth
    x = np.clip(synth.pileup_inputs(batch, seed=seed), -127, 127).astype(np.int64)
    r = np.random.default_rng(seed)
    n_cols = batch + 40
    cols = r.integers(0, 128, size=(n_cols, 18)).astype(np.int64)
    starts = r.integers(-40, n_cols + 8, size=batch).astype(np.int64)
    lo = starts + r.integers(0, 12, size=batch)
    hi = starts + kr.T - r.integers(0, 12, size=batch)
    return x, cols, starts, np.stack([lo, hi], axis=1).astype(np.int64)


@pytest.mark.parametrize("tile", [16, 32])
@pytest.mark.parametrize("batch", BATCHES)
def test_lstm2_split_bit_identical(batch, tile):
    m = _model(lstm_tile=tile)
    x, cols, starts, bounds = _counts(batch, 700 + batch)
    for dt in DTYPES:
        xd = torch.from_numpy(x).to(dt).cuda()
        _same(_runs(m, lambda: m(xd)), "dense %s, tile %d, batch %d" % (dt, tile, batch))
        c = torch.from_numpy(cols).to(dt).cuda()
        s = torch.from_numpy(starts).cuda()
        b = torch.from_numpy(bounds).cuda()
        _same(_runs(m, lambda: m.forward_windows(c, s, bounds=b)), "windows %s, tile %d, batch %d" % (dt, tile, batch))


@pytest.mark.parametrize("batch", [33, 1025, 2600])
def test_lstm2_split_default_tiles_and_mufu16(batch):
    """The library's tile choice (device-resident: stream-ordered; host tensor: latency rule), and lstm_mufu16 = 1."""
    x, _, _, _ = _counts(batch, 900 + batch)
    xh = torch.from_numpy(x.astype(np.int32))
    xd = xh.cuda()
    m = _model()
    _same(_runs(m, lambda: m(xd)), "device-resident, batch %d" % batch)
    _same(_runs(m, lambda: m(xh)), "host tensor, batch %d" % batch)
    m16 = _model(lstm_mufu16=1)
    _same(_runs(m16, lambda: m16(xd)), "lstm_mufu16, batch %d" % batch)
