"""The GPU counter's window verdicts and the bounded window gather against the reference's own candidate loop
(``preprocess/CreateTensorPileupFromCffi.py:343-397``), read from tests/golden/pileup_window_cases.npz (minted from the reference
by tests/golden/make_pileup_window_golden.py; the reference checkout is not needed here).  ``pytest -m gpu`` on an H100.

For every case of tests/plp_window_cases.py:
  - ``cand_ok`` of ``PileupCounter.count(...).fetch()`` selects exactly the positions the reference keeps, and the run bounds
    (``c3b_plp_window_bounds``) equal the C oracle's;
  - ``PileupCounter.forward`` gathers every window straight from the device-resident matrix with those bounds: LSTM1's input
    operand (tap ``lstm1_x``) of the kept rows equals ``kernel_ref.lstm1_x`` of the reference's tensors bit for bit, so the
    gather and its zero padding are exact, and the probabilities equal Clair3_P on the reference's tensors.
The fp32 debug path (precision 1) and the host-buffer path of ``Clair3_P.forward_windows(..., bounds=...)`` gather the same
windows."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import kernel_ref as kr  # noqa: E402
import plp_window_cases as cases  # noqa: E402
from test_pileup_windows_cpu import fixture  # noqa: E402

pytestmark = pytest.mark.gpu

GAP_CASES = [n for n in cases.IDS if "gap" in n or "zero_column" in n or n.startswith(("random_", "ctg_start", "run_"))]


@pytest.fixture(scope="module")
def counter():
    from clair3_b200 import pileup_counts as pc
    c = pc.PileupCounter(0)
    yield c
    c.close()


def _model(precision):
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_P
    m = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    m.set_option("precision", precision)
    m.set_option("taps", 1)
    m.set_option("chunk_sites", 4096)            # every candidate of a case in one pass: the taps cover all of them
    m.to(torch.device("cuda:0"))
    m.eval()
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=3).items()})
    return m


@pytest.fixture(scope="module")
def model():
    return _model(0)


def _count(counter, name):
    from oracle import pileup_oracle as po
    case = cases.BUILD[name]()
    s, e = cases.counter_region(case)
    got = counter.count(case["records"], s, e, case["ref"], case["ref_start"], **case["kw"]).fetch()
    want = po.clair3_pileup(case["records"], s, e, case["ref"], case["ref_start"], **case["kw"])
    return got, want


@pytest.mark.parametrize("name", cases.IDS)
def test_gpu_windows_equal_reference(counter, model, name):
    got, want = _count(counter, name)
    want_pos, want_t, _ = fixture(name)
    ok = got["cand_ok"].astype(bool)
    pos = got["major"][got["cand_cols"][ok]] + 1
    assert np.array_equal(pos, want_pos), "%s: the GPU keeps %s, the reference %s" % (name, pos.tolist(), want_pos.tolist())
    assert np.array_equal(counter.window_bounds(), want["window_bounds"]), name
    n = len(ok)
    if n == 0:
        return
    y, ok2 = counter.forward(model)
    torch.cuda.synchronize()
    assert np.array_equal(ok2, got["cand_ok"])
    xop = model.tap("lstm1_x").reshape(n, kr.T, kr.X1_COLS).astype(np.float64)
    sel = np.nonzero(ok)[0]
    if len(sel) == 0:
        return
    xwant = kr.lstm1_x(want_t)
    d = np.argwhere(xop[sel] != xwant)
    assert len(d) == 0, "%s: lstm1_x of the window at position %d differs at row %d, column %d" % (
        name, want_pos[d[0][0]], d[0][1], d[0][2])
    y = y.cpu().numpy()[sel]
    yref = model(torch.from_numpy(want_t).to("cuda:0")).cpu().numpy()
    assert float(np.abs(y - yref).max()) < 1e-5, name      # same kernels on the same operands (cf. the chained-forward test)


def test_fp32_path_and_host_bounds_gather_the_same_windows(counter):
    """precision 1 (kernels_common.cu's gather) through PileupCounter.forward, and Clair3_P.forward_windows with host matrix,
    starts and bounds, both equal the forward over the reference's tensors."""
    m32 = _model(1)
    m16 = _model(0)
    checked = 0
    for name in GAP_CASES:
        got, want = _count(counter, name)
        want_pos, want_t, _ = fixture(name)
        sel = np.nonzero(got["cand_ok"])[0]
        if len(sel) == 0:
            continue
        y32, _ = counter.forward(m32)
        yref32 = m32(torch.from_numpy(want_t).to("cuda:0")).cpu().numpy()
        assert float(np.abs(y32.cpu().numpy()[sel] - yref32).max()) < 1e-5, name
        starts = got["cand_cols"] - 16
        bounds = counter.window_bounds()
        yh = m16.forward_windows(got["matrix"], starts, bounds=bounds).numpy()
        yref16 = m16(torch.from_numpy(want_t).to("cuda:0")).cpu().numpy()
        assert float(np.abs(yh[sel] - yref16).max()) < 1e-5, name
        checked += len(sel)
    assert checked > 100
