"""Which candidates get a 33-row tensor, and what it holds: the C oracle's ``cand_ok`` and window bounds
(oracle/pileup_oracle.c) against the reference's OWN candidate loop, ``CreateTensorPileup`` of
``preprocess/CreateTensorPileupFromCffi.py:343-397``, run unmodified from the reference checkout by
oracle/pileup_tensor_ref.py on the cases of tests/plp_window_cases.py.

The oracle keeps a candidate's window when ``cand_ok`` is 1; the tensor is the window's rows of the count matrix, with zeros
outside ``window_bounds`` (the candidate's contiguous run).  Both must equal the reference's kept positions, in its order, and
its tensors element for element.  tests/golden/pileup_window_cases.npz keeps the reference's output, so the cases stay checked
where the reference checkout is absent; the GPU counter and the bounded gather are held to it by
tests/test_gpu_pileup_windows.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import pileup_oracle as po  # noqa: E402
import plp_window_cases as cases  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pileup_window_cases.npz")
FLANK, T = 16, 33
P1 = cases.P + 1                  # the targeted candidate's 1-based position

_fixture = None


def fixture(name):
    """(positions, tensors, pos_info) the reference kept on case `name`, from the committed fixture."""
    global _fixture
    if _fixture is None:
        _fixture = np.load(GOLDEN)
    return tuple(_fixture["%s/%s" % (name, k)] for k in ("positions", "tensors", "pos_info"))


def reference():
    from oracle import pileup_tensor_ref
    if not pileup_tensor_ref.available():
        pytest.skip("needs the reference checkout (its preprocess/ Python, and oracle/_ref/libclair3_pileup_ref.so built from "
                    "its src/): CLAIR3_REFERENCE")
    return pileup_tensor_ref


def oracle_windows(case):
    """The oracle's kept windows: (1-based positions, tensors int64 [k, 33, 18], the oracle's full output)."""
    s, e = cases.counter_region(case)
    o = po.clair3_pileup(case["records"], s, e, case["ref"], case["ref_start"], **case["kw"])
    kept = np.nonzero(o["cand_ok"])[0]
    cols = o["cand_cols"][kept]
    tensors = np.zeros((len(kept), T, 18), np.int64)
    for i, (j, c) in enumerate(zip(kept, cols)):
        lo, hi = o["window_bounds"][j]
        tensors[i, lo - (c - FLANK):hi - (c - FLANK)] = o["matrix"][lo:hi]
    return o["major"][cols] + 1, tensors, o


def check_windows(name, pos, tensors, want_pos, want_tensors, who):
    assert np.array_equal(pos, want_pos), "%s: %s keeps %s, the reference %s" % (name, who, pos.tolist(), want_pos.tolist())
    assert tensors.shape == want_tensors.shape, (name, tensors.shape, want_tensors.shape)
    d = np.argwhere(tensors != want_tensors)
    assert len(d) == 0, "%s: %s's window at position %d differs from the reference's at %d cells, first [row %d, feature %d]" % (
        name, who, want_pos[d[0][0]], len(d), d[0][1], d[0][2])


@pytest.mark.parametrize("name", cases.IDS)
def test_oracle_windows_equal_reference(name):
    """The live reference's kept windows equal the oracle's, and the committed fixture."""
    ptr = reference()
    case = cases.BUILD[name]()
    tensors, pos_info, _ = ptr.create_tensor_pileup(case["records"], case["ref"], case["ref_start"], case["ctg_start"],
                                                    case["ctg_end"], **case["kw"])
    want_pos = ptr.kept_positions(pos_info)
    pos, got, _ = oracle_windows(case)
    check_windows(name, pos, got, want_pos, tensors, "the oracle")
    fpos, ftensors, finfo = fixture(name)
    assert np.array_equal(fpos, want_pos) and np.array_equal(ftensors, tensors) and list(finfo) == pos_info, \
        "%s: tests/golden/pileup_window_cases.npz is stale (re-mint it with tests/golden/make_pileup_window_golden.py)" % name


@pytest.mark.parametrize("name", cases.IDS)
def test_oracle_windows_equal_fixture(name):
    """The same comparison against the reference's committed output (no reference checkout needed)."""
    pos, got, _ = oracle_windows(cases.BUILD[name]())
    want_pos, want, _ = fixture(name)
    check_windows(name, pos, got, want_pos, want, "the oracle")


def _run(o, c):
    """The rows [first, last] of the contiguous run (consecutive positions) that holds matrix row c."""
    m = o["major"]
    lo, hi = c, c
    while lo > 0 and m[lo - 1] == m[lo] - 1:
        lo -= 1
    while hi + 1 < len(m) and m[hi + 1] == m[hi] + 1:
        hi += 1
    return lo, hi


@pytest.mark.parametrize("name", cases.IDS)
def test_window_bounds_are_the_candidates_run(name):
    """window_bounds of EVERY candidate (kept or not) = its 33-row window intersected with its contiguous run."""
    _, _, o = oracle_windows(cases.BUILD[name]())
    for j, c in enumerate(o["cand_cols"]):
        first, last = _run(o, int(c))
        want = (max(first, c - FLANK), min(last, c + FLANK) + 1)
        assert tuple(o["window_bounds"][j]) == want, (name, int(c), tuple(o["window_bounds"][j]), want)


def _zero_rows(t):
    z = ~t.any(axis=1)
    lead = int(np.argmin(z)) if not z.all() else len(z)
    trail = int(np.argmin(z[::-1])) if not z.all() else len(z)
    return lead, trail, np.nonzero(z)[0].tolist()


def _kept(name):
    pos, tensors, _ = fixture(name)
    return pos.tolist(), tensors


def _is_candidate(name, pos1):
    _, _, o = oracle_windows(cases.BUILD[name]())
    return pos1 - 1 in set(o["major"][o["cand_cols"]].tolist())


def test_cases_are_aimed():
    """Each targeted case reaches the branch it cites, read off the reference's own output (the fixture)."""
    # :358 end <= last - the run must reach c0 + 18, two columns past the window
    for right, kept in ((15, []), (16, []), (17, []), (18, [P1]), (19, [P1])):
        name = "run_ends_at_c0+%d" % right
        assert _kept(name)[0] == kept, name
        assert _is_candidate(name, P1), name
    # :384-392 with call_ht every one is kept; zero rows behind the run only when it ends before c0 + 16
    for right in range(15, 20):
        pos, t = _kept("run_ends_at_c0+%d_call_ht" % right)
        assert pos == [P1]
        assert _zero_rows(t[0])[1] == max(0, FLANK - right), right
    # :358 start - 1 >= first / :374 the head window
    assert _kept("run_starts_at_c0-15")[0] == [] and not _is_candidate("run_starts_at_c0-15", P1)
    for left in (16, 17):
        assert _kept("run_starts_at_c0-%d" % left)[0] == [P1]
        pos, t = _kept("run_starts_at_c0-%d_call_ht" % left)
        assert pos == [P1] and _zero_rows(t[0])[:2] == (0, 0)
    pos, t = _kept("run_starts_at_c0-15_call_ht")
    assert pos == [P1] and _zero_rows(t[0])[:2] == (1, 0)
    # :371 the run's last column is skipped; the column before it gets 15 zero rows; the first column 16 in front
    assert _kept("candidate_on_last_column_call_ht")[0] == [] and _is_candidate("candidate_on_last_column_call_ht", P1)
    pos, t = _kept("candidate_on_second_to_last_column_call_ht")
    assert pos == [P1] and _zero_rows(t[0])[:2] == (0, 15)
    pos, t = _kept("candidate_on_first_column_call_ht")
    assert pos == [P1] and _zero_rows(t[0])[:2] == (16, 0)
    # :379 / :392 short on both sides
    assert _kept("run_shorter_than_window_call_ht")[0] == [] and _is_candidate("run_shorter_than_window_call_ht", P1)
    # one-column gaps: the reference's zeros where the count matrix holds the neighbouring run's columns
    for name, lead, trail in (("one_column_gap_after_call_ht", 0, 11), ("one_column_gap_before_call_ht", 12, 0)):
        pos, t = _kept(name)
        assert pos == [P1] and _zero_rows(t[0])[:2] == (lead, trail), name
        _, _, o = oracle_windows(cases.BUILD[name]())
        c = int(o["cand_cols"][0])
        naive = o["matrix"][c - FLANK:c + FLANK + 1]
        assert naive.shape == (T, 18) and naive.any(axis=1).all() and not np.array_equal(naive, t[0]), name
    assert _kept("one_column_gap_after")[0] == [] and _is_candidate("one_column_gap_after", P1)
    # :365 an all-zero column (stats bit 1) drops the plain window; the head / tail windows keep it
    for name in ("all_zero_column_plain", "all_zero_column_plain_call_ht", "all_zero_column_tail_call_ht",
                 "all_zero_column_head_call_ht"):
        _, _, o = oracle_windows(cases.BUILD[name]())
        zc = int(np.searchsorted(o["major"], cases.P + 5))
        assert o["major"][zc] == cases.P + 5 and o["stats"][zc, 5] & 2 and not o["matrix"][zc].any(), name
        assert _is_candidate(name, P1), name
    assert _kept("all_zero_column_plain")[0] == [] and _kept("all_zero_column_plain_call_ht")[0] == []
    pos, t = _kept("all_zero_column_tail_call_ht")
    assert pos == [P1] and _zero_rows(t[0]) == (0, 0, [FLANK + 5])
    pos, t = _kept("all_zero_column_head_call_ht")
    assert pos == [P1] and _zero_rows(t[0]) == (6, 0, list(range(6)) + [FLANK + 5])
    # ctgStart = 1: head windows overhanging matrix row 0
    assert _kept("ctg_start_1")[0] == [18, 31]
    pos, t = _kept("ctg_start_1_call_ht")
    assert pos == [6, 17, 18, 31] and _zero_rows(t[0])[:2] == (11, 0) and _zero_rows(t[1])[:2] == (0, 0)
    pos, t = _kept("ctg_start_inside_run_call_ht")
    assert pos == [P1 - 40] and _zero_rows(t[0])[:2] == (13, 0)
    # the seeded regions with gaps: call_ht keeps windows the plain branch drops
    for s in (0, 6):
        assert len(_kept("random_%d_call_ht" % s)[0]) > len(_kept("random_%d" % s)[0]), s
