"""Test helper: the candidate-window cases, shared by tests/test_pileup_windows_cpu.py (the C oracle against the reference's own
``CreateTensorPileup``, oracle/pileup_tensor_ref.py) and tests/test_gpu_pileup_windows.py (the CUDA counter and the bounded
window gather, against the committed fixture tests/golden/pileup_window_cases.npz).

Between the counter and Clair3_P the reference slices one 33-row tensor per candidate it keeps: the candidate loop of
``preprocess/CreateTensorPileupFromCffi.py:343-397`` over the contiguous chunks that ``__enforce_pileup_chunk_contiguity``
(``:180-236``) cuts from the count matrix.  Every case is ``(name, build)``; ``build()`` returns a dict with ``records``, ``ref``,
``ref_start``, ``ctg_start`` / ``ctg_end`` (the 1-based contig slice of ``CreateTensorPileup``) and ``kw`` (the keyword arguments of
``PileupCounter.count``; the counter's region is ``pileup_counts.counting_region(ctg_start, ctg_end)``).  The targeted cases
place one SNP candidate at column P (0-based) and cite the line they aim at.  With ``pos = P + 1`` the reference's window is
``start, end = pos - 16, pos + 17``:
    :358  ``start - 1 >= first and end <= last`` - the run covers P - 16 and reaches P + 18, two columns past the window;
    :365  no all-zero row in the window;
    :371  with call_ht, ``pos > last`` skips a candidate on the run's last column;
    :374  with call_ht, the head window: zero rows in front of a run that starts after P - 16;
    :384-392  with call_ht, the tail window: zero rows behind a run that ends before P + 16 (none when it ends at P + 16 or
          P + 17), and a shape check that drops windows short on both sides.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from clair3_b200 import synth_reads as sr  # noqa: E402

import plp_ref_cases as prc  # noqa: E402

REF, P, FLANK = prc.REF, prc.P, prc.FLANK
CTG = (1, 360)                   # ctgStart, ctgEnd: the counter region is [0, 393), the whole of REF


def _reads(lo, hi, n=6, n_alt=4, snp=P, skip=None, ref=REF):
    """n reads covering the 0-based columns [lo, hi] inclusive, strands alternating, the first n_alt with a SNP at `snp`.
    skip: a column every read jumps with a one-base reference skip (N), which leaves that column covered but all-zero
    (src/clair3_pileup.c skips refskip reads before counting them)."""
    out = []
    for i in range(n):
        subst = {snp: prc._other(ref[snp])} if i < n_alt and snp is not None else None
        if skip is None or not lo < skip < hi:
            out.append(prc._match(ref, lo, hi - lo + 1, flag=16 * (i & 1), subst=subst))
            continue
        seq = list(ref[lo:hi + 1].upper())
        for p, b in (subst or {}).items():
            seq[p - lo] = b
        seq = "".join(seq[:skip - lo] + seq[skip - lo + 1:])
        out.append((lo, 16 * (i & 1), 60, [("M", skip - lo), ("N", 1), ("M", hi - skip)], seq))
    return out


def _block(lo, hi, n=3):
    """A second covered block without candidates (reads of the reference bases over [lo, hi])."""
    return _reads(lo, hi, n=n, n_alt=0, snp=None)


def _case(items, call_ht, ctg=CTG, ref=REF, ref_start=0, **kw):
    return {"records": sr.records_from_lists(items), "ref": ref, "ref_start": ref_start, "ctg_start": ctg[0], "ctg_end": ctg[1],
            "kw": dict(kw, call_ht=bool(call_ht))}


def _ht(call_ht):
    return "_call_ht" if call_ht else ""


def _targeted():
    out = []
    for ht in (False, True):
        # :358 end <= last / :384-392 the tail window: the run ends at P + 15 .. P + 19, a second block after a gap
        for right in range(15, 20):
            out.append(("run_ends_at_c0+%d%s" % (right, _ht(ht)),
                        lambda right=right, ht=ht: _case(_reads(P - 40, P + right) + _block(P + right + 10, P + right + 50), ht)))
        # :358 start - 1 >= first / :374 the head window: the run starts at P - 17 .. P - 15, a first block before a gap
        for left in range(15, 18):
            out.append(("run_starts_at_c0-%d%s" % (left, _ht(ht)),
                        lambda left=left, ht=ht: _case(_block(P - left - 50, P - left - 10) + _reads(P - left, P + 40), ht)))
        # :371 pos > last: the candidate on the run's last column; :384-389 the one before it (15 zero rows behind)
        out.append(("candidate_on_last_column%s" % _ht(ht),
                    lambda ht=ht: _case(_reads(P - 40, P) + _block(P + 10, P + 50), ht, min_depth=1)))
        out.append(("candidate_on_second_to_last_column%s" % _ht(ht),
                    lambda ht=ht: _case(_reads(P - 40, P + 1) + _block(P + 10, P + 50), ht, min_depth=1)))
        # :374-378 the candidate on the run's first column (16 zero rows in front)
        out.append(("candidate_on_first_column%s" % _ht(ht),
                    lambda ht=ht: _case(_block(P - 50, P - 10) + _reads(P, P + 40), ht, min_depth=1)))
        # :379 / :392 the shape checks: a 21-column run, short of both window edges
        out.append(("run_shorter_than_window%s" % _ht(ht), lambda ht=ht: _case(_reads(P - 10, P + 10), ht)))
        # :384-391 a one-column coverage gap behind the candidate, and :374-378 one in front of it: the window's rows past the gap
        # are zeros in the reference's tensor, the neighbouring run's columns in the count matrix
        out.append(("one_column_gap_after%s" % _ht(ht),
                    lambda ht=ht: _case(_reads(P - 40, P + 5) + _block(P + 7, P + 50), ht)))
        out.append(("one_column_gap_before%s" % _ht(ht),
                    lambda ht=ht: _case(_block(P - 50, P - 6) + _reads(P - 4, P + 40), ht)))
        # :365 an all-zero column at P + 5 inside an otherwise complete window: dropped, call_ht or not
        out.append(("all_zero_column_plain%s" % _ht(ht), lambda ht=ht: _case(_reads(P - 40, P + 40, skip=P + 5), ht)))
        # ctgStart = 1: the counter region starts at 0 and the first run at matrix row 0; candidates 5, 16, 17 and 30 columns in
        # (:374 head windows that overhang row 0, and the plain branch just past them)
        out.append(("ctg_start_1%s" % _ht(ht), lambda ht=ht: _case(
            [prc._match(REF, 0, 70, flag=16 * (i & 1), subst={p: prc._other(REF[p]) for p in (5, 16, 17, 30)} if i < 3 else None)
             for i in range(6)], ht)))
    # :384-392 the tail window and :374-378 the head window skip the all-zero test: the zero column stays in the kept tensor
    out.append(("all_zero_column_tail_call_ht", lambda: _case(_reads(P - 40, P + 17, skip=P + 5) + _block(P + 27, P + 60), True)))
    out.append(("all_zero_column_head_call_ht", lambda: _case(_block(P - 60, P - 20) + _reads(P - 10, P + 40, skip=P + 5), True)))
    # a slice that starts inside the reads: the counter region starts at ctgStart - 35, so its first row is the run's first
    out.append(("ctg_start_inside_run_call_ht", lambda: _case(_reads(P - 60, P + 40, snp=P - 40), True, ctg=(P - 8, 360))))
    return out


def _seeded():
    """Every configuration of plp_ref_cases.SEEDED with a coverage gap (``random_<s>``, s % 3 == 0), call_ht both ways: the
    1-based slice is chosen so that the counter's region is the configuration's region where the contig allows it."""
    out = []
    for s in (0, 3, 6, 9):
        for ht in (False, True):
            def build(s=s, ht=ht):
                rec, ref, rs, start, end, kw = prc._random(s)
                kw = {k: v for k, v in kw.items() if k in ("min_depth", "min_mq", "call_snp_only")}
                return {"records": rec, "ref": ref, "ref_start": rs, "ctg_start": max(1, start + 35), "ctg_end": end - 33,
                        "kw": dict(kw, call_ht=ht)}
            out.append(("random_%d%s" % (s, _ht(ht)), build))
    return out


TARGETED = _targeted()
SEEDED = _seeded()
ALL = TARGETED + SEEDED
IDS = [n for n, _ in ALL]
BUILD = dict(ALL)


def counter_region(case):
    from clair3_b200.pileup_counts import counting_region
    return counting_region(case["ctg_start"], case["ctg_end"])
