"""CPU-side checks of the full-alignment tensor builder: the glibc rand() restatement, the khash bucket order with int keys, the
C-ABI header, and known answers of the reference's own calculate_clair3_full_alignment (compiled by oracle/fa_ref.py; those
tests skip where oracle/_ref has not been built) - each expected number follows from the cited source lines of
src/clair3_full_alignment_dwell.{c,h}."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from clair3_b200 import fa_tensor as ft
from clair3_b200 import synth_reads as sr
from clair3_b200.pileup_counts import khash_iteration_order
from fa_golden import load_fa_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle():
    from oracle import fa_ref
    if fa_ref.build() is None:
        pytest.skip("oracle/_ref/libclair3_fa_ref.so is not built (set CLAIR3_REFERENCE)")
    return fa_ref


@pytest.mark.parametrize("seed,skip", [(1, 0), (1, 37), (42, 1000), (0, 5), (4000000000, 12345)])
def test_glibc_rand_restatement_matches_libc(seed, skip):
    libc = ctypes.CDLL(None)
    libc.srand(ctypes.c_uint(seed))
    want = [libc.rand() for _ in range(skip + 80)][skip:]
    assert ft.glibc_rand(seed, skip, 80).tolist() == want


def test_khash_int_keys_known_order():
    # identity hash: 4 buckets, 5 & 3 = 1, 1 & 3 = 1 -> probe 2; 9 & 3 = 1 -> probe 2, then 0
    assert khash_iteration_order([5, 1, 9]) == [2, 0, 1]
    # a fourth put of a present key grows the full (3 of 4) table to 8 buckets; kh_resize moves the keys in old bucket order,
    # kicking out keys not yet moved: 9 -> 1 (kicks 5 -> 5), then 1 -> 1 taken -> 2
    assert khash_iteration_order([5, 1, 9], put_after_last=True) == [2, 1, 0]


def _run(rec_items, cand, ref, **kw):
    fa_ref = _oracle()
    return fa_ref.full_alignment(sr.records_from_lists(rec_items), cand, ref, **kw)


REF = "ACGT" * 25      # 100 bases


def test_known_answers_basic_channels():
    # one forward read, 40M from position 10, mapq 30, qualities absent (0xFF -> normalize_bq 100), reads the reference except
    # an N at position 30 (query 20)
    q = list(REF[10:50])
    q[20] = "N"
    m, alt, draws = _run([(10, 0, 30, [("M", 40)], "".join(q))], [30], REF, matrix_depth=5)
    row = m[0, 2]                                  # one read, depth 5: padding 4 -> 2 rows on top (:139-150)
    assert (m[0, [0, 1, 3, 4]] == 0).all()
    c = 16                                         # the candidate column
    assert row[c, 0] == 75                         # reference G (num2countbase_fa['G' - 'A'], .h:39-44)
    assert row[c, 1] == 100                        # read base N -> alt value 100
    assert row[c, 2] == 100 and row[c, 3] == 50 and row[c, 4] == 100 and row[c, 7] == 60   # strand, mq 30 -> 50, bq, unphased
    assert row[c, 5] == 100                        # AF: 1 of depth 1
    assert alt == ["31-1-G-XA 1 "]                 # N counts as A (acgt2num); ref count 0 -> no R field


def test_known_answers_indels_filter_dedup_lowercase():
    ref = REF[:40] + REF[40:60].lower() + REF[60:]
    reads = [
        (10, 0, 60, [("M", 21), ("I", 2), ("M", 20)], REF[10:31] + "TT" + REF[31:51]),   # insertion after position 30
        (12, 16, 60, [("M", 19), ("D", 3), ("M", 20)], REF[12:31] + REF[34:54]),         # deletion after position 30
        (12, 0, 60, [("M", 40)], REF[12:52]),                                            # same name as read 1: dropped
        (14, 256, 60, [("M", 40)], REF[14:54]),                                          # secondary (2316 & 256): dropped
        (14, 0, 2, [("M", 40)], REF[14:54]),                                             # mapq below min_mq 5: dropped
    ]
    fa_ref = _oracle()
    rec = sr.records_from_lists(reads)
    names = [b"a", b"b", b"b", b"c", b"d"]
    rec["qname"] = np.frombuffer(b"".join(names), np.uint8).copy()
    rec["qname_off"] = np.array([0, 1, 2, 3, 4, 5], np.int64)
    m, alt, _ = fa_ref.full_alignment(rec, [30], ref, matrix_depth=4)
    # two kept reads at depth 4: one padding row on top, rows sorted by read index (both unphased)
    ins_row, del_row = m[0, 1], m[0, 2]
    assert (m[0, 0] == 0).all() and (m[0, 3] == 0).all()
    assert ins_row[16, 1] == -50 and ins_row[16, 6] == 50 and ins_row[17, 6] == 50      # I at the anchor, spill of "TT"
    assert del_row[16, 1] == -100 and (del_row[17:20, 0] == 0).all()                    # D marks the base before; deleted columns unwritten
    assert del_row[16, 2] == 50                                                         # reverse strand
    assert ins_row[16, 5] == 50 and del_row[16, 5] == 50                                # AF 1/2 each
    assert alt == ["31-2-G-IGTT 1 DTAC 1 "]                                             # ref count 2 - 1 - 1 = 0
    assert ins_row[26, 0] == 100                   # position 40 is soft-masked 'a': the matrix upper-cases it (:848)


def test_golden_fixture_equals_fresh_oracle_output():
    fa_ref = _oracle()
    rec, ref, cand, var, params, m, alt, draws = load_fa_golden()
    m2, alt2, draws2 = fa_ref.full_alignment(rec, cand, ref, variants=var, **params)
    assert np.array_equal(m, m2) and alt == alt2 and draws == draws2


def test_fa_header_compiles_as_c99_and_links(tmp_path):
    src = tmp_path / "use_fa.c"
    src.write_text('#include "clair3_b200_fa.h"\n#include "clair3_b200.h"\n'
                   "int main(void) {\n  c3b_fa *w = 0;\n  c3b_fa_params p = {89, 1, 5, 0, 1, 0, 0};\n"
                   "  if (c3b_fa_create(&w, 0)) return (int)p.matrix_depth;\n  c3b_fa_destroy(w);\n  return 0;\n}\n")
    from clair3_b200 import build
    lib = build.build_library()
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), lib,
                        "-o", str(tmp_path / "use_fa")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
