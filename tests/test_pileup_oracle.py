"""CPU checks of the pileup feature counter's oracle (oracle/pileup_oracle.c, the plain-C restatement of
``calculate_clair3_pileup``, HKU-BAL/Clair3 src/clair3_pileup.c:142-476) and of the host side of the GPU counter.

The oracle is pinned against the reference's own calculate_clair3_pileup, compiled by oracle/pileup_ref.py, in
tests/test_pileup_reference_cpu.py.  Here it is also checked against hand-worked known-answer cases (every expected number below
is derived in the comments from the reference's source lines) and an independent random-access Python model (tests/plp_model.py)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from clair3_b200 import synth_reads as sr
from oracle import pileup_oracle as po
from plp_model import model_pileup

KEYS = ("matrix", "major", "stats", "cand_cols", "cand_ok", "window_bounds")


def case_indels():
    """ref 0..19 = AACCGGTTAACCGGTTAACC, region [0, 20).
    r1 pos 2 fwd 5M       CCGGT          matches ref 2..6
    r2 pos 2 rev 3M2D2M   CCG--AA        deletion of ref 5,6; A (mismatch) on ref 7, A on ref 8
    r3 pos 4 fwd 2M1I2M   GG[T]TT        insertion 'T' after ref 5
    r4 secondary (flag 256): dropped by the reader (src/medaka_bamiter.c:22)
    r5 mapq 3 < min_mq 5: dropped (:24)"""
    ref = "AACCGGTTAACCGGTTAACC"
    rec = sr.records_from_lists([
        (2, 0, 60, [("M", 5)], "CCGGT"),
        (2, 16, 60, [("M", 3), ("D", 2), ("M", 2)], "CCGAA"),
        (4, 0, 60, [("M", 2), ("I", 1), ("M", 2)], "GGTTT"),
        (3, 256, 60, [("M", 6)], "CCGGTT"),
        (3, 0, 3, [("M", 6)], "TTTTTT"),
    ])
    #            A   C   G   T  Ia  Ib  Da  Db   D | a   c   g   t  ia  ib  da  db   d
    matrix = np.array([
        [0, -1, 0, 0, 0, 0, 0, 0, 0, 0, -1, 0, 0, 0, 0, 0, 0, 0],      # pos 2, ref C: C+ 1, c- 1 -> -sum on both strands (:368-369)
        [0, -1, 0, 0, 0, 0, 0, 0, 0, 0, -1, 0, 0, 0, 0, 0, 0, 0],      # pos 3, ref C
        [0, 0, -2, 0, 0, 0, 0, 0, 0, 0, 0, -1, 0, 0, 0, 1, 1, 0],      # pos 4, ref G: r1,r3 G+, r2 g- and its 2D starts next: da=db=1
        [0, 0, -2, 0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1],       # pos 5, ref G: r1,r3 G+ (r3 + insertion T: Ia=Ib=1), r2 deleted: d- 1
        [0, 0, 0, -2, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1],       # pos 6, ref T: r1,r3 T+, r2 deleted
        [0, 0, 0, -1, 0, 0, 0, 0, 0, 1, 0, 0, -1, 0, 0, 0, 0, 0],      # pos 7, ref T: r3 T+, r2 a-: T+ = -fwd sum, t- = -rev sum (= -1!)
        [0, 0, 0, 0, 0, 0, 0, 0, 0, -1, 0, 0, 0, 0, 0, 0, 0, 0],       # pos 8, ref A: r2 a- only
    ], dtype=np.int64)
    major = np.arange(2, 9, dtype=np.int64)
    #                 depth ref alt del ins
    stats5 = np.array([[2, 2, 0, 0, 0], [2, 2, 0, 0, 0], [3, 3, 0, 1, 0], [3, 2, 0, 0, 1], [3, 2, 0, 0, 0], [2, 1, 1, 0, 0],
                       [1, 1, 0, 0, 0]], dtype=np.int32)
    # call_ht (no flanking requirement), min_depth 2, snp 0.08, indel 0.15: pos 4 (del 1/3), pos 5 (ins 1/3), pos 7 (alt 1/2)
    cand = np.array([2, 3, 5], dtype=np.int64)
    return rec, ref, matrix, major, stats5, cand


def case_quirks():
    """ref 0..11 = ACGTACGTACGT, region [0, 12).
    rA pos 0 fwd 4M      ANGT   N on column 1: feature index -1 -> the PREVIOUS column's feature 17 (src/clair3_pileup.c:280)
    rB pos 0 fwd 2M3N2M  ACCG   reference skip over 2,3,4 (is_refskip: counted by htslib as covering, skipped by :251)"""
    ref = "ACGTACGTACGT"
    rec = sr.records_from_lists([
        (0, 0, 60, [("M", 4)], "ANGT"),
        (0, 0, 60, [("M", 2), ("N", 3), ("M", 2)], "ACCG"),
    ])
    matrix = np.zeros((7, 18), dtype=np.int64)
    matrix[0, 0] = -2          # pos 0 ref A: two A+
    matrix[0, 17] = 1          # ... plus column 1's N
    matrix[1, 1] = -1          # pos 1 ref C: rB C+ (rA's N went to column 0)
    matrix[2, 2] = -1          # pos 2 ref G: rA G+, rB skipped
    matrix[3, 3] = -1          # pos 3 ref T
    #       pos 4: only rB, reference-skipped: covered, all features zero
    matrix[5, 1] = -1          # pos 5 ref C: rB C+
    matrix[6, 2] = -1          # pos 6 ref G
    major = np.arange(0, 7, dtype=np.int64)
    stats5 = np.array([[2, 2, 0, 0, 0], [2, 1, 0, 0, 0], [1, 1, 0, 0, 0], [1, 1, 0, 0, 0], [1, 0, 0, 0, 0], [1, 1, 0, 0, 0],
                       [1, 1, 0, 0, 0]], dtype=np.int32)      # depth counts the N base (:287); an all-skip column has depth max(1, 0)
    zero_rows = np.array([0, 0, 0, 0, 1, 0, 0], dtype=bool)
    return rec, ref, matrix, major, stats5, zero_rows


def test_known_answer_indels():
    rec, ref, matrix, major, stats5, cand = case_indels()
    r = po.clair3_pileup(rec, 0, 20, ref, 0, call_ht=True)
    assert np.array_equal(r["major"], major)
    assert np.array_equal(r["matrix"], matrix)
    assert np.array_equal(r["stats"][:, :5], stats5)
    assert np.array_equal(r["cand_cols"], cand)
    assert not r["cand_ok"].any()                     # 7 columns: no candidate has 16 columns on each side
    # without call_ht nothing has 16 contiguous columns before it (:385-387)
    assert len(po.clair3_pileup(rec, 0, 20, ref, 0)["cand_cols"]) == 0


def test_known_answer_quirks():
    rec, ref, matrix, major, stats5, zero_rows = case_quirks()
    r = po.clair3_pileup(rec, 0, 12, ref, 0, call_ht=True, min_depth=1)
    assert np.array_equal(r["major"], major)
    assert np.array_equal(r["matrix"], matrix)
    assert np.array_equal(r["stats"][:, :5], stats5)
    assert np.array_equal((r["stats"][:, 5] & 2) != 0, zero_rows)


def test_adjacent_deletions_merge_and_insertion_after_deletion():
    """resolve_cigar2: '1D2D' is one 3-base deletion seen from the preceding base; an insertion right after a deletion is reported
    on the deletion's last column with the inserted bases starting at qpos (first = 0, src/clair3_pileup.c:294)."""
    ref = "ACGTACGTACGTACGT"
    rec = sr.records_from_lists([
        (0, 0, 60, [("M", 2), ("D", 1), ("D", 2), ("M", 2)], "ACCG"),           # deletion of 2,3,4
        (0, 0, 60, [("M", 2), ("D", 3), ("M", 2)], "ACCG"),                     # the same deletion as one operation
        (0, 16, 60, [("M", 3), ("D", 2), ("I", 2), ("M", 1)], "ACGTTG"),        # deletion of 3,4 then insertion TT, then ref 5
    ])
    r = po.clair3_pileup(rec, 0, 16, ref, 0, call_ht=True)
    m = r["matrix"]
    assert m[1, 6] == 2 and m[1, 7] == 2              # both forward reads: ONE deletion length (3) -> all 2, best 2
    assert m[2, 15] == 1 and m[2, 16] == 1            # reverse read's 2D seen from column 2
    assert m[4, 13] == 1 and m[4, 14] == 1            # its insertion is on the deletion's last column (4), reverse strand
    assert m[2, 8] == 2 and m[3, 8] == 2 and m[4, 8] == 2 and m[3, 17] == 1 and m[4, 17] == 1


@pytest.mark.parametrize("seed", range(8))
def test_oracle_matches_random_access_model_with_reference_windows(seed):
    """Every output, including the window verdict and bounds of the reference's candidate loop
    (preprocess/CreateTensorPileupFromCffi.py:356-396; tests/test_pileup_windows_cpu.py holds both to the reference itself)."""
    wild = seed % 2 == 0
    origin = [1000, 0, 5, 300][seed % 4]
    gaps = [(origin + 100, origin + 160)] if seed % 3 == 0 else ()
    rec, ref, rs = sr.random_alignment(260, depth=[3, 10, 25][seed % 3], read_len=[60, 150, 300][seed % 3], seed=seed, wild=wild,
                                       origin=origin, gaps=gaps, indel_rate=0.08, n_rate=0.01)
    kw = dict(min_depth=[2, 4][seed % 2], min_mq=[5, 20][seed % 2], call_snp_only=seed % 5 == 0, call_ht=seed % 7 == 0)
    a = po.clair3_pileup(rec, origin, origin + 260, ref, rs, **kw)
    b = model_pileup(rec, origin, origin + 260, ref, rs, **kw)
    for k in KEYS:
        assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), k


def test_properties_on_a_larger_region():
    rec, ref, rs = sr.random_alignment(6000, depth=30, read_len=1500, seed=11)
    r = po.clair3_pileup(rec, 1000, 7000, ref, rs, gvcf=True)
    m, st = r["matrix"], r["stats"]
    assert len(r["major"]) == 6000 and (np.diff(r["major"]) == 1).all()
    assert (m[:, [5, 7, 14, 16]] <= m[:, [4, 6, 13, 15]]).all()                 # best <= all
    assert (st[:, 3] == m[:, 6] + m[:, 15]).all() and (st[:, 4] == m[:, 4] + m[:, 13]).all()
    up = np.frombuffer(ref.upper().encode(), np.uint8)[r["major"] - rs]
    idx = np.select([up == ord("C"), up == ord("G"), up == ord("T")], [1, 2, 3], 0)
    rows = np.arange(len(m))
    # the reference-base feature holds minus the strand's A+C+G+T total (:368-369): the four base features of a strand sum to
    # 2 * (that feature) ... i.e. others - total = -ref count
    for base in (0, 9):
        four = m[:, base:base + 4].copy()
        refcol = four[rows, idx].copy()
        four[rows, idx] = 0
        assert (refcol <= 0).all() and (-refcol >= four.sum(axis=1)).all()
    assert len(r["cand_cols"]) > 10 and (np.diff(r["cand_cols"]) > 0).all()
    assert (r["pos_total_count"] >= r["pos_ref_count"]).all()


def test_host_side_validation_and_symbols():
    from clair3_b200 import _ffi, pileup_counts as pc
    rec, ref, rs = sr.random_alignment(300, 5, 100, seed=1)
    b = pc.BamRecords.from_dict(rec)
    assert b.n_reads == len(rec["pos"]) and b.nbytes() > 0
    bad = dict(rec)
    bad["pos"] = rec["pos"][::-1].copy()
    with pytest.raises(_ffi.C3BError, match="sorted"):
        pc.BamRecords.from_dict(bad)
    bad = dict(rec)
    bad["cigar_off"] = rec["cigar_off"][:-1]
    with pytest.raises(_ffi.C3BError, match="n_reads \\+ 1"):
        pc.BamRecords.from_dict(bad)
    for name in ("c3b_plp_create", "c3b_plp_count", "c3b_plp_sizes", "c3b_plp_fetch", "c3b_plp_device", "c3b_plp_last_ms", "c3b_plp_destroy"):
        assert name in _ffi.DECLARED_FUNCTIONS
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(_ffi.C3BError, match="no CUDA device|no CPU"):
            pc.PileupCounter(0)


def test_chunk_and_counting_regions():
    """preprocess/CreateTensorPileupFromCffi.py:281-292,305-311,55 restated: the chunks tile the contig, the counting region is the
    slice widened by 33 positions on each side, shifted by the two 1-based -> 0-based conversions on its way into C."""
    from clair3_b200 import _ffi, pileup_counts as pc
    L, n = 1_000_003, 7
    cuts = [pc.chunk_region(L, i, n) for i in range(1, n + 1)]
    assert cuts[0][0] == 0 and cuts[-1][1] >= L and all(a[1] == b[0] for a, b in zip(cuts, cuts[1:]))
    assert pc.chunk_region(700, 2, 7) == (100, 200)
    assert pc.counting_region(0, 100) == (0, 133)                 # start clipped at 1, then at 0 twice
    assert pc.counting_region(1000, 2000) == (965, 2033)          # 1000 - 33 = 967 (1-based) -> "966" -> 965 (0-based)
    with pytest.raises(_ffi.C3BError):
        pc.chunk_region(100, 0, 4)


LINEAR = [f for f in range(18) if f not in (5, 7, 14, 16)]           # every feature but the four "best allele" maxima


def split_by_parity(rec):
    """Two record sets: the even-numbered and the odd-numbered reads."""
    from clair3_b200 import synth_reads as sr
    out = []
    for par in (0, 1):
        idx = np.arange(par, len(rec["pos"]), 2)
        cig = [rec["cigar"][rec["cigar_off"][i]:rec["cigar_off"][i + 1]] for i in idx]
        seq = [rec["seq"][rec["seq_off"][i]:rec["seq_off"][i + 1]] for i in idx]
        out.append({"pos": rec["pos"][idx], "flag": rec["flag"][idx], "mapq": rec["mapq"][idx], "l_qseq": rec["l_qseq"][idx],
                    "cigar_off": np.concatenate([[0], np.cumsum([len(c) for c in cig])]).astype(np.int64),
                    "cigar": np.concatenate(cig) if cig else np.zeros(0, np.uint32),
                    "seq_off": np.concatenate([[0], np.cumsum([len(q) for q in seq])]).astype(np.int64),
                    "seq": np.concatenate(seq) if seq else np.zeros(0, np.uint8)})
    return out


def check_additivity(count, rec, start, end, ref, rs):
    """Size-independent property of the counter: with no non-ACGT read bases (no index -1 spill-over between columns), every
    feature except the best-allele maxima is LINEAR in the set of reads - on the columns both halves cover, counts(all reads) =
    counts(even reads) + counts(odd reads), minus-the-strand-total reference features included; the maxima are sub-additive."""
    a, b = split_by_parity(rec)
    whole, ra, rb = count(rec), count(a), count(b)
    common = np.intersect1d(ra["major"], rb["major"])
    assert len(common) > 0.9 * (end - start)
    iw, ia, ib = (np.searchsorted(r["major"], common) for r in (whole, ra, rb))
    mw, ma, mb = whole["matrix"][iw], ra["matrix"][ia], rb["matrix"][ib]
    assert np.array_equal(mw[:, LINEAR], ma[:, LINEAR] + mb[:, LINEAR])
    best = [5, 7, 14, 16]
    assert (mw[:, best] <= ma[:, best] + mb[:, best]).all() and (mw[:, best] >= np.maximum(ma[:, best], mb[:, best])).all()
    sw, sa, sb = whole["stats"][iw], ra["stats"][ia], rb["stats"][ib]
    assert np.array_equal(sw[:, [0, 3, 4]], sa[:, [0, 3, 4]] + sb[:, [0, 3, 4]])          # depth, del_count, ins_count
    return int(len(common))


def test_counts_are_additive_over_read_subsets():
    rec, ref, rs = sr.random_alignment(3000, depth=30, read_len=700, seed=13, n_rate=0.0, filtered_frac=0.0)
    rec["mapq"][:] = 60
    check_additivity(lambda r: po.clair3_pileup(r, 1000, 4000, ref, rs), rec, 1000, 4000, ref, rs)


@pytest.mark.parametrize("seed", range(6))
def test_host_formatter_text_matches_oracle(seed):
    """The all_alt_info strings (src/clair3_pileup.c:391-450): the product's host formatter (clair3_b200.pileup_counts.format_alt_info,
    with its own restatement of khash's bucket order), fed with allele lists in the layout the GPU exports (taken here from the
    random-access model) - including the last read with an insertion on the column, from which the formatter replays the growth of a
    full khash table on a put of a present string (src/khash.h:310-318; it reorders seeds 1 and 5) - against the C oracle's text
    (which restates khash separately)."""
    from clair3_b200 import pileup_counts as pc
    wild = seed % 2 == 0
    rec, ref, rs = sr.random_alignment(400, depth=[15, 40, 28][seed % 3], read_len=[100, 300, 200][seed % 3], seed=40 + seed, wild=wild,
                                       indel_rate=[0.08, 0.15][seed % 2], n_rate=0.01)
    max_indel = [50, 5][seed % 2]
    want = po.clair3_pileup(rec, 1000, 1400, ref, rs, alt_info=True, max_indel_length=max_indel, call_ht=seed == 5)
    m = model_pileup(rec, 1000, 1400, ref, rs, call_ht=seed == 5)
    assert np.array_equal(m["cand_cols"], want["cand_cols"]) and len(want["alt_info"]) == len(want["cand_cols"]) >= 1
    host = pc.BamRecords.from_dict(rec)
    refb = ref.encode()
    got = []
    for ci in m["cand_cols"]:
        al = m["alleles"][ci]
        cols = [np.array([a[j] for a in al], dtype=np.uint32) for j in range(4)]
        got.append(pc.format_alt_info(int(m["major"][ci]), m["matrix"][ci], m["stats"][ci], refb, rs, max_indel, *cols, host,
                                      ins_last=int(m["ins_last"][ci]), fetch_end=1400 + pc.FETCH_EXPAND + 1))
    assert got == want["alt_info"]


def test_alt_info_known_answer():
    rec, ref, *_ = case_indels()
    r = po.clair3_pileup(rec, 0, 20, ref, 0, call_ht=True, alt_info=True)
    # pos 4 (1-based 5): depth 3, ref G, r2's deletion of ref 5,6 = "GT" once, reference depth 3 - 1; pos 5: r3's insertion T after G;
    # pos 7: one A against ref T
    assert r["alt_info"] == ["5-3-G-DGT 1 RG 2 ", "6-3-G-IGT 1 RG 1 ", "8-2-T-XA 1 RT 1 "]


def test_alt_info_many_insertion_alleles_follow_khash_bucket_order():
    """40 distinct insertion alleles on one column take the reference's string counter through its 4 -> 8 -> 16 -> 32 -> 64 bucket
    growth (kick-out rehash each time): the text lists them in bucket order, identically in the oracle (C restatement of khash) and
    in the product's host formatter (Python restatement)."""
    from clair3_b200 import pileup_counts as pc
    rng = np.random.default_rng(3)
    ref = "ACGTACGTACGTACGTACGTACGT"
    items, seen = [], set()
    while len(items) < 60:
        k = int(rng.integers(1, 7))
        insert = "".join("ACGT"[i] for i in rng.integers(0, 4, k))
        if len(seen) >= 40 and insert not in seen:
            continue
        seen.add(insert)
        items.append((0, 16 if rng.random() < 0.4 else 0, 60, [("M", 4), ("I", k), ("M", 4)], "ACGT" + insert + "ACGT"))
    rec = sr.records_from_lists(items)
    want = po.clair3_pileup(rec, 0, 24, ref, 0, call_ht=True, alt_info=True)
    m = model_pileup(rec, 0, 24, ref, 0, call_ht=True)
    ci = int(np.nonzero(m["major"] == 3)[0][0])
    assert ci in m["cand_cols"].tolist()
    al = m["alleles"][ci]
    assert len({a[0] & 0x3FFFFFFF for a in al}) >= 5 and len(seen) == 40
    cols = [np.array([a[j] for a in al], dtype=np.uint32) for j in range(4)]
    text = pc.format_alt_info(3, m["matrix"][ci], m["stats"][ci], ref.encode(), 0, 50, *cols, pc.BamRecords.from_dict(rec),
                              ins_last=int(m["ins_last"][ci]))
    assert text == want["alt_info"][m["cand_cols"].tolist().index(ci)]
    assert text.count(" IT") + text.startswith("4-60-T-IT") == 40
    first_seen = []
    for it in items:
        if it[4][4:-4] not in first_seen:
            first_seen.append(it[4][4:-4])
    printed = [tok[2:] for tok in text.split("-", 3)[3].split(" ") if tok.startswith("IT")]
    assert sorted(printed) == sorted(first_seen) and printed != first_seen            # bucket order, not insertion order


def test_host_post_processing_mirrors_the_reference_caller():
    """enforce_chunk_contiguity / alt_info_list restate preprocess/CreateTensorPileupFromCffi.py:180-236 and :66-73 on the counter's
    outputs (fed here from the oracle): chunks split at coverage holes, one tuple per candidate string."""
    from clair3_b200 import pileup_counts as pc
    rec, ref, rs = sr.random_alignment(900, depth=8, read_len=120, seed=17, gaps=[(1300, 1420), (1700, 1760)])
    r = po.clair3_pileup(rec, 1000, 1900, ref, rs, alt_info=True)
    positions = np.zeros(len(r["major"]), dtype=[("major", int), ("minor", int)])
    positions["major"] = r["major"]
    chunks = pc.enforce_chunk_contiguity(r["matrix"], positions)
    assert len(chunks) >= 3 and sum(len(c[1]) for c in chunks) == len(positions)
    for counts, pos in chunks:
        assert len(counts) == len(pos) and (np.diff(pos["major"]) == 1).all()
    for (_, a), (_, b) in zip(chunks, chunks[1:]):
        assert b["major"][0] - a["major"][-1] > 1
    tup = pc.alt_info_list(r["alt_info"], "chr20")
    assert len(tup) == len(r["alt_info"]) > 0
    p0, name, alt = tup[0]
    assert p0 == int(r["major"][r["cand_cols"][0]]) + 1 and name.startswith("chr20:%d:" % p0) and alt.split("-")[0].isdigit()
    assert pc.enforce_chunk_contiguity(r["matrix"][:0], positions[:0]) == []


def test_forward_argument_checks_without_a_gpu():
    """PileupCounter.forward refuses a model without weights, the full-alignment network and a model on another device before it
    touches the library (the checks themselves need no GPU)."""
    import types
    import torch
    from clair3_b200 import _ffi, pileup_counts as pc
    ctr = object.__new__(pc.PileupCounter)
    ctr._device = torch.device("cuda", 0)
    ok = types.SimpleNamespace(_handle=object(), _kind=_ffi.CONSTANTS["C3B_PILEUP"], input_channels=18, _device=torch.device("cuda:0"), out_dim=24)
    for bad, msg in ((dict(_handle=None), "no device"), (dict(_kind=_ffi.CONSTANTS["C3B_FULL_ALIGNMENT"]), "pileup network"),
                     (dict(input_channels=8), "pileup network"), (dict(_device=torch.device("cuda", 1)), "lives on")):
        m = types.SimpleNamespace(**{**vars(ok), **bad})
        with pytest.raises(_ffi.C3BError, match=msg):
            pc.PileupCounter.forward(ctr, m)
    with pytest.raises(AttributeError):            # a valid model passes every check and only then reaches the (absent) workspace
        pc.PileupCounter.forward(ctr, ok)
    ctr._h = None                                  # so that __del__ has nothing to release


@pytest.mark.parametrize("block", range(4))
def test_arbitrary_operation_orders_with_reference_windows(block):
    """CIGARs with the nine operations in ANY order (leading deletions / skips / pads, trailing insertions, runs of the same
    operation, clips in the middle): the oracle's incremental htslib cursor and the random-access model still agree on every output,
    the reference's window verdict and bounds included."""
    ops_all = "MIDNSHP=X"
    for seed in range(block * 15, block * 15 + 15):
        rng = np.random.default_rng(1000 + seed)
        ref = sr.random_reference(400, seed=seed)
        items = []
        for _ in range(int(rng.integers(3, 25))):
            ops = [(ops_all[int(rng.integers(0, 9))], int(rng.integers(1, 6))) for _ in range(int(rng.integers(1, 9)))]
            if not any(o in "MDN=X" for o, _ in ops):
                ops.insert(int(rng.integers(0, len(ops) + 1)), ("M", int(rng.integers(1, 6))))
            lq = sum(l for o, l in ops if o in "MIS=X")
            seq = "".join("ACGTN"[int(i)] for i in rng.choice(5, lq, p=[.24, .24, .24, .24, .04])) if lq else ""
            items.append((int(rng.integers(0, 60)), int(rng.choice([0, 16])), 60, ops, seq))
        rec = sr.records_from_lists(items)
        start = int(rng.integers(0, 20))
        end = start + int(rng.integers(30, 120))
        kw = dict(call_ht=bool(seed % 2), min_depth=int(rng.integers(1, 4)))
        a = po.clair3_pileup(rec, start, end, ref, 0, **kw)
        b = model_pileup(rec, start, end, ref, 0, **kw)
        for k in KEYS:
            assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), (seed, k)


def load_counts_golden(tag):
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pileup_counts.npz"))
    rec = {k: z["%s_rec_%s" % (tag, k)] for k in ("pos", "flag", "mapq", "cigar_off", "cigar", "seq_off", "seq", "l_qseq")}
    start, end, rs, gvcf, call_ht, max_indel = (int(v) for v in z["%s_meta" % tag])
    want = {k: z["%s_%s" % (tag, k)] for k in ("matrix", "major", "stats", "cand_cols", "cand_ok", "pos_ref_count", "pos_total_count")}
    want["alt_info"] = [str(x) for x in z["%s_alt_info" % tag]]
    return rec, z["%s_ref" % tag].tobytes().decode(), rs, start, end, dict(gvcf=bool(gvcf), call_ht=bool(call_ht), max_indel_length=max_indel), want


@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_against_reference_confirmed_vectors_and_windows(tag):
    """tests/golden/pileup_counts.npz (tests/golden/make_pileup_counts_golden.py): records in, every output array and the
    all_alt_info strings out, minted from the reference's own calculate_clair3_pileup.  stats, which the reference does not have,
    come from the oracle after it was checked equal on everything else; cand_ok is the oracle's window verdict after it was
    checked equal to the positions the reference's own CreateTensorPileup keeps."""
    rec, ref, rs, start, end, kw, want = load_counts_golden(tag)
    got = po.clair3_pileup(rec, start, end, ref, rs, alt_info=True, **kw)
    for k in ("matrix", "major", "stats", "cand_cols", "cand_ok") + (("pos_ref_count", "pos_total_count") if kw["gvcf"] else ()):
        assert np.array_equal(got[k], want[k]), k
    assert got["alt_info"] == want["alt_info"] and len(want["alt_info"]) > 5
