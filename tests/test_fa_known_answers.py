"""More known answers of the reference's calculate_clair3_full_alignment (compiled by oracle/fa_ref.py; skipped where
oracle/_ref is not built), each derived from the cited lines of src/clair3_full_alignment_dwell.{c,h}, plus the bed / VCF helpers
and the BAM round trip of the full-alignment record fields."""
import ctypes
import gzip
import os

import numpy as np
import pytest

from clair3_b200 import bam_io
from clair3_b200 import fa_tensor as ft
from clair3_b200 import synth_reads as sr

REF = "ACGT" * 50          # 200 bases: position p holds "ACGT"[p % 4]
C = 16                     # the candidate column of a 33-column window


def _oracle():
    from oracle import fa_ref
    if fa_ref.build() is None:
        pytest.skip("oracle/_ref/libclair3_fa_ref.so is not built (no reference checkout found)")
    return fa_ref


def _run(items, cand, ref=REF, **kw):
    return _oracle().full_alignment(sr.records_from_lists(items), cand, ref, **kw)


def _sub(s, i, b):
    return s[:i] + b + s[i + 1:]


def test_haplotag_hap1_hap2_unphased():
    # variant at 120 (ref 'A', alt 'C'), phase set 7, genotype 1 (0|1).  realign_read (:262-313) compares the read around the
    # variant with ref and with alt over overhang 10 bases each side: a read showing ref -> allele 1 == genotype -> cost +1 ->
    # HAP_1 (channel 7 = 30); a read showing alt -> allele 2 -> cost -1 -> HAP_2 (90); a read with mapq < 20 is not tagged (60).
    var = [(120, "A", "C", 1, 7)]
    ref_read = REF[100:160]
    alt_read = _sub(REF[100:160], 20, "C")
    items = [(100, 0, 60, [("M", 60)], alt_read), (100, 0, 60, [("M", 60)], ref_read), (100, 0, 10, [("M", 60)], ref_read)]
    m, _, _ = _run(items, [130], variants=var, need_haplotagging=True, matrix_depth=3)
    # rows sorted by (haplotype, read index) (:92-103): unphased read 2, HAP_1 read 1, HAP_2 read 0
    assert m[0, :, C, 7].tolist() == [60, 30, 90]
    assert m[0, 2, 120 - 114, 1] == 25            # the HAP_2 row shows the alt base C at position 120 (column 120 - (130 - 16))


def test_haplotag_lowercase_reference_never_matches():
    # realign_read takes the RAW reference bytes (get_ref_seq, :207-215): over a soft-masked stretch no read base matches the
    # reference string.  A read showing the reference base: 21 mismatches against ref and against alt -> allele 0, no cost ->
    # unphased (60; the same read is HAP_1 over upper-case bases).  A read showing the alt base matches alt's one upper-case base
    # -> allele 2 -> genotype 1 gives cost -1 -> HAP_2 (90).
    ref = REF[:105] + REF[105:136].lower() + REF[136:]
    var = [(120, "A", "C", 1, 7)]
    items = [(100, 0, 60, [("M", 60)], REF[100:160]), (100, 0, 60, [("M", 60)], _sub(REF[100:160], 20, "C"))]
    m, _, _ = _run(items, [130], ref=ref, variants=var, need_haplotagging=True, matrix_depth=2)
    assert m[0, :, C, 7].tolist() == [60, 90]


def test_haplotag_variant_on_last_base_appends_alt():
    # variant on the read's last aligned base: the right-hand cigar_prefix_length (:158-205) runs out of CIGAR before overhang + 1
    # bases and leaves 0 / 0, so the query stops before the variant and alt = ref[v-10, v) + alt base, appended at
    # alt[left_ref_bases] (:292-295).  The query equals ref -> distance 0 < 1 -> allele 1 whatever the read shows there.
    var = [(139, "T", "A", 1, 3)]
    read = _sub(REF[100:140], 39, "A")           # shows the alt base on its last base
    m, _, _ = _run([(100, 0, 60, [("M", 40)], read)], [130], variants=var, need_haplotagging=True, matrix_depth=1)
    assert m[0, 0, C, 7] == 30                    # allele 1 == genotype 1 -> HAP_1


def test_reference_n_and_alt_channel_precedence():
    # ref N -> channel 0 = 100 (num2countbase_fa['N' - 'A'], .h:39-44).  On one base, insertion (-50) beats deletion start (-100),
    # which beats a mismatch (:855-896)
    ref = _sub(REF, 130, "N")
    ins_del = [(110, 0, 60, [("M", 21), ("I", 2), ("D", 3), ("M", 20)], _sub(REF[110:131], 20, "G") + "TT" + REF[134:154])]
    del_only = [(110, 0, 60, [("M", 21), ("D", 3), ("M", 20)], _sub(REF[110:131], 20, "G") + REF[134:154])]
    snp = [(110, 0, 60, [("M", 40)], _sub(REF[110:150], 20, "G"))]
    for items, alt_v in ((ins_del, -50), (del_only, -100), (snp, 75)):
        m, _, _ = _run(items, [130], ref=ref, matrix_depth=1)
        assert m[0, 0, C, 0] == 100 and m[0, 0, C, 1] == alt_v


def test_dwell_without_mv_and_int8_wrap():
    # channel 8 = (int8_t) of the per-base signal length (:905-911): no mv tag -> 0; 200 samples on a base -> -56
    fa_ref = _oracle()
    rec = sr.records_from_lists([(100, 0, 60, [("M", 40)], REF[100:140]), (100, 0, 60, [("M", 40)], REF[100:140])])
    moves = np.ones(1 + 40, np.int32)
    moves[0] = 5
    # base 30 (position 130) gets 200 samples: its move 1 followed by 199 zeros
    mv = np.concatenate([moves[:32], np.zeros(199, np.int32), moves[32:]])
    rec["mv"], rec["mv_off"] = mv, np.array([0, 0, len(mv)], np.int64)
    m, _, _ = fa_ref.full_alignment(rec, [130], REF, matrix_depth=2, enable_dwell_time=True)
    assert m[0, 0, C, 8] == 0 and m[0, 1, C, 8] == -56 and m[0, 1, C - 1, 8] == 1


def test_draws_per_candidate_and_chaining_against_libc():
    # sort_read_name_by_haplotype draws n - 1 rand() values for every candidate with n > depth reads (:117-134), in candidate
    # order; rand_skip continues the process-global stream
    fa_ref = _oracle()
    items = [(100 + (i % 3), 0, 60, [("M", 60)], REF[100 + (i % 3):160 + (i % 3)]) for i in range(12)]
    rec = sr.records_from_lists(items)
    m1, _, d1 = fa_ref.full_alignment(rec, [130, 140], REF, matrix_depth=5)
    assert d1 == 2 * (12 - 1)
    m2, _, d2 = fa_ref.full_alignment(rec, [140], REF, matrix_depth=5, rand_skip=11)
    assert d2 == 11 and np.array_equal(m2[0], m1[1])
    libc = ctypes.CDLL(None)
    libc.srand(1)
    assert ft.glibc_rand(1, 11, 11).tolist() == [libc.rand() for _ in range(22)][11:]


def test_candidates_from_bed(tmp_path):
    p = tmp_path / "fa.bed"
    p.write_text("ctg\t100\t133\nctg\t0\t40\nother\t500\t533\nctg\t300\t301\tA-C-1-7\nctg\t200\t233\n")
    cand, lo, hi = ft.candidates_from_bed(str(p), "ctg")
    # centres (:73-78): start 100 -> 101 + 33 // 2 - 1 = 116 -> 0-based 115; start 0 -> 41 - 16 - 2 = 23 -> 22; 200 -> 215
    assert cand == [22, 115, 215] and (lo, hi) == (1, 302)
    assert ft.candidates_from_bed(str(p), "none") == ([], None, None)


def test_phased_variants_from_vcf(tmp_path):
    body = ("##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tS\n"
            "ctg\t101\t.\tA\tC\t30\tPASS\t.\tGT:PS\t0|1:77\n"
            "ctg\t150\t.\tG\tT\t30\tPASS\t.\tGT:PS\t1|0:77\n"
            "ctg\t160\t.\tG\tT\t30\tPASS\t.\tGT\t0/1\n"
            "chr2\t10\t.\tA\tG\t30\tPASS\t.\tGT:PS\t0|1:5\n")
    p = tmp_path / "p.vcf.gz"
    with gzip.open(p, "wt") as f:
        f.write(body)
    assert ft.phased_variants_from_vcf(str(p), "ctg") == [(100, "A", "C", 1, 77), (149, "G", "T", 2, 77)]
    q = tmp_path / "p.vcf"
    q.write_text(body)
    assert len(ft.phased_variants_from_vcf(str(q))) == 3


def test_bam_round_trip_of_full_alignment_fields(tmp_path):
    rec, ref, cand, var = sr.random_fa_case(5, depth=15, dwell=True)
    rec["mv"] = rec["mv"].copy()
    rec["mv"][int(rec["mv_off"][3])] = 300          # a value beyond int8: written as mv:B:i
    path = str(tmp_path / "fa.bam")
    bam_io.write_bam(path, rec, [("ctg", len(ref))])
    got, refs = bam_io.read_bam(path, fa_fields=True)
    for k in ("pos", "flag", "mapq", "cigar_off", "cigar", "seq_off", "seq", "l_qseq", "qual", "qual_off", "qname", "qname_off",
              "mv", "mv_off"):
        assert np.array_equal(np.asarray(got[k]), np.asarray(rec[k])), k
    plain, _ = bam_io.read_bam(path)
    assert not any(k in plain for k in ("qual", "qname", "mv"))
