"""Test helper: the full-alignment tensor builder's cases checked against the reference's own ``calculate_clair3_full_alignment``
(compiled by oracle/fa_ref.py), shared by tests/test_fa_reference_cpu.py (the compiled reference and the committed fixture) and
tests/test_gpu_fa_reference.py (the CUDA builder) so that the two lists cannot drift apart.

Every case is ``(name, build)``; ``build()`` returns ``(records, ref_seq, candidates, variants, params)`` where ``params`` are the
keyword arguments of ``oracle.fa_ref.full_alignment`` (``fa_golden.builder_kwargs`` turns them into ``FullAlignmentBuilder.build``'s).
The seeded cases are random regions from ``synth_reads.random_fa_case``; each targeted case aims at one place of
src/clair3_full_alignment_dwell.c (cited; ``.h`` is src/clair3_full_alignment_dwell.h).  ``LARGE_SKIP`` names the cases whose
``rand_skip`` is 2^31 or more: the reference needs that many glibc ``rand()`` calls before it starts."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from clair3_b200 import synth_reads as sr  # noqa: E402

FLANK = 16


def params(need_haplotagging=False, min_mq=5, matrix_depth=8, max_indel_length=50, enable_dwell_time=False, rand_seed=1, rand_skip=0):
    return dict(need_haplotagging=need_haplotagging, min_mq=min_mq, matrix_depth=matrix_depth, max_indel_length=max_indel_length,
                enable_dwell_time=enable_dwell_time, rand_seed=rand_seed, rand_skip=rand_skip)


# ------------------------------------------------------------------------------------------------------------ seeded regions
GEN = [  # seed, random_fa_case arguments, parameters
    (1, dict(depth=30), dict(need_haplotagging=True, matrix_depth=89, enable_dwell_time=False)),
    (2, dict(depth=30), dict(need_haplotagging=False, matrix_depth=89, enable_dwell_time=False)),
    (3, dict(depth=40, dwell=True), dict(need_haplotagging=True, matrix_depth=89, enable_dwell_time=True)),
    (4, dict(depth=40, dwell=True), dict(need_haplotagging=False, matrix_depth=55, enable_dwell_time=True)),
    (5, dict(depth=150), dict(need_haplotagging=True, matrix_depth=89, enable_dwell_time=False)),
    (6, dict(depth=150, dwell=True), dict(need_haplotagging=True, matrix_depth=89, enable_dwell_time=True)),
    (7, dict(depth=90, dup_frac=0.3), dict(need_haplotagging=True, matrix_depth=55, enable_dwell_time=False)),
    (8, dict(depth=60, clip_frac=0.9), dict(need_haplotagging=True, matrix_depth=55, enable_dwell_time=False)),
    (9, dict(depth=50, long_ins=True, n_var=40), dict(need_haplotagging=True, matrix_depth=89, enable_dwell_time=False)),
    (10, dict(depth=50, long_ins=False, n_base_rate=0.02), dict(need_haplotagging=True, matrix_depth=89, enable_dwell_time=False)),
    (11, dict(depth=200, read_len=3000, n_cand=80), dict(need_haplotagging=True, matrix_depth=89, enable_dwell_time=False)),
    (12, dict(depth=20, n_var=0), dict(need_haplotagging=True, matrix_depth=89, enable_dwell_time=False, min_mq=20)),
    (13, dict(depth=120, dwell=True, dup_frac=0.2), dict(need_haplotagging=True, matrix_depth=55, enable_dwell_time=True,
                                                         max_indel_length=5)),
    # random_alignment(wild=True): = / X runs, pads, adjacent deletions, insertion after deletion, 1I2I (no reference skips)
    (21, dict(depth=40, wild=True, n_var=30), dict(need_haplotagging=True, matrix_depth=89, enable_dwell_time=False)),
    (22, dict(depth=120, wild=True, dwell=True, read_len=400), dict(need_haplotagging=True, matrix_depth=55, enable_dwell_time=True)),
    (23, dict(depth=60, wild=True, dup_frac=0.2, n_cand=120), dict(need_haplotagging=False, matrix_depth=89, enable_dwell_time=False,
                                                                    max_indel_length=5)),
]


def _seeded(seed, gen, prm):
    rec, ref, cand, var = sr.random_fa_case(seed, **gen)
    return rec, ref, cand, var, params(**dict(dict(matrix_depth=89), **prm))


SEEDED = [("%s_%d" % ("wild" if g.get("wild") else "seeded", s), (lambda s=s, g=g, p=p: _seeded(s, g, p))) for s, g, p in GEN]


# ------------------------------------------------------------------------------------------------------------ builders
REF = sr.random_reference(700, seed=11, lower_frac=0.0, n_frac=0.0)       # upper-case A/C/G/T only
C = 300                                                                     # the candidate most cases aim at
SNP = {"A": "C", "C": "G", "G": "T", "T": "A"}


def read(pos, ops, seq, flag=0, mapq=60, name=None, qual=None, mv=None):
    return dict(pos=pos, ops=ops, seq=seq, flag=flag, mapq=mapq, name=name, qual=qual, mv=mv)


def match(pos, n, ref=REF, subst=None, **kw):
    """n matching bases from pos; subst: {reference position: read base}."""
    s = list(ref[pos:pos + n].upper())
    for p, b in (subst or {}).items():
        if pos <= p < pos + n:
            s[p - pos] = b
    return read(pos, [("M", n)], "".join(s), **kw)


def ins_read(p, ins, ref=REF, left=20, right=20, **kw):
    """A read whose last base before the insertion `ins` is on p."""
    return read(p - left + 1, [("M", left), ("I", len(ins)), ("M", right)],
                ref[p - left + 1:p + 1].upper() + ins + ref[p + 1:p + 1 + right].upper(), **kw)


def del_read(p, n, ref=REF, left=20, right=20, **kw):
    """A read whose last base before an n-base deletion is on p."""
    return read(p - left + 1, [("M", left), ("D", n), ("M", right)],
                ref[p - left + 1:p + 1].upper() + ref[p + 1 + n:p + 1 + n + right].upper(), **kw)


def records(reads, with_qual=True, dwell=False):
    """Record arrays (sorted by position, stably) with base qualities, names (``r<i>`` in list order unless given) and mv tags."""
    reads = [dict(r, name=r["name"] if r["name"] is not None else "r%d" % i) for i, r in enumerate(reads)]
    reads.sort(key=lambda r: r["pos"])
    rec = sr.records_from_lists([(r["pos"], r["flag"], r["mapq"], r["ops"], r["seq"]) for r in reads])
    lq = rec["l_qseq"].astype(np.int64)
    if with_qual:
        q = [np.asarray(r["qual"], np.uint8) if r["qual"] is not None else (np.arange(int(n)) * 7 % 41).astype(np.uint8)
             for r, n in zip(reads, lq)]
        rec["qual"] = np.concatenate(q) if q else np.zeros(0, np.uint8)
        rec["qual_off"] = np.concatenate([[0], np.cumsum(lq)]).astype(np.int64)
    enc = [r["name"].encode() for r in reads]
    rec["qname"] = np.frombuffer(b"".join(enc), dtype=np.uint8).copy()
    rec["qname_off"] = np.concatenate([[0], np.cumsum([len(e) for e in enc])]).astype(np.int64)
    if dwell:
        mv = [np.asarray(r["mv"] if r["mv"] is not None else [], np.int32) for r in reads]
        rec["mv"] = np.concatenate(mv) if mv else np.zeros(0, np.int32)
        rec["mv_off"] = np.concatenate([[0], np.cumsum([len(m) for m in mv])]).astype(np.int64)
    return rec


def case(reads, cands, ref=REF, variants=(), with_qual=True, **kw):
    p = params(**kw)
    return records(reads, with_qual, p["enable_dwell_time"]), ref, np.array(cands, np.int64), list(variants), p


def cover(n, p0=C - 20, n_bases=41, **kw):
    """n plain reads over [p0, p0 + n_bases)."""
    return [match(p0, n_bases, **kw) for _ in range(n)]


# ------------------------------------------------------------------------------------------------------------ targeted cases
def _filter_cases():
    out = []
    for fl in (4, 8, 256, 2048):                        # each bit of SAMTOOLS_VIEW_FILTER_FLAG = 2316 drops the read (:539-540)
        out.append(("flag_%d_dropped" % fl, lambda fl=fl: case(
            cover(3) + [match(C - 20, 41, subst={C: SNP[REF[C]]}, flag=fl | 16 * (i & 1)) for i in range(3)], [C])))
    for fl in (1, 2, 16, 64, 128, 512, 1024):           # every other flag keeps it (:539)
        out.append(("flag_%d_kept" % fl, lambda fl=fl: case(
            cover(3) + [match(C - 20, 41, subst={C: SNP[REF[C]]}, flag=fl) for i in range(3)], [C])))
    for mq in (19, 20):                                  # alignment->core.qual < min_mq (:542)
        out.append(("mapq_%d_min_20" % mq, lambda mq=mq: case(
            cover(3) + [match(C - 20, 41, subst={C: SNP[REF[C]]}, mapq=mq) for _ in range(3)], [C], min_mq=20)))
    # read names (:547-559): the first read of a name claims it when it passes the filters, overlapping a window or not
    out.append(("name_first_filtered", lambda: case(
        [match(C - 30, 41, name="dup", flag=4), match(C - 20, 41, name="dup", subst={C: SNP[REF[C]]})] + cover(2), [C])))
    out.append(("name_first_low_mapq", lambda: case(
        [match(C - 30, 41, name="dup", mapq=3), match(C - 20, 41, name="dup", subst={C: SNP[REF[C]]})] + cover(2), [C])))
    out.append(("name_first_without_overlap", lambda: case(
        [match(C - 100, 30, name="dup"), match(C - 20, 41, name="dup", subst={C: SNP[REF[C]]})] + cover(2), [C])))
    out.append(("name_prefixes", lambda: case(
        [match(C - 20 + i, 30, name=nm, subst={C: SNP[REF[C]]} if i % 2 else None)
         for i, nm in enumerate(["r1", "r10", "r1", "r100", "r10", "r", "r1"])], [C])))
    long_a, long_b = "q" * 249 + "a", "q" * 249 + "b"
    out.append(("name_250_bytes", lambda: case(
        [match(C - 20 + i, 30, name=nm, flag=16 * (i & 1)) for i, nm in enumerate([long_a, long_b, long_a, long_b + "", "q" * 250])],
        [C])))

    def many_names():                                    # the open-addressing name table at load 1/2, long probe chains
        rng = np.random.default_rng(5)
        ref = sr.random_reference(4400, seed=12, lower_frac=0.0, n_frac=0.0)
        reads = [match(int(p), 8, ref=ref, name="n%05d" % i) for i, p in enumerate(np.sort(rng.integers(0, 4000, 4080)))]
        reads += [match(4100 + (i % 20), 30, ref=ref, name="n%05d" % int(rng.integers(0, 4080)) if i % 3 else "late%d" % i,
                        subst={4125: SNP[ref[4125]]} if i % 2 else None) for i in range(16)]
        return case(reads, [50, 2000, 3990, 4125], ref=ref)
    out.append(("names_4096_distinct", many_names))
    return out


def _window_cases():
    out = []
    out.append(("candidate_at_16", lambda: case([match(0, 40, subst={16: SNP[REF[16]]} if i < 2 else None) for i in range(5)], [16, 40])))
    for gap in (1, 32, 33, 34):                          # flanking windows overlap / touch / are apart (:501-533)
        out.append(("candidates_%d_apart" % gap, lambda gap=gap: case(
            [match(C - 40, 120, subst={C: SNP[REF[C]], C + gap: SNP[REF[C + gap]]} if i % 2 else None) for i in range(5)]
            + [ins_read(C + gap, "TG"), del_read(C + gap - 1, 2)], [C, C + gap])))
    # read_start >= end_pos is excluded, read_end <= start_pos too (:808-811); the reads one base inside are kept
    out.append(("read_bounds_at_window_edges", lambda: case(
        [match(C + 17, 20, subst={C + 17: "A"}), match(C - 36, 20), match(C + 16, 20, subst={C + 16: SNP[REF[C + 16]]}),
         match(C - 35, 20, subst={C - 16: SNP[REF[C - 16]]})] + cover(2), [C])))
    out.append(("read_starts_with_deletion", lambda: case(
        [read(C - 5, [("D", 3), ("M", 20)], REF[C - 2:C + 18]), read(C, [("D", 1), ("M", 10)], REF[C + 1:C + 11])] + cover(3), [C])))
    out.append(("read_starts_with_insertion", lambda: case(
        [read(C, [("I", 3), ("M", 20)], "GGT" + REF[C:C + 20]), read(C + 1, [("S", 2), ("I", 2), ("M", 8)], "AC" + "TT" + REF[C + 1:C + 9])]
        + cover(3), [C])))
    out.append(("read_on_one_flanking_position", lambda: case(
        [match(C - 16, 1), match(C + 16, 1, subst={C + 16: SNP[REF[C + 16]]}), match(C - 30, 15), match(C + 17, 10)] + cover(2), [C])))
    short = REF[:C + 10]
    out.append(("candidates_near_contig_end", lambda: case(
        [match(C - 30, 40, ref=short, subst={C + 5: SNP[short[C + 5]]} if i % 2 else None) for i in range(5)]
        + [read(C - 10, [("M", 15), ("D", 5)], short[C - 10:C + 5])], [C - 8, C, C + 5, C + 9], ref=short)))
    return out


def _cigar_cases():
    q = lambda a, b: REF[a:b]                            # noqa: E731
    x = SNP[REF[C]]
    shapes = {                                           # the CIGAR walk (:654-765)
        "equal_and_diff_runs": [read(C - 10, [("=", 10), ("X", 1), ("=", 10)], q(C - 10, C) + x + q(C + 1, C + 11)),
                                read(C - 8, [("X", 3), ("=", 15)], "".join(SNP[b] for b in q(C - 8, C - 5)) + q(C - 5, C + 10))],
        "clips_both_ends": [read(C - 10, [("H", 5), ("S", 3), ("M", 20), ("S", 4), ("H", 2)], "GGG" + q(C - 10, C + 10) + "TTTT"),
                            read(C - 10, [("S", 2), ("M", 20), ("H", 3)], "AC" + q(C - 10, C + 10), flag=16)],
        "pads_between_operations": [read(C - 10, [("M", 11), ("P", 3), ("M", 8)], q(C - 10, C + 9)),
                                    read(C - 10, [("M", 11), ("P", 1), ("D", 2), ("P", 2), ("M", 8)], q(C - 10, C + 1) + q(C + 3, C + 11))],
        "deletion_then_insertion": [read(C - 10, [("M", 11), ("D", 2), ("I", 3), ("M", 8)], q(C - 10, C + 1) + "ACG" + q(C + 3, C + 11))] * 2,
        "insertion_then_deletion": [read(C - 10, [("M", 11), ("I", 2), ("D", 3), ("M", 8)], q(C - 10, C + 1) + "TT" + q(C + 4, C + 12))] * 2,
        # the second deletion is anchored on the first one's last base (:692-696)
        "deletion_then_deletion": [read(C - 10, [("M", 11), ("D", 1), ("D", 2), ("M", 8)], q(C - 10, C + 1) + q(C + 4, C + 12)),
                                   read(C - 10, [("M", 10), ("D", 2), ("D", 3), ("M", 8)], q(C - 10, C) + q(C + 5, C + 13))],
        "deletion_over_the_window": [read(C - 30, [("M", 10), ("D", 45), ("M", 10)], q(C - 30, C - 20) + q(C + 25, C + 35))] * 2,
        "insertion_2I1I_on_candidate": [read(C - 10, [("M", 11), ("I", 2), ("I", 1), ("M", 8)], q(C - 10, C + 1) + "GAT" + q(C + 1, C + 9)),
                                        read(C - 10, [("M", 11), ("I", 1), ("M", 8)], q(C - 10, C + 1) + "T" + q(C + 1, C + 9))],
        "insertion_1I1P1I_on_candidate": [read(C - 10, [("M", 11), ("I", 1), ("P", 1), ("I", 1), ("M", 8)], q(C - 10, C + 1) + "CA" + q(C + 1, C + 9)),
                                          read(C - 10, [("M", 11), ("I", 1), ("M", 8)], q(C - 10, C + 1) + "C" + q(C + 1, C + 9))],
        # the overwritten insertion shares its string with another read's: the counter, hence the AF channel, counts it
        "insertion_2I1I_shared_string": [read(C - 10, [("M", 11), ("I", 2), ("I", 1), ("M", 8)], q(C - 10, C + 1) + "GAT" + q(C + 1, C + 9)),
                                         read(C - 9, [("M", 10), ("I", 2), ("M", 8)], q(C - 9, C + 1) + "GA" + q(C + 1, C + 9)),
                                         read(C - 8, [("M", 9), ("I", 1), ("I", 2), ("I", 1), ("M", 8)], q(C - 8, C + 1) + "TGAC" + q(C + 1, C + 9))],
        # the last put of a present string after the last new one grows the counter's table (khash.h:310-318)
        "insertion_2I1I_repeat_after_last_new": [read(C - 10 + i, [("M", 11 - i), ("I", 1), ("I", 1), ("M", 8)],
                                                      q(C - 10 + i, C + 1) + s + q(C + 1, C + 9)) for i, s in enumerate(["GA", "CT", "AG", "TT"])],
    }
    out = [("cigar_" + k, lambda v=v: case(v + cover(2), [C])) for k, v in shapes.items()]
    for rel in (-16, 0, 16):                             # indels anchored on c - 16, c and c + 16 (:692, :725)
        out.append(("insertion_anchored_c%+d" % rel, lambda rel=rel: case(
            [ins_read(C + rel, "AC" * (i + 1)) for i in range(3)] + cover(2, C - 40, 80), [C])))
        out.append(("deletion_anchored_c%+d" % rel, lambda rel=rel: case(
            [del_read(C + rel, 2 + i) for i in range(3)] + cover(2, C - 40, 80), [C])))
    return out


def _insertion_strings(n, seed):
    rng = np.random.default_rng(seed)
    seen, out = set(), []
    while len(out) < n:
        s = "".join("ACGTN"[int(i)] for i in rng.choice(5, int(rng.integers(1, 7)), p=[.235, .235, .235, .235, .06]))
        if s not in seen:
            seen.add(s)
            out.append(s)
    return out


def _alt_text_cases():
    out = []
    for mx in (5, 50):                                   # strlen(key) <= max_indel_length, key <= max_indel_length (:970, :990)
        for n in (mx, mx + 1):
            out.append(("insertion_len_%d_max_%d" % (n, mx), lambda n=n, mx=mx: case(
                [ins_read(C, "ACGTT" * (n // 5) + "G" * (n % 5), flag=16 * i) for i in range(2)] + [ins_read(C, "T")] + cover(2), [C],
                max_indel_length=mx)))
            ref = sr.random_reference(900, seed=13, lower_frac=0.1, n_frac=0.0)
            out.append(("deletion_len_%d_max_%d" % (n, mx), lambda n=n, mx=mx, ref=ref: case(
                [del_read(C, n, ref=ref, flag=16 * i) for i in range(2)] + [del_read(C, 1, ref=ref)] + cover(2, ref=ref), [C], ref=ref,
                max_indel_length=mx)))
    # distinct insertion strings / deletion lengths: the khash counters grow through 4, 8, 16, 32, 64 buckets, and with 3, 6, 12,
    # 25 or 49 keys a later put of a present key grows the full table first (khash.h:310-318) - the alleles' order (:963-1001)
    for n in (3, 6, 12, 25, 49):
        for trailing in (False, True):
            def ins_case(n=n, trailing=trailing):
                strs = _insertion_strings(n, seed=n)
                reads = [ins_read(C, s, name="i%03d" % i) for i, s in enumerate(strs)]
                reads += [ins_read(C, strs[i % n], name="j%03d" % i) for i in range(2)] if trailing else []
                if not trailing:
                    reads.insert(n - 1, ins_read(C, strs[0], name="k"))
                return case(reads, [C])
            out.append(("insertions_%d_distinct%s" % (n, "_repeat_after_last" if trailing else ""), ins_case))
            def del_case(n=n, trailing=trailing):
                ref = sr.random_reference(900, seed=14, lower_frac=0.0, n_frac=0.0)
                reads = [del_read(C, 1 + i, ref=ref, right=10) for i in range(n)]
                reads += [del_read(C, 1 + (7 * i) % n, ref=ref, right=10) for i in range(2)] if trailing else []
                if not trailing:
                    reads.insert(n - 1, del_read(C, 1, ref=ref, right=10))
                return case(reads, [C], ref=ref)
            out.append(("deletions_%d_distinct%s" % (n, "_repeat_after_last" if trailing else ""), del_case))
    short = REF[:C + 12]                                 # "D%.*s" runs to the contig end (:998)
    out.append(("deletion_text_to_contig_end", lambda: case(
        [read(C - 10, [("M", 11), ("D", 11)], short[C - 10:C + 1])] * 2 + [match(C - 20, 32, ref=short)], [C], ref=short)))
    for rb in "acgtNn":                                  # upper_base, acgt2num of the centre (:953-961)
        def ref_case(rb=rb):
            ref = REF[:C] + rb + REF[C + 1:]
            reads = [match(C - 20, 41, ref=ref, subst={C: "ACGT"[i % 4]}) for i in range(6)] + [ins_read(C, "TT", ref=ref),
                                                                                                del_read(C, 3, ref=ref)]
            return case(reads, [C], ref=ref)
        out.append(("ref_base_%s" % rb, ref_case))
    return out


def _depth_cases():
    out = []
    for extra in (0, 1):                                 # n == matrix_depth draws nothing, n == matrix_depth + 1 draws n - 1 (:121-134)
        out.append(("reads_depth_plus_%d" % extra, lambda extra=extra: case(
            [match(C - 20 + i, 30, subst={C: SNP[REF[C]]} if i % 3 == 0 else None, flag=16 * (i & 1)) for i in range(8 + extra)], [C])))
    for n in (3, 4):                                     # prefix padding (depth - n) >> 1 (:139-150)
        out.append(("padding_%d_of_8" % n, lambda n=n: case([match(C - 20 + i, 30) for i in range(n)], [C])))
    for md in (1, 8, 55, 89):
        out.append(("matrix_depth_%d" % md, lambda md=md: case(
            [match(C - 20 + i % 19, 30, subst={C: "ACGT"[i % 4]}, flag=16 * (i % 3 == 0)) for i in range(md + 7)], [C], matrix_depth=md)))
    out.append(("reads_1536_on_one_window", lambda: case(
        [match(C - 16 + i % 20, 20, subst={C: "ACGT"[i % 4]} if i % 5 == 0 else None) for i in range(1536)], [C])))

    def ten(**kw):                                       # ten consecutive shuffling candidates: the draw offsets add up
        cands = [200 + 40 * k for k in range(10)]
        reads = [match(c - 20 + i % 7, 30, subst={c: "ACGT"[(i + k) % 4]} if i % 2 else None, flag=16 * (i % 3 == 0))
                 for k, c in enumerate(cands) for i in range(9 + k)]
        return case(reads, cands, **kw)
    out.append(("ten_shuffling_candidates", lambda: ten()))
    for seed in (0, 42, 4294967295):
        out.append(("rand_seed_%d" % seed, lambda seed=seed: ten(rand_seed=seed)))
    for skip in LARGE_SKIPS:
        out.append(("rand_skip_%d" % skip, lambda skip=skip: ten(rand_skip=skip)))
    return out


LARGE_SKIPS = (2 ** 31 - 1, 2 ** 31, 2 ** 32 - 5, 2 ** 32 + 12345)
LARGE_SKIP = ["rand_skip_%d" % s for s in LARGE_SKIPS]


def _norm_cases():
    out = []

    def mapq_sweep():                                    # normalize_mq (.h:11) at every mapq, one read per matrix row
        cands = [100 + 40 * k for k in range(32)]
        ref = sr.random_reference(1500, seed=15, lower_frac=0.0, n_frac=0.0)
        reads = [match(c - 16, 33, ref=ref, mapq=8 * k + i, subst={c: SNP[ref[c]]} if i % 2 else None)
                 for k, c in enumerate(cands) for i in range(8)]
        return case(reads, cands, ref=ref, min_mq=0)
    out.append(("mapq_0_to_255", mapq_sweep))

    def bq_sweep(with_qual):                             # normalize_bq (.h:12) at every base quality; absent qualities are 0xFF
        reads = [match(C - 16, 33, qual=[(33 * i + k) % 256 for k in range(33)]) for i in range(8)]
        return case(reads, [C], with_qual=with_qual)
    out.append(("base_quality_0_to_255", lambda: bq_sweep(True)))
    out.append(("base_quality_absent", lambda: bq_sweep(False)))

    def af_grid(lo, hi):                                 # normalize_af(count / (float)depth) (.h:13, :915-948) for depth lo..hi
        cands, reads = [], []
        ref = sr.random_reference(300 * (hi - lo + 1) + 400, seed=16, lower_frac=0.0, n_frac=0.0)
        k = 0
        for d in range(lo, hi + 1):
            # counts whose 100 c / d is an integer first (there float32 may round below it), then spread over 0..d
            crit = [c for c in range(1, d) if 100 * c % d == 0]
            want = sorted(set(crit[::-1][:3] + [d // 3, d // 7, 1, d] + ([53, 59] if d == 100 else [])) - {0}, key=lambda c: -c)
            groups = [[]]
            for c in want:
                if sum(groups[-1]) + c > d:
                    groups.append([])
                groups[-1].append(c)
            for g in groups:
                c0 = 100 + 100 * k
                k += 1
                cands.append(c0)
                kinds = ["snp_%s" % b for b in "ACGT" if b != ref[c0]] + ["del_%d" % L for L in range(1, 40)]
                for c, kind in zip(g, kinds):
                    for _ in range(c):
                        if kind.startswith("snp"):
                            reads.append(match(c0, 1, ref=ref, subst={c0: kind[-1]}))
                        else:
                            L = int(kind[4:])
                            reads.append(read(c0, [("M", 1), ("D", L), ("M", 1)], ref[c0] + ref[c0 + 1 + L]))
                reads += [match(c0, 1, ref=ref) for _ in range(d - sum(g))]
        if len(ref) < cands[-1] + 100:
            raise AssertionError("af_grid reference too short")
        return case(reads, cands, ref=ref, matrix_depth=hi)             # every read is a matrix row
    for lo, hi in ((1, 40), (41, 80), (81, 120)):
        out.append(("af_grid_depth_%d_to_%d" % (lo, hi), lambda lo=lo, hi=hi: af_grid(lo, hi)))
    return out


def _hap_cases():
    """haplotag_read / realign_read / cigar_prefix_length (:158-422), run for reads with mapq >= 20 (:629-632)."""
    out = []
    v = C - 8
    alt = SNP[REF[v]]

    def hap_reads(n=4, **kw):
        return [match(C - 20, 41, subst={v: alt} if i % 2 else None, flag=16 * (i % 3 == 0), **kw) for i in range(n)]
    for mq in (19, 20):
        out.append(("haplotag_mapq_%d" % mq, lambda mq=mq: case(hap_reads(mapq=mq) + cover(2), [C], variants=[(v, REF[v], alt, 1, 7)],
                                                                 need_haplotagging=True)))
    spots = {   # where the variant lies in the read
        "first_aligned_base": [match(v, 30, subst={v: alt}), match(v, 30)],
        "last_aligned_base": [match(v - 29, 30, subst={v: alt}), match(v - 29, 30)],
        "inside_deletion": [read(v - 10, [("M", 8), ("D", 5), ("M", 20)], REF[v - 10:v - 2] + REF[v + 3:v + 23])] * 2,
        "at_insertion": [read(v - 10, [("M", 10), ("I", 2), ("M", 20)], REF[v - 10:v] + "GG" + REF[v:v + 20]),
                         read(v - 10, [("M", 10), ("I", 1), ("M", 20)], REF[v - 10:v] + alt + REF[v:v + 20])],
        "in_soft_clip": [read(v + 3, [("S", 5), ("M", 25)], "ACGTA" + REF[v + 3:v + 28])] * 2,
        # the skip [v - 70, v - 20) overlaps no candidate window
        "in_ref_skip": [read(v - 90, [("M", 20), ("N", 50), ("M", 40)], REF[v - 90:v - 70] + REF[v - 20:v + 20]),
                        read(v - 90, [("M", 20), ("N", 45), ("M", 30)], REF[v - 90:v - 70] + REF[v - 25:v + 5])],
    }
    for k, rs in spots.items():
        vv = v - 50 if k == "in_ref_skip" else v
        out.append(("haplotag_variant_" + k, lambda rs=rs, vv=vv: case(
            rs + hap_reads(), [C], variants=[(vv, REF[vv], SNP[REF[vv]], 1, 7), (v + 1, REF[v + 1], SNP[REF[v + 1]], 2, 7)],
            need_haplotagging=True)))
    # two phase sets with opposite costs; max == |min| gives HAP_2 (:396-421)
    for gts in ((1, 1), (1, 2), (2, 2)):
        out.append(("haplotag_two_phase_sets_gt_%d%d" % gts, lambda gts=gts: case(
            [match(C - 20, 41, subst={v: alt, v + 4: SNP[REF[v + 4]]} if i == 0 else {v: alt} if i == 1 else None) for i in range(3)] + cover(2),
            [C], variants=[(v, REF[v], alt, gts[0], 7), (v + 4, REF[v + 4], SNP[REF[v + 4]], gts[1], 9)], need_haplotagging=True)))

    def ps64():                                          # 64 phase sets on one read: the most the library keeps per read
        var = [(C - 32 + i, REF[C - 32 + i], SNP[REF[C - 32 + i]], 1 + i % 2, 100 + i) for i in range(64)]
        return case([match(C - 32, 70, subst={p: a for p, _, a, _, _ in var[::3]}), match(C - 32, 70)] + cover(2), [C],
                    variants=var, need_haplotagging=True)
    out.append(("haplotag_64_phase_sets", ps64))

    def lower():                                         # lower-case reference under the variant (realign_read's ref string)
        ref = REF[:v - 3] + REF[v - 3:v + 4].lower() + REF[v + 4:]
        return case(hap_reads(), [C], ref=ref, variants=[(v, REF[v], alt, 2, 7)], need_haplotagging=True)
    out.append(("haplotag_lower_case_reference", lower))
    return out


def _dwell_cases():
    """compute_signal_lengths_from_mv_tag (:20-74) and the signal channel (:669-672, :734-744, :905-911)."""
    out = []

    def mv_for(n_bases, runs, lead=0, stride=5):
        m = [stride] + [0] * lead
        for r in runs[:]:
            m += [1] + [0] * (r - 1)
        return m
    reads = {
        "no_tag_and_length_1": [match(C - 20, 41, mv=None), match(C - 20, 41, mv=[5]), match(C - 20, 41, mv=mv_for(41, [3] * 41))],
        "leading_zero_moves": [match(C - 20, 41, mv=mv_for(41, [2] * 41, lead=4)), match(C - 20, 41, mv=[5, 0, 0, 0])],
        "more_moves_than_bases": [match(C - 20, 41, mv=mv_for(41, [2] * 60)), match(C - 20, 41, mv=mv_for(41, [4] * 30))],
        "reverse_strand": [match(C - 20, 41, flag=16, mv=mv_for(41, list(range(1, 42)))), match(C - 20, 41, mv=mv_for(41, list(range(1, 42))))],
        "insertion_signal_wraps": [dict(ins_read(C, "ACGTA"), mv=mv_for(46, [30] * 46)), dict(ins_read(C - 3, "GG"), mv=mv_for(42, [100] * 42)),
                                   dict(ins_read(C + 2, "T"), mv=mv_for(41, [127] * 41), flag=16)],
    }
    for k, rs in reads.items():
        out.append(("dwell_" + k, lambda rs=rs: case(rs + [dict(match(C - 20, 41), mv=None)], [C], enable_dwell_time=True)))
    return out


TARGETED = (_filter_cases() + _window_cases() + _cigar_cases() + _alt_text_cases() + _depth_cases() + _norm_cases() + _hap_cases()
            + _dwell_cases())

ALL = SEEDED + TARGETED
IDS = [n for n, _ in ALL]
BUILD = dict(ALL)
assert len(BUILD) == len(ALL), "case names must be unique"
