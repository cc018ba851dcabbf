"""Test helper: the pileup feature counter's cases checked against the reference's own ``calculate_clair3_pileup`` (compiled by
oracle/pileup_ref.py), shared by tests/test_pileup_reference_cpu.py (the C oracle) and tests/test_gpu_pileup_reference.py (the
CUDA counter) so that the two lists cannot drift apart.

Every case is ``(name, build)``; ``build()`` returns ``(records, ref_seq, ref_start, start, end, kwargs)`` where the kwargs are
those of ``oracle.pileup_oracle.clair3_pileup`` / ``PileupCounter.count``.  The seeded cases repeat every ``random_alignment``
configuration of tests/test_gpu_pileup_counts.py; the targeted ones each aim at one line of src/clair3_pileup.c (cited)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from clair3_b200 import synth_reads as sr  # noqa: E402

FLANK = 16


# ------------------------------------------------------------------------------------------------------------ seeded regions
def _random(seed):
    origin = [1000, 0, 5, 300][seed % 4]
    width = [700, 256, 1025, 513][seed % 4]
    gaps = [(origin + 100, origin + 190)] if seed % 3 == 0 else ()
    rec, ref, rs = sr.random_alignment(width, depth=[4, 12, 35][seed % 3], read_len=[60, 150, 400][seed % 3], seed=100 + seed,
                                       wild=seed % 2 == 0, origin=origin, gaps=gaps, indel_rate=0.08, n_rate=0.01)
    kw = dict(min_depth=[2, 4][seed % 2], min_mq=[5, 20][seed % 2], call_snp_only=seed % 5 == 0, call_ht=seed % 7 == 0,
              gvcf=seed % 2 == 1)
    return rec, ref, rs, origin, origin + width, kw


def _alt_info(seed):
    width = [700, 3000, 513, 20000][seed]
    rec, ref, rs = sr.random_alignment(width, depth=[15, 40, 300, 30][seed], read_len=[100, 600, 300, 3000][seed], seed=60 + seed,
                                       wild=seed == 0, indel_rate=[0.08, 0.06, 0.12, 0.05][seed], n_rate=0.01)
    return rec, ref, rs, 1000, 1000 + width, dict(max_indel_length=[50, 5, 50, 50][seed], call_ht=seed == 0, gvcf=seed == 1)


def _long_reads():
    rec, ref, rs = sr.random_alignment(40000, depth=30, read_len=5000, seed=7, indel_rate=0.05)
    return rec, ref, rs, 1000, 41000, dict(gvcf=True)


def _deep_indel_rich():
    rec, ref, rs = sr.random_alignment(600, depth=300, read_len=300, seed=9, indel_rate=0.12, wild=False)
    return rec, ref, rs, 1000, 1600, {}


def _golden(tag):
    from test_pileup_oracle import load_counts_golden
    rec, ref, rs, start, end, kw, _ = load_counts_golden(tag)
    return rec, ref, rs, start, end, kw


SEEDED = ([("random_%d" % s, (lambda s=s: _random(s))) for s in range(12)]
          + [("alt_info_%d" % s, (lambda s=s: _alt_info(s))) for s in range(4)]
          + [("long_reads_40k", _long_reads), ("deep_indel_rich", _deep_indel_rich),
             ("golden_a", lambda: _golden("a")), ("golden_b", lambda: _golden("b"))])


# ------------------------------------------------------------------------------------------------------------ targeted cases
REF = sr.random_reference(400, seed=5, lower_frac=0.0, n_frac=0.0)       # upper-case A/C/G/T only
P = 200                                                                     # the column most cases aim at


def _other(b):
    return {"A": "C", "C": "G", "G": "T", "T": "A"}[b.upper()]


def _match(ref, pos, n, flag=0, mapq=60, subst=None):
    """A read of n matching bases from pos; subst: {reference position: read base} (positions outside the read are ignored)."""
    s = list(ref[pos:pos + n].upper())
    for p, b in (subst or {}).items():
        if pos <= p < pos + n:
            s[p - pos] = b
    return (pos, flag, mapq, [("M", n)], "".join(s))


def _snp_column(n_alt, depth, ref=REF, p=P, span=40):
    """depth reads over [p - span, p + span), n_alt of them with a non-reference base at p; strands alternate."""
    return [_match(ref, p - span, 2 * span, flag=16 * (i & 1), subst={p: _other(ref[p])} if i < n_alt else None)
            for i in range(depth)]


def _ins_read(ref, p, ins, flag=0, left=30, right=30):
    """A read whose last base before the insertion `ins` is on column p."""
    return (p - left + 1, flag, 60, [("M", left), ("I", len(ins)), ("M", right)], ref[p - left + 1:p + 1].upper() + ins + ref[p + 1:p + 1 + right].upper())


def _del_read(ref, p, n, flag=0, left=30, right=30):
    """A read whose last base before an n-base deletion is on column p."""
    return (p - left + 1, flag, 60, [("M", left), ("D", n), ("M", right)], ref[p - left + 1:p + 1].upper() + ref[p + 1 + n:p + 1 + n + right].upper())


def _case(items, start, end, ref=REF, **kw):
    return sr.records_from_lists(items), ref, 0, start, end, kw


def _af_cases():
    out = []
    for n_alt, depth in ((2, 25), (1, 25), (4, 50), (3, 50), (8, 100), (7, 100)):
        for snp_only in (False, True):
            out.append(("af_snp_%d_of_%d%s" % (n_alt, depth, "_snp_only" if snp_only else ""),
                        lambda n_alt=n_alt, depth=depth, snp_only=snp_only: _case(
                            _snp_column(n_alt, depth), P - 40, P + 40, call_snp_only=snp_only, call_ht=True)))
    for md in (24, 25, 26):                                          # pass_min_depth at depth 25 (:375)
        out.append(("af_snp_min_depth_%d" % md, lambda md=md: _case(_snp_column(2, 25), P - 40, P + 40, min_depth=md, call_ht=True)))
    for kind in ("ins", "del"):                                      # 3/20 and 2/20 against min_indel_af 0.15 (:384)
        for n_ev in (3, 2):
            def build(kind=kind, n_ev=n_ev):
                items = [_match(REF, P - 40, 80, flag=16 * (i & 1)) for i in range(20 - n_ev)]
                for i in range(n_ev):
                    items.append(_ins_read(REF, P, "GA", flag=16 * (i & 1)) if kind == "ins" else _del_read(REF, P, 2, flag=16 * (i & 1)))
                return _case(items, P - 40, P + 40, call_ht=True, min_snp_af=0.5)
            out.append(("af_%s_%d_of_20" % (kind, n_ev), build))
            out.append(("af_%s_%d_of_20_snp_only" % (kind, n_ev),
                        lambda build=build: (lambda c: c[:5] + ({**c[5], "call_snp_only": True},))(build())))
    return out


def _equal_majority_cases():
    """ref_count == alt_count, decided only by `ref_base - major_alt_base < 0` (:378): AF thresholds out of reach."""
    out = []
    for alt in "ACGT":
        def build(alt=alt):
            items = [_match(REF, P - 40, 80, flag=16 * (i & 1), subst={P: alt} if i < 5 else None) for i in range(10)]
            return _case(items, P - 40, P + 40, call_ht=True, min_snp_af=0.9, min_indel_af=0.9)
        if alt != REF[P]:
            out.append(("equal_majority_alt_%s_ref_%s" % (alt, REF[P]), build))
    return out


def _insertion_strings(n, seed, with_n=True, long_len=0):
    rng = np.random.default_rng(seed)
    seen, out = set(), []
    while len(out) < n:
        k = int(rng.integers(1, 7))
        s = "".join("ACGTN"[int(i)] if with_n else "ACGT"[int(i) % 4] for i in rng.choice(5, k, p=[.235, .235, .235, .235, .06]))
        if len(out) % 5 == 4 and long_len:
            s = "".join("ACGT"[int(i)] for i in rng.integers(0, 4, long_len))
        if s not in seen:
            seen.add(s)
            out.append(s)
    return out


def _many_insertions_cases():
    """Many distinct insertion alleles on one column: the reference's khash string counter (src/khash.h) grows through 4, 8, 16,
    32 and 64 buckets, and the alleles are printed in its bucket order (:428-442).  With 3 and 25 distinct strings the table is
    full after the last new key, so a later put of a present key still grows it first (khash.h:310-318)."""
    out = []
    for n in (1, 3, 4, 6, 7, 12, 13, 25, 40):
        for trailing in (False, True):
            def build(n=n, trailing=trailing):
                rng = np.random.default_rng(1000 + n)
                strs = _insertion_strings(n, seed=n, long_len=12)
                items = [_ins_read(REF, P, s, flag=16 * int(rng.random() < 0.4)) for s in strs]
                if trailing:                                              # present keys again, after the last new one
                    items += [_ins_read(REF, P, strs[int(rng.integers(0, n))], flag=16 * int(rng.random() < 0.5)) for _ in range(3)]
                else:                                                     # repeats only before the last new key
                    items = items[:-1] + [_ins_read(REF, P, strs[0], flag=16)] + items[-1:]
                items += [_match(REF, P - 40, 80) for _ in range(4)]
                # records_from_lists sorts stably by position: every insertion read starts at P - 29, so their order is kept
                return _case(items, P - 40, P + 40, call_ht=True, max_indel_length=10)
            out.append(("insertions_%d_distinct%s" % (n, "_trailing_puts" if trailing else ""), build))
    return out


def _deletion_cases():
    out = []
    ref = sr.random_reference(1400, seed=8, lower_frac=0.1, n_frac=0.0)
    for n in (31, 32, 33, 64, 65, 200):                              # the dels_f / dels_r growth (:258-265)
        def build(n=n):
            items = [_del_read(ref, P, n, flag=16 * (i % 3 == 0), left=40, right=40) for i in range(3)]
            items += [_del_read(ref, P, 5, flag=16), _match(ref, P - 39, 300), _match(ref, P - 39, 300, flag=16)]
            return _case(items, P - 39, P + 60, ref=ref, call_ht=True, max_indel_length=250)
        out.append(("deletion_len_%d" % n, build))
    for n in (50, 51):                                               # `i+1 <= max_indel_length` (:416)
        out.append(("deletion_len_%d_max_50" % n, lambda n=n: _case(
            [_del_read(ref, P, n, left=40, right=40) for _ in range(3)] + [_match(ref, P - 39, 120)], P - 39, P + 40, ref=ref, call_ht=True)))
    # a deletion whose text runs to the last base of the contig: the read ends with it
    short = ref[:300]
    out.append(("deletion_text_to_contig_end", lambda: _case(
        [(280, 0, 60, [("M", 5), ("D", 15)], short[280:285].upper())] * 2 + [_match(short, 270, 30)], 260, 300, ref=short, call_ht=True)))
    # a deletion longer than 1000 after the region's last column: the reference's text stops at its fetch window, end + 1000
    # inclusive (:189-190, :423)
    long_ref = sr.random_reference(3200, seed=9, lower_frac=0.05, n_frac=0.0)
    end = 1200
    out.append(("long_deletion_at_region_end", lambda: _case(
        [_del_read(long_ref, end - 1, 1500, left=20, right=10) for _ in range(3)] + [_match(long_ref, end - 40, 39)],
        end - 40, end, ref=long_ref, call_ht=True, max_indel_length=2000)))
    return out


def _odd_base_cases():
    """Read bases that are not A/C/G/T (N, IUPAC codes, '=') map to feature index -1 (src/clair3_pileup.h:66-71): the count lands
    on the PREVIOUS emitted column's feature 17, and on the first emitted column in front of the matrix (:286)."""
    out = []
    for code in "NRY=":
        def build(code=code):
            items = [_match(REF, P, 20, subst={P: code}), _match(REF, P, 20, flag=16), _match(REF, P, 20, subst={P + 1: code}),
                     # a coverage gap of 5 columns, then the first column after it (previous emitted column != pos - 1)
                     _match(REF, P + 25, 20, subst={P + 25: code}), _match(REF, P + 25, 20, flag=16),
                     _match(REF, P + 25, 20, flag=16, subst={P + 44: code})]                 # ... and on the last column
            return _case(items, P - 5, P + 60, call_ht=True, min_depth=1)
        out.append(("read_base_%s" % {"=": "eq"}.get(code, code), build))
    return out


def _ref_base_cases():
    """Lower-case, N and IUPAC reference bases under candidate-like columns: upper_base, then base2index maps every non-ACGT base to
    A (src/clair3_pileup.h:36-41) and the candidate test requires A/C/G/T (:376)."""
    out = []
    for rb in "acgtNRYKnr":
        def build(rb=rb):
            ref = REF[:P] + rb + REF[P + 1:]
            items = [_match(ref, P - 40, 80, flag=16 * (i & 1), subst={P: "ACGT"[i % 4]} if i < 6 else None) for i in range(10)]
            items.append(_ins_read(ref, P, "TT"))
            items.append(_del_read(ref, P, 3, flag=16))
            return _case(items, P - 40, P + 40, ref=ref, call_ht=True)
        out.append(("ref_base_%s" % rb, build))
    return out


def _edge_cases():
    out = []
    ref = REF
    for start in (0, 1):                                             # the `pre_pos == 0` reset (:225)
        def build(start=start):
            alts = {p: _other(ref[p]) for p in (16, 17, 30)}        # 16 flanking columns before column 17, 15 before column 16
            items = [_match(ref, 0, 60, flag=16 * (i & 1), subst=alts if i < 3 else None) for i in range(6)]
            return _case(items, start, 60, gvcf=True)
        out.append(("region_start_%d" % start, build))
    out.append(("region_starts_inside_reads", lambda: _case(
        [_match(ref, P - 60, 120, flag=16 * (i & 1), subst={P - 14: _other(ref[P - 14]), P - 13: _other(ref[P - 13]), P + 1: _other(ref[P + 1])}
                if i < 4 else None) for i in range(8)], P - 30, P + 40)))
    for gap in (1, 15, 16, 17):                                      # contiguous_flanking_num around a candidate (:225-229, :388-390)
        for call_ht in (False, True):
            def build(gap=gap, call_ht=call_ht):
                b = P + 6                                            # first column after the gap [b - gap, b)
                alts = {p: _other(ref[p]) for p in (b - gap - 1, b, b + 15, b + 16, b + 17)}
                items = [_match(ref, P - 40, b - gap - (P - 40), flag=16 * (i & 1), subst=alts if i < 3 else None) for i in range(6)]
                items += [_match(ref, b, 60, flag=16 * (i & 1), subst=alts if i < 3 else None) for i in range(6)]
                return _case(items, P - 40, P + 70, call_ht=call_ht)
            out.append(("coverage_gap_%d%s" % (gap, "_call_ht" if call_ht else ""), build))
    out.append(("reads_ending_at_start", lambda: _case(
        [_match(ref, P - 30, 30) for _ in range(4)] + [_match(ref, P - 30, 31, flag=16)] +
        [_match(ref, P, 40, subst={P + 2: _other(ref[P + 2])} if i < 2 else None) for i in range(4)], P, P + 40, call_ht=True)))
    return out


def _cigar_cases():
    ref = REF
    q = lambda a, b: ref[a:b].upper()                                # noqa: E731
    shapes = {
        "soft_hard_clips": [(P - 10, 0, 60, [("H", 5), ("S", 3), ("M", 20), ("S", 4), ("H", 2)], "GGG" + q(P - 10, P + 10) + "TTTT"),
                            (P - 10, 16, 60, [("S", 2), ("M", 20), ("H", 3)], "AC" + q(P - 10, P + 10))],
        "insertion_first_and_last": [(P - 10, 0, 60, [("I", 3), ("M", 11)], "TTT" + q(P - 10, P + 1)),
                                     (P - 10, 16, 60, [("S", 2), ("I", 2), ("M", 11), ("I", 4)], "CCGG" + q(P - 10, P + 1) + "ACGT"),
                                     (P - 10, 0, 60, [("M", 11), ("I", 4), ("S", 2)], q(P - 10, P + 1) + "GGTA" + "CC")],
        "deletion_then_insertion": [(P - 10, 0, 60, [("M", 11), ("D", 2), ("I", 3), ("M", 8)], q(P - 10, P + 1) + "ACG" + q(P + 3, P + 11))] * 2,
        "insertion_then_deletion": [(P - 10, 16, 60, [("M", 11), ("I", 2), ("D", 3), ("M", 8)], q(P - 10, P + 1) + "TT" + q(P + 4, P + 12))] * 2,
        "deletions_1D2D": [(P - 10, 0, 60, [("M", 11), ("D", 1), ("D", 2), ("M", 8)], q(P - 10, P + 1) + q(P + 4, P + 12)),
                           (P - 10, 16, 60, [("M", 11), ("D", 3), ("M", 8)], q(P - 10, P + 1) + q(P + 4, P + 12))],
        "pads_2I1P1I": [(P - 10, 0, 60, [("M", 11), ("I", 2), ("P", 1), ("I", 1), ("M", 8)], q(P - 10, P + 1) + "GAT" + q(P + 1, P + 9)),
                        (P - 10, 16, 60, [("M", 11), ("P", 2), ("I", 2), ("M", 8)], q(P - 10, P + 1) + "CA" + q(P + 1, P + 9)),
                        (P - 10, 0, 60, [("M", 11), ("I", 3), ("M", 8)], q(P - 10, P + 1) + "GAT" + q(P + 1, P + 9))],
        "pad_between_matches": [(P - 10, 0, 60, [("M", 11), ("P", 3), ("M", 8)], q(P - 10, P + 9))] * 2,
        "refskip_spanning_start": [(P - 20, 0, 60, [("M", 10), ("N", 30), ("M", 10)], q(P - 20, P - 10) + q(P + 20, P + 30)),
                                   (P + 5, 16, 60, [("M", 5)], q(P + 5, P + 10))],
        "all_refskip_column": [(P - 10, 0, 60, [("M", 5), ("N", 10), ("M", 5)], q(P - 10, P - 5) + q(P + 5, P + 10)),
                               (P - 10, 16, 60, [("M", 5), ("N", 10), ("M", 5)], q(P - 10, P - 5) + q(P + 5, P + 10))],
        "equal_and_diff_ops": [(P - 10, 0, 60, [("=", 5), ("X", 1), ("=", 5)], q(P - 10, P - 5) + _other(ref[P - 5]) + q(P - 4, P + 1)),
                               (P - 10, 16, 60, [("=", 11)], q(P - 10, P + 1))],
        "no_reference_operation": [(P - 10, 0, 60, [("S", 4), ("I", 3)], "ACGTACG"), (P - 10, 0, 60, [("M", 8)], q(P - 10, P - 2)),
                                   (P - 9, 0, 60, [("H", 4)], "")],
    }
    out = []
    for name, items in shapes.items():
        start = P if name == "refskip_spanning_start" else P - 12
        out.append(("cigar_" + name, lambda items=items, start=start: _case(items, start, P + 30, call_ht=True, min_depth=1)))
    return out


def _filter_cases():
    """src/medaka_bamiter.c:20-22: UNMAP, SECONDARY, QCFAIL, DUP and SUPPLEMENTARY reads are dropped, every other flag kept, then
    MAPQ < min_mq dropped."""
    out = []
    for fl in (4, 256, 512, 1024, 2048, 1, 2, 8, 32, 64, 128, 1 | 2 | 64 | 16):
        out.append(("flag_%d" % fl, lambda fl=fl: _case(
            [_match(REF, P - 40, 80) for _ in range(3)] + [_match(REF, P - 40, 80, flag=fl, subst={P: _other(REF[P])}) for _ in range(3)],
            P - 40, P + 40, call_ht=True)))
    for mq in (19, 20):
        out.append(("mapq_%d_min_20" % mq, lambda mq=mq: _case(
            [_match(REF, P - 40, 80) for _ in range(3)] + [_match(REF, P - 40, 80, mapq=mq, subst={P: _other(REF[P])}) for _ in range(3)],
            P - 40, P + 40, call_ht=True, min_mq=20)))
    return out


def _deep_column():
    """About 5000 reads on one column: the counters and the %zu / %i fields of the text."""
    rng = np.random.default_rng(77)
    items = []
    for i in range(5000):
        r = rng.random()
        if r < 0.25:
            items.append(_match(REF, P - 30, 60, flag=16 * (i & 1), subst={P: "ACGT"[i % 4]}))
        elif r < 0.35:
            items.append(_ins_read(REF, P, "ACGT"[i % 4] * (1 + i % 3), flag=16 * (i & 1)))
        elif r < 0.45:
            items.append(_del_read(REF, P, 1 + i % 4, flag=16 * (i & 1)))
        else:
            items.append(_match(REF, P - 30, 60, flag=16 * (i & 1)))
    return _case(items, P - 30, P + 30, call_ht=True, gvcf=True)


TARGETED = (_af_cases() + _equal_majority_cases() + _many_insertions_cases() + _deletion_cases() + _odd_base_cases()
            + _ref_base_cases() + _edge_cases() + _cigar_cases() + _filter_cases() + [("deep_column_5000", _deep_column)])

ALL = SEEDED + TARGETED
IDS = [n for n, _ in ALL]
BUILD = dict(ALL)


def past_contig_end():
    """Reads that reach past the contig end, with the region ending at it: the reference would read its reference sequence out
    of bounds; the GPU counter and the C oracle treat the missing bases as 'N' (DESIGN.md: the pileup counter's deviation)."""
    ref = REF[:230]
    items = [_match(REF, 200, 40, flag=16 * (i & 1), subst={232: _other(REF[232])} if i < 3 else None) for i in range(6)]
    return _case(items, 190, 240, ref=ref, call_ht=True)
