"""Synthetic coordinate-sorted alignment records in htslib's in-memory layout (bam1_core_t fields, ``len << 4 | op`` CIGAR words,
4-bit packed sequences) for the pileup feature counter (``clair3_b200.pileup_counts``): there is no BAM, FASTA or htslib in this
image, so tests and ``bench.py`` feed records of the right shape.  Pure numpy, seeded.
"""
from __future__ import annotations

import numpy as np

OP = {"M": 0, "I": 1, "D": 2, "N": 3, "S": 4, "H": 5, "P": 6, "=": 7, "X": 8}
NT16 = "=ACMGRSVTWYHKDBN"                       # htslib seq_nt16_str
_CODE = {c: i for i, c in enumerate(NT16)}
_QUERY = {0, 1, 4, 7, 8}                        # operations that consume the query
_REF = {0, 2, 3, 7, 8}                          # operations that consume the reference


def pack_seq(codes):
    """nt16 codes (one per base) -> bam_get_seq() bytes: two bases per byte, high nibble first."""
    codes = np.asarray(codes, dtype=np.uint8)
    if len(codes) & 1:
        codes = np.concatenate([codes, np.zeros(1, np.uint8)])
    return ((codes[0::2] << 4) | codes[1::2]).astype(np.uint8)


def records_from_lists(items):
    """items: iterable of (pos, flag, mapq, [(op_char, len), ...], sequence string or nt16 codes) -> the record arrays.
    Sorted by pos (stable) as a coordinate-sorted BAM is."""
    items = sorted(items, key=lambda t: t[0])
    pos, flag, mapq, cig, coff, seq, soff, lq = [], [], [], [], [0], [], [0], []
    for p, f, q, ops, s in items:
        pos.append(p)
        flag.append(f)
        mapq.append(q)
        for o, l in ops:
            cig.append((int(l) << 4) | OP[o])
        coff.append(len(cig))
        codes = np.array([_CODE[c] for c in s], dtype=np.uint8) if isinstance(s, str) else np.asarray(s, dtype=np.uint8)
        packed = pack_seq(codes)
        seq.append(packed)
        soff.append(soff[-1] + len(packed))
        lq.append(len(codes))
    return {"pos": np.array(pos, np.int64), "flag": np.array(flag, np.uint16), "mapq": np.array(mapq, np.uint8),
            "cigar_off": np.array(coff, np.int64), "cigar": np.array(cig, np.uint32),
            "seq_off": np.array(soff, np.int64), "seq": np.concatenate(seq) if seq else np.zeros(0, np.uint8),
            "l_qseq": np.array(lq, np.int32)}


def random_reference(n, seed=0, lower_frac=0.05, n_frac=0.002):
    rng = np.random.default_rng(seed)
    s = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, n)].copy()
    low = rng.random(n) < lower_frac
    s[low] += 32                                 # soft-masked (lower-case) stretches: the counter upper-cases them
    s[rng.random(n) < n_frac] = ord("N")
    return s.tobytes().decode()


_JUNCTIONS_WILD = [
    [("I", 1)], [("I", 2)], [("I", 7)], [("I", 23)], [("D", 1)], [("D", 3)], [("D", 40)], [("D", 1), ("D", 2)], [("N", 25)],
    [("I", 2), ("P", 1), ("I", 1)], [("P", 2), ("I", 3)], [("D", 2), ("I", 2)], [("I", 1), ("D", 1)], [("N", 5), ("D", 2)],
    [("D", 4), ("N", 3)], [("P", 1)], [("I", 1), ("I", 2)],
]
# the same without reference skips: a skip over a full-alignment candidate window is input the reference leaves undefined
_JUNCTIONS_WILD_NO_SKIP = [j for j in _JUNCTIONS_WILD if all(o != "N" for o, _ in j)]


def random_alignment(region_len, depth, read_len=2000, seed=0, indel_rate=0.04, sub_rate=0.03, n_rate=0.002, wild=False,
                     origin=1000, gaps=(), filtered_frac=0.08, clip_frac=0.3, short_ins=False, ref_skips=True):
    """Reads of mean length ``read_len`` tiling [origin - read_len, origin + region_len + read_len) at mean depth ``depth`` on a
    random reference.  ``wild``: junctions between match segments are drawn from a list of awkward operation runs (adjacent
    deletions, pads, skips, insertion after deletion) - slower, for tests; ``ref_skips=False`` leaves the skips (N) out of it.
    ``gaps``: (begin, end) intervals no read may start in (coverage holes).  Returns (records, ref_seq, ref_start)."""
    junctions = _JUNCTIONS_WILD if ref_skips else _JUNCTIONS_WILD_NO_SKIP
    rng = np.random.default_rng(seed)
    lo = max(0, origin - read_len)
    hi = origin + region_len + read_len
    ref_start = max(0, lo - 50)
    ref = random_reference(hi + 4 * read_len + 200 - ref_start, seed=seed + 1)
    ref_codes = np.zeros(len(ref), np.uint8)
    rb = np.frombuffer(ref.upper().encode(), dtype=np.uint8)
    for ch, code in (("A", 1), ("C", 2), ("G", 4), ("T", 8), ("N", 15)):
        ref_codes[rb == ord(ch)] = code
    n_reads = max(1, int(depth * (hi - lo) / read_len))
    starts = np.sort(rng.integers(lo, hi, n_reads))
    for g0, g1 in gaps:
        starts = starts[(starts < g0 - read_len * 2) | (starts >= g1)]
    n_reads = len(starts)
    mean_seg = max(2.0, 1.0 / max(indel_rate, 1e-6))
    pos = starts.astype(np.int64)
    flag = np.where(rng.random(n_reads) < 0.5, 16, 0).astype(np.uint16)
    bad = rng.random(n_reads) < filtered_frac
    flag[bad] |= rng.choice(np.array([4, 256, 512, 1024, 2048], np.uint16), int(bad.sum()))
    mapq = rng.integers(0, 61, n_reads).astype(np.uint8)
    cig_all, coff, seq_all, soff, lq = [], [0], [], [0], []
    for r in range(n_reads):
        L = int(max(30, rng.normal(read_len, read_len * 0.3)))
        k = max(1, int(L / mean_seg))
        seg = rng.geometric(1.0 / mean_seg, k).astype(np.int64)
        if wild:
            ops, lens = [], []
            for i in range(k):
                ops.append(rng.choice([0, 7, 8], p=[0.8, 0.1, 0.1]))
                lens.append(int(seg[i]))
                if i + 1 < k:
                    for o, l in junctions[rng.integers(0, len(junctions))]:
                        ops.append(OP[o])
                        lens.append(l)
            ops = np.array(ops, np.int64)
            lens = np.array(lens, np.int64)
        else:
            ops = np.zeros(2 * k - 1, np.int64)
            lens = np.zeros(2 * k - 1, np.int64)
            lens[0::2] = seg
            j = rng.random(k - 1) < 0.5
            ops[1::2] = np.where(j, 1, 2)
            jl = rng.geometric(0.6, k - 1)
            if not short_ins:
                big = rng.random(k - 1) < 0.03
                jl = np.where(big, rng.integers(8, 40, k - 1), jl)
            lens[1::2] = jl
        if rng.random() < clip_frac:
            c = rng.integers(1, 30)
            ops = np.concatenate([[4 if rng.random() < 0.7 else 5], ops])
            lens = np.concatenate([[c], lens])
        if rng.random() < clip_frac:
            c = rng.integers(1, 30)
            ops = np.concatenate([ops, [4 if rng.random() < 0.7 else 5]])
            lens = np.concatenate([lens, [c]])
        qcons = np.isin(ops, list(_QUERY))
        rcons = np.isin(ops, list(_REF))
        ql = np.where(qcons, lens, 0)
        rl = np.where(rcons, lens, 0)
        y0 = np.cumsum(ql) - ql
        x0 = np.cumsum(rl) - rl
        nq = int(ql.sum())
        q = np.frombuffer(b"\x01\x02\x04\x08", dtype=np.uint8)[rng.integers(0, 4, nq)].copy()
        mm = np.isin(ops, [0, 7, 8])
        ml = lens[mm]
        tot = int(ml.sum())
        if tot:
            ar = np.arange(tot) - np.repeat(np.cumsum(ml) - ml, ml)
            qi = np.repeat(y0[mm], ml) + ar
            ri = np.repeat(x0[mm], ml) + ar + (int(pos[r]) - ref_start)
            ri = np.minimum(ri, len(ref_codes) - 1)
            copy = rng.random(tot) >= sub_rate
            q[qi[copy]] = ref_codes[ri[copy]]
        q[rng.random(nq) < n_rate] = rng.choice(np.array([15, 0, 3, 5], np.uint8))
        packed = pack_seq(q)
        cig_all.append(((lens.astype(np.uint32) << 4) | ops.astype(np.uint32)).astype(np.uint32))
        coff.append(coff[-1] + len(ops))
        seq_all.append(packed)
        soff.append(soff[-1] + len(packed))
        lq.append(nq)
    rec = {"pos": pos, "flag": flag, "mapq": mapq, "cigar_off": np.array(coff, np.int64),
           "cigar": np.concatenate(cig_all) if cig_all else np.zeros(0, np.uint32), "seq_off": np.array(soff, np.int64),
           "seq": np.concatenate(seq_all) if seq_all else np.zeros(0, np.uint8), "l_qseq": np.array(lq, np.int32)}
    return rec, ref, ref_start


def aligned_bases(rec):
    """Reference bases covered by all records (the counter's unit of work)."""
    ops = rec["cigar"] & 15
    lens = rec["cigar"] >> 4
    return int(lens[np.isin(ops, list(_REF))].sum())


def random_fa_case(seed, region_len=3000, depth=30, read_len=1500, n_cand=40, n_var=12, dup_frac=0.05, dwell=False, n_base_rate=0.003,
                   long_ins=True, clip_frac=0.3, mv_missing_frac=0.1, wild=False):
    """A full-alignment test case on a contig that starts at position 0: records with base qualities, read names (``dup_frac`` of
    them repeating an earlier name) and, with ``dwell``, ``mv`` move tables; strictly ascending candidates (>= 16) and sorted
    phased heterozygous SNPs ``(position, ref_base, alt_base, genotype, phase_set)``.  Query bases are A/C/G/T with a few N; the
    reference has soft-masked (lower-case) stretches and a few N.  ``wild``: ``random_alignment``'s awkward operation runs, without
    reference skips.  Returns (records, ref_seq, candidates, variants)."""
    rng = np.random.default_rng(seed + 7919)
    rec, ref, rs = random_alignment(region_len, depth, read_len=read_len, seed=seed, n_rate=0.0, origin=read_len,
                                    clip_frac=clip_frac, short_ins=not long_ins, wild=wild, ref_skips=False)
    assert rs == 0
    n = len(rec["pos"])
    lq = rec["l_qseq"].astype(np.int64)
    seq = rec["seq"].copy()
    for r in range(n):                                    # a few N read bases (nt16 15): alt 100, counted as A
        k = rng.binomial(int(lq[r]), n_base_rate)
        for q in rng.integers(0, max(int(lq[r]), 1), k):
            b = int(rec["seq_off"][r]) + int(q >> 1)
            seq[b] = (seq[b] & 0x0F) | 0xF0 if q % 2 == 0 else (seq[b] & 0xF0) | 0x0F
    rec["seq"] = seq
    rec["qual"] = rng.integers(0, 61, int(lq.sum())).astype(np.uint8)
    rec["qual_off"] = np.concatenate([[0], np.cumsum(lq)]).astype(np.int64)
    names = []
    for r in range(n):
        names.append(names[rng.integers(0, r)] if r and rng.random() < dup_frac else "read_%d_%d" % (seed, r))
    enc = [s.encode() for s in names]
    rec["qname"] = np.frombuffer(b"".join(enc), dtype=np.uint8).copy()
    rec["qname_off"] = np.concatenate([[0], np.cumsum([len(e) for e in enc])]).astype(np.int64)
    if dwell:
        mv, off = [], [0]
        for r in range(n):
            if rng.random() < mv_missing_frac:
                off.append(off[-1])
                continue
            runs = rng.geometric(0.3, int(lq[r]) + int(rng.integers(-3, 4)))      # samples per base, a few bases more or less
            runs[rng.random(len(runs)) < 0.01] += 140                             # > 127: the int8 channel wraps
            m = np.zeros(1 + int(runs.sum()), np.int32)
            m[0] = 5                                                              # the stride element
            m[1 + np.concatenate([[0], np.cumsum(runs)[:-1]])] = 1
            mv.append(m)
            off.append(off[-1] + len(m))
        rec["mv"] = np.concatenate(mv) if mv else np.zeros(0, np.int32)
        rec["mv_off"] = np.array(off, np.int64)
    lo, hi = read_len, read_len + region_len
    cand = np.unique(rng.integers(lo, hi, n_cand)).astype(np.int64)
    vpos = np.unique(rng.integers(lo - 200, hi + 200, n_var))
    variants = []
    for p in vpos:
        rb = ref[int(p)].upper()
        ab = "ACGT".replace(rb, "")[int(rng.integers(0, 3))] if rb in "ACGT" else "A"
        variants.append((int(p), rb, ab, int(rng.integers(1, 3)), int(1000 + (p // 700))))
    return rec, ref, cand, variants
