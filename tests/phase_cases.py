"""Seeded phasing cases: random fragments for the DP, and a synthetic diploid contig - two haplotypes of heterozygous SNPs, reads
drawn from each with substitution errors and small indels - with its records, its VCF rows and the true phase."""
from __future__ import annotations

import numpy as np

from clair3_b200 import phasing
from clair3_b200.synth_reads import records_from_lists

_BASES = "ACGT"


def random_fragments(seed, n_reads, n_var, max_span=None, min_entries=2):
    """Fragments of ``n_reads`` reads over ``n_var`` variants: each read a random run of variants with a few left out, random
    alleles and weights."""
    rng = np.random.default_rng(seed)
    max_span = max_span or n_var
    out = [[], [], [], []]
    for r in range(n_reads):
        span = int(rng.integers(min_entries, max(min_entries, max_span) + 1))
        a = int(rng.integers(0, max(n_var - span, 0) + 1))
        vs = np.arange(a, min(a + span, n_var))
        vs = vs[(rng.random(len(vs)) > 0.2) | (vs == vs[0]) | (vs == vs[-1])]
        if len(vs) < min_entries:
            continue
        out[0].append(np.full(len(vs), r, np.int64))
        out[1].append(vs.astype(np.int32))
        out[2].append(rng.integers(0, 2, len(vs)).astype(np.uint8))
        out[3].append(rng.integers(1, 41, len(vs)).astype(np.uint8))
    if not out[0]:
        return phasing.empty_fragments()
    return phasing.Fragments(*(np.concatenate(a) for a in out))


def diploid_contig(seed, length, depth, read_len, het_rate=1e-3, err=0.03, indel_every=400, ctg="chr1", low_mapq_frac=0.05,
                   flagged_frac=0.03, start=0):
    """(records dict with qual / qname, reference string, VCF rows of the contig, true haplotype-0 allele per het SNP in row
    order) of a diploid contig.  The rows hold the het SNPs (GT 0/1) and, between them, rows phasing leaves alone: a 0/0
    reference call, a 1/1 SNP, a 0/1 deletion and a multi-allelic row."""
    rng = np.random.default_rng(seed)
    ref = np.array(list(_BASES))[rng.integers(0, 4, length)]
    het = np.unique(rng.integers(50, max(length - 50, 51), max(1, int(length * het_rate))))
    alt = np.array([_BASES.replace(ref[p], "")[rng.integers(0, 3)] for p in het])
    truth = rng.integers(0, 2, len(het)).astype(np.uint8)          # haplotype 0's allele
    haps = [ref.copy(), ref.copy()]
    for p, a, t in zip(het, alt, truth):
        haps[int(t)][p] = a                                          # haplotype t carries ALT
    n_reads = max(1, int(depth * length / read_len))
    items, quals = [], []
    for _ in range(n_reads):
        h = int(rng.integers(0, 2))
        L = int(max(200, min(length - start - 1, rng.normal(read_len, read_len * 0.2))))
        p = int(rng.integers(start, max(start + 1, length - L)))
        ops, seq, x = [], [], p
        while x < min(p + L, length):
            m = int(min(rng.geometric(1.0 / indel_every), min(p + L, length) - x))
            m = max(m, 1)
            seg = haps[h][x:x + m].copy()
            e = rng.random(len(seg)) < err
            seg[e] = np.array(list(_BASES))[rng.integers(0, 4, int(e.sum()))]
            ops.append(("M", len(seg)))
            seq.extend(seg.tolist())
            x += len(seg)
            if x >= min(p + L, length) - 2:
                break
            if rng.random() < 0.5:
                d = int(rng.integers(1, 4))
                ops.append(("D", d))
                x += d
            else:
                n_ins = int(rng.integers(1, 4))
                ops.append(("I", n_ins))
                seq.extend(np.array(list(_BASES))[rng.integers(0, 4, n_ins)].tolist())
        if rng.random() < 0.2:
            ops = [("S", 5)] + ops
            seq = list("ACGTA") + seq
        flag = 16 if rng.random() < 0.5 else 0
        if rng.random() < flagged_frac:
            flag |= int(rng.choice([256, 1024, 2048]))
        mapq = int(rng.integers(0, 20)) if rng.random() < low_mapq_frac else int(rng.integers(20, 61))
        items.append((p, flag, mapq, ops, "".join(seq)))
        quals.append(rng.integers(5, 41, len(seq)).astype(np.uint8))
    order = sorted(range(len(items)), key=lambda i: items[i][0])
    rec = records_from_lists([items[i] for i in order])
    q = [quals[i] for i in order]
    rec["qual"] = np.concatenate(q)
    rec["qual_off"] = np.concatenate([[0], np.cumsum([len(x) for x in q])]).astype(np.int64)
    names = [("r%d_%d" % (seed, i)).encode() for i in range(len(order))]
    rec["qname"] = np.frombuffer(b"".join(names), np.uint8).copy()
    rec["qname_off"] = np.concatenate([[0], np.cumsum([len(x) for x in names])]).astype(np.int64)
    rows = []
    fmt = "GT:GQ:DP:AD:AF"
    for i, (p, a) in enumerate(zip(het.tolist(), alt.tolist())):
        filt = "LowQual" if i % 7 == 3 else "PASS"
        rows.append("%s\t%d\t.\t%s\t%s\t%.2f\t%s\tP\t%s\t0/1:%d:%d:%d,%d:0.5000\n" % (ctg, p + 1, ref[p], a, 10 + i % 9, filt, fmt,
                                                                                    20, depth, depth // 2, depth // 2))
        q0 = p + 20
        if i % 5 == 1 and q0 < length and q0 not in het:
            kind = i // 5 % 4
            if kind == 0:
                rows.append("%s\t%d\t.\t%s\t.\t5.00\tRefCall\tP\t%s\t0/0:5:%d:%d:0.0000\n" % (ctg, q0 + 1, ref[q0], fmt, depth, depth))
            elif kind == 1:
                b = _BASES.replace(ref[q0], "")[0]
                rows.append("%s\t%d\t.\t%s\t%s\t30.00\tPASS\tF\t%s\t1/1:30:%d:0,%d:1.0000\n" % (ctg, q0 + 1, ref[q0], b, fmt, depth, depth))
            elif kind == 2:
                rows.append("%s\t%d\t.\t%s%s\t%s\t12.00\tPASS\tF\t%s\t0/1:12:%d:10,10:0.5000\n"
                            % (ctg, q0 + 1, ref[q0], ref[q0 + 1] if q0 + 1 < length else "A", ref[q0], fmt, depth))
            else:
                b, c = _BASES.replace(ref[q0], "")[:2]
                rows.append("%s\t%d\t.\t%s\t%s,%s\t15.00\tPASS\tF\tGT:GQ:DP:AD:AF\t1/2:15:%d:0,9,9:0.5,0.5\n"
                            % (ctg, q0 + 1, ref[q0], b, c, depth))
    return rec, "".join(ref.tolist()), rows, truth
