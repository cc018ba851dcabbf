"""Crafted alignment records for the phasing observations (``phasing.fragments``, ``phase_fragment_kernel``): each case is a
contig with heterozygous SNP rows and reads at the record edges - every CIGAR operation, zero-length operations, CIGARs of
31 to 65 operations and one past 65,535 (written through the CG tag), qualities 0 / 1 / 93 / 0xFF, N and IUPAC bases at a
variant, a CIGAR longer than its sequence, MAPQ 19 / 20 / 255, each FLAG bit alone, reads of one and two entries, and
variants and reads at the contig's and the decode spans' edges."""
from __future__ import annotations

import re

import numpy as np

from clair3_b200.synth_reads import NT16, records_from_lists

_ACGT = "ACGT"
_CODE = {c: i for i, c in enumerate(NT16)}


class Read:
    """One record: pos, CIGAR text, flag, MAPQ; at each variant it covers with an aligned base it shows allele
    ``(variant index + hap) % 2`` unless ``bases`` gives that variant's nt16 code; ``qual`` one quality for every base (None:
    a pattern); ``lq`` cuts the sequence to that many bases."""

    def __init__(self, pos, cigar, flag=0, mapq=60, hap=0, bases=None, qual=None, lq=None):
        self.pos, self.flag, self.mapq, self.hap = pos, flag, mapq, hap
        self.ops = [(o, int(n)) for n, o in re.findall(r"(\d+)([MIDNSHP=X])", cigar)] if isinstance(cigar, str) else cigar
        self.bases, self.qual, self.lq = bases or {}, qual, lq


class Case:
    """A contig of ``length`` random bases with 0/1 SNP rows at ``var_pos`` and the records of ``reads``; ``spans`` are the
    decode spans to run it at."""

    def __init__(self, length, var_pos, reads, spans=(1 << 30,), seed=0, ctg="chr1"):
        rng = np.random.default_rng(seed)
        self.length, self.ctg, self.spans = length, ctg, tuple(spans)
        self.ref = "".join(_ACGT[i] for i in rng.integers(0, 4, length))
        self.var_pos = [int(p) for p in var_pos]
        assert self.var_pos == sorted(set(self.var_pos)) and self.var_pos[-1] < length
        self.alt = [_ACGT[(_ACGT.index(self.ref[p]) + 1 + int(rng.integers(0, 3))) % 4] for p in self.var_pos]
        self.rows = ["%s\t%d\t.\t%s\t%s\t30\tPASS\tP\tGT:GQ\t0/1:30\n" % (ctg, p + 1, self.ref[p], a)
                     for p, a in zip(self.var_pos, self.alt)]
        self.reads = sorted(reads, key=lambda r: r.pos)          # as records_from_lists orders them (stable)
        self.rec = self._records()

    def _seq(self, r):
        vidx = {p: i for i, p in enumerate(self.var_pos)}
        out, x = [], r.pos
        for op, n in r.ops:
            if op in "M=X":
                for y in range(x, x + n):
                    base = _CODE[self.ref[y]]
                    if op == "X":
                        base = _CODE[_ACGT[(_ACGT.index(self.ref[y]) + 2) % 4]]
                    if y in vidx:
                        v = vidx[y]
                        base = r.bases.get(v, _CODE[self.alt[v] if (v + r.hap) % 2 else self.ref[y]])
                    out.append(base)
                x += n
            elif op in "DN":
                x += n
            elif op in "IS":
                out.extend([_CODE["C"]] * n)
        assert x <= self.length, "a read past the contig's end"
        return np.array(out if r.lq is None else out[:r.lq], np.uint8)

    def _records(self):
        items, quals = [], []
        for i, r in enumerate(self.reads):
            s = self._seq(r)
            items.append((r.pos, r.flag, r.mapq, r.ops, s))
            q = (np.arange(len(s)) * 7 + 5 * i) % 60 + 1 if r.qual is None else np.full(len(s), r.qual)
            quals.append(q.astype(np.uint8))
        rec = records_from_lists(items)
        rec["qual"] = np.concatenate(quals) if quals else np.zeros(0, np.uint8)
        rec["qual_off"] = np.concatenate([[0], np.cumsum([len(q) for q in quals])]).astype(np.int64)
        return rec


def _cover(lo, hi, hap, step=60):
    """Plain M reads of both haplotypes tiling [lo, hi): they link the variants there into blocks."""
    return [Read(p, "%dM" % min(2 * step, hi - p), hap=(hap + i) % 2) for i, p in enumerate(range(lo, hi - 1, step))]


def ops_case():
    """= and X reads, mixed M = X, an N skip and a D over a variant, H and P inside a read, zero-length operations, a leading I."""
    var = [100, 110, 120, 130, 140, 300, 305, 310, 330, 340, 500, 510, 520, 530, 700, 705, 710, 720, 900, 905, 910, 915, 1100,
           1110, 1120]
    reads = [Read(95, "50="), Read(95, "5=1X9=1X9=1X24=", hap=1), Read(98, "2M3=1X4M10=5X20M"),
             Read(295, "10M15N20M"), Read(295, "12M5D30M", hap=1),
             Read(495, "5H10M2P10M3I1P15M5H"),
             Read(690, "0M10M0=5=0X5X0D0N12M3=0M", hap=1),
             Read(895, "3I25M"), Read(1095, "2S4I30M", hap=1)]
    for lo, hi in ((80, 160), (280, 360), (480, 550), (680, 740), (880, 930), (1080, 1140)):
        reads += _cover(lo, hi, 0, step=30)
    return Case(1300, var, reads, spans=(1 << 30, 300))


def edges_case():
    """Variants on the first and last reference base of every aligned operation, and of the read."""
    var = [200, 209, 210, 217, 218, 220, 225, 227, 230, 233, 236, 242]
    reads = [Read(200, "10M3I8=2D6X4N1M5D7M"), Read(200, "43M", hap=1), Read(195, "5S48M"), Read(200, "10=33X", hap=1)]
    return Case(400, var, reads, spans=(1 << 30, 210))


def _ops_of(n):
    """n CIGAR operations, the last an M: M / I / M / D cycles."""
    cyc = [("M", 3), ("I", 1), ("M", 2), ("D", 1)]
    return [cyc[i % 4] for i in range(n - 1)] + [("M", 3)]


def ciglen_case():
    """CIGARs of exactly 31, 32, 33, 64 and 65 operations, and one of 70,001 through the CG tag."""
    var, reads = [], []
    for i, n in enumerate((31, 32, 33, 64, 65)):
        p = 100 + 300 * i
        ops = _ops_of(n)
        span = sum(x for o, x in ops if o in "MD")
        var += list(range(p, p + span, 4)) + [p + span - 1]
        reads += [Read(p, ops), Read(p, "%dM" % span, hap=1)]
    p0, n_big = 2000, 70001
    big = [("M", 1) if i % 2 == 0 else ("I", 1) for i in range(n_big)]
    span = (n_big + 1) // 2
    var += list(range(p0 + 3, p0 + span, 97)) + [p0 + span - 1]
    reads.append(Read(p0, big))
    reads += [Read(p, "%dM" % min(3000, p0 + span - p), hap=1) for p in range(p0, p0 + span - 1, 1500)]
    return Case(p0 + span + 500, sorted(set(var)), reads, spans=(1 << 30, 7000))


def qual_case():
    """Reads of quality 0, 1, 93 and 0xFF (the bytes of a record written without qualities) at every base."""
    var = [100, 110, 120, 300, 310, 320, 500, 510, 520, 700, 710, 720]
    reads = []
    for i, q in enumerate((0, 1, 93, 0xFF)):
        p = 95 + 200 * i
        reads += [Read(p, "40M", qual=q), Read(p, "40M", hap=1), Read(p + 2, "35M", qual=q, hap=1)]
    return Case(900, var, reads)


def bases_case():
    """N, IUPAC codes and '=' at a variant (no entry), and CIGARs that run past the sequence (l_qseq)."""
    var = [100, 110, 120, 130, 300, 310, 320, 330, 500, 510, 520, 530]
    iupac = {c: _CODE[c] for c in "NRYMKSWBDHV="}
    reads = [Read(95, "40M", bases={0: iupac["N"], 2: iupac["R"]}), Read(95, "40M", bases={1: iupac["Y"], 3: iupac["="]}, hap=1),
             Read(95, "40M", bases={0: iupac["M"], 1: iupac["K"], 2: iupac["S"]}), Read(95, "40M", hap=1),
             Read(295, "40M", bases={4: iupac["W"], 5: iupac["B"], 6: iupac["D"], 7: iupac["H"]}),
             Read(295, "40M", bases={4: iupac["V"]}, hap=1), Read(295, "40M"),
             Read(495, "40M", lq=26), Read(495, "10M2I28M", lq=27, hap=1), Read(495, "5S35M", lq=31), Read(495, "40M", hap=1)]
    return Case(700, var, reads)


FLAG_BITS = (0x1, 0x2, 0x4, 0x8, 0x10, 0x20, 0x40, 0x80, 0x100, 0x200, 0x400, 0x800)


def flags_case():
    """MAPQ 19, 20 and 255, and each FLAG bit alone on a read of three entries."""
    var = [100, 110, 120, 300, 310, 320]
    reads = [Read(95, "40M", mapq=q, hap=i % 2) for i, q in enumerate((19, 20, 255))]
    reads += [Read(295, "40M", flag=f, hap=i % 2) for i, f in enumerate(FLAG_BITS)]
    reads += [Read(95, "40M", hap=1), Read(295, "40M", hap=1)]
    return Case(500, var, reads)


def few_case():
    """A read of exactly one entry (dropped) and one of exactly two."""
    var = [100, 110, 300, 310]
    reads = [Read(95, "10M"), Read(95, "20M", hap=1), Read(95, "30M"), Read(295, "10M5D8M", bases={3: _CODE["N"]}),
             Read(295, "20M", hap=1), Read(290, "30M")]
    return Case(500, var, reads)


def span_case():
    """Variants at contig positions 0 and length - 1, a read across three decode spans, reads starting on span edges."""
    L = 3000
    var = [0, 5, 10, 490, 500, 510, 600, 990, 1000, 1010, 1490, 1500, 1510, 2490, 2500, 2510, 2990, 2995, 2999]
    reads = [Read(0, "20M"), Read(0, "12M", hap=1), Read(2980, "20M"), Read(2985, "15M", hap=1), Read(480, "40M"),
             Read(500, "20M", hap=1), Read(600, "1000M"), Read(1000, "20M"), Read(1480, "40M", hap=1), Read(1500, "20M"),
             Read(2480, "40M"), Read(2500, "20M", hap=1), Read(985, "30M", hap=1)]
    return Case(L, var, reads, spans=(500, 499, 1 << 30))


def last_span_case():
    """A contig whose only reads start in its last decode span."""
    var = [2810, 2820, 2830, 2900, 2950, 2990]
    reads = [Read(2800, "60M"), Read(2805, "50M", hap=1), Read(2825, "100M"), Read(2890, "105M", hap=1), Read(2940, "60M")]
    return Case(3000, var, reads, spans=(700, 1000))


CASES = {"ops": ops_case, "edges": edges_case, "ciglen": ciglen_case, "qual": qual_case, "bases": bases_case,
         "flags": flags_case, "few": few_case, "span": span_case, "last_span": last_span_case}
