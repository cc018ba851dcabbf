"""Seeded FASTA files for the tests of the bgzip-compressed reference: plain FASTAs of chosen line widths and line ends, and
their BGZF copies with the ``.fai`` and the ``.gzi`` that ``samtools faidx`` writes, the blocks cut where a test wants them
and compressed by zlib or a chosen ``deflate_craft`` mode."""
from __future__ import annotations

import os
import shutil
import struct

import numpy as np

import bam_craft as bc
import deflate_craft as dc
from clair3_b200 import bam_io

# bases as references hold them: mostly upper-case ACGT, soft-masked runs in lower case, N and the other IUPAC codes
_LETTERS = np.frombuffer(b"ACGTacgtNnRYKMSWBDHV", np.uint8)
_WEIGHTS = np.array([20, 20, 20, 20, 6, 6, 6, 6, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1], float)


def random_sequence(n, rng):
    return _LETTERS[rng.choice(len(_LETTERS), n, p=_WEIGHTS / _WEIGHTS.sum())].tobytes().decode()


def write_fasta(path, seqs, width=60, eol="\n"):
    """``seqs`` [(name, bases)] as a FASTA of ``width`` bases per line (None: one line per sequence), lines ended by ``eol``."""
    with open(path, "w", newline="") as f:
        for name, seq in seqs:
            f.write(">%s desc\t%d%s" % (name, len(seq), eol))
            w = width or max(len(seq), 1)
            for i in range(0, len(seq), w):
                f.write(seq[i:i + w] + eol)
    bam_io.write_fai(path)
    return path


def write_gzi(path, starts):
    """htslib's ``.gzi`` of a BGZF file whose blocks start at ``starts`` [(compressed, uncompressed offset)], the first
    (0, 0) included: the count, then one pair per block after the first."""
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(starts) - 1))
        for c, u in starts[1:]:
            f.write(struct.pack("<QQ", c, u))
    return path


def bgzip(src, dst, cuts=None, mode=None):
    """``src`` (a plain FASTA with its ``.fai``) as the BGZF file ``dst`` with ``dst.fai`` and ``dst.gzi``.  Without ``cuts``
    the blocks are ``bam_io.write_bgzf``'s; with them, the block boundaries are those uncompressed offsets (``bam_craft``)
    and each block is compressed by ``deflate_craft`` mode ``mode`` (zlib when None).  Returns the block starts."""
    data = open(src, "rb").read()
    if cuts is None:
        voff = bam_io.write_bgzf(dst, data)
        starts = [(voff(u) >> 16, u) for u in range(0, len(data), 0xFF00)]
    else:
        pts = bc.cut_points(len(data), cuts)
        with open(dst, "wb") as f:
            starts = []
            for i, (a, b) in enumerate(zip(pts[:-1], pts[1:])):
                starts.append((f.tell(), a))
                payload = data[a:b]
                f.write(bc.bgzf(payload, None if mode is None else dc.encode_mode(payload, mode, np.random.default_rng(i))))
            f.write(bam_io._EOF)
    shutil.copy(src + ".fai", dst + ".fai")
    write_gzi(dst + ".gzi", starts or [(0, 0)])
    return starts


def base_at_offset(fai_row, u):
    """The first base of the ``.fai`` row whose uncompressed byte offset is at or after ``u`` (its length when none is)."""
    _, length, off, lb, lw = fai_row
    i = np.arange(length, dtype=np.int64)
    return int(np.searchsorted(off + i // lb * lw + i % lb, u))


def windows(fai_row, block_starts, rng, n_random=12):
    """[(start, end)] of one sequence: random ones, and ones that start or end on a line end, on a block edge and at the
    sequence's end, plus empty and reversed ones."""
    name, length, off, lb, lw = fai_row
    out = [(0, length), (length, length), (5, 5), (7, 3), (length - 1, length + 10), (max(length - 61, 0), length)]
    for _ in range(n_random):
        a = int(rng.integers(0, length + 3))
        out.append((a, int(rng.integers(a, length + 8))))
    for k in range(1, min(length // max(lb, 1), 4) + 1):     # on line ends
        e = k * lb
        out += [(e - 1, e), (e, e + 1), (max(e - 70, 0), e), (e, min(e + 70, length)), (e - 1, e + 1)]
    for _, u in block_starts[1:]:                           # on block edges
        s = base_at_offset(fai_row, u)
        if 0 < s < length:
            out += [(s - 1, s), (s, s + 1), (max(s - 100, 0), s), (s, min(s + 100, length)), (s - 1, s + 1)]
    return out


def sequences(seed, n, lo, hi):
    rng = np.random.default_rng(seed)
    return [("s%d_%d" % (seed, i), random_sequence(int(rng.integers(lo, hi)), rng)) for i in range(n)]


# (name, FASTA writer arguments, sequences seed / count / length range, BGZF cuts: None = write_bgzf, else (step range, mode))
CASES = [
    ("w60", {"width": 60}, (1, 4, 1, 4000), (100, 900, None)),
    ("w61_crlf", {"width": 61, "eol": "\r\n"}, (2, 3, 500, 3000), (50, 700, None)),
    ("w80", {"width": 80}, (3, 4, 20000, 40000), None),
    ("one_line", {"width": None}, (4, 3, 200, 3000), (64, 500, None)),
    ("stored", {"width": 60}, (5, 2, 300, 1500), (80, 600, "stored")),
    ("fixed", {"width": 61, "eol": "\r\n"}, (6, 2, 300, 1500), (80, 600, "fixed")),
    ("dynamic", {"width": 80}, (7, 2, 300, 1500), (80, 600, "dynamic15")),
]


def make_case(d, case):
    """(plain path, BGZF path, block starts, [(name, bases)]) of one of ``CASES`` under directory ``d``."""
    name, fmt, (seed, n, lo, hi), blocks = case
    seqs = sequences(seed, n, lo, hi)
    plain = write_fasta(os.path.join(d, name + ".fa"), seqs, **fmt)
    cuts = None
    if blocks is not None:
        rng = np.random.default_rng(seed + 100)
        size, cuts, c = os.path.getsize(plain), [], 0
        while c < size:
            c += int(rng.integers(blocks[0], blocks[1]))
            cuts.append(c)
    starts = bgzip(plain, plain + ".gz", cuts, None if blocks is None else blocks[2])
    return plain, plain + ".gz", starts, seqs
