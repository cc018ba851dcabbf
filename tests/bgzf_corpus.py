"""Payloads for the BGZF writer's tests: the cases that reach each rule of zlib's level-6 compressor that ``deflate.cuh``
restates, real VCF text, and seeded mixtures.  ``payloads()`` is [(name, bytes)], every payload at most one BGZF block's
0xFF00 bytes; ``texts()`` are whole-file texts that span many blocks."""
import os
import shutil
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from clair3_b200 import bam_io  # noqa: E402

PAYLOAD = bam_io._BGZF_PAYLOAD
MIN_LOOKAHEAD = 258 + 3 + 1
SLIDE_AT = 32768 + 32768 - MIN_LOOKAHEAD        # fill_window slides once strstart reaches w_size + MAX_DIST
ZLIB_VERSION = "1.3"                            # the zlib these payloads were made byte-identical against


def build_host_deflater(out_dir):
    """Compiles tests/deflate_host.cpp with AddressSanitizer and UBSan into ``out_dir``; its path, or None without g++."""
    cxx = shutil.which("g++")
    if cxx is None:
        return None
    exe = os.path.join(out_dir, "deflate_host")
    r = subprocess.run([cxx, "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-fno-omit-frame-pointer", "-I", os.path.join(os.path.dirname(HERE), "clair3_b200", "csrc"),
                        os.path.join(HERE, "deflate_host.cpp"), "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def vcf_text(n_rows, seed, contigs=("chr1", "chr2", "chrX")):
    """VCF text shaped like the genome route's files: a header, then rows with Clair3's INFO / FORMAT fields."""
    rng = np.random.default_rng(seed)
    head = ["##fileformat=VCFv4.2", "##source=Clair3", '##INFO=<ID=P,Number=0,Type=Flag,Description="pileup">',
            '##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">']
    head += ["##contig=<ID=%s,length=%d>" % (c, 1000000 + 7919 * i) for i, c in enumerate(contigs)]
    head.append("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE")
    rows, pos = [], 0
    bases = np.array(list("ACGT"))
    for i in range(n_rows):
        c = contigs[min(i * len(contigs) // max(n_rows, 1), len(contigs) - 1)]
        pos += int(rng.integers(1, 400))
        ref = "".join(rng.choice(bases, int(rng.choice([1, 1, 1, 2, 5]))))
        alt = "".join(rng.choice(bases, int(rng.choice([1, 1, 1, 3]))))
        gt = rng.choice(["0/1", "1/1", "0/0", "1/2"])
        q = rng.random() * 40
        dp = int(rng.integers(2, 90))
        af = rng.random()
        rows.append("%s\t%d\t.\t%s\t%s\t%.2f\t%s\tP\tGT:GQ:DP:AF\t%s:%d:%d:%.4f" % (
            c, pos, ref, alt, q, "PASS" if q > 8 else "LowQual", gt, int(q), dp, af))
    return "\n".join(head + rows) + "\n"


def _fib_text(rng, n):
    """Bytes whose literal counts follow the Fibonacci numbers, shuffled, then random bytes: skewed symbol counts, which in
    the mixtures make the literal / length code want lengths past 15 bits, so gen_bitlen's overflow repair runs."""
    counts, a, b = [], 1, 1
    while sum(counts) + a <= n and len(counts) < 40:
        counts.append(a)
        a, b = b, a + b
    syms = np.concatenate([np.full(c, s, np.uint8) for s, c in enumerate(counts)])
    rng.shuffle(syms)
    pad = rng.integers(64, 256, n - len(syms)).astype(np.uint8)
    return bytes(np.concatenate([syms, pad]))


def payloads(seed=0, mixtures=0):
    rng = np.random.default_rng(seed)
    rnd = lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes()  # noqa: E731
    text = vcf_text(3000, seed).encode()
    out = [("empty", b""), ("1 byte", b"A"), ("2 bytes", b"AC"), ("3 bytes", b"ACG"), ("3 equal bytes", b"AAA"),
           ("4 equal bytes", b"AAAA"),
           ("text, 0xFF00 bytes", text[:PAYLOAD]), ("text, 0xFF00 - 1 bytes", text[:PAYLOAD - 1]),
           ("random, 0xFF00 bytes", rnd(PAYLOAD)), ("random, 0xFF00 - 1 bytes", rnd(PAYLOAD - 1)), ("random, 1000", rnd(1000)),
           ("one byte, 0xFF00", b"A" * PAYLOAD), ("one byte, 259", b"T" * 259), ("two bytes alternating", b"AC" * (PAYLOAD // 2))]
    for end in (MIN_LOOKAHEAD - 1, MIN_LOOKAHEAD, MIN_LOOKAHEAD + 1):
        for n in (PAYLOAD, 9000):
            out.append(("run ending %d bytes before the end of %d" % (end, n), rnd(n - end - 3000) + b"G" * 3000 + rnd(end)))
    for at in (SLIDE_AT - 2, SLIDE_AT - 1, SLIDE_AT, SLIDE_AT + 1, SLIDE_AT + 3):
        out.append(("run ending at %d" % at, rnd(at - 5000) + b"C" * 5000 + text[:PAYLOAD - at]))
        out.append(("text then random, switch at %d" % at, text[:at] + rnd(PAYLOAD - at)))
    for k in range(4):
        n = [PAYLOAD, 40000, 20000, 8000][k]
        out.append(("Fibonacci literal counts, %d bytes" % n, _fib_text(rng, n)))
    out.append(("symbol buffer flushes several times", bytes(rng.integers(0, 16, PAYLOAD, dtype=np.uint8) + 65)))
    out.append(("short matches, far apart", b"".join(rnd(5000) + b"xyz" for _ in range(12))[:PAYLOAD]))
    out.append(("VCF rows", text[PAYLOAD:2 * PAYLOAD]))
    for i in range(mixtures):
        out.append(("mixture %d" % i, mixture(rng, text)))
    return out


def mixture(rng, text):
    """A seeded payload of up to 0xFF00 bytes made of pieces of the cases above."""
    n = int(rng.choice([rng.integers(0, 64), rng.integers(0, PAYLOAD + 1), PAYLOAD, PAYLOAD - 1]))
    parts, have = [], 0
    while have < n:
        k = int(rng.integers(1, 9000))
        kind = int(rng.integers(0, 5))
        if kind == 0:
            p = rng.integers(0, 256, k, dtype=np.uint8).tobytes()
        elif kind == 1:
            p = bytes([int(rng.integers(0, 256))]) * k
        elif kind == 2:
            o = int(rng.integers(0, len(text) - k))
            p = text[o:o + k]
        elif kind == 3:
            p = bytes(rng.integers(0, int(rng.integers(1, 8)), k, dtype=np.uint8) + 97)
        else:
            p = _fib_text(rng, k)
        parts.append(p)
        have += len(p)
    return b"".join(parts)[:n]


def texts(seed=0):
    """Whole-file texts: [(name, bytes)]."""
    rng = np.random.default_rng(seed)
    return [("empty", b""), ("one row", b"chr1\t5\t.\tA\tC\t3.1\tPASS\tP\tGT\t0/1\n"),
            ("VCF, 40 blocks", vcf_text(40000, seed + 1).encode()),
            ("VCF, exactly 3 blocks", vcf_text(3000, seed + 2).encode()[:3 * PAYLOAD]),
            ("random, 5 blocks and a bit", rng.integers(0, 256, 5 * PAYLOAD + 17, dtype=np.uint8).tobytes())]
