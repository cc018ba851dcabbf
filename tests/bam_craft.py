"""Hand-made BAM streams for tests: records with any auxiliary bytes, CIGAR and header, BGZF blocks cut where a test wants them
and compressed by a chosen ``deflate_craft`` mode (or zlib)."""
from __future__ import annotations

import struct
import zlib

import numpy as np

from clair3_b200 import bam_io

_NT = np.array([1, 2, 4, 8], np.uint8)             # A C G T as BAM's 4-bit codes


def record(pos, cigar, l_seq, aux=b"", tid=0, name=b"r", seq=None, qual=None, flag=0, mapq=60):
    """One record, block_size first.  ``cigar``: uint32 words; ``seq``: packed bytes ((l_seq + 1) // 2); ``qual``: l_seq bytes."""
    cig = np.asarray(cigar, dtype="<u4")
    seq = bytes((l_seq + 1) // 2) if seq is None else bytes(seq)
    qual = b"\xff" * l_seq if qual is None else bytes(qual)
    nm = name + b"\0"
    body = bam_io._CORE.pack(tid, pos, len(nm), mapq, 4680, len(cig), flag, l_seq, -1, -1, 0) + nm + cig.tobytes() + seq + qual + aux
    return struct.pack("<i", len(body)) + body


def header(refs, text=b"@HD\tVN:1.6\tSO:coordinate\n"):
    out = bytearray(b"BAM\x01" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs)))
    for name, length in refs:
        nb = name.encode() + b"\0"
        out += struct.pack("<i", len(nb)) + nb + struct.pack("<i", length)
    return bytes(out)


def bgzf(payload, stream=None):
    """One BGZF block of ``payload``; ``stream``: its raw DEFLATE data (default zlib level 6)."""
    if stream is None:
        c = zlib.compressobj(6, zlib.DEFLATED, -15)
        stream = c.compress(payload) + c.flush()
    head = struct.pack("<BBBBIBBHBBHH", 0x1F, 0x8B, 8, 4, 0, 0, 0xFF, 6, 0x42, 0x43, 2, len(stream) + 25)
    return head + stream + struct.pack("<II", zlib.crc32(payload) & 0xFFFFFFFF, len(payload))


def cut_points(n, cuts, step=0xFF00):
    """Block boundaries of an n-byte stream: the given cut offsets, and more every ``step`` bytes between them."""
    pts, prev = [0], 0
    for c in sorted(set(c for c in cuts if 0 < c < n)) + [n]:
        while c - prev > step:
            prev += step
            pts.append(prev)
        pts.append(c)
        prev = c
    return pts


def write_blocks(path, stream, cuts, encode=None):
    """Writes ``stream`` as BGZF blocks between consecutive ``cuts`` (offsets, 0 and len included) and the EOF block;
    ``encode(payload, i)`` gives block i's raw DEFLATE data (default zlib)."""
    with open(path, "wb") as f:
        for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
            f.write(bgzf(stream[a:b], None if encode is None else encode(stream[a:b], i)))
        f.write(bam_io._EOF)
    return path


def pack_seq(codes):
    codes = np.asarray(codes, np.uint8)
    if len(codes) % 2:
        codes = np.concatenate([codes, [0]]).astype(np.uint8)
    return (codes[0::2] << 4 | codes[1::2]).astype(np.uint8).tobytes()


def long_read(ref, ref_start, pos, n_cycles, rng, sub_rate=0.03):
    """An alignment at ``pos`` of ``n_cycles`` x (kM 1I kM 1D), k in 4..12 - four CIGAR operations per cycle - with substitutions:
    (CIGAR words, 4-bit base codes)."""
    ops, bases, r = [], [], pos - ref_start
    refc = np.frombuffer(ref.upper().encode(), np.uint8)
    lut = np.zeros(256, np.uint8)
    for ch, v in zip(b"ACGT", _NT):
        lut[ch] = v
    lut[ord("N")] = 15
    for _ in range(n_cycles):
        for kind in (0, 1, 0, 2):
            if kind == 0:
                k = int(rng.integers(4, 13))
                b = lut[refc[r:r + k]].copy()
                sub = rng.random(k) < sub_rate
                b[sub] = _NT[rng.integers(0, 4, int(sub.sum()))]
                bases.append(b)
                ops.append(k << 4)
                r += k
            elif kind == 1:
                bases.append(_NT[rng.integers(0, 4, 1)])
                ops.append(1 << 4 | 1)
            else:
                ops.append(1 << 4 | 2)
                r += 1
    return np.array(ops, np.uint32), np.concatenate(bases)
