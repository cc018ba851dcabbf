"""A small DEFLATE (RFC 1951) encoder for tests: every block type, explicit or length-limited Huffman codes, and the stream
features that zlib's compressor never writes but other encoders do (libdeflate, which htslib usually links, among them):

- code-length runs (symbols 16 / 17 / 18) that cross from the literal/length lengths into the distance lengths (``joint=True``,
  as libdeflate codes the two arrays; zlib codes them apart);
- codes of 11 to 15 bits (explicit code lengths; or a length limit on codes built from the symbol counts);
- a distance code with exactly one used code, or with none;
- the fewest code-length codes and HLIT = 257;
- stored, fixed and dynamic blocks in one member, and empty stored blocks (sync-flush markers);
- length 258 coded as 285 or as 284 plus 31 extra bits; distance 32768; overlapping copies at distance 1 and 2.

A block is a dict: ``kind`` ("stored", "fixed", "dynamic"), ``syms`` (literal byte values and ``Match(length, dist, code)``
tuples; a stored block takes ``data`` bytes), and for dynamic blocks optional ``lit`` / ``dist`` code lengths, ``limit`` (the
length limit of the codes built from the symbol counts), ``joint`` and ``hclen``.  ``encode(blocks)`` returns the raw stream and
``replay(blocks)`` the bytes the symbols mean, computed without any decoder.  ``corpus()`` and ``malformed()`` are the streams the
inflater tests run.
"""
from __future__ import annotations

import heapq
import os
import shutil
import struct
import subprocess
import zlib
from collections import namedtuple

import numpy as np

Match = namedtuple("Match", "length dist code", defaults=(None,))      # code: force the length symbol (284 for 258)

ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
LEN_BASE = (3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258)
LEN_EXTRA = (0,) * 8 + tuple(i // 4 for i in range(4, 24)) + (0,)
DIST_BASE = (1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
             8193, 12289, 16385, 24577)
DIST_EXTRA = (0, 0, 0, 0) + tuple(i // 2 for i in range(2, 28))
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32

# the inflater's statuses (clair3_b200/csrc/inflate.cuh, c3b_inflate::Status)
STATUS = {"OK": 0, "BAD_BLOCK_TYPE": 1, "BAD_STORED_LENGTH": 2, "BAD_CODE_LENGTHS": 3, "BAD_CODE": 4, "BAD_DISTANCE": 5,
          "OUTPUT_OVERFLOW": 6, "INPUT_OVERRUN": 7}


class Bits:
    """LSB-first bit writer."""

    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, k):
        self.acc |= (v & ((1 << k) - 1)) << self.n
        self.n += k
        while self.n >= 8:
            self.out.append(self.acc & 0xFF)
            self.acc >>= 8
            self.n -= 8

    def code(self, c, k):               # Huffman codes go MSB first
        self.put(int("{:0{}b}".format(c, k)[::-1], 2) if k else 0, k)

    def align(self):
        if self.n:
            self.put(0, 8 - self.n)

    def bytes(self):
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


def canonical(lengths):
    """The canonical codes (RFC 1951 3.2.2) of a list of code lengths."""
    count = [0] * 16
    for x in lengths:
        count[x] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = []
    for x in lengths:
        out.append(nxt[x] if x else None)
        if x:
            nxt[x] += 1
    return out


def limited_lengths(freq, limit):
    """Optimal code lengths of at most ``limit`` bits for symbol counts ``freq`` (package-merge).  One used symbol gets length
    1; none gives all zeros."""
    used = [i for i, f in enumerate(freq) if f]
    lengths = [0] * len(freq)
    if len(used) == 1:
        lengths[used[0]] = 1
    if len(used) < 2:
        return lengths
    assert len(used) <= 1 << limit
    leaves = sorted((freq[i], (i,)) for i in used)
    cur = list(leaves)
    for _ in range(limit - 1):
        pk = [(cur[j][0] + cur[j + 1][0], cur[j][1] + cur[j + 1][1]) for j in range(0, len(cur) - 1, 2)]
        cur = list(heapq.merge(leaves, pk, key=lambda t: t[0]))
    for _, syms in cur[:2 * len(used) - 2]:
        for s in syms:
            lengths[s] += 1
    return lengths


def length_code(n, force=None):
    """(symbol, extra bits, extra value) of match length n; ``force`` = 284 codes 258 as 284 plus 31."""
    if force == 284:
        assert n == 258
        return 284, 5, 31
    if n == 258:
        return 285, 0, 0
    i = max(j for j in range(28) if LEN_BASE[j] <= n)
    return 257 + i, LEN_EXTRA[i], n - LEN_BASE[i]


def dist_code(d):
    i = max(j for j in range(30) if DIST_BASE[j] <= d)
    return i, DIST_EXTRA[i], d - DIST_BASE[i]


def _counts(syms):
    lit, dist = [0] * 286, [0] * 30
    for s in syms:
        if isinstance(s, Match):
            lit[length_code(s.length, s.code)[0]] += 1
            dist[dist_code(s.dist)[0]] += 1
        else:
            lit[s] += 1
    lit[256] += 1
    return lit, dist


def _rle(lengths):
    """Code-length symbols [(symbol, extra bits, extra value)] for a list of lengths, zlib-style runs."""
    out, i, n = [], 0, len(lengths)
    while i < n:
        v, j = lengths[i], i
        while j < n and lengths[j] == v:
            j += 1
        run = j - i
        if v == 0:
            while run >= 11:
                k = min(run, 138)
                out.append((18, 7, k - 11))
                run -= k
            if run >= 3:
                out.append((17, 3, run - 3))
                run = 0
            out += [(0, 0, 0)] * run
        else:
            out.append((v, 0, 0))
            run -= 1
            while run >= 3:
                k = min(run, 6)
                out.append((16, 2, k - 3))
                run -= k
            out += [(v, 0, 0)] * run
        i = j
    return out


def dynamic_header(lit, dist, joint=True, hclen=None, cl_lengths=None):
    """The bits of a dynamic block's header after BTYPE, and the runs' crossing flag: HLIT, HDIST, HCLEN, the code-length code
    and the run-length-coded lengths (``joint``: one run sequence over both arrays)."""
    nlit = max(257, max(i for i, x in enumerate(lit) if x) + 1)
    used_d = [i for i, x in enumerate(dist) if x]
    ndist = max(1, used_d[-1] + 1 if used_d else 1)
    L, D = list(lit[:nlit]), list(dist[:ndist])
    runs = _rle(L + D) if joint else _rle(L) + _rle(D)
    crossing, at = False, 0
    for s, _, v in runs:
        k = 3 + v if s == 16 else 3 + v if s == 17 else 11 + v if s == 18 else 1
        crossing |= at < nlit < at + k
        at += k
    assert at == nlit + ndist
    if cl_lengths is None:
        f = [0] * 19
        for s, _, _ in runs:
            f[s] += 1
        cl_lengths = limited_lengths(f, 7)
    ncl = max(4, max(ORDER.index(s) for s in range(19) if cl_lengths[s]) + 1)
    if hclen is not None:
        assert hclen >= ncl
        ncl = hclen
    b = Bits()
    b.put(nlit - 257, 5)
    b.put(ndist - 1, 5)
    b.put(ncl - 4, 4)
    for s in ORDER[:ncl]:
        b.put(cl_lengths[s], 3)
    codes = canonical(cl_lengths)
    ops = [("c", codes[s], cl_lengths[s], eb, ev) for s, eb, ev in runs]
    return b, ops, crossing, nlit, ndist


def _emit_ops(w, ops):
    for _, c, k, eb, ev in ops:
        w.code(c, k)
        w.put(ev, eb)


def _emit_syms(w, syms, lit, dist):
    lc, dc = canonical(lit), canonical(dist)
    for s in syms:
        if isinstance(s, Match):
            sym, eb, ev = length_code(s.length, s.code)
            w.code(lc[sym], lit[sym])
            w.put(ev, eb)
            ds, eb, ev = dist_code(s.dist)
            w.code(dc[ds], dist[ds])
            w.put(ev, eb)
        else:
            w.code(lc[s], lit[s])
    w.code(lc[256], lit[256])


def block_lengths(blk):
    """(literal/length lengths, distance lengths) a dynamic block codes with."""
    lit, dist = _counts(blk.get("syms", []))
    L = blk.get("lit") or limited_lengths(lit, blk.get("limit", 15))
    D = blk.get("dist")
    if D is None:
        D = limited_lengths(dist, blk.get("limit", 15))
    return list(L), list(D)


def encode(blocks):
    """The raw DEFLATE stream of ``blocks``; the last block is final unless a block says ``final``."""
    w = Bits()
    for i, blk in enumerate(blocks):
        final = blk.get("final", i == len(blocks) - 1)
        kind = blk["kind"]
        w.put(int(final), 1)
        if kind == "stored":
            w.put(0, 2)
            w.align()
            data = blk["data"]
            w.put(len(data), 16)
            w.put(~len(data) & 0xFFFF, 16)
            for x in data:
                w.put(x, 8)
        elif kind == "fixed":
            w.put(1, 2)
            _emit_syms(w, blk["syms"], FIXED_LIT, FIXED_DIST)
        else:
            w.put(2, 2)
            L, D = block_lengths(blk)
            hb, ops, _, _, _ = dynamic_header(L, D, blk.get("joint", True), blk.get("hclen"))
            _splice(w, hb)
            _emit_ops(w, ops)
            _emit_syms(w, blk["syms"], L, D)
    return w.bytes()


def _splice(w, b):
    for i in range(len(b.out) * 8 + b.n):
        byte = b.out[i >> 3] if i >> 3 < len(b.out) else b.acc
        w.put(byte >> (i & 7) & 1, 1)


def replay(blocks):
    """The bytes the blocks' symbols mean (copies byte by byte, so a distance below the length repeats what it wrote)."""
    out = bytearray()
    for blk in blocks:
        if blk["kind"] == "stored":
            out += blk["data"]
            continue
        for s in blk["syms"]:
            if isinstance(s, Match):
                assert 3 <= s.length <= 258 and 1 <= s.dist <= min(len(out), 32768)
                for _ in range(s.length):
                    out.append(out[-s.dist])
            else:
                out.append(s)
    return bytes(out)


def lz77(data, start=0, window=32768, max_chain=8):
    """Greedy LZ77 symbols of data[start:] with data[:start] as history of the same block (it must be emitted first)."""
    syms, heads, i, n = [], {}, start, len(data)
    for j in range(max(0, start - window), start):
        heads.setdefault(data[j:j + 3], []).append(j)
    while i < n:
        best, bd = 0, 0
        if i + 3 <= n:
            for j in reversed(heads.get(data[i:i + 3], [])[-max_chain:]):
                if i - j > window:
                    break
                k = 3
                while k < 258 and i + k < n and data[j + k] == data[i + k]:
                    k += 1
                if k > best:
                    best, bd = k, i - j
        step = best if best >= 3 else 1
        if best >= 3:
            syms.append(Match(best, bd))
        else:
            syms.append(data[i])
        for j in range(i, i + step):
            heads.setdefault(data[j:j + 3], []).append(j)
        i += step
    return syms


def check(blocks):
    """(stream, bytes): the stream, checked both ways - zlib inflates it to what the symbols replay to."""
    s = encode(blocks)
    want = replay(blocks)
    got = zlib.decompress(s, -15)
    assert got == want, "crafted stream does not inflate to its symbols"
    return s, want


# ---- the corpus ----

def corpus(seed=0):
    """[(name, blocks)]: valid streams, each with the features its name gives."""
    rng = np.random.default_rng(seed)
    out = []
    text = bytes(rng.integers(0, 4, 3000).astype(np.uint8) + 65) + b"ACGT" * 200
    syms = lz77(text)
    out.append(("fixed", [dict(kind="fixed", syms=syms)]))
    out.append(("dynamic joint runs", [dict(kind="dynamic", syms=syms, joint=True)]))
    out.append(("dynamic separate runs", [dict(kind="dynamic", syms=syms, joint=False)]))
    # a run of 5s across the literal/length -> distance boundary: lengths 280..285 and distance codes 0..5 all 5 bits
    lit = _complete([9] * 256 + [6] * 16 + [7] * 8 + [5] * 6)
    dist = [5] * 6 + [4] * 2 + [5] * 22
    run = [Match(3 + j, 1 + j) for j in range(6)]
    lit_syms = [int(x) for x in rng.integers(0, 256, 40)] + run + [Match(258, 6), Match(258, 5, 284)]
    out.append(("run crosses into distances", [dict(kind="dynamic", syms=lit_syms, lit=lit, dist=dist, joint=True)]))
    # long codes: one literal/length and one distance code of every length 1..15 (two of 15), each used many times
    lit = [0] * 286
    for k, sym in enumerate((65, 66, 67, 68, 69, 70, 71, 72, 73, 74, 257, 258, 259, 75, 256, 76)):
        lit[sym] = min(k + 1, 15)
    dist = [min(k + 1, 15) for k in range(16)]
    picks = rng.integers(0, 14, 3000)
    long_syms = [65 + i for i in range(12)] * 40
    for v in picks:
        long_syms.append(Match(3 + int(v) % 3, DIST_BASE[int(v)]) if v >= 10 else 65 + int(v) if v < 11 else 75)
    long_syms += [Match(3 + k % 3, DIST_BASE[k]) for k in range(16)] + [75, 76] * 5
    out.append(("codes of 11-15 bits", [dict(kind="dynamic", syms=long_syms, lit=_complete(lit), dist=dist)]))
    # a single distance code (length 1, an incomplete code zlib allows), and no distance code at all
    one = [66, 67, 68] + [Match(10 + j % 40, 3) for j in range(50)]
    out.append(("one distance code", [dict(kind="dynamic", syms=one)]))
    out.append(("no distance code", [dict(kind="dynamic", syms=[int(x) for x in rng.integers(0, 256, 500)])]))
    # HLIT = 257 (literals and end-of-block only) with the fewest code-length codes: lengths 6..9 only (HCLEN field 4)
    lit257 = [6] + [8] * 248 + [9] * 8
    out.append(("HLIT 257, 8 code-length codes", [dict(kind="dynamic", syms=[int(x) for x in rng.integers(0, 256, 300)],
                                                       lit=lit257, dist=[0], joint=True)]))
    # block types mixed in one member, with empty stored blocks (sync-flush markers) between them
    data = bytes(rng.integers(0, 256, 700).astype(np.uint8))
    mixed = [dict(kind="stored", data=data[:100]), dict(kind="stored", data=b""), dict(kind="fixed", syms=list(data[100:300])),
             dict(kind="dynamic", syms=list(data[300:500]) + [Match(50, 200), Match(258, 1)]), dict(kind="stored", data=b""),
             dict(kind="stored", data=data[500:]), dict(kind="fixed", syms=[Match(258, 7), Match(258, 7, 284)]),
             dict(kind="stored", data=b"")]
    out.append(("stored, fixed, dynamic and empty stored blocks", mixed))
    # length 258 both ways, distances 1 and 2 overlapping, distance 32768
    big = bytes(rng.integers(0, 256, 32768).astype(np.uint8))
    far = [dict(kind="stored", data=big[:30000]), dict(kind="stored", data=big[30000:]),
           dict(kind="dynamic", syms=[Match(258, 32768), Match(258, 32768, 284), Match(3, 32768), 7, Match(258, 1), 8, 9,
                                      Match(257, 2), Match(258, 2, 284), Match(4, 1)])]
    out.append(("length 258 as 285 and 284+31, distance 32768, distance 1 and 2", far))
    # a full 64 KiB block of each kind, and random mixes
    full = bytes(rng.integers(0, 3, 65536).astype(np.uint8) + 97)
    fsyms = lz77(full)
    out.append(("64 KiB dynamic", [dict(kind="dynamic", syms=fsyms, limit=15)]))
    out.append(("64 KiB fixed", [dict(kind="fixed", syms=fsyms)]))
    out.append(("64 KiB stored", [dict(kind="stored", data=full[:65535]), dict(kind="stored", data=full[65535:])]))
    for k in range(6):
        out.append(("random mix %d" % k, random_blocks(bytes(rng.integers(0, 6, int(rng.integers(1, 9000))).astype(np.uint8) + 65),
                                                      rng)))
    out.append(("empty", [dict(kind="stored", data=b"")]))
    out.append(("empty fixed", [dict(kind="fixed", syms=[])]))
    return out


def _complete(lit):
    """``lit`` padded with zeros to 286 entries after checking that its code is complete."""
    assert sum(2.0 ** -x for x in lit if x) == 1.0 and len(lit) <= 286, "incomplete or over-subscribed"
    return list(lit) + [0] * (286 - len(lit))


def random_blocks(data, rng, modes=("stored", "fixed", "dynamic", "dynamic15", "separate")):
    """``data`` as 1 to 4 blocks of random kinds; matches may reach into earlier blocks."""
    n = len(data)
    cuts = sorted(set([0, n] + [int(x) for x in rng.integers(0, n + 1, int(rng.integers(0, 4)))]))
    blocks = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        m = modes[int(rng.integers(0, len(modes)))]
        if m == "stored":
            for c in range(a, b, 65535):
                blocks.append(dict(kind="stored", data=data[c:min(b, c + 65535)]))
            continue
        syms = lz77(data[:b], start=a)
        if m == "fixed":
            blocks.append(dict(kind="fixed", syms=syms))
        else:
            blocks.append(dict(kind="dynamic", syms=syms, limit=15 if m == "dynamic15" else 12, joint=m != "separate"))
    if not blocks:
        blocks.append(dict(kind="stored", data=b""))
    return blocks


def encode_mode(data, mode, rng=None):
    """``data`` as one crafted stream of the named mode (the GPU tests compress each payload one way)."""
    rng = rng or np.random.default_rng(len(data))
    if mode == "stored":
        blocks = [dict(kind="stored", data=data[c:c + 65535]) for c in range(0, len(data), 65535)] or [dict(kind="stored", data=b"")]
    elif mode == "fixed":
        blocks = [dict(kind="fixed", syms=lz77(data))]
    elif mode == "dynamic15":
        blocks = [dict(kind="dynamic", syms=lz77(data), limit=15)]
    elif mode == "separate":
        blocks = [dict(kind="dynamic", syms=lz77(data), limit=15, joint=False)]
    elif mode == "flushed":                      # an empty stored block after every piece, as a sync flush writes
        blocks = []
        for c in range(0, max(len(data), 1), 4096):
            blocks += [dict(kind="dynamic", syms=lz77(data[:c + 4096], start=c)), dict(kind="stored", data=b"")]
    else:
        blocks = random_blocks(data, rng)
    return check(blocks)[0]


MODES = ("stored", "fixed", "dynamic15", "separate", "flushed", "mixed")


# ---- malformed streams: zlib rejects each; the inflater must return the named status ----

def _raw(*fields):
    b = Bits()
    for v, k in fields:
        b.put(v, k)
    return b


def malformed():
    """[(name, stream, output capacity, status name)]."""
    out = []
    ok_text = bytes(range(65, 91)) * 4
    good, _ = check([dict(kind="fixed", syms=list(ok_text))])
    # BTYPE 11
    out.append(("BTYPE 11", _raw((1, 1), (3, 2), (0, 16)).bytes(), 100, "BAD_BLOCK_TYPE"))
    # stored LEN / NLEN
    b = _raw((1, 1), (0, 2))
    b.align()
    b.put(5, 16)
    b.put(0x1234, 16)
    out.append(("stored NLEN mismatch", b.bytes() + b"hello", 100, "BAD_STORED_LENGTH"))
    # over-subscribed literal/length lengths: 257 symbols of 1 bit
    out.append(("over-subscribed lengths", _dyn_raw([1] * 257, [1]), 1000, "BAD_CODE_LENGTHS"))
    # an over-subscribed code-length code
    b = _raw((1, 1), (2, 2), (0, 5), (0, 5), (15, 4), *[(1, 3)] * 19)
    out.append(("over-subscribed code-length code", b.bytes() + bytes(8), 1000, "BAD_CODE_LENGTHS"))
    # a 16 (repeat the previous length) first
    out.append(("repeat code first", _dyn_custom([(16, 2, 0)]), 1000, "BAD_CODE_LENGTHS"))
    # a zero run past HLIT + HDIST
    out.append(("repeat past HLIT+HDIST", _dyn_custom([(8, 0, 0)] * 256 + [(18, 7, 127)]), 1000, "BAD_CODE_LENGTHS"))
    # no end-of-block code; and only the four code-length codes 16, 17, 18, 0 (every length then is 0)
    out.append(("no end-of-block code", _dyn_custom([(8, 0, 0)] * 256 + [(0, 0, 0), (1, 0, 0)]), 1000, "BAD_CODE_LENGTHS"))
    b = _raw((1, 1), (2, 2), (0, 5), (0, 5), (0, 4), (0, 3), (0, 3), (1, 3), (1, 3))
    out.append(("HCLEN 4", b.bytes() + bytes(40), 1000, "BAD_CODE_LENGTHS"))
    # HLIT 287 / HDIST 31
    out.append(("HLIT 287", _raw((1, 1), (2, 2), (30, 5), (0, 5), (15, 4), *[(3, 3)] * 19).bytes() + bytes(40), 1000,
                "BAD_CODE_LENGTHS"))
    out.append(("HDIST 31", _raw((1, 1), (2, 2), (0, 5), (30, 5), (15, 4), *[(3, 3)] * 19).bytes() + bytes(40), 1000,
                "BAD_CODE_LENGTHS"))
    # fixed-code symbols 286 / 287 and distance codes 30 / 31
    lc = canonical(FIXED_LIT)
    for sym in (286, 287):
        w = _raw((1, 1), (1, 2))
        w.code(lc[65], 8)
        w.code(lc[sym], 8)
        out.append(("fixed symbol %d" % sym, w.bytes() + bytes(4), 1000, "BAD_CODE"))
    dc = canonical(FIXED_DIST)
    for ds in (30, 31):
        w = _raw((1, 1), (1, 2))
        w.code(lc[65], 8)
        w.code(lc[257], 7)
        w.code(dc[ds], 5)
        out.append(("fixed distance code %d" % ds, w.bytes() + bytes(4), 1000, "BAD_CODE"))
    # a distance before the block's start
    s = encode([dict(kind="fixed", syms=[65, 66, Match(5, 3)])])
    out.append(("distance before the start", s, 1000, "BAD_DISTANCE"))
    # a match in a block whose distance code is empty
    lit = _complete([8] * 254 + [9] * 4)                 # 256: end-of-block, 257: length 3
    out.append(("match without distance codes", _dyn_syms(lit, [0], [65, 66, 67], [(257, None)]), 1000, "BAD_CODE"))
    # truncated: a stored block cut inside its data, and a fixed block cut in its symbols (the zeros read past the end decode
    # as end-of-block)
    st = encode([dict(kind="stored", data=ok_text)])
    out.append(("truncated stored block", st[:len(st) - 20], 1000, "INPUT_OVERRUN"))
    out.append(("truncated fixed block", good[:len(good) // 2], 1000, "INPUT_OVERRUN"))
    out.append(("truncated dynamic header", encode([dict(kind="dynamic", syms=list(ok_text))])[:6], 1000, "INPUT_OVERRUN"))
    out.append(("truncated stored header", encode([dict(kind="fixed", syms=[65], final=False), dict(kind="stored", data=b"AB")])[:4],
                1000, "INPUT_OVERRUN"))
    out.append(("empty input", b"", 1000, "INPUT_OVERRUN"))
    # output past the capacity (ISIZE): by literals, by a copy and by a stored block
    out.append(("literals past ISIZE", good, len(ok_text) - 1, "OUTPUT_OVERFLOW"))
    out.append(("copy past ISIZE", encode([dict(kind="fixed", syms=[65, Match(258, 1)])]), 200, "OUTPUT_OVERFLOW"))
    out.append(("stored past ISIZE", st, len(ok_text) - 1, "OUTPUT_OVERFLOW"))
    for name, s, cap, status in out:
        try:
            got = zlib.decompress(s, -15)
        except zlib.error:
            continue
        # zlib knows no output size: these streams are valid DEFLATE and malformed only against their BGZF block's ISIZE
        assert status == "OUTPUT_OVERFLOW" and len(got) > cap, "zlib accepts the malformed stream %r" % name
    return out


def _dyn_custom(runs, cl=None):
    """A final dynamic block of HLIT 286, HDIST 30 whose code-length symbols are ``runs`` (then zero padding)."""
    cl = cl or [4] * 13 + [5] * 6
    codes = canonical(cl)
    b = _raw((1, 1), (2, 2), (29, 5), (29, 5), (15, 4))
    for s in ORDER:
        b.put(cl[s], 3)
    for s, eb, ev in runs:
        b.code(codes[s], cl[s])
        b.put(ev, eb)
    return b.bytes() + bytes(64)


def _dyn_raw(lit, dist):
    """A final dynamic block with these lengths, coded without checks, then zeros."""
    b = Bits()
    b.put(1, 1)
    b.put(2, 2)
    hb, ops, _, _, _ = dynamic_header(lit + [0] * (286 - len(lit)), dist, True)
    _splice(b, hb)
    _emit_ops(b, ops)
    return b.bytes() + bytes(64)


def _dyn_syms(lit, dist, literals, lens):
    """A final dynamic block with these lengths that codes ``literals`` and then length symbols without distances."""
    b = Bits()
    b.put(1, 1)
    b.put(2, 2)
    hb, ops, _, _, _ = dynamic_header(lit, dist, True)
    _splice(b, hb)
    _emit_ops(b, ops)
    lc = canonical(lit)
    for x in literals:
        b.code(lc[x], lit[x])
    for sym, _ in lens:
        b.code(lc[sym], lit[sym])
    return b.bytes() + bytes(8)


# ---- the host build of inflate.cuh (tests/inflate_host.cpp), with AddressSanitizer and UBSan ----

_TESTS = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(_TESTS), "clair3_b200", "csrc")
_SAN_ENV = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")


def build_host_inflater(out_dir):
    """Compiles tests/inflate_host.cpp into ``out_dir``; its path, or None without g++."""
    cxx = shutil.which("g++")
    if cxx is None:
        return None
    exe = os.path.join(out_dir, "inflate_host")
    r = subprocess.run([cxx, "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-fno-omit-frame-pointer", "-I", _CSRC, os.path.join(_TESTS, "inflate_host.cpp"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def run_host(exe, mode, payload):
    """The driver's stdout; fails on a non-zero exit or any sanitizer report.  ``mode``: its arguments, split on spaces."""
    r = subprocess.run([exe] + mode.split(), input=payload, capture_output=True, env=_SAN_ENV, timeout=600)
    err = r.stderr.decode(errors="replace")
    assert r.returncode == 0 and "Sanitizer" not in err and "runtime error" not in err, err[-4000:]
    return r.stdout


def run_host_inflater(exe, cases):
    """[(status, output bytes)] of the host inflater for [(stream, capacity)]."""
    out = run_host(exe, "inflate", b"".join(struct.pack("<II", len(s), cap) + s for s, cap in cases))
    res, o = [], 0
    for _ in cases:
        st, n = struct.unpack_from("<ii", out, o)
        o += 8
        res.append((st, out[o:o + max(n, 0)]))
        o += max(n, 0)
    assert o == len(out)
    return res
