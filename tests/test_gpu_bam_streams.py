"""The GPU BAM reader on the streams and records real BAM writers produce, against ``bam_io.read_bam`` (which inflates through zlib):

- BGZF blocks compressed by ``deflate_craft`` in every mode (stored, fixed, 15-bit-limited dynamic codes, code-length runs coded
  apart, sync-flushed, mixed block types), with payload sizes at every residue mod 32; malformed blocks reported by number and
  reason, each sent to the GPU only after the sanitized host build of the same inflater has run it;
- record-start speculation forced down its hard paths by fake record headers planted in ``B,C`` arrays, qualities and header
  text, with the BGZF cuts placed so that a fake is the first plausible offset of its block;
- records whose CIGAR is in a ``CG`` tag: the decoder against ``read_bam``, and one ~300 kb read of more than 65,535 operations
  through the pileup counter and the full-alignment builder against the same records with the CIGAR inline."""
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bam_craft as bc  # noqa: E402
import deflate_craft as dc  # noqa: E402
from clair3_b200 import bam_io  # noqa: E402
from clair3_b200 import synth_reads as sr  # noqa: E402
from clair3_b200._ffi import C3BError  # noqa: E402
from clair3_b200.bam_decode import BamDecoder  # noqa: E402
from clair3_b200.fa_tensor import FullAlignmentBuilder  # noqa: E402
from clair3_b200.pileup_counts import PileupCounter  # noqa: E402
from test_bam_cg_cpu import CONVERTED, UNCONVERTED, ultra_long_case  # noqa: E402

pytestmark = pytest.mark.gpu

# bam_decode.cu's status_name
REASON = {"BAD_BLOCK_TYPE": "bad DEFLATE block type", "BAD_STORED_LENGTH": "stored block length does not match its complement",
          "BAD_CODE_LENGTHS": "malformed Huffman code lengths", "BAD_CODE": "invalid Huffman code",
          "BAD_DISTANCE": "back-reference distance reaches before the block's start", "OUTPUT_OVERFLOW": "inflates past its ISIZE",
          "INPUT_OVERRUN": "DEFLATE stream runs past the block's compressed data"}


@pytest.fixture(scope="module")
def dec():
    d = BamDecoder(0)
    yield d
    d.close()


def _same(got, path, ctg, start, end, fa_fields):
    want, _ = bam_io.read_bam(path, ctg, start, end, fa_fields=fa_fields)
    h = got.host()
    keys = [k for k in want if k != "tid"]
    assert sorted(keys) == sorted(h)
    for k in keys:
        assert h[k].dtype == want[k].dtype and np.array_equal(h[k], want[k]), (k, start, end, fa_fields)
    return len(want["pos"])


def _all_blocks(path):
    refs, vo = bam_io.read_bam_header(path)
    return open(path, "rb").read()[vo >> 16:], vo & 0xFFFF


def _check(dec, path, regions, index=True):
    n = 0
    data, u0 = _all_blocks(path)
    if index:
        bam_io.write_bai(path)
    for start, end in regions:
        for fa in (False, True):
            n += _same(dec.decode_bytes(data, u0, -1, 0, start, end, fa_fields=fa), path, "ctg", start, end, fa)
            if index:
                _same(dec.decode(path, "ctg", start, end, fa_fields=fa), path, "ctg", start, end, fa)
    return n


def _stream(path):
    raw = open(path, "rb").read()
    return b"".join(bam_io._inflate_block(raw, o)[1] for o, _, _ in bam_io.bgzf_blocks(raw))


# ---- A: crafted DEFLATE streams ----

def test_crafted_blocks_of_every_mode(tmp_path, dec):
    rec, _, _, _ = sr.random_fa_case(12, dwell=True, read_len=700, depth=12)
    src = str(tmp_path / "src.bam")
    bam_io.write_bam(src, rec, [("ctg", 10000)])
    s = _stream(src)
    rng = np.random.default_rng(4)
    sizes = [32 * int(rng.integers(1, 200)) + r for r in rng.permutation(32)]     # every residue mod 32
    cuts = [0]
    for z in sizes:
        if cuts[-1] + z >= len(s):
            break
        cuts.append(cuts[-1] + z)
    assert len(cuts) > 32
    cuts = bc.cut_points(len(s), cuts[1:], step=40000)
    dst = bc.write_blocks(str(tmp_path / "crafted.bam"), s, cuts,
                          lambda p, i: dc.encode_mode(p, dc.MODES[i % len(dc.MODES)], np.random.default_rng(i)))
    assert sorted({(b - a) % 32 for a, b in zip(cuts[:-1], cuts[1:])}) == list(range(32))
    assert _check(dec, dst, [(None, None), (1200, 2500), (4000, 4001)]) > 0


def test_malformed_blocks_are_reported_by_number_and_reason(tmp_path, dec):
    exe = dc.build_host_inflater(str(tmp_path))
    if exe is None:
        pytest.skip("needs g++ for the sanitized host run that must precede the GPU run")
    cases = dc.malformed()
    host = dc.run_host_inflater(exe, [(s, cap) for _, s, cap, _ in cases])
    for (name, _, _, status), (st, _) in zip(cases, host):
        assert st == dc.STATUS[status], (name, st, status)          # the host build ran it first, without a sanitizer report
    rec, _, _ = sr.random_alignment(3000, depth=10, read_len=400, seed=8)
    path = str(tmp_path / "m.bam")
    bam_io.write_bam(path, rec, [("ctg", 10000)])
    data, u0 = _all_blocks(path)
    blocks = bam_io.bgzf_blocks(data)
    assert len(blocks) >= 3
    for k, (name, s, cap, status) in enumerate(cases):
        j = 1 + k % (len(blocks) - 1)
        o, size, _ = blocks[j]
        bad = data[:o] + bc.bgzf(b"\0" * cap, s) + data[o + size:]
        with pytest.raises(C3BError, match="BGZF block %d \\(at byte %d of the data\\): %s" % (j, o, REASON[status])):
            dec.decode_bytes(bad, u0, -1, 0)
    _same(dec.decode_bytes(data, u0, -1, 0), path, "ctg", None, None, False)      # the workspace stays usable


# ---- B: adversarial record starts ----

def fields_bytes(U, o):
    """bam_decode.cu's fields_bytes, restated."""
    l_name = U[o + 12]
    n_cig, = struct.unpack_from("<H", U, o + 16)
    l_seq, = struct.unpack_from("<i", U, o + 20)
    if l_name < 1 or l_seq < 0:
        return -1
    return 32 + l_name + 4 * n_cig + (l_seq + 1) // 2 + l_seq


def looks_like_record(U, o, end_u):
    """bam_decode.cu's looks_like_record, restated: the test plants fakes that pass it."""
    if o + 36 > end_u:
        return False
    bs, = struct.unpack_from("<i", U, o)
    need = fields_bytes(U, o)
    if need < 0 or bs < need or o + 4 + bs > end_u:
        return False
    if min(struct.unpack_from("<iiii", U, o + 4)[:2] + struct.unpack_from("<ii", U, o + 24)) < -1:
        return False
    l_name = U[o + 12]
    if U[o + 36 + l_name - 1] != 0:
        return False
    return all(0x21 <= c <= 0x7E and c != ord("@") for c in U[o + 36:o + 36 + l_name - 1])


def first_hit(U, lo, hi, end_u):
    return next((o for o in range(lo, hi) if looks_like_record(U, o, end_u)), None)


def fake(bs):
    """A fake record header that passes looks_like_record when bs >= 34 and the bytes it claims exist: refID 0, a 2-byte name."""
    return struct.pack("<i", bs) + bam_io._CORE.pack(0, 1234, 2, 60, 4680, 0, 0, 0, -1, -1, 0) + b"f\0"


class Layout:
    """Records with fixed-size B,C arrays (and qualities) whose bytes are filled after the offsets are known."""

    def __init__(self, n, arr=200, seed=0, long_at=None, long_len=150000, text=b"@HD\tVN:1.6\tSO:coordinate\n"):
        rng = np.random.default_rng(seed)
        self.text_fake = len(b"BAM\x01") + 4 + len(text)                         # where a fake in the header text goes
        text = text + b"@CO\t" + bytes(60) + b"\n"
        self.head = bytearray(bc.header([("ctg", 1 << 20)], text))
        self.text_fake += 4
        self.recs, self.start, self.arr, self.qual = [], [], [], []
        off = len(self.head)
        for i in range(n):
            l_seq = long_len if i == long_at else int(rng.integers(50, 120))
            qual = rng.integers(0, 60, l_seq).astype(np.uint8).tobytes()
            aux = b"XBBC" + struct.pack("<i", arr) + bytes(arr)
            r = bytearray(bc.record(100 + 37 * i, [l_seq << 4], l_seq, aux, name=b"q%d" % i, qual=qual,
                                    seq=rng.integers(0, 256, (l_seq + 1) // 2).astype(np.uint8).tobytes()))
            self.start.append(off)
            self.arr.append(off + len(r) - arr)
            self.qual.append(off + len(r) - arr - 8 - l_seq)
            self.recs.append(r)
            off += len(r)
        self.end = off
        self.buf = None

    def stream(self):
        if self.buf is None:
            self.buf = bytearray(self.head + b"".join(self.recs))
        return self.buf

    def put(self, at, b):
        s = self.stream()
        assert self.start[0] <= at or at + len(b) <= len(self.head)
        s[at:at + len(b)] = b


def test_record_start_speculation_cannot_be_fooled(tmp_path, dec):
    L = Layout(60, long_at=40)
    S, cuts, planted = L.stream(), [], []
    # (a) a fake in record 5's B,C array chains to record 7's start: the true chain enters at record 6 and meets it there
    a = L.arr[5] + 8
    L.put(a, fake(L.start[7] - a - 4))
    planted.append(("a", a))
    cuts.append(a - 3)
    # the same in record 16's qualities, chaining to record 18
    q = L.qual[16] + 5
    L.put(q, fake(L.start[18] - q - 4))
    planted.append(("a, in qualities", q))
    cuts.append(q - 3)
    # (b) a fake in record 12's array whose chain leaves the block one byte after the true chain does
    b = L.arr[12] + 8
    cuts += [b - 3, L.start[14] + 10]
    L.put(b, fake(L.start[15] + 1 - b - 4))
    planted.append(("b", b))
    # (c) a fake chain in record 22's array that marks twice and then breaks on a block_size below 32
    c = L.arr[22] + 8
    L.put(c, fake(60))
    L.put(c + 64, struct.pack("<i", 40))
    L.put(c + 108, struct.pack("<i", 5))
    planted.append(("c", c))
    cuts.append(c - 3)
    # (d) a block wholly inside record 40 (150 kb of sequence and qualities) that starts at a fake
    d = L.qual[40] + 70000
    L.put(d, fake(5000))
    L.put(d + 5004, fake(9000))
    planted.append(("d", d))
    cuts += [d - 3, d + 20000]
    # (e) a fake in the header text, before the first record: the first block starts just before it
    e = L.text_fake
    L.put(e, fake(40))
    cuts.append(e - 3)
    S = bytes(L.stream())
    pts = bc.cut_points(len(S), cuts, step=30000)
    path = bc.write_blocks(str(tmp_path / "fakes.bam"), S, pts)
    assert bam_io.read_bam(path, "ctg")[0]["pos"].size == 60
    # every fake is the first offset its block's speculation would take (block ranges as bam_speculate_kernel clips them)
    data, u0 = _all_blocks(path)
    base = pts[[i for i, p in enumerate(pts) if p <= e][-1]]                      # uncompressed offset of the data's first byte
    U, first = S[base:], L.start[0] - base
    assert first == u0
    for name, o in planted:
        blk = max(p for p in pts if p <= o)
        hi = min(p for p in pts if p > o)
        lo = max(blk, L.start[0])
        assert first_hit(S, lo, hi, len(S)) == o, name
    assert first_hit(S, e - 3, L.start[0], len(S)) == e and e < L.start[0]      # (e): before first_uoff
    blk_d = max(p for p in pts if p <= d)
    assert L.start[40] < blk_d and min(p for p in pts if p > d) < L.start[41]   # (d): no record starts in the block
    assert _check(dec, path, [(None, None), (100 + 37 * 6, 100 + 37 * 30), (100 + 37 * 39, 100 + 37 * 41), (4000, 4100)]) > 0


# ---- C: CIGARs in CG tags ----

def test_cg_records_decode_as_read_bam_reads_them(tmp_path, dec):
    recs, n = [], 0
    for j, (_, cig, aux) in enumerate(CONVERTED + UNCONVERTED):
        for rep in range(3):
            recs.append(bc.record(100 + 10 * n, cig, 20, aux, name=b"v%d_%d" % (j, rep), qual=bytes(range(20)), seq=bytes(range(10))))
            n += 1
    S = bc.header([("ctg", 100000)]) + b"".join(recs)
    path = bc.write_blocks(str(tmp_path / "cg.bam"), S, bc.cut_points(len(S), [len(S) // 3, len(S) // 2]))
    want, _ = bam_io.read_bam(path, "ctg")
    assert (np.diff(want["cigar_off"]) == 5).sum() == 3 * len(CONVERTED)
    assert _check(dec, path, [(None, None), (150, 400), (300, 301)]) > 0


def _subset(rec, idx):
    out = {f: rec[f][idx] for f in ("pos", "flag", "mapq", "l_qseq")}
    for off, v in (("cigar_off", "cigar"), ("seq_off", "seq"), ("qual_off", "qual"), ("qname_off", "qname"), ("mv_off", "mv")):
        parts = [rec[v][rec[off][i]:rec[off][i + 1]] for i in idx]
        out[v] = np.concatenate(parts).astype(rec[v].dtype)
        out[off] = np.concatenate([[0], np.cumsum([len(x) for x in parts])]).astype(np.int64)
    return out


def test_ultra_long_read_counts_as_its_inline_cigar(tmp_path, dec):
    rec, ref, rs, k = ultra_long_case()
    n_ops = int(rec["cigar_off"][k + 1] - rec["cigar_off"][k])
    assert n_ops > 65535 and rec["l_qseq"][k] > 250000
    path = str(tmp_path / "ul.bam")
    bam_io.write_bam(path, rec, [("ctg", 400000)])
    bam_io.write_bai(path)
    start, end = 20000, 50000
    # the records of the region with their CIGARs inline, straight from the arrays that were written
    cig = [rec["cigar"][rec["cigar_off"][i]:rec["cigar_off"][i + 1]] for i in range(len(rec["pos"]))]
    span = np.array([int((c >> 4)[np.isin(c & 15, (0, 2, 3, 7, 8))].sum()) for c in cig])
    idx = np.nonzero((rec["pos"] < end) & (rec["pos"] + np.maximum(span, 1) > start))[0]
    assert k in idx
    inline = _subset(rec, idx)
    dev = dec.decode(path, "ctg", start, end, fa_fields=True, ref_seq=ref)
    h = dev.host()
    for f in h:
        assert np.array_equal(h[f], inline[f]), f
    ctr = PileupCounter(0)
    a = ctr.count(inline, start, end, ref, rs, alt_info=True)
    ma, ta = a.fetch(), a.alt_text().alt_text_fetch()["text"]
    b = ctr.count(dev, start, end, None, rs, alt_info=True)
    mb, tb = b.fetch(), b.alt_text().alt_text_fetch()["text"]
    for f in ma:
        assert np.array_equal(ma[f], mb[f]), f
    assert ta == tb and len(ta) > 0
    ctr.close()
    assert rs == 0
    cand = np.arange(start + 101, end - 100, 293, dtype=np.int64)
    bld = FullAlignmentBuilder(0)
    x = bld.build(inline, cand, ref, rs)
    mx, ax = x.fetch(), bld.alt_info_strings()
    y = bld.build(dev, cand, None, rs)
    my, ay = y.fetch(), bld.alt_info_strings()
    assert mx.shape[0] == len(cand) and np.array_equal(mx, my) and ax == ay and np.count_nonzero(mx) > 0
    bld.close()
