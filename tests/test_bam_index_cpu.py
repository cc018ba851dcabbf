"""The host half of the GPU BAM reader: BGZF header checks, header reading and the .bai index (clair3_b200/bam_io.py).

``write_bai`` -> ``read_bai`` -> ``bai_range`` must give a byte range whose records, filtered as ``read_bam`` filters them, are
exactly ``read_bam``'s: the GPU reader decodes that range and applies the same filter on the device."""
import struct
import zlib

import numpy as np
import pytest

from clair3_b200 import bam_io
from clair3_b200 import synth_reads as sr


def _host_filter(buf, first, end_u, tid, start, end):
    """read_bam's filter over the records chained from ``first`` to ``end_u`` of an uncompressed range: (pos list, names)."""
    lo = -1 if start is None else start
    hi = 1 << 62 if end is None else end
    off, out = first, []
    while off < end_u:
        bs, = struct.unpack_from("<i", buf, off)
        t, p, l_name, _, _, n_cig = struct.unpack_from("<iiBBHH", buf, off + 4)
        rec0, off = off + 4, off + 4 + bs
        if t < 0 or t != tid:
            if t > tid:
                break
            continue
        if p >= hi:
            break
        cig = np.frombuffer(buf, dtype="<u4", count=n_cig, offset=rec0 + 32 + l_name)
        span = int((cig >> 4)[np.isin(cig & 15, (0, 2, 3, 7, 8))].sum()) if n_cig else 0
        if p + max(span, 1) <= lo:
            continue
        out.append((p, bytes(buf[rec0 + 32:rec0 + 32 + l_name - 1])))
    return out


def _inflate_range(raw, c0, c1):
    sub = raw[c0:c1]
    return b"".join(bam_io._inflate_block(sub, o)[1] for o, _, _ in bam_io.bgzf_blocks(sub))


def _two_contig_bam(tmp_path, seed=3, read_len=2000):
    rec0, _, _ = sr.random_alignment(20000, depth=6, read_len=read_len, seed=seed)
    rec1, _, _ = sr.random_alignment(9000, depth=4, read_len=read_len, seed=seed + 1)
    n0, n1 = len(rec0["pos"]), len(rec1["pos"])
    rec = {"pos": np.concatenate([rec0["pos"], rec1["pos"]]), "flag": np.concatenate([rec0["flag"], rec1["flag"]]),
           "mapq": np.concatenate([rec0["mapq"], rec1["mapq"]]), "l_qseq": np.concatenate([rec0["l_qseq"], rec1["l_qseq"]]),
           "cigar": np.concatenate([rec0["cigar"], rec1["cigar"]]),
           "cigar_off": np.concatenate([rec0["cigar_off"], rec1["cigar_off"][1:] + rec0["cigar_off"][-1]]),
           "seq": np.concatenate([rec0["seq"], rec1["seq"]]),
           "seq_off": np.concatenate([rec0["seq_off"], rec1["seq_off"][1:] + rec0["seq_off"][-1]]),
           "tid": np.concatenate([np.zeros(n0, np.int32), np.full(n1, 2, np.int32)])}
    path = str(tmp_path / "two.bam")
    bam_io.write_bam(path, rec, [("c0", 40000), ("empty", 5000), ("c2", 30000)],
                     names=["q%d" % i for i in range(n0 + n1)])
    return path, rec


REGIONS = [(None, None), (0, 10), (0, 500), (1000, 1001), (2500, 9000), (12345, 12346), (20000, 21000), (25000, 40000),
           (39000, 40000), (100000, 200000), (500, 400)]


@pytest.mark.parametrize("read_len", [150, 2000])
def test_index_range_gives_read_bam_records(tmp_path, read_len):
    path, rec = _two_contig_bam(tmp_path, read_len=read_len)
    bai = bam_io.write_bai(path)
    idx = bam_io.read_bai(bai)
    assert len(idx) == 3 and idx[1]["bins"] == {} and bam_io._PSEUDO_BIN not in idx[0]["bins"]
    raw = open(path, "rb").read()
    # region edges on read starts and ends of the first contig
    p0 = int(rec["pos"][5])
    span = int((rec["cigar"][rec["cigar_off"][5]:rec["cigar_off"][6]] >> 4)[np.isin(rec["cigar"][rec["cigar_off"][5]:rec["cigar_off"][6]] & 15, (0, 2, 3, 7, 8))].sum())
    regions = REGIONS + [(p0, p0 + 1), (p0 - 1, p0), (p0 + span, p0 + span + 5), (p0 + span - 1, p0 + span)]
    for ctg, tid in (("c0", 0), ("empty", 1), ("c2", 2)):
        for start, end in regions:
            want, _ = bam_io.read_bam(path, ctg, start, end, with_names=True)
            c0, c1, u0, u1 = bam_io.bai_range(idx, tid, 0 if start is None else start, (1 << 29) if end is None else end, path)
            got = _host_filter(_inflate_range(raw, c0, c1), u0, u1, tid, start, end) if c1 > c0 else []
            assert [p for p, _ in got] == want["pos"].tolist(), (ctg, start, end)
            assert [n.decode() for _, n in got] == want["names"], (ctg, start, end)


def test_header_spanning_several_blocks(tmp_path):
    rec, _, _ = sr.random_alignment(3000, depth=3, read_len=500, seed=9)
    refs = [("contig_%05d" % i, 1000 + i) for i in range(9000)]          # ~180 kB of header: three blocks and more
    path = str(tmp_path / "big_header.bam")
    bam_io.write_bam(path, rec, refs, tid=7)
    got_refs, vo = bam_io.read_bam_header(path)
    assert got_refs == refs
    raw = open(path, "rb").read()
    blocks = bam_io.bgzf_blocks(raw)
    assert len([b for b in blocks if b[0] < vo >> 16]) >= 3
    buf = b"".join(bam_io._inflate_block(raw, o)[1] for o, _, _ in blocks)
    _, hdr_end = bam_io.read_header(buf)
    before = sum(isize for o, _, isize in blocks if o < vo >> 16)
    assert before + (vo & 0xFFFF) == hdr_end
    want, _ = bam_io.read_bam(path, "contig_00007")
    got = _host_filter(_inflate_range(raw, vo >> 16, len(raw)), vo & 0xFFFF, len(buf) - before, 7, None, None)
    assert [p for p, _ in got] == want["pos"].tolist()


def _block(payload=b"abc", magic=b"\x1f\x8b\x08\x04", extra=None, bsize=None, isize=None):
    data = zlib.compressobj(6, zlib.DEFLATED, -15)
    data = data.compress(payload) + data.flush()
    extra = struct.pack("<BBHH", 66, 67, 2, 0) if extra is None else extra
    size = 12 + len(extra) + len(data) + 8
    if b"BC" in extra[:2] or extra[:2] == b"BC":
        extra = extra[:4] + struct.pack("<H", size - 1 if bsize is None else bsize) + extra[6:]
    head = magic + b"\x00\x00\x00\x00\x00\xff" + struct.pack("<H", len(extra)) + extra
    return head + data + struct.pack("<II", zlib.crc32(payload), len(payload) if isize is None else isize)


def test_bgzf_header_checks():
    good = _block()
    assert bam_io.bgzf_blocks(good) == [(0, len(good), 3)]
    # a BC subfield after another subfield is found
    other = struct.pack("<BBH", 65, 66, 3) + b"xyz"
    blk = _block(extra=other + struct.pack("<BBHH", 66, 67, 2, 0))
    size = len(blk)
    blk = blk[:12 + 7 + 4] + struct.pack("<H", size - 1) + blk[12 + 7 + 6:]
    assert bam_io.bgzf_blocks(blk) == [(0, size, 3)]
    plain = zlib.compressobj(6, zlib.DEFLATED, 31)
    plain = plain.compress(b"abc") + plain.flush()                     # ordinary gzip: no FEXTRA
    with pytest.raises(ValueError, match="not a BGZF block"):
        bam_io.bgzf_blocks(plain)
    with pytest.raises(ValueError, match="no BC subfield"):
        bam_io.bgzf_blocks(_block(extra=struct.pack("<BBH", 65, 66, 2) + b"zz"))
    with pytest.raises(ValueError, match="BSIZE .* out of range"):
        bam_io.bgzf_blocks(_block(bsize=len(good) + 10))
    with pytest.raises(ValueError, match="BSIZE .* out of range"):
        bam_io.bgzf_blocks(_block(bsize=10))
    with pytest.raises(ValueError, match="ISIZE .* exceeds 65536"):
        bam_io.bgzf_blocks(_block(isize=65537))
    with pytest.raises(ValueError, match="trailing bytes"):
        bam_io.bgzf_blocks(good + good[:10])
