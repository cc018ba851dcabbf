"""Host-side BAM / FASTA reading: the plain-Python record reader, and the header, index and byte ranges the GPU reader takes.

The reference decodes alignments with htslib inside libclair3 (``sam_itr_next`` / ``bam_mplp_auto``, HKU-BAL/Clair3
``src/medaka_bamiter.c:13-55``, ``src/clair3_pileup.c:160-176``) and fetches the reference with ``faidx_fetch_seq`` (``:184-186``).
Two readers produce the records the GPU counter and builder take:

- ``clair3_b200.bam_decode.BamDecoder`` inflates the BGZF blocks and parses the records on the GPU, into device-resident records.
  This module gives it what the host has to know first: the header and the first record's virtual offset
  (``read_bam_header``), the ``.bai`` index (``read_bai``) and the compressed byte range of a region (``bai_range``), and the
  checked BGZF block headers (``bgzf_blocks``).
- ``read_bam`` is the plain-Python reader: it inflates the whole file with ``gzip`` (BGZF blocks are gzip members) and parses the
  records per the SAM/BAM specification, section 4.2, on the CPU.  It states the region filter both readers apply, and the tests
  hold the GPU reader to it.

A writer is included so that tests (and users without samtools) can produce valid files, and ``write_bai`` indexes them as the
specification's section 5.2 describes.  CRAM and CSI indexes are not handled.  The reference bases come out of a FASTA file
(``read_fasta``, or ``fetch_fasta`` at random access through its ``.fai``).  ``idxstats`` reads the mapped counts of the
``.bai``; ``write_bgzf`` and ``write_tbi`` write a bgzipped, tabix-indexed VCF as ``bgzip`` and ``tabix -p vcf`` do.
"""
from __future__ import annotations

import bisect
import gzip
import os
import struct
import zlib

import numpy as np

_REF_CONSUMING = (0, 2, 3, 7, 8)
_CORE = struct.Struct("<iiBBHHHiiii")          # refID pos l_read_name mapq bin n_cigar_op flag l_seq next_refID next_pos tlen
_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")      # the 28-byte BGZF end-of-file block


def read_header(buf):
    """(references [(name, length)], offset of the first alignment) of an uncompressed BAM byte string."""
    if buf[:4] != b"BAM\x01":
        raise ValueError("not a BAM stream (magic %r)" % buf[:4])
    l_text, = struct.unpack_from("<i", buf, 4)
    off = 8 + l_text
    n_ref, = struct.unpack_from("<i", buf, off)
    off += 4
    refs = []
    for _ in range(n_ref):
        l_name, = struct.unpack_from("<i", buf, off)
        name = buf[off + 4:off + 4 + l_name - 1].decode()
        l_ref, = struct.unpack_from("<i", buf, off + 4 + l_name)
        refs.append((name, l_ref))
        off += 8 + l_name
    return refs, off


_AUX_SIZE = {ord("A"): 1, ord("c"): 1, ord("C"): 1, ord("s"): 2, ord("S"): 2, ord("i"): 4, ord("I"): 4, ord("f"): 4}
_B_DTYPE = {ord("c"): "<i1", ord("C"): "<u1", ord("s"): "<i2", ord("S"): "<u2", ord("i"): "<i4", ord("I"): "<u4"}


def _aux_mv(buf, p, e):
    """The values of the ``mv`` B-array among the auxiliary fields buf[p:e] (SAM/BAM specification 4.2.4), widened to int32, or
    None when the record has no such tag."""
    while p + 3 <= e:
        tag, t = buf[p:p + 2], buf[p + 2]
        if t == ord("B"):
            sub = buf[p + 3]
            cnt, = struct.unpack_from("<i", buf, p + 4)
            if tag == b"mv" and sub in _B_DTYPE:
                return np.frombuffer(buf, dtype=_B_DTYPE[sub], count=cnt, offset=p + 8).astype(np.int32)
            p += 8 + cnt * (_AUX_SIZE.get(sub, 4))
        elif t in (ord("Z"), ord("H")):
            z = buf.index(b"\0", p + 3)
            p = z + 1
        else:
            p += 3 + _AUX_SIZE[t]
    return None


_CG_MAX = 1 << 29             # htslib moves a CG tag of fewer words than this


def _aux_find(buf, p, e, tag):
    """(offset, type byte) of the first auxiliary field named ``tag`` in buf[p:e], or None when there is none or the fields
    before it are malformed (htslib's ``bam_aux_get``)."""
    while p + 3 <= e:
        t = buf[p + 2]
        if buf[p:p + 2] == tag:
            return p, t
        if t == ord("B"):
            if p + 8 > e:
                return None
            cnt, = struct.unpack_from("<i", buf, p + 4)
            q = p + 8 + cnt * _AUX_SIZE.get(buf[p + 3], 4)
            if cnt < 0 or q > e:
                return None
            p = q
        elif t in (ord("Z"), ord("H")):
            z = buf.find(b"\0", p + 3, e)
            if z < 0:
                return None
            p = z + 1
        elif t in _AUX_SIZE:
            p += 3 + _AUX_SIZE[t]
        else:
            return None
    return None


def _cg_cigar(buf, core, c0, aux0, e):
    """The real CIGAR of a record whose operations did not fit the 16-bit ``n_cigar_op``, or None.  A writer stores such a
    record's CIGAR as the placeholder ``<l_seq>S<ref_len>N`` and the real one in a ``CG:B,I`` tag (SAM/BAM specification 4.2.2);
    htslib's ``bam_tag2cigar`` moves it back when the record has a position, its first operation is ``S`` of length l_seq, and the
    first ``CG`` tag is a ``B,I`` or ``B,i`` array of at least n_cigar_op (and fewer than 2^29) words."""
    tid, p, _, _, _, n_cig, _, l_seq = core[:8]
    if n_cig == 0 or tid < 0 or p < 0:
        return None
    w0, = struct.unpack_from("<I", buf, c0)
    if w0 & 15 != 4 or w0 >> 4 != l_seq:
        return None
    hit = _aux_find(buf, aux0, e, b"CG")
    if hit is None or hit[1] != ord("B") or hit[0] + 8 > e or buf[hit[0] + 3] not in (ord("I"), ord("i")):
        return None
    cnt, = struct.unpack_from("<I", buf, hit[0] + 4)
    if cnt < n_cig or cnt >= _CG_MAX or hit[0] + 8 + 4 * cnt > e:
        return None
    return np.frombuffer(buf, dtype="<u4", count=cnt, offset=hit[0] + 8)


def read_bam(path, ref_name=None, start=None, end=None, with_names=False, fa_fields=False):
    """Alignment records of a coordinate-sorted BAM as the arrays of ``clair3_b200.records.BamRecords`` (plus ``tid``), in
    file order.  ``ref_name`` / ``start`` / ``end`` (0-based, end-exclusive) keep what an indexed fetch of that region returns:
    records of that contig whose alignment overlaps [start, end).  Unmapped-without-position records (refID -1) are skipped.
    A record of more than 65,535 CIGAR operations, stored as a placeholder CIGAR and a ``CG`` tag, gets its real CIGAR back as
    htslib reads it (``_cg_cigar``).
    ``fa_fields``: also the fields the full-alignment tensor builder reads (``clair3_b200.fa_tensor``): ``qual`` / ``qual_off``
    (bam_get_qual), ``qname`` / ``qname_off`` (read names without the NUL, concatenated bytes) and ``mv`` / ``mv_off`` (the
    ``mv`` B-array including its leading stride element, any integer subtype widened to int32; an empty range when the record has
    no ``mv`` tag).  Returns (records dict, [(reference name, length)])."""
    with gzip.open(path, "rb") as f:
        buf = f.read()
    refs, off = read_header(buf)
    want_tid = None
    if ref_name is not None:
        names = [n for n, _ in refs]
        if ref_name not in names:
            raise ValueError("contig %r is not in the BAM header" % ref_name)
        want_tid = names.index(ref_name)
    lo = -1 if start is None else int(start)
    hi = 1 << 62 if end is None else int(end)
    pos, flag, mapq, lq, tids, names_out = [], [], [], [], [], []
    quals, qnames, mvs = [], [], []
    cig_parts, seq_parts, coff, soff = [], [], [0], [0]
    n = len(buf)
    while off + 4 <= n:
        block_size, = struct.unpack_from("<i", buf, off)
        rec0 = off + 4
        off = rec0 + block_size
        if off > n:
            raise ValueError("truncated BAM record")
        tid, p, l_name, mq, _bin, n_cig, fl, l_seq, _, _, _ = _CORE.unpack_from(buf, rec0)
        if tid < 0 or (want_tid is not None and tid != want_tid):
            if want_tid is not None and tid > want_tid:
                break                                        # sorted: nothing of the wanted contig follows
            continue
        if p >= hi and want_tid is not None:
            break
        c0 = rec0 + 32 + l_name
        cig = np.frombuffer(buf, dtype="<u4", count=n_cig, offset=c0)
        cg = _cg_cigar(buf, (tid, p, l_name, mq, _bin, n_cig, fl, l_seq), c0, c0 + 4 * n_cig + (l_seq + 1) // 2 + l_seq, off)
        s0 = c0 + 4 * n_cig
        if cg is not None:
            cig, n_cig = cg, len(cg)
        span = int((cig >> 4)[np.isin(cig & 15, _REF_CONSUMING)].sum()) if n_cig else 0
        if p + max(span, 1) <= lo:
            continue
        nb = (l_seq + 1) // 2
        pos.append(p)
        flag.append(fl)
        mapq.append(mq)
        lq.append(l_seq)
        tids.append(tid)
        cig_parts.append(cig)
        seq_parts.append(buf[s0:s0 + nb])
        coff.append(coff[-1] + n_cig)
        soff.append(soff[-1] + nb)
        if with_names:
            names_out.append(buf[rec0 + 32:rec0 + 32 + l_name - 1].decode())
        if fa_fields:
            q0 = s0 + nb
            quals.append(buf[q0:q0 + l_seq])
            qnames.append(buf[rec0 + 32:rec0 + 32 + l_name - 1])
            mv = _aux_mv(buf, q0 + l_seq, off)
            mvs.append(mv if mv is not None else np.zeros(0, np.int32))
    rec = {"pos": np.array(pos, np.int64), "flag": np.array(flag, np.uint16), "mapq": np.array(mapq, np.uint8),
           "l_qseq": np.array(lq, np.int32), "cigar_off": np.array(coff, np.int64),
           "cigar": np.concatenate(cig_parts).astype(np.uint32) if cig_parts else np.zeros(0, np.uint32),
           "seq_off": np.array(soff, np.int64), "seq": np.frombuffer(b"".join(seq_parts), dtype=np.uint8).copy(),
           "tid": np.array(tids, np.int32)}
    if with_names:
        rec["names"] = names_out
    if fa_fields:
        def offsets(parts):
            return np.concatenate([[0], np.cumsum([len(x) for x in parts], dtype=np.int64)]).astype(np.int64)
        rec["qual"] = np.frombuffer(b"".join(quals), dtype=np.uint8).copy()
        rec["qual_off"] = offsets(quals)
        rec["qname"] = np.frombuffer(b"".join(qnames), dtype=np.uint8).copy()
        rec["qname_off"] = offsets(qnames)
        rec["mv"] = np.concatenate(mvs).astype(np.int32) if mvs else np.zeros(0, np.int32)
        rec["mv_off"] = offsets(mvs)
    return rec, refs


def _reg2bin(beg, end):
    """The UCSC binning scheme of the BAM specification (section 5.3)."""
    end -= 1
    for shift, base in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> shift == end >> shift:
            return base + (beg >> shift)
    return 0


def _bgzf_block(payload):
    comp = zlib.compressobj(6, zlib.DEFLATED, -15)
    data = comp.compress(payload) + comp.flush()
    bsize = len(data) + 25                                   # total block size - 1
    header = struct.pack("<BBBBIBBHBBHH", 0x1F, 0x8B, 8, 4, 0, 0, 0xFF, 6, 0x42, 0x43, 2, bsize)
    return header + data + struct.pack("<II", zlib.crc32(payload) & 0xFFFFFFFF, len(payload))


def write_bam(path, rec, refs, tid=0, names=None, header_text=None):
    """Writes the records (arrays as ``read_bam`` returns them; every record on contig ``tid`` unless ``rec['tid']`` is given) as a
    BGZF-compressed BAM: ``refs`` = [(name, length)].  Without ``rec['qual']`` the qualities are written as 0xFF (absent); read names
    come from ``names``, else ``rec['qname']`` / ``rec['qname_off']``, else ``r<i>``; ``rec['mv']`` / ``rec['mv_off']`` become an
    ``mv:B:c`` tag (``mv:B:i`` when a value does not fit int8) on every record with a non-empty range, as ``read_bam(...,
    fa_fields=True)`` returns them.  A record of more than 65,535 CIGAR operations is written as htslib writes it: the placeholder
    CIGAR ``<l_seq>S<ref_len>N`` and the real one in a ``CG:B,I`` tag after the other tags."""
    text = (header_text or "@HD\tVN:1.6\tSO:coordinate\n" + "".join("@SQ\tSN:%s\tLN:%d\n" % r for r in refs)).encode()
    out = bytearray(b"BAM\x01" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs)))
    for name, length in refs:
        nb = name.encode() + b"\x00"
        out += struct.pack("<i", len(nb)) + nb + struct.pack("<i", length)
    n = len(rec["pos"])
    tids = rec.get("tid", np.full(n, tid, np.int32))
    for i in range(n):
        cig = np.ascontiguousarray(rec["cigar"][rec["cigar_off"][i]:rec["cigar_off"][i + 1]], dtype="<u4")
        seq = bytes(rec["seq"][rec["seq_off"][i]:rec["seq_off"][i + 1]])
        l_seq = int(rec["l_qseq"][i])
        if names:
            nm = names[i].encode() + b"\x00"
        elif rec.get("qname_off") is not None:
            nm = bytes(rec["qname"][rec["qname_off"][i]:rec["qname_off"][i + 1]]) + b"\x00"
        else:
            nm = ("r%d" % i).encode() + b"\x00"
        if rec.get("qual_off") is not None:
            qual = bytes(np.asarray(rec["qual"][rec["qual_off"][i]:rec["qual_off"][i + 1]], dtype=np.uint8))
        else:
            qual = b"\xff" * l_seq
        aux = b""
        if rec.get("mv_off") is not None and rec["mv_off"][i + 1] > rec["mv_off"][i]:
            mv = np.asarray(rec["mv"][rec["mv_off"][i]:rec["mv_off"][i + 1]], dtype=np.int64)
            small = mv.min() >= -128 and mv.max() <= 127
            aux = b"mvB" + (b"c" if small else b"i") + struct.pack("<i", len(mv)) + mv.astype("<i1" if small else "<i4").tobytes()
        p = int(rec["pos"][i])
        span = int((cig >> 4)[np.isin(cig & 15, _REF_CONSUMING)].sum())
        if len(cig) > 0xFFFF:                                 # as htslib writes it: the placeholder, and the CIGAR in CG:B,I last
            aux += b"CGBI" + struct.pack("<I", len(cig)) + cig.tobytes()
            cig = np.array([l_seq << 4 | 4, span << 4 | 3], dtype="<u4")
        body = _CORE.pack(int(tids[i]), p, len(nm), int(rec["mapq"][i]), _reg2bin(p, p + max(span, 1)), len(cig), int(rec["flag"][i]),
                          l_seq, -1, -1, 0) + nm + cig.tobytes() + seq[:(l_seq + 1) // 2] + qual + aux
        out += struct.pack("<i", len(body)) + body
    with open(path, "wb") as f:
        _write_bgzf_blocks(f, out)


_BGZF_PAYLOAD = 0xFF00        # payload per block, as bgzip and htslib cut it


def _write_bgzf_blocks(f, data):
    """Writes ``data`` to the open file ``f`` as BGZF blocks of ``_BGZF_PAYLOAD`` bytes and the EOF block; returns the file
    offset of each block."""
    offsets = []
    for b0 in range(0, len(data), _BGZF_PAYLOAD):           # BGZF: at most 64 KiB of payload per block
        offsets.append(f.tell())
        f.write(_bgzf_block(bytes(data[b0:b0 + _BGZF_PAYLOAD])))
    f.write(_EOF)
    return offsets


def write_bgzf(path, data):
    """Writes ``data`` (bytes or str) as a BGZF file with the end-of-file block, as ``bgzip`` does (the blocks ``write_bam``
    writes).  Returns the virtual offset (SAM/BAM specification 4.1.1) of every uncompressed byte position as a function
    ``voffset(u)``, which ``write_tbi`` indexes with."""
    data = data.encode() if isinstance(data, str) else bytes(data)
    with open(path, "wb") as f:
        offsets = _write_bgzf_blocks(f, data)
        end = f.tell() - len(_EOF)

    def voffset(u):
        i = u // _BGZF_PAYLOAD
        return offsets[i] << 16 | (u - i * _BGZF_PAYLOAD) if i < len(offsets) else end << 16
    return voffset


def read_fasta(path, name, start=0, end=None):
    """Bases [start, end) of sequence ``name`` (first word of the '>' line) of a plain or gzip-compressed FASTA file, case kept
    (the counter upper-cases where the reference does).  A linear scan: no .fai needed."""
    opener = gzip.open if str(path).endswith(".gz") else open
    parts, on, have = [], False, 0
    with opener(path, "rt") as f:
        for line in f:
            if line.startswith(">"):
                if on:
                    break
                on = line[1:].split()[0] == name if line[1:].split() else False
                continue
            if on:
                line = line.strip()
                parts.append(line)
                have += len(line)
                if end is not None and have >= end:
                    break
    if not parts and not on:
        raise ValueError("sequence %r not found in %s" % (name, path))
    seq = "".join(parts)
    return seq[start:end]


def write_fasta(path, seqs, width=60):
    with open(path, "w") as f:
        for name, seq in seqs:
            f.write(">%s\n" % name)
            for i in range(0, len(seq), width):
                f.write(seq[i:i + width] + "\n")


def write_fai(fasta_path, fai_path=None):
    """Writes the ``.fai`` of a plain FASTA (default ``fasta_path + ".fai"``) as ``samtools faidx`` does: per sequence its name,
    length, the byte offset of its first base, bases per line and bytes per line.  Every line but a sequence's last must be
    full.  Returns the path written."""
    rows, cur = [], None
    with open(fasta_path, "rb") as f:
        if f.read(2) == b"\x1f\x8b":
            raise ValueError("%s: a compressed FASTA cannot be indexed here; decompress it first" % fasta_path)
        f.seek(0)
        off = 0
        for line in f:
            if line.startswith(b">"):
                cur = [line[1:].split()[0].decode(), 0, off + len(line), 0, 0]
                rows.append(cur)
            elif cur is not None:
                n = len(line.rstrip(b"\r\n"))
                if cur[3] == 0:
                    cur[3], cur[4] = n, len(line)
                cur[1] += n
            off += len(line)
    path = fai_path or str(fasta_path) + ".fai"
    with open(path, "w") as f:
        f.write("".join("%s\t%d\t%d\t%d\t%d\n" % tuple(r) for r in rows))
    return path


def read_fai(path):
    """The rows of a ``.fai`` index in file order: [(name, length, offset, line bases, line bytes)]."""
    out = []
    with open(path) as f:
        for row in f:
            c = row.rstrip("\n").split("\t")
            if len(c) >= 5:
                out.append((c[0], int(c[1]), int(c[2]), int(c[3]), int(c[4])))
    return out


def fetch_fasta(path, name, start=0, end=None, fai=None):
    """Bases [start, end) of sequence ``name`` of a plain FASTA through its ``.fai`` (default ``path + ".fai"``), clipped to the
    sequence, case kept: what ``read_fasta`` returns, read at random access as ``faidx_fetch_seq`` reads it.  A bgzip-compressed
    FASTA is refused (ValueError)."""
    rows = {r[0]: r for r in read_fai(fai or str(path) + ".fai")}
    if name not in rows:
        raise ValueError("sequence %r not found in the index of %s" % (name, path))
    _, length, off, lb, lw = rows[name]
    start = max(0, int(start))
    end = length if end is None else min(int(end), length)
    if end <= start:
        return ""
    with open(path, "rb") as f:
        if f.read(2) == b"\x1f\x8b":
            raise ValueError("%s: compressed FASTA is not supported; decompress it (and re-index it)" % path)
        a = off + start // lb * lw + start % lb
        b = off + (end - 1) // lb * lw + (end - 1) % lb + 1
        f.seek(a)
        raw = f.read(b - a)
    return raw.replace(b"\n", b"").replace(b"\r", b"").decode()


# ---- BGZF blocks, the header and the .bai index: what the GPU reader (clair3_b200.bam_decode) needs from the host ----

BGZF_MAX = 65536             # a BGZF block holds at most 64 KiB, compressed or not (SAM/BAM specification 4.1)


def bgzf_block(buf, off):
    """(total size, payload offset, payload size, ISIZE) of the BGZF block at ``buf[off:]``, after the checks the GPU reader's
    ``c3b_bam_decode`` makes: the gzip magic ``1f 8b 08 04``, a ``BC`` subfield anywhere in the extra field, a ``BSIZE`` that
    covers the header and footer and fits the data, and ``ISIZE <= 65536``.  Raises ValueError naming the block's offset."""
    if len(buf) - off < 18:
        raise ValueError("%d trailing bytes at offset %d are not a BGZF block" % (len(buf) - off, off))
    if bytes(buf[off:off + 4]) != b"\x1f\x8b\x08\x04":
        raise ValueError("the block at offset %d is not a BGZF block (gzip header %s, want 1f 8b 08 04)"
                         % (off, bytes(buf[off:off + 4]).hex(" ")))
    xlen, = struct.unpack_from("<H", buf, off + 10)
    if off + 12 + xlen > len(buf):
        raise ValueError("the extra field of the block at offset %d runs past the data" % off)
    bsize, x = None, 0
    while x + 4 <= xlen:
        si1, si2, slen = struct.unpack_from("<BBH", buf, off + 12 + x)
        if x + 4 + slen > xlen:
            break
        if si1 == 66 and si2 == 67 and slen == 2:
            bsize, = struct.unpack_from("<H", buf, off + 16 + x)
            break
        x += 4 + slen
    if bsize is None:
        raise ValueError("the block at offset %d has no BC subfield" % off)
    size = bsize + 1
    if size < 12 + xlen + 8 or off + size > len(buf):
        raise ValueError("BSIZE %d of the block at offset %d is out of range" % (bsize, off))
    isize, = struct.unpack_from("<I", buf, off + size - 4)
    if isize > BGZF_MAX:
        raise ValueError("ISIZE %d of the block at offset %d exceeds 65536" % (isize, off))
    return size, off + 12 + xlen, size - 12 - xlen - 8, isize


def bgzf_blocks(buf):
    """[(offset, total size, ISIZE)] of the BGZF blocks that make up ``buf`` (whole blocks only), checked as ``bgzf_block``."""
    out, off = [], 0
    while off < len(buf):
        size, _, _, isize = bgzf_block(buf, off)
        out.append((off, size, isize))
        off += size
    return out


def _inflate_block(buf, off):
    size, p0, n, isize = bgzf_block(buf, off)
    data = zlib.decompress(bytes(buf[p0:p0 + n]), -15)
    if len(data) != isize:
        raise ValueError("the block at offset %d inflates to %d bytes, not its ISIZE %d" % (off, len(data), isize))
    return size, data


def _read_block(f, off):
    """(total size, the block's bytes) of the BGZF block at byte ``off`` of the open file ``f``; (0, b"") at the end of the file."""
    f.seek(off)
    head = f.read(18)
    if not head:
        return 0, b""
    xlen, = struct.unpack_from("<H", head, 10) if len(head) >= 12 else (0,)
    head += f.read(max(0, 12 + xlen - len(head)))
    size = bgzf_block(head + bytes(BGZF_MAX), 0)[0]     # the header alone decides the size; the padding stands in for the rest
    return size, head + f.read(size - len(head))


def read_bam_header(path):
    """(references [(name, length)], virtual offset of the first record) of a BAM file, inflating only the blocks that hold the
    header.  The virtual offset is ``block offset << 16 | offset in the block's data`` (SAM/BAM specification 4.1.1)."""
    with open(path, "rb") as f:
        data, starts, off = bytearray(), [], 0
        while True:
            size, block = _read_block(f, off)
            if not size:
                raise ValueError("%s: the file ends inside the BAM header" % path)
            starts.append((off, len(data)))
            data += _inflate_block(block, 0)[1]
            off += size
            if len(data) < 4 or data[:4] != b"BAM\x01":
                if len(data) >= 4:
                    raise ValueError("not a BAM stream (magic %r)" % bytes(data[:4]))
                continue
            try:
                refs, end = read_header(data)
            except (struct.error, UnicodeDecodeError):
                continue
            if end == len(data):                   # the header ends with the block: the first record starts the next one
                return refs, off << 16
            c, u = starts[bisect.bisect_right([u for _, u in starts], end) - 1]
            return refs, c << 16 | (end - u)


_PSEUDO_BIN = 37450          # the .bai pseudo-bin that holds a reference's offsets and mapped / unmapped counts


def _reg2bins(beg, end):
    """Every bin that can hold a record overlapping [beg, end) (SAM/BAM specification 5.3, reg2bins)."""
    end -= 1
    bins = [0]
    for shift, base in ((26, 1), (23, 9), (20, 73), (17, 585), (14, 4681)):
        bins.extend(range(base + (beg >> shift), base + (end >> shift) + 1))
    return bins


def read_bai(path):
    """A ``.bai`` index (SAM/BAM specification 5.2) as one dict per reference: ``bins`` {bin: [(begin, end) virtual offsets]}
    without the pseudo-bin 37450, and ``linear``, the 16 kb linear index (uint64 virtual offsets)."""
    with open(path, "rb") as f:
        buf = f.read()
    if buf[:4] != b"BAI\x01":
        raise ValueError("%s: not a BAI index (magic %r)" % (path, buf[:4]))
    n_ref, = struct.unpack_from("<i", buf, 4)
    off, out = 8, []
    for _ in range(n_ref):
        n_bin, = struct.unpack_from("<i", buf, off)
        off += 4
        bins = {}
        for _ in range(n_bin):
            b, n_chunk = struct.unpack_from("<Ii", buf, off)
            off += 8
            chunks = np.frombuffer(buf, dtype="<u8", count=2 * n_chunk, offset=off).reshape(-1, 2)
            off += 16 * n_chunk
            if b != _PSEUDO_BIN:
                bins[b] = [(int(x), int(y)) for x, y in chunks]
        n_intv, = struct.unpack_from("<i", buf, off)
        off += 4
        linear = np.frombuffer(buf, dtype="<u8", count=n_intv, offset=off).astype(np.uint64)
        off += 8 * n_intv
        out.append({"bins": bins, "linear": linear})
    return out


def _bai_span(index, tid, start, end):
    """(first virtual offset, end virtual offset) covering every record of contig ``tid`` the index puts in [start, end), or
    None: the chunks of the bins of reg2bins, less those that end before the linear index's offset for ``start``."""
    if tid >= len(index):
        return None
    beg = max(int(start), 0)
    hi = min(int(end), 1 << 29)
    if hi <= beg:                                  # read_bam keeps pos < end and pos + span > start: those start before end
        beg, hi = 0, hi
    if hi <= 0:
        return None
    ref = index[tid]
    lin = ref["linear"]
    min_off = int(lin[min(beg >> 14, len(lin) - 1)]) if len(lin) else 0
    chunks = [c for b in _reg2bins(beg, hi) for c in ref["bins"].get(b, ()) if c[1] > min_off]
    if not chunks:
        return None
    return min(c[0] for c in chunks), max(c[1] for c in chunks)


def bai_range(index, tid, start, end, bam_path):
    """One compressed byte range of whole BGZF blocks ``(coff_begin, coff_end, first_uoff, end_uoff)`` that holds every record of
    contig ``tid`` overlapping [start, end), from the index (``read_bai``): the union of the chunks of the bins of
    ``reg2bins(start, end)``, pruned by the linear index.  ``first_uoff`` is the first record's offset in the first block's data
    and ``end_uoff`` where the records end, counted from the range's first uncompressed byte: the arguments of
    ``c3b_bam_decode``.  The union is a superset of the region's records; the decoder's filter makes it exact.  The block sizes
    come from the headers of the range's blocks in ``bam_path``.  (0, 0, 0, 0) when the index holds nothing there."""
    span = _bai_span(index, tid, start, end)
    if span is None:
        return 0, 0, 0, 0
    (c0, u0), (ce, ue) = divmod(span[0], 1 << 16), divmod(span[1], 1 << 16)
    acc, c = 0, c0
    with open(bam_path, "rb") as f:
        while c < ce:
            size, block = _read_block(f, c)
            if not size:
                break
            acc += bgzf_block(block, 0)[3]
            c += size
        if c != ce:
            raise ValueError("%s: the index's offset %d is not the start of a BGZF block" % (bam_path, ce))
        if ue == 0:
            return c0, ce, u0, acc
        size, block = _read_block(f, ce)
        return c0, ce + size, u0, acc + ue


def write_bai(bam_path, bai_path=None):
    """Writes the ``.bai`` index of a coordinate-sorted BAM (default ``bam_path + ".bai"``) as the SAM/BAM specification (5.2)
    describes it: per reference the bins of reg2bin(pos, pos + max(span, 1)) with their chunks of virtual offsets (adjacent
    records of a bin merged into one chunk), the pseudo-bin 37450 (offsets of the reference's records, mapped and unmapped
    counts) and the 16 kb linear index, then the number of records without a coordinate.  Returns the path written."""
    with open(bam_path, "rb") as f:
        raw = f.read()
    blocks = bgzf_blocks(raw)
    parts, ustart, u = [], [], 0
    for off, _, isize in blocks:
        ustart.append(u)
        parts.append(_inflate_block(raw, off)[1])
        u += isize
    buf = b"".join(parts)

    def voff(x):
        i = bisect.bisect_right(ustart, x) - 1
        return blocks[i][0] << 16 | (x - ustart[i])

    refs, off = read_header(buf)
    idx = [_index_ref() for _ in refs]
    n_no_coor = 0
    while off + 4 <= len(buf):
        block_size, = struct.unpack_from("<i", buf, off)
        tid, p, l_name, _, _, n_cig, fl = struct.unpack_from("<iiBBHHH", buf, off + 4)
        beg, nxt = voff(off), voff(off + 4 + block_size)
        cig = np.frombuffer(buf, dtype="<u4", count=n_cig, offset=off + 36 + l_name)
        off += 4 + block_size
        if tid < 0 or p < 0:
            n_no_coor += 1
            continue
        span = int((cig >> 4)[np.isin(cig & 15, _REF_CONSUMING)].sum()) if n_cig else 0
        _index_push(idx[tid], p, p + max(span, 1), beg, nxt, not fl & 4)
    out = bytearray(b"BAI\x01" + struct.pack("<i", len(refs)))
    for r in idx:
        out += _index_ref_bytes(r)
    out += struct.pack("<Q", n_no_coor)
    path = bai_path or str(bam_path) + ".bai"
    with open(path, "wb") as f:
        f.write(out)
    return path


# ---- the binning and linear index one reference of a .bai or a .tbi holds (SAM/BAM specification 5.2, tabix 1.1) ----

def _index_ref():
    return {"bins": {}, "lin": {}, "first": None, "last": 0, "mapped": 0, "unmapped": 0}


def _index_push(r, beg, end, voff_beg, voff_end, mapped=True):
    """Adds the record [beg, end) stored at virtual offsets [voff_beg, voff_end) to one reference's index: its bin's chunks
    (adjacent records of a bin merged into one chunk), the 16 kb windows it overlaps and the pseudo-bin's offsets and counts."""
    chunks = r["bins"].setdefault(_reg2bin(beg, end), [])
    if chunks and chunks[-1][1] == voff_beg:
        chunks[-1][1] = voff_end
    else:
        chunks.append([voff_beg, voff_end])
    for w in range(beg >> 14, ((end - 1) >> 14) + 1):
        r["lin"].setdefault(w, voff_beg)
    r["first"] = voff_beg if r["first"] is None else r["first"]
    r["last"] = voff_end
    r["mapped" if mapped else "unmapped"] += 1


def _index_ref_bytes(r):
    """One reference's bins (with the pseudo-bin 37450) and linear index, serialised."""
    bins = dict(r["bins"])
    if r["first"] is not None:
        bins[_PSEUDO_BIN] = [[r["first"], r["last"]], [r["mapped"], r["unmapped"]]]
    out = bytearray(struct.pack("<i", len(bins)))
    for b, chunks in bins.items():
        out += struct.pack("<Ii", b, len(chunks)) + b"".join(struct.pack("<QQ", x, y) for x, y in chunks)
    n_intv = max(r["lin"]) + 1 if r["lin"] else 0
    lin, prev = [], r["first"] or 0             # windows before the first record's: its offset; gaps: the previous window's
    for w in range(n_intv):
        prev = r["lin"].get(w, prev)
        lin.append(prev)
    out += struct.pack("<i", n_intv) + b"".join(struct.pack("<Q", x) for x in lin)
    return bytes(out)


def _read_index_refs(buf, off, n_ref):
    """(per reference {"bins": {bin: [(beg, end)]} without the pseudo-bin, "linear": uint64 [], "mapped", "unmapped"}, end
    offset) of the reference sections of a .bai / .tbi starting at ``buf[off:]``."""
    out = []
    for _ in range(n_ref):
        n_bin, = struct.unpack_from("<i", buf, off)
        off += 4
        bins, mapped, unmapped = {}, 0, 0
        for _ in range(n_bin):
            b, n_chunk = struct.unpack_from("<Ii", buf, off)
            off += 8
            chunks = np.frombuffer(buf, dtype="<u8", count=2 * n_chunk, offset=off).reshape(-1, 2)
            off += 16 * n_chunk
            if b == _PSEUDO_BIN:
                mapped, unmapped = (int(x) for x in chunks[1]) if n_chunk >= 2 else (0, 0)
            else:
                bins[b] = [(int(x), int(y)) for x, y in chunks]
        n_intv, = struct.unpack_from("<i", buf, off)
        off += 4
        linear = np.frombuffer(buf, dtype="<u8", count=n_intv, offset=off).astype(np.uint64)
        off += 8 * n_intv
        out.append({"bins": bins, "linear": linear, "mapped": mapped, "unmapped": unmapped})
    return out, off


def idxstats(bam_path, bai_path=None):
    """``samtools idxstats`` without its last ``*`` row: [(name, length, mapped, unmapped)] per reference of the BAM header, the
    counts read from the ``.bai`` pseudo-bin (default ``bam_path + ".bai"``; 0 and 0 for a reference without one).  A missing
    index is an error (FileNotFoundError), as there."""
    bai_path = bai_path or str(bam_path) + ".bai"
    if not os.path.exists(bai_path):
        raise FileNotFoundError("%s: no BAM index (.bai) found; index the BAM first (a CSI index is not supported)" % bai_path)
    refs, _ = read_bam_header(bam_path)
    with open(bai_path, "rb") as f:
        buf = f.read()
    if buf[:4] != b"BAI\x01":
        raise ValueError("%s: not a BAI index (magic %r)" % (bai_path, buf[:4]))
    n_ref, = struct.unpack_from("<i", buf, 4)
    idx, _ = _read_index_refs(buf, 8, n_ref)
    return [(name, length, idx[i]["mapped"] if i < n_ref else 0, idx[i]["unmapped"] if i < n_ref else 0)
            for i, (name, length) in enumerate(refs)]


# ---- tabix (.tbi) over a BGZF-compressed VCF ----

TBI_VCF = (2, 1, 2, 0, ord("#"), 0)     # format (VCF), col_seq, col_beg, col_end, meta char, skip: ``tabix -p vcf``


def write_tbi(vcf_gz_path, text, voffset, tbi_path=None):
    """Writes the tabix index (``tabix -p vcf``) of a VCF whose text ``text`` was written by ``write_bgzf`` (``voffset``: what it
    returned).  Rows starting with ``#`` are skipped; a record covers [POS - 1, POS - 1 + len(REF)); the contigs are named in
    the order the file first holds them.  The index is BGZF-compressed as tabix writes it.  Returns the path written."""
    data = text.encode() if isinstance(text, str) else bytes(text)
    names, idx, u = [], {}, 0
    for line in data.splitlines(keepends=True):
        nxt = u + len(line)
        if not line.startswith(b"#") and line.strip():
            c = line.rstrip(b"\r\n").split(b"\t")
            ctg, beg = c[0].decode(), int(c[1]) - 1
            end = beg + max(len(c[3]) if len(c) > 3 else 1, 1)
            if ctg not in idx:
                names.append(ctg)
                idx[ctg] = _index_ref()
            _index_push(idx[ctg], beg, end, voffset(u), voffset(nxt))
        u = nxt
    nm = b"".join(n.encode() + b"\0" for n in names)
    out = bytearray(b"TBI\x01" + struct.pack("<i", len(names)) + struct.pack("<6i", *TBI_VCF) + struct.pack("<i", len(nm)) + nm)
    for n in names:
        out += _index_ref_bytes(idx[n])
    out += struct.pack("<Q", 0)
    path = tbi_path or str(vcf_gz_path) + ".tbi"
    write_bgzf(path, bytes(out))
    return path


def read_tbi(path):
    """A tabix index: {"header": (format, col_seq, col_beg, col_end, meta, skip), "names": [...], "refs": per contig as
    ``_read_index_refs``, "n_no_coor"}."""
    with gzip.open(path, "rb") as f:
        buf = f.read()
    if buf[:4] != b"TBI\x01":
        raise ValueError("%s: not a tabix index (magic %r)" % (path, buf[:4]))
    n_ref, = struct.unpack_from("<i", buf, 4)
    header = struct.unpack_from("<6i", buf, 8)
    l_nm, = struct.unpack_from("<i", buf, 32)
    names = [n.decode() for n in buf[36:36 + l_nm].split(b"\0")[:n_ref]]
    refs, off = _read_index_refs(buf, 36 + l_nm, n_ref)
    n_no_coor = struct.unpack_from("<Q", buf, off)[0] if off + 8 <= len(buf) else None
    return {"header": header, "names": names, "refs": refs, "n_no_coor": n_no_coor}


def tbi_chunks(tbi, ctg, start, end):
    """The chunks [(begin, end) virtual offsets] a tabix query of the 0-based [start, end) on ``ctg`` reads: the chunks of the
    bins of reg2bins(start, end), less those that end before the linear index's offset for ``start``."""
    if ctg not in tbi["names"]:
        return []
    ref = tbi["refs"][tbi["names"].index(ctg)]
    lin = ref["linear"]
    min_off = int(lin[min(start >> 14, len(lin) - 1)]) if len(lin) else 0
    return sorted(c for b in _reg2bins(max(start, 0), max(end, start + 1)) for c in ref["bins"].get(b, ()) if c[1] > min_off)
