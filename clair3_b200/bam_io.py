"""Host-side BAM / FASTA reading for the pileup feature counter when htslib is not at hand.

The reference decodes alignments with htslib inside libclair3 (``sam_itr_next`` / ``bam_mplp_auto``, HKU-BAL/Clair3
``src/medaka_bamiter.c:13-55``, ``src/clair3_pileup.c:160-176``) and fetches the reference with ``faidx_fetch_seq`` (``:184-186``).  The GPU
counter (``clair3_b200.pileup_counts``) starts from DECODED records; this module is the plain-Python way to get them out of a
coordinate-sorted ``.bam`` (BGZF blocks are gzip members, so ``gzip`` decodes the container; the records are parsed per the SAM/BAM
specification, section 4.2) and the reference bases out of a FASTA file - decoding stays on the CPU, as in the reference.  A writer
is included so that tests (and users without samtools) can produce valid files.  CRAM and the ``.bai`` index are not handled: the
file is scanned, which is what a chunk-per-process deployment amortises poorly - with htslib available, fill ``BamRecords`` from
``bam1_t`` directly (INTEGRATION.md).
"""
from __future__ import annotations

import gzip
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


def read_bam(path, ref_name=None, start=None, end=None, with_names=False, fa_fields=False):
    """Alignment records of a coordinate-sorted BAM as the arrays of ``clair3_b200.pileup_counts.BamRecords`` (plus ``tid``), in
    file order.  ``ref_name`` / ``start`` / ``end`` (0-based, end-exclusive) keep what an indexed fetch of that region returns:
    records of that contig whose alignment overlaps [start, end).  Unmapped-without-position records (refID -1) are skipped.
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
        span = int((cig >> 4)[np.isin(cig & 15, _REF_CONSUMING)].sum()) if n_cig else 0
        if p + max(span, 1) <= lo:
            continue
        s0 = c0 + 4 * n_cig
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
    fa_fields=True)`` returns them."""
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
        body = _CORE.pack(int(tids[i]), p, len(nm), int(rec["mapq"][i]), _reg2bin(p, p + max(span, 1)), len(cig), int(rec["flag"][i]),
                          l_seq, -1, -1, 0) + nm + cig.tobytes() + seq[:(l_seq + 1) // 2] + qual + aux
        out += struct.pack("<i", len(body)) + body
    with open(path, "wb") as f:
        for b0 in range(0, len(out), 0xFF00):                # BGZF: at most 64 KiB of payload per block
            f.write(_bgzf_block(bytes(out[b0:b0 + 0xFF00])))
        f.write(_EOF)


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
