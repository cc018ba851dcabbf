"""Records of more than 65,535 CIGAR operations, which BAM's 16-bit ``n_cigar_op`` cannot hold.  Since htslib 1.7 a writer stores
such a record's CIGAR as the placeholder ``<l_seq>S<ref_len>N`` and the real one in a ``CG:B,I`` tag, and htslib's reader
(``bam_read1`` -> ``bam_tag2cigar``) moves it back, so every tool reading through htslib sees the real alignment.
``bam_io.write_bam`` writes such records that way and ``bam_io.read_bam`` applies the same rule: a record with a position, a
first operation ``S`` of length l_seq, and a first ``CG`` tag of type ``B,I`` or ``B,i`` holding at least n_cigar_op words.

The rule is stated from htslib's source (``bam_tag2cigar`` in ``sam.c``) and the SAM specification section 4.2.2; no htslib is at
hand to run against, so these tests hold the reader to that statement, with hand-made records for the cases a writer would not
produce."""
import gzip
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bam_craft as bc  # noqa: E402
from clair3_b200 import bam_io  # noqa: E402
from clair3_b200 import synth_reads as sr  # noqa: E402

FIELDS = ("pos", "flag", "mapq", "l_qseq", "cigar_off", "cigar", "seq_off", "seq", "qual_off", "qual", "qname_off", "qname",
          "mv_off", "mv")


def ultra_long_case(seed=3, n_cycles=17500):
    """Short reads around one read of 4 * n_cycles CIGAR operations (~300 kb with the default), in position order, with
    qualities, names and mv tables: (records, ref, ref_start, index of the long read)."""
    rec, ref, rs = sr.random_alignment(320000, depth=2, read_len=3000, seed=seed, origin=3000)
    rng = np.random.default_rng(seed)
    p = 5000
    cig, codes = bc.long_read(ref, rs, p, n_cycles, rng)
    k = int(np.searchsorted(rec["pos"], p))
    out = {}
    for f in ("pos", "flag", "mapq", "l_qseq"):
        out[f] = np.insert(rec[f], k, {"pos": p, "flag": 0, "mapq": 60, "l_qseq": len(codes)}[f]).astype(rec[f].dtype)
    for off, v, mine in (("cigar_off", "cigar", cig), ("seq_off", "seq", np.frombuffer(bc.pack_seq(codes), np.uint8))):
        out[v] = np.concatenate([rec[v][:rec[off][k]], mine, rec[v][rec[off][k]:]]).astype(rec[v].dtype)
        out[off] = np.concatenate([rec[off][:k + 1], rec[off][k:] + len(mine)]).astype(np.int64)
    lq = out["l_qseq"].astype(np.int64)
    out["qual"] = rng.integers(0, 60, int(lq.sum())).astype(np.uint8)
    out["qual_off"] = np.concatenate([[0], np.cumsum(lq)]).astype(np.int64)
    names = [b"read%d" % i for i in range(len(lq))]
    out["qname"] = np.frombuffer(b"".join(names), np.uint8).copy()
    out["qname_off"] = np.concatenate([[0], np.cumsum([len(x) for x in names])]).astype(np.int64)
    mvn = rng.integers(0, 4, len(lq)) * (rng.random(len(lq)) < 0.7)
    out["mv"] = rng.integers(0, 2, int(mvn.sum())).astype(np.int32)
    out["mv_off"] = np.concatenate([[0], np.cumsum(mvn)]).astype(np.int64)
    return out, ref, rs, k


def _same(got, want, fields=FIELDS):
    for f in fields:
        assert got[f].dtype == want[f].dtype and np.array_equal(got[f], want[f]), f


def test_ultra_long_cigar_round_trips_through_the_cg_tag(tmp_path):
    rec, _, _, k = ultra_long_case(n_cycles=17000)
    n_ops = int(rec["cigar_off"][k + 1] - rec["cigar_off"][k])
    assert n_ops > 65535
    path = str(tmp_path / "cg.bam")
    bam_io.write_bam(path, rec, [("ctg", 400000)])
    # on disk: the placeholder <l_seq>S<ref_len>N, and the real CIGAR in CG:B,I after the other tags
    with open(path, "rb") as f:
        buf = gzip.decompress(f.read())
    _, off = bam_io.read_header(buf)
    for _ in range(k):
        off += 4 + struct.unpack_from("<i", buf, off)[0]
    bs, = struct.unpack_from("<i", buf, off)
    tid, p, l_name, _, bin_, n_cig, _, l_seq = bam_io._CORE.unpack_from(buf, off + 4)[:8]
    cig = rec["cigar"][rec["cigar_off"][k]:rec["cigar_off"][k + 1]]
    span = int((cig >> 4)[np.isin(cig & 15, (0, 2, 3, 7, 8))].sum())
    assert n_cig == 2 and l_seq == rec["l_qseq"][k]
    assert list(np.frombuffer(buf, "<u4", 2, off + 36 + l_name)) == [l_seq << 4 | 4, span << 4 | 3]
    assert bin_ == bam_io._reg2bin(p, p + span)
    tail = buf[off + 4 + bs - 8 - 4 * n_ops:off + 4 + bs]
    assert tail[:8] == b"CGBI" + struct.pack("<I", n_ops) and np.array_equal(np.frombuffer(tail[8:], "<u4"), cig)
    got, _ = bam_io.read_bam(path, "ctg", fa_fields=True)
    _same(got, rec)
    # region filtering takes the real CIGAR's span: a window just before the read's end keeps it, one just after drops it
    end = int(rec["pos"][k]) + span
    for lo, hi, kept in ((end - 1, end + 5, True), (end, end + 5, False)):
        sub, _ = bam_io.read_bam(path, "ctg", lo, hi)
        assert (int(rec["pos"][k]) in sub["pos"].tolist() and n_ops in np.diff(sub["cigar_off"]).tolist()) == kept


def _cg_file(path, cig, aux):
    """One 20-base record at position 100 with these CIGAR words and aux bytes, between two plain records."""
    recs = [bc.record(50, [20 << 4], 20, name=b"a"), bc.record(100, cig, 20, aux, name=b"v", qual=bytes(range(20)), seq=bytes(range(10))),
            bc.record(300, [20 << 4], 20, name=b"b")]
    with open(path, "wb") as f:
        f.write(bc.bgzf(bc.header([("ctg", 100000)]) + b"".join(recs)))
        f.write(bam_io._EOF)


REAL = np.array([5 << 4 | 4, 8 << 4, 2 << 4 | 1, 3 << 4 | 2, 5 << 4], np.uint32)      # 5S8M2I3D5M: 20 bases, span 16
PLACE = [20 << 4 | 4, 16 << 4 | 3]
MV = b"mvBc" + struct.pack("<i", 3) + bytes([5, 1, 0])


def _cg(sub=b"I", words=REAL, count=None):
    return b"CGB" + sub + struct.pack("<I", len(words) if count is None else count) + np.asarray(words, "<u4").tobytes()


CONVERTED = [
    ("B,I", PLACE, _cg()),
    ("B,i", PLACE, _cg(b"i")),
    ("after mv and other tags", PLACE, b"XZZabc\0" + MV + b"XiC\x07" + _cg()),
    ("before mv", PLACE, _cg() + MV),
    ("count equal to n_cigar_op", [20 << 4 | 4, 16 << 4 | 3, 0 << 4 | 3, 0 << 4 | 3, 0 << 4 | 3], _cg()),
]
UNCONVERTED = [
    ("S length is not l_seq", [19 << 4 | 4, 16 << 4 | 3], _cg()),
    ("first operation is not S", [20 << 4 | 0, 16 << 4 | 3], _cg()),
    ("B,S type", PLACE, b"CGBS" + struct.pack("<I", 5) + bytes(10)),
    ("B,C type", PLACE, b"CGBC" + struct.pack("<I", 5) + bytes(5)),
    ("Z type", PLACE, b"CGZ5S8M\0"),
    ("count below n_cigar_op", PLACE, _cg(words=REAL[:1])),
    ("a later CG tag", PLACE, b"CGZx\0" + _cg()),
    ("no CG tag", PLACE, MV),
]


@pytest.mark.parametrize("name,cig,aux", CONVERTED, ids=[c[0] for c in CONVERTED])
def test_cg_record_reads_as_its_inline_cigar(tmp_path, name, cig, aux):
    a, b = str(tmp_path / "cg.bam"), str(tmp_path / "inline.bam")
    _cg_file(a, cig, aux)
    rest = aux.replace(_cg(), b"").replace(_cg(b"i"), b"")
    assert rest != aux
    _cg_file(b, REAL, rest)
    for region in ((None, None), (115, 116), (116, 117)):
        got, _ = bam_io.read_bam(a, "ctg", *region, fa_fields=True)
        want, _ = bam_io.read_bam(b, "ctg", *region, fa_fields=True)
        _same(got, want)
    got, _ = bam_io.read_bam(a, "ctg", fa_fields=True)
    assert np.array_equal(got["cigar"][1:6], REAL)


@pytest.mark.parametrize("name,cig,aux", UNCONVERTED, ids=[c[0] for c in UNCONVERTED])
def test_records_outside_the_rule_keep_their_cigar(tmp_path, name, cig, aux):
    path = str(tmp_path / "x.bam")
    _cg_file(path, cig, aux)
    got, _ = bam_io.read_bam(path, "ctg", fa_fields=True)
    assert np.array_equal(got["cigar"][got["cigar_off"][1]:got["cigar_off"][2]], np.array(cig, np.uint32))


def test_unplaced_record_keeps_its_cigar(tmp_path):
    """pos -1 on a placed contig: htslib moves the CG tag only for a record with a position."""
    path = str(tmp_path / "u.bam")
    with open(path, "wb") as f:
        f.write(bc.bgzf(bc.header([("ctg", 1000)]) + bc.record(-1, PLACE, 20, _cg())))
        f.write(bam_io._EOF)
    got, _ = bam_io.read_bam(path, "ctg")
    assert np.array_equal(got["cigar"], np.array(PLACE, np.uint32))
