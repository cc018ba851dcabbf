"""The GPU BAM reader (``clair3_b200.bam_decode``, ``include/clair3_b200_bam.h``) against ``bam_io.read_bam`` on the same file and
arguments: every field, dtype included, with and without ``fa_fields`` and the index; blocks re-compressed every way zlib
writes them; auxiliary fields of every type; malformed input reported with a clear message; and the records through the pileup
counter and the full-alignment builder to call records."""
import struct
import zlib

import numpy as np
import pytest
import torch

from clair3_b200 import bam_io, decode, synth
from clair3_b200 import synth_reads as sr
from clair3_b200._ffi import C3BError
from clair3_b200.bam_decode import BamDecoder
from clair3_b200.fa_tensor import FullAlignmentBuilder
from clair3_b200.model import Clair3_F, Clair3_P
from clair3_b200.pileup_counts import PileupCounter

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dec():
    d = BamDecoder(0)
    yield d
    d.close()


def _same(got, path, ctg, start, end, fa_fields):
    want, _ = bam_io.read_bam(path, ctg, start, end, fa_fields=fa_fields)
    h = got.host()
    keys = [k for k in want if k != "tid"]
    assert sorted(keys) == sorted(h), (sorted(keys), sorted(h))
    for k in keys:
        assert h[k].dtype == want[k].dtype, (k, h[k].dtype, want[k].dtype)
        assert np.array_equal(h[k], want[k]), (k, ctg, start, end, fa_fields)
    return len(want["pos"])


def _check(dec, path, ctg, regions, fa=(False, True), index=(None, False)):
    n = 0
    for start, end in regions:
        for fa_fields in fa:
            for ix in index:                     # None: decode() (with path + ".bai" when it exists); False: every block
                if ix is False:
                    got = dec.decode_bytes(*_all_blocks(path, ctg), start=start, end=end, fa_fields=fa_fields)
                else:
                    got = dec.decode(path, ctg, start, end, fa_fields=fa_fields)
                n += _same(got, path, ctg, start, end, fa_fields)
    return n


def _all_blocks(path, ctg=None):
    """(bytes after the header, first_uoff, -1, tid of ctg or 0): the decode without an index."""
    refs, vo = bam_io.read_bam_header(path)
    raw = open(path, "rb").read()
    tid = [n for n, _ in refs].index(ctg) if ctg else 0
    return raw[vo >> 16:], vo & 0xFFFF, -1, tid


REGIONS = [(None, None), (0, 10), (1000, 1001), (2500, 9000), (12345, 12346), (20000, 21000), (100000, 200000)]


@pytest.mark.parametrize("read_len,wild", [(150, False), (8000, False), (2000, True)])
def test_random_alignment_matches_read_bam(tmp_path, dec, read_len, wild):
    rec, _, _ = sr.random_alignment(20000, depth=8, read_len=read_len, seed=11, wild=wild)
    path = str(tmp_path / "a.bam")
    bam_io.write_bam(path, rec, [("ctg", 60000)])
    bam_io.write_bai(path)
    assert _check(dec, path, "ctg", REGIONS) > 0


def test_fa_case_with_dwell_names_quals(tmp_path, dec):
    rec, _, _, _ = sr.random_fa_case(5, dwell=True)
    path = str(tmp_path / "fa.bam")
    bam_io.write_bam(path, rec, [("ctg", 10000)])
    bam_io.write_bai(path)
    assert _check(dec, path, "ctg", [(None, None), (1500, 3000), (4000, 4001)]) > 0
    got = dec.decode(path, "ctg", fa_fields=True).host()
    assert (np.diff(got["mv_off"]) == 0).any() and (np.diff(got["mv_off"]) > 0).any()


def _multi_contig(tmp_path, unsorted=False):
    parts, tids = [], []
    for t, seed in ((0, 1), (2, 2), (3, 3)):
        r, _, _ = sr.random_alignment(8000, depth=5, read_len=600, seed=seed)
        parts.append(r)
        tids.append(np.full(len(r["pos"]), t, np.int32))
    r, _, _ = sr.random_alignment(2000, depth=2, read_len=300, seed=4)      # refID -1 records at the end
    parts.append(r)
    tids.append(np.full(len(r["pos"]), -1, np.int32))
    rec = {k: np.concatenate([p[k] for p in parts]) for k in ("pos", "flag", "mapq", "l_qseq", "cigar", "seq")}
    for k, v in (("cigar_off", "cigar"), ("seq_off", "seq")):
        off, acc = [0], 0
        for p in parts:
            off.extend((p[k][1:] + acc).tolist())
            acc += len(p[v])
        rec[k] = np.array(off, np.int64)
    rec["tid"] = np.concatenate(tids)
    if unsorted:
        rng = np.random.default_rng(0)
        perm = rng.permutation(len(rec["pos"]))
        rec = _permute(rec, perm)
    path = str(tmp_path / ("unsorted.bam" if unsorted else "multi.bam"))
    bam_io.write_bam(path, rec, [("c0", 20000), ("none", 100), ("c2", 20000), ("c3", 20000)])
    return path


def _permute(rec, perm):
    out = {k: rec[k][perm] for k in ("pos", "flag", "mapq", "l_qseq", "tid")}
    for k, v in (("cigar_off", "cigar"), ("seq_off", "seq")):
        pieces = [rec[v][rec[k][i]:rec[k][i + 1]] for i in perm]
        out[v] = np.concatenate(pieces)
        out[k] = np.concatenate([[0], np.cumsum([len(x) for x in pieces])]).astype(np.int64)
    return out


def test_contigs_empty_contig_and_unplaced(tmp_path, dec):
    path = _multi_contig(tmp_path)
    bam_io.write_bai(path)
    for ctg in ("c0", "none", "c2", "c3"):
        for start, end in [(None, None), (0, 100), (3000, 5000), (9500, 9600)]:
            for fa_fields in (False, True):
                _same(dec.decode(path, ctg, start, end, fa_fields=fa_fields), path, ctg, start, end, fa_fields)
                data, u0, u1, tid = _all_blocks(path, ctg)
                _same(dec.decode_bytes(data, u0, u1, tid, start, end, fa_fields=fa_fields), path, ctg, start, end, fa_fields)


def test_unsorted_file_stops_where_read_bam_stops(tmp_path, dec):
    path = _multi_contig(tmp_path, unsorted=True)
    for ctg in ("c0", "c2", "c3"):
        for start, end in [(None, None), (0, 4000), (5000, 6000)]:
            data, u0, u1, tid = _all_blocks(path, ctg)
            _same(dec.decode_bytes(data, u0, u1, tid, start, end, fa_fields=True), path, ctg, start, end, True)


# ---- re-compressed blocks ----

def _bgzf(payload, level=6, strategy=zlib.Z_DEFAULT_STRATEGY):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy)
    data = c.compress(payload) + c.flush()
    header = struct.pack("<BBBBIBBHBBHH", 0x1F, 0x8B, 8, 4, 0, 0, 0xFF, 6, 0x42, 0x43, 2, len(data) + 25)
    return header + data + struct.pack("<II", zlib.crc32(payload) & 0xFFFFFFFF, len(payload))


def _stream(path):
    raw = open(path, "rb").read()
    return b"".join(bam_io._inflate_block(raw, o)[1] for o, _, _ in bam_io.bgzf_blocks(raw))


def _reblock(src, dst, cuts=None, step=0xFF00, **kw):
    """Writes the uncompressed stream of src as new BGZF blocks: payload sizes from `cuts` first, then `step` each."""
    s = _stream(src)
    out, o = bytearray(), 0
    for c in list(cuts or []):
        out += _bgzf(s[o:o + c], **kw)
        o += c
    while o < len(s):
        out += _bgzf(s[o:o + step], **kw)
        o += step
    out += bam_io._EOF
    with open(dst, "wb") as f:
        f.write(out)


@pytest.mark.parametrize("kw", [dict(level=0), dict(level=1), dict(level=9), dict(strategy=zlib.Z_FIXED),
                                dict(strategy=zlib.Z_HUFFMAN_ONLY), dict(strategy=zlib.Z_RLE)])
def test_recompressed_blocks(tmp_path, dec, kw):
    rec, _, _, _ = sr.random_fa_case(8, dwell=True, read_len=800, depth=10)
    src, dst = str(tmp_path / "s.bam"), str(tmp_path / "d.bam")
    bam_io.write_bam(src, rec, [("ctg", 10000)])
    _reblock(src, dst, **kw)
    _check(dec, dst, "ctg", [(None, None), (900, 2000)], index=(False,))


def test_block_boundaries(tmp_path, dec):
    """1-byte payloads, a 65,536-byte payload, empty blocks mid-file, a read of over 64 kb (sequence and qualities) spanning
    several blocks, and a block_size field split across two blocks."""
    rec, _, _ = sr.random_alignment(4000, depth=4, read_len=500, seed=21)
    big, _, _ = sr.random_alignment(10, depth=1, read_len=200000, seed=22, indel_rate=0.001)
    k = int(np.argmax(big["l_qseq"]))
    assert big["l_qseq"][k] > 65536
    rec = _insert_read(rec, big, k)
    src = str(tmp_path / "s.bam")
    bam_io.write_bam(src, rec, [("ctg", 500000)])
    s = _stream(src)
    _, hdr = bam_io.read_header(s)
    rec_len = struct.unpack_from("<i", s, hdr)[0] + 4
    cuts = [1, 1, 1, hdr - 3 + 2, 0, 1, 0, 65536, 0, rec_len + 7, 3, 0]         # a cut inside the first record's block_size
    dst = str(tmp_path / "d.bam")
    _reblock(src, dst, cuts=cuts, step=40000)
    blocks = bam_io.bgzf_blocks(open(dst, "rb").read())
    assert 65536 in [b[2] for b in blocks] and 0 in [b[2] for b in blocks[:-1]]
    bam_io.write_bai(dst)
    _check(dec, dst, "ctg", [(None, None), (0, 2000), (3000, 3500)], index=(None, False))


def _insert_read(rec, other, k):
    """rec with read k of `other` placed in position order."""
    p = int(other["pos"][k])
    i = int(np.searchsorted(rec["pos"], p))
    out = {}
    for f in ("pos", "flag", "mapq", "l_qseq"):
        out[f] = np.concatenate([rec[f][:i], other[f][k:k + 1], rec[f][i:]])
    for off, v in (("cigar_off", "cigar"), ("seq_off", "seq")):
        mine = other[v][other[off][k]:other[off][k + 1]]
        out[v] = np.concatenate([rec[v][:rec[off][i]], mine, rec[v][rec[off][i]:]])
        out[off] = np.concatenate([rec[off][:i + 1], rec[off][i:] + len(mine)]).astype(np.int64)
    return out


# ---- auxiliary fields ----

_AUX = [b"XAAz", b"Xcc\x85", b"XCC\xf0", b"Xss" + struct.pack("<h", -300), b"XSS" + struct.pack("<H", 60000),
        b"Xii" + struct.pack("<i", -70000), b"XII" + struct.pack("<I", 4000000000), b"Xff" + struct.pack("<f", 1.5),
        b"XZZhello\x00", b"XHH0AFF\x00", b"XBBf" + struct.pack("<i", 2) + struct.pack("<ff", 1, 2),
        b"XbBS" + struct.pack("<i", 3) + struct.pack("<HHH", 1, 2, 3), b"mvBf" + struct.pack("<i", 1) + struct.pack("<f", 3.0)]
_MV_TYPES = {"c": "<i1", "C": "<u1", "s": "<i2", "S": "<u2", "i": "<i4", "I": "<u4"}


def _aux_bam(path, n=60, seed=0):
    """A BAM whose records carry every SAM aux type before and after an mv B-array of each integer subtype, or no mv."""
    rng = np.random.default_rng(seed)
    text = b"@HD\tVN:1.6\tSO:coordinate\n"
    out = bytearray(b"BAM\x01" + struct.pack("<i", len(text)) + text + struct.pack("<i", 1) + struct.pack("<i", 4) + b"ctg\x00"
                    + struct.pack("<i", 100000))
    for i in range(n):
        l_seq = int(rng.integers(0, 40))
        cig = np.array([l_seq << 4 | 0] if l_seq else [], dtype="<u4")
        nm = b"r%d\x00" % i
        seq = rng.integers(0, 256, (l_seq + 1) // 2, dtype=np.uint8).tobytes()
        qual = rng.integers(0, 60, l_seq, dtype=np.uint8).tobytes()
        before = b"".join(_AUX[j] for j in rng.permutation(len(_AUX))[:int(rng.integers(0, len(_AUX)))])
        after = b"".join(_AUX[j] for j in rng.permutation(len(_AUX))[:int(rng.integers(0, 4))])
        sub = "cCsSiI"[i % 6]
        if i % 7 == 3:
            mv = b""
        else:
            vals = rng.integers(0, 100, int(rng.integers(0, 12)))
            if sub in "cs":
                vals = vals - 50
            mv = b"mvB" + sub.encode() + struct.pack("<i", len(vals)) + vals.astype(_MV_TYPES[sub]).tobytes()
        pos = 100 + 10 * i
        body = bam_io._CORE.pack(0, pos, len(nm), 60, 4681, len(cig), 0, l_seq, -1, -1, 0) + nm + cig.tobytes() + seq + qual + before + mv + after
        out += struct.pack("<i", len(body)) + body
    with open(path, "wb") as f:
        for b0 in range(0, len(out), 997):
            f.write(_bgzf(bytes(out[b0:b0 + 997])))
        f.write(bam_io._EOF)


def test_aux_fields_and_mv_subtypes(tmp_path, dec):
    path = str(tmp_path / "aux.bam")
    _aux_bam(path)
    got = dec.decode(path, "ctg", fa_fields=True).host()
    want, _ = bam_io.read_bam(path, "ctg", fa_fields=True)
    assert (np.diff(want["mv_off"]) == 0).sum() >= 8 and len(want["mv"]) > 50
    _check(dec, path, "ctg", [(None, None), (300, 500)], index=(None, False))


# ---- malformed input ----

def test_malformed_input_is_reported(tmp_path, dec):
    rec, _, _ = sr.random_alignment(3000, depth=30, read_len=400, seed=31)
    path = str(tmp_path / "m.bam")
    bam_io.write_bam(path, rec, [("ctg", 10000)])
    data, u0, u1, tid = _all_blocks(path)
    blocks = bam_io.bgzf_blocks(data)
    assert len(blocks) >= 3
    o, size, _ = blocks[1]

    def expect(buf, pattern, first=u0, end=u1):
        with pytest.raises(C3BError, match=pattern):
            dec.decode_bytes(buf, first, end, tid)
        _same(dec.decode_bytes(data, u0, u1, tid), path, "ctg", None, None, False)      # the workspace stays usable

    bad = bytearray(data)
    bad[o + size - 8] ^= 0x01                                                            # CRC32
    expect(bad, "BGZF block 1 .*CRC32 mismatch")
    bad = bytearray(data)
    struct.pack_into("<I", bad, o + size - 4, struct.unpack_from("<I", bad, o + size - 4)[0] - 1)     # ISIZE
    expect(bad, "BGZF block 1 .*(ISIZE|CRC32)")
    bad = bytearray(data)
    for j in range(40, 48):                                                              # the Huffman stream
        bad[o + 18 + j] ^= 0xA5
    expect(bad, "BGZF block 1 ")
    total = sum(b[2] for b in blocks)
    expect(data, "truncated record", end=total - 30)
    with pytest.raises(C3BError, match="not a BGZF block"):
        dec.decode_bytes(b"\x1f\x8b\x08\x00" + data[4:], u0, u1, tid)


# ---- end to end: file -> call records ----

def test_file_to_call_records(tmp_path, dec):
    rec, ref, rs = sr.random_alignment(6000, depth=20, read_len=3000, seed=41, origin=4000)
    path = str(tmp_path / "e.bam")
    bam_io.write_bam(path, rec, [("ctg", 40000)])
    bam_io.write_bai(path)
    start, end = 4000, 10000
    host, _ = bam_io.read_bam(path, "ctg", start, end)
    devrec = dec.decode(path, "ctg", start, end, ref_seq=ref)
    dev = torch.device("cuda:0")
    model = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    model.to(dev)
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()})
    cfg = decode.replay_config(pileup=True, add_indel_length=False)
    ctr = PileupCounter(0)
    a = ctr.count(host, start, end, ref, rs, alt_info=True)
    ma = a.fetch()
    ta = a.alt_text().alt_text_fetch()["text"]
    ra = a.call(model, cfg, "ctg")
    b = ctr.count(devrec, start, end, None, rs, alt_info=True)
    mb = b.fetch()
    tb = b.alt_text().alt_text_fetch()["text"]
    rb = b.call(model, cfg, "ctg")
    for k in ma:
        assert np.array_equal(ma[k], mb[k]), k
    assert ta == tb and len(ta) > 0
    assert np.array_equal(ra["calls"], rb["calls"]) and decode.calls_text(ra, cfg) == decode.calls_text(rb, cfg)
    ctr.close()

    frec, fref, cand, var = sr.random_fa_case(6, dwell=True)
    fpath = str(tmp_path / "f.bam")
    bam_io.write_bam(fpath, frec, [("ctg", len(fref))])
    fhost, _ = bam_io.read_bam(fpath, "ctg", fa_fields=True)
    fdev = dec.decode(fpath, "ctg", fa_fields=True, ref_seq=fref)
    fm = Clair3_F(add_indel_length=True, predict=True, input_channels=9)
    fm.to(dev)
    fm.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=9, seed=1).items()})
    fcfg = decode.replay_config(pileup=False, add_indel_length=True)._replace(quality_score_for_pass=None)
    bld = FullAlignmentBuilder(0)
    x = bld.build(fhost, cand, fref, 0, variants=var, dwell=True)
    mx, kx = x.fetch(), x.kept_reads()
    rx = x.call(fm, fcfg, "ctg")
    y = bld.build(fdev, cand, None, 0, variants=var, dwell=True)
    my, ky = y.fetch(), y.kept_reads()
    ry = y.call(fm, fcfg, "ctg")
    assert np.array_equal(mx, my) and all(np.array_equal(p, q) for p, q in zip(kx, ky))
    assert np.array_equal(rx["calls"], ry["calls"]) and decode.calls_text(rx, fcfg) == decode.calls_text(ry, fcfg)
    bld.close()


def test_decoded_tensors_survive_later_decodes(tmp_path, dec):
    rec, _, _ = sr.random_alignment(3000, depth=6, read_len=400, seed=51)
    path = str(tmp_path / "k.bam")
    bam_io.write_bam(path, rec, [("ctg", 10000)])
    first = dec.decode(path, "ctg", 0, 2000)
    dec.decode(path, "ctg", 1500, 4000, fa_fields=True)
    _same(first, path, "ctg", 0, 2000, False)
    ms, launches = dec.last_ms()
    assert ms > 0 and launches == 14
