"""A bgzip-compressed reference FASTA on the host (clair3_b200/bam_io.py): the ``.gzi`` reader against a writer kept here, the
``.fai`` + ``.gzi`` fetch against ``read_fasta`` over the whole decompressed file, the refusals, the genome route's input
checks, and ``--keep_iupac_bases`` reaching both output configs."""
import gzip
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bgzf_fasta as bf  # noqa: E402
from clair3_b200 import bam_io, genome, run_clair3  # noqa: E402


def test_read_gzi_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    for n in (0, 1, 7, 300):
        c = np.cumsum(rng.integers(28, 70000, n))
        u = np.cumsum(rng.integers(0, 65537, n))
        starts = [(0, 0)] + list(zip(c.tolist(), u.tolist()))
        p = bf.write_gzi(str(tmp_path / ("r%d.gzi" % n)), starts)
        got = bam_io.read_gzi(p)
        assert got.dtype == np.int64 and got.shape == (n, 2)
        assert got.tolist() == [list(x) for x in starts[1:]]


def test_read_gzi_refuses_malformed(tmp_path):
    good = bf.write_gzi(str(tmp_path / "g.gzi"), [(0, 0), (100, 65280), (200, 130560)])
    raw = open(good, "rb").read()
    cases = {"empty": b"", "short count": raw[:5], "truncated": raw[:-3], "extra bytes": raw + b"\0",
             "count too large": struct.pack("<Q", 3) + raw[8:],
             "descending compressed": struct.pack("<QQQQQ", 2, 200, 65280, 100, 130560),
             "descending uncompressed": struct.pack("<QQQQQ", 2, 100, 130560, 200, 65280),
             "repeated compressed": struct.pack("<QQQQQ", 2, 100, 65280, 100, 130560)}
    for name, buf in cases.items():
        p = tmp_path / "bad.gzi"
        p.write_bytes(buf)
        with pytest.raises(ValueError, match="gzi"):
            bam_io.read_gzi(str(p))


@pytest.mark.parametrize("case", bf.CASES, ids=[c[0] for c in bf.CASES])
def test_fetch_matches_read_fasta(tmp_path, case):
    plain, gz, starts, seqs = bf.make_case(str(tmp_path), case)
    assert bam_io.is_bgzf(gz) and not bam_io.is_bgzf(plain)
    assert gzip.open(gz, "rb").read() == open(plain, "rb").read()
    if case[3] is not None:
        assert len(starts) > 3
    rng = np.random.default_rng(len(case[0]))
    rows = {r[0]: r for r in bam_io.read_fai(gz + ".fai")}
    n = 0
    for name, seq in seqs:
        for a, b in bf.windows(rows[name], starts, rng):
            want = bam_io.read_fasta(gz, name, a, b) if b >= a else ""
            assert want == seq[a:b]
            assert bam_io.fetch_fasta(gz, name, a, b) == want, (name, a, b)
            assert bam_io.fetch_fasta(plain, name, a, b) == want
            n += 1
    assert n > 50


def test_fasta_span_covers_the_window(tmp_path):
    """The compressed range holds whole blocks from the one that holds the window's first byte to the one that holds its last."""
    plain, gz, starts, seqs = bf.make_case(str(tmp_path), bf.CASES[0])
    gzi = bam_io.read_gzi(gz + ".gzi")
    raw = open(gz, "rb").read()
    blocks = bam_io.bgzf_blocks(raw)
    ustart = np.cumsum([0] + [b[2] for b in blocks])
    for row in bam_io.read_fai(gz + ".fai"):
        for s, e in ((0, 1), (0, row[1]), (row[1] // 2, row[1] // 2 + 300)):
            a, b, c0, c1, u0 = bam_io.fasta_span(row, s, min(e, row[1]), gzi)
            first = [i for i, blk in enumerate(blocks) if blk[0] == c0][0]
            assert ustart[first] <= a < ustart[first + 1] and u0 == a - ustart[first]
            if c1 is None:                                          # to the end of the file: the last block with data
                last = max(i for i, blk in enumerate(blocks) if blk[2])
            else:
                last = [i for i, blk in enumerate(blocks) if blk[0] == c1][0] - 1
            assert ustart[last] < b <= ustart[last + 1]


def test_refusals(tmp_path):
    plain, gz, _, _ = bf.make_case(str(tmp_path), bf.CASES[0])
    name = bam_io.read_fai(plain + ".fai")[0][0]
    # plain gzip (no BGZF extra field): refused as samtools faidx refuses it
    pg = tmp_path / "plain.fa.gz"
    pg.write_bytes(gzip.compress(open(plain, "rb").read()))
    (tmp_path / "plain.fa.gz.fai").write_text(open(plain + ".fai").read())
    assert not bam_io.is_bgzf(str(pg))
    with pytest.raises(ValueError, match="compressed FASTA"):
        bam_io.fetch_fasta(str(pg), name, 0, 10)
    # a missing .gzi
    os.rename(gz + ".gzi", gz + ".gzi.away")
    with pytest.raises(FileNotFoundError, match="samtools faidx"):
        bam_io.fetch_fasta(gz, name, 0, 10)
    assert bam_io.fetch_fasta(gz, name, 0, 10, gzi=gz + ".gzi.away") == bam_io.fetch_fasta(plain, name, 0, 10)
    # a corrupt .gzi
    (tmp_path / (os.path.basename(gz) + ".gzi")).write_bytes(b"\x05" + bytes(10))
    with pytest.raises(ValueError, match="gzi"):
        bam_io.fetch_fasta(gz, name, 0, 10)


def _genome_inputs(tmp_path):
    seqs = bf.sequences(9, 3, 2000, 6000)
    seqs = [("chr%d" % (i + 1), s) for i, (_, s) in enumerate(seqs)]
    plain = bf.write_fasta(str(tmp_path / "ref.fa"), seqs)
    gz = plain + ".gz"
    bf.bgzip(plain, gz, cuts=[1000, 5000])
    for p in ("in.bam", "in.bam.bai"):
        (tmp_path / p).write_bytes(b"")
    return plain, gz, str(tmp_path / "in.bam"), seqs


def test_check_inputs_and_plan_accept_bgzf(tmp_path):
    plain, gz, bam, seqs = _genome_inputs(tmp_path)
    assert genome.check_inputs(bam, gz) == bam + ".bai"
    stats = [(n, len(s), 1, 0) for n, s in seqs]
    assert genome.plan(bam, gz, chunk_size=2500, idxstats=stats) == genome.plan(bam, plain, chunk_size=2500, idxstats=stats)
    head = genome.header(gz)
    assert "##reference=%s\n" % gz in head and head.replace(gz, plain) == genome.header(plain)
    os.remove(gz + ".gzi")
    with pytest.raises(FileNotFoundError, match="gzi"):
        genome.check_inputs(bam, gz)
    pg = tmp_path / "p.fa.gz"
    pg.write_bytes(gzip.compress(open(plain, "rb").read()))
    (tmp_path / "p.fa.gz.fai").write_text(open(plain + ".fai").read())
    with pytest.raises(ValueError, match="compressed FASTA"):
        genome.check_inputs(bam, str(pg))


def test_keep_iupac_bases_option():
    args = run_clair3.parser().parse_args(["--bam_fn", "b", "--ref_fn", "r", "--model_path", "m", "--platform", "ont",
                                           "--output", "o"])
    assert args.keep_iupac_bases is False
    for extra, want in ((["--keep_iupac_bases"], True), (["--keep_iupac_bases", "True"], True),
                        (["--keep_iupac_bases", "False"], False)):
        args = run_clair3.parser().parse_args(["--bam_fn", "b", "--ref_fn", "r", "--model_path", "m", "--platform", "ont",
                                               "--output", "o"] + extra)
        assert args.keep_iupac_bases is want
    for long_indel in (False, True):
        on = genome.output_configs(long_indel, keep_iupac_bases=True)
        off = genome.output_configs(long_indel)
        assert [c.keep_iupac_bases for c in on] == [True, True] and [c.keep_iupac_bases for c in off] == [False, False]
        assert [c._replace(keep_iupac_bases=False) for c in on] == list(off)
