"""The BGZF writer on the GPU (``c3b_bgzf_compress`` through ``BamDecoder.compress_bgzf`` / ``write_bgzf``) against the host
writer ``bam_io.write_bgzf``, which is zlib level 6: equal bytes on the corpus of ``bgzf_corpus`` from host and device
sources; the files inflate through zlib and through the decoder's own inflater; the same ``voffset`` at every row start; and
``genome.call_genome``'s ``.vcf.gz`` and ``.tbi`` files, now compressed on the device, byte-identical to what the host writer
makes of the same texts."""
import gzip
import os
import sys
import zlib

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import bgzf_corpus as bc  # noqa: E402
from clair3_b200 import bam_io, genome  # noqa: E402
from clair3_b200._ffi import C3BError  # noqa: E402
from clair3_b200.bam_decode import BamDecoder  # noqa: E402

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(zlib.ZLIB_RUNTIME_VERSION != bc.ZLIB_VERSION,
                                 reason="byte equality is held to zlib %s; this Python links zlib %s"
                                 % (bc.ZLIB_VERSION, zlib.ZLIB_RUNTIME_VERSION))]
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def dec():
    d = BamDecoder(0)
    yield d
    d.close()


def _host_file(tmp_path, data):
    path = str(tmp_path / "host.gz")
    voff = bam_io.write_bgzf(path, data)
    with open(path, "rb") as f:
        return f.read(), voff


def test_blocks_equal_the_host_writer(dec):
    """Every payload of the corpus and 400 seeded mixtures as one block each, from host bytes and from a device tensor."""
    for name, p in bc.payloads(2, mixtures=400):
        want = bam_io._bgzf_block(p) if p else b""
        image, off = dec.compress_bgzf(p)
        assert image == want, (name, len(p))
        assert off == ([0, len(want)] if p else [0])
        d_image, d_off = dec.compress_bgzf(torch.frombuffer(bytearray(p), dtype=torch.uint8).to(DEV) if p
                                           else torch.empty(0, dtype=torch.uint8, device=DEV))
        assert (d_image, d_off) == (image, off), name


def test_files_equal_inflate_and_index_alike(dec, tmp_path):
    """Multi-block texts: the same file bytes and voffset at every row start as the host writer; the file inflates through
    zlib and, block by block, through the decoder's own inflater (c3b_fasta_fetch with one line as long as the text)."""
    for name, t in bc.texts(4):
        want, voff_h = _host_file(tmp_path, t)
        path = str(tmp_path / "dev.gz")
        voff_d = dec.write_bgzf(path, t)
        with open(path, "rb") as f:
            got = f.read()
        assert got == want, name
        assert gzip.decompress(got) == t
        if t:
            body = got[:-len(bam_io._EOF)]
            back = dec.fetch_fasta_bytes(body, 0, 0, len(t), len(t), len(t))
            assert bytes(back.cpu().numpy()) == t, name
        starts = [0] + [i + 1 for i, c in enumerate(t) if c == 10] + [len(t)]
        assert [voff_d(u) for u in starts] == [voff_h(u) for u in starts], name


def test_device_source_of_many_blocks(dec):
    t = bc.vcf_text(20000, 9).encode()
    host, off = dec.compress_bgzf(t)
    dev, d_off = dec.compress_bgzf(torch.frombuffer(bytearray(t), dtype=torch.uint8).to(DEV))
    assert dev == host and d_off == off and len(off) == -(-len(t) // bc.PAYLOAD) + 1
    with pytest.raises(C3BError):
        dec.compress_bgzf(torch.zeros(4, dtype=torch.int32, device=DEV))


@pytest.fixture(scope="module")
def genome_setup(tmp_path_factory):
    import test_gpu_genome as tg
    from clair3_b200 import cascade
    d = str(tmp_path_factory.mktemp("genome"))
    ws = cascade.Workspaces(0)
    yield tg, tg.make_genome(d), tg._models(), ws
    ws.close()


@pytest.mark.parametrize("case", ["plain", "bed", "long_indel"])
def test_call_genome_files_equal_the_host_writer(genome_setup, case, tmp_path):
    """call_genome's pileup, full_alignment and merge_output .vcf.gz and .tbi files against bam_io.write_bgzf / write_tbi
    of the texts it returns, byte for byte, in the plain, BED and --enable_long_indel cases."""
    tg, (bam, fa, seqs), (m_p, m_f), ws = genome_setup
    kw = tg._call_kw({"long_indel": True} if case == "long_indel" else {})
    if case == "bed":
        kw["bed_fn"] = tg._targets("bed", seqs)
    out = str(tmp_path / "dev")
    res = genome.call_genome(bam, fa, m_p, m_f, out, cmdline="run --x", include_all_ctgs=True, min_contig_size=tg.MIN_SIZE,
                             chunk_size=tg.CHUNK, split_bed_size=tg.SPLIT, workspaces=ws, **kw)
    assert "compress" in res["stages"] and "write" in res["stages"]
    assert {"pileup", "merge_output"} <= set(res["texts"])
    if case != "bed":
        assert "full_alignment" in res["texts"]
    host = tmp_path / "host"
    host.mkdir()
    for n, t in res["texts"].items():
        hp = str(host / (n + ".vcf.gz"))
        genome.write_vcf_gz(hp, t)
        for suffix in ("", ".tbi"):
            with open(os.path.join(out, n + ".vcf.gz" + suffix), "rb") as f:
                got = f.read()
            with open(hp + suffix, "rb") as f:
                want = f.read()
            assert got == want, (case, n, suffix)
