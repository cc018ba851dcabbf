"""The GPU BGZF writer (``c3b_bgzf_compress``) where real files take it: texts of more blocks than the grid has CTAs, so a CTA
of ``bgzf_deflate_kernel`` compresses a second, third, ... block on the window, head, prev, trees and symbol-buffer slot the
block before left it, with only ``reset_block`` between.  Every block must still be exactly zlib level 6's
(``bam_io._bgzf_block``, ``bam_io.write_bgzf``): at block counts around multiples of the grid and past the size scan's
1,024-entry step, with every corpus payload placed on a CTA that has just compressed a full block, across a workspace history
that mixes in FASTA fetches and BAM decodes, from device sources on another stream and at a storage offset, and for a VCF
over chr1-length contigs whose ``.tbi`` must find every row."""
import gzip
import os
import sys
import zlib

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import bgzf_corpus as bc  # noqa: E402
import bgzf_fasta as bf  # noqa: E402
from clair3_b200 import bam_io, genome  # noqa: E402
from clair3_b200 import synth_reads as sr  # noqa: E402
from clair3_b200.bam_decode import BamDecoder  # noqa: E402

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(zlib.ZLIB_RUNTIME_VERSION != bc.ZLIB_VERSION,
                                 reason="byte equality is held to zlib %s; this Python links zlib %s"
                                 % (bc.ZLIB_VERSION, zlib.ZLIB_RUNTIME_VERSION))]
DEV = torch.device("cuda:0")
P = bc.PAYLOAD
SCAN_STEP = 1024                        # block_scan_kernel's step: the size scan carries between steps past this many blocks


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid(nb):
    """c3b_bgzf_compress's launch: min(nb, SMs) CTAs of bgzf_deflate_kernel, and CTA c compresses blocks c, c + grid,
    c + 2 grid, ...: block b runs on CTA b % grid(nb) as its (b // grid(nb) + 1)-th block."""
    return min(nb, sms())


KINDS = ("random", "runs", "VCF rows", "Fibonacci counts")


def kind_of(b, nb):
    """Block b's kind: consecutive blocks of one CTA, and neighbouring blocks of one round, differ in kind."""
    g = grid(nb)
    return (b // g + b % g) % len(KINDS)


class Maker:
    """Payloads of each kind: random bytes (stored blocks), long runs of one byte (long match chains; a full block slides the
    window), VCF rows, and bytes with Fibonacci symbol counts (gen_bitlen's overflow repair)."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.vcf = bc.vcf_text(30000, seed).encode()

    def payload(self, kind, n):
        rng = self.rng
        if kind == 0:
            return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        if kind == 1:
            out, have = [], 0
            while have < n:
                k = int(rng.integers(300, 20000))
                out.append(bytes([int(rng.integers(0, 256))]) * k)
                have += k
            return b"".join(out)[:n]
        if kind == 2:
            o = int(rng.integers(0, len(self.vcf) - n))
            return self.vcf[o:o + n]
        return bc._fib_text(rng, n)

    def text(self, nb, last):
        """nb blocks, each of kind_of(b, nb), the last one ``last`` bytes long."""
        return b"".join(self.payload(kind_of(b, nb), P if b < nb - 1 else last) for b in range(nb))


def host_file(tmp_path, data, name="host.gz"):
    """bam_io.write_bgzf's file of ``data``: (bytes, voffset, its blocks' offsets before the EOF block)."""
    path = str(tmp_path / name)
    voff = bam_io.write_bgzf(path, data)
    with open(path, "rb") as f:
        raw = f.read()
    return raw, voff, [o for o, _, _ in bam_io.bgzf_blocks(raw)][:-1]


def check_text(dec, tmp_path, t, host=None):
    """The device writer against the host writer on text t: each block of the image against bam_io._bgzf_block of its
    payload as write_bgzf wrote it (naming its CTA, round and kind on a mismatch), the offsets, the whole file, the voffset
    of every row start, and the file inflated by gzip and by the decoder's own inflater."""
    nb = -(-len(t) // P)
    raw, voff_h, hoff = host or host_file(tmp_path, t)
    image, off = dec.compress_bgzf(t)
    assert len(off) == nb + 1 and off[-1] == len(image)
    for b in range(nb):
        assert image[off[b]:off[b + 1]] == raw[hoff[b]:hoff[b + 1] if b + 1 < nb else len(raw) - len(bam_io._EOF)], \
            ("block", b, "of", nb, "CTA", b % grid(nb), "round", b // grid(nb), KINDS[kind_of(b, nb)])
    assert off[:-1] == hoff
    assert image + bam_io._EOF == raw
    path = str(tmp_path / "dev.gz")
    voff_d = dec.write_bgzf(path, t)
    with open(path, "rb") as f:
        got = f.read()
    assert got == raw
    assert gzip.decompress(got) == t
    back = dec.fetch_fasta_bytes(image, 0, 0, len(t), len(t), len(t))
    assert torch.equal(back, torch.frombuffer(bytearray(t), dtype=torch.uint8).to(DEV))
    del back
    starts = np.concatenate([[0], np.flatnonzero(np.frombuffer(t, np.uint8) == 10) + 1, [len(t)]]).tolist()
    assert [voff_d(u) for u in starts] == [voff_h(u) for u in starts]


@pytest.fixture(scope="module")
def dec():
    d = BamDecoder(0)
    yield d
    d.close()


@pytest.fixture(scope="module")
def big(tmp_path_factory):
    """A text of more than SCAN_STEP blocks (over 66.9 MB) and its host file."""
    nb = SCAN_STEP + sms() + 5
    t = Maker(101).text(nb, 4321)
    assert nb > SCAN_STEP and len(t) > SCAN_STEP * P
    return t, host_file(tmp_path_factory.mktemp("big"), t)


# ---------------------------------------------------------------------------------------------- 1. block counts around the grid
@pytest.mark.parametrize("extra", ["S-1", "S", "S+1", "2S+1", "3S+7"])
def test_block_counts_around_the_grid(dec, tmp_path, extra):
    s = sms()
    nb = {"S-1": s - 1, "S": s, "S+1": s + 1, "2S+1": 2 * s + 1, "3S+7": 3 * s + 7}[extra]
    t = Maker(nb).text(nb, 1 + nb * 7919 % (P - 1))
    check_text(dec, tmp_path, t)


def test_more_blocks_than_the_size_scan_step(dec, tmp_path, big):
    t, host = big
    check_text(dec, tmp_path, t, host)


# ---------------------------------------------------------------------------------------------- 2. the corpus on a reused CTA
@pytest.fixture(scope="module")
def prefix():
    """2S - 1 full blocks of every kind in turn, compressed once on the host: the shared start of the calls below.  (payloads,
    their host blocks, the blocks' offsets, the payloads joined)"""
    s = sms()
    m = Maker(202)
    blocks = [m.payload(b % len(KINDS), P) for b in range(2 * s - 1)]
    want = [bam_io._bgzf_block(p) for p in blocks]
    return blocks, want, np.concatenate([[0], np.cumsum([len(w) for w in want])]).tolist(), b"".join(blocks)


def mixtures(seed, count, keep):
    """``count`` seeded corpus mixtures whose lengths ``keep`` accepts."""
    rng = np.random.default_rng(seed)
    text = bc.vcf_text(3000, seed).encode()
    out = []
    while len(out) < count:
        m = bc.mixture(rng, text)
        if keep(len(m)):
            out.append(m)
    return out


def test_full_corpus_payloads_on_reused_ctas(dec, prefix):
    """Every full-size corpus payload and 300 full-size mixtures at block indices >= S: each on a CTA's second or later block,
    after whatever the block before it on that CTA was."""
    s = sms()
    pre, pre_want, _, _ = prefix
    full = [p for _, p in bc.payloads(6) if len(p) == P] + mixtures(303, 300, lambda n: n == P)
    nb = s + len(full)
    image, off = dec.compress_bgzf(b"".join(pre[:s] + full))
    assert len(off) == nb + 1
    for b in range(nb):
        want = pre_want[b] if b < s else bam_io._bgzf_block(full[b - s])
        assert image[off[b]:off[b + 1]] == want, ("block", b, "CTA", b % s, "round", b // s)


def test_short_corpus_payloads_after_a_full_block(dec, prefix):
    """Every short corpus payload and 200 short mixtures as the last block of a call of S + j blocks: it lands on CTA j - 1
    as that CTA's second block, right after the full prefix block j - 1 (j cycles so every kind comes before)."""
    s = sms()
    _, pre_want, pre_off, pre_text = prefix
    pre_image = b"".join(pre_want)
    short = [p for _, p in bc.payloads(7) if 0 < len(p) < P] + mixtures(404, 200, lambda n: 0 < n < P)
    for i, p in enumerate(short):
        j = 1 + (37 * i) % s
        nb = s + j
        assert grid(nb) == s and (nb - 1) % grid(nb) == j - 1
        image, off = dec.compress_bgzf(pre_text[:(nb - 1) * P] + p)
        assert off[:-1] == pre_off[:nb] and image[:off[-2]] == pre_image[:pre_off[nb - 1]], (i, j)
        assert image[off[-2]:] == bam_io._bgzf_block(p), (i, len(p), "CTA", j - 1, "after a", KINDS[(j - 1) % len(KINDS)])


# ---------------------------------------------------------------------------------------------- 3. workspace history
@pytest.fixture(scope="module")
def reads(tmp_path_factory):
    """A bgzip-compressed FASTA (with .fai and .gzi) and a small indexed BAM for the fetches and decodes between writes."""
    d = tmp_path_factory.mktemp("reads")
    rng = np.random.default_rng(505)
    seqs = [("s1", bf.random_sequence(300000, rng)), ("s2", bf.random_sequence(70000, rng))]
    plain = bf.write_fasta(str(d / "ref.fa"), seqs)
    gz = str(d / "ref.fa.gz")
    bf.bgzip(plain, gz)
    rec, _, _ = sr.random_alignment(20000, depth=8, read_len=800, seed=505)
    bam = str(d / "a.bam")
    bam_io.write_bam(bam, rec, [("ctg", 60000)])
    bam_io.write_bai(bam)
    return gz, dict(seqs), bam


def _fetch_and_decode(d, reads, a, b):
    """As genome._read_span queues them: the FASTA window without a wait, the decode on the same stream, then the status."""
    gz, seqs, bam = reads
    ref = d.fetch_fasta(gz, "s1", a, b, wait=False)
    got = d.decode(bam, "ctg", 1000 + a // 50, 9000 + a // 50, fa_fields=True, ref_seq=ref)
    d.fasta_status()
    assert ref.cpu().numpy().tobytes().decode() == seqs["s1"][a:b]
    want, _ = bam_io.read_bam(bam, "ctg", 1000 + a // 50, 9000 + a // 50, fa_fields=True)
    h = got.host()
    assert len(want["pos"]) > 0
    for k in want:
        if k != "tid":
            assert np.array_equal(h[k], want[k]), k


def test_workspace_history(tmp_path, big, reads):
    s = sms()
    d = BamDecoder(0)
    try:
        m = Maker(606)
        t, host = big
        check_text(d, tmp_path, t, host)
        _fetch_and_decode(d, reads, 12345, 212345)
        check_text(d, tmp_path, m.text(1, 777))
        assert d.compress_bgzf(b"") == (b"", [0])
        _fetch_and_decode(d, reads, 100, 50000)
        check_text(d, tmp_path, m.text(s + 1, P))
        _fetch_and_decode(d, reads, 250000, 300000)
        assert d.compress_bgzf(b"") == (b"", [0])
        check_text(d, tmp_path, m.text(s - 1, 1))
    finally:
        d.close()


# ---------------------------------------------------------------------------------------------- 4. device sources
def test_tensor_made_on_another_stream(dec):
    """A uint8 tensor built by torch ops on a non-default stream, compressed while that stream is current: the kernels queue
    behind the ops that wrote it."""
    s = sms()
    n = (s + 3) * P + 999
    st = torch.cuda.Stream(DEV)
    g = torch.Generator(device=DEV).manual_seed(707)
    with torch.cuda.stream(st):
        runs = torch.randint(0, 256, ((n >> 9) + 1,), generator=g, device=DEV, dtype=torch.uint8).repeat_interleave(512)[:n]
        noise = torch.randint(0, 256, (n,), generator=g, device=DEV, dtype=torch.uint8)
        keep = torch.arange(n, device=DEV) % (3 * P) < 2 * P            # runs for two blocks, noise for one
        t = torch.where(keep, runs, noise)
        image, off = dec.compress_bgzf(t)
    st.synchronize()
    assert (image, off) == dec.compress_bgzf(t.cpu().numpy().tobytes())


def test_view_at_a_storage_offset(dec):
    s = sms()
    base = torch.frombuffer(bytearray(Maker(808).text(s + 4, P)), dtype=torch.uint8).to(DEV)
    v = base[12345:12345 + (s + 1) * P + 2 * 4321 + 1]
    assert v.storage_offset() == 12345 and v.numel() % 2 == 1
    assert dec.compress_bgzf(v) == dec.compress_bgzf(v.cpu().numpy().tobytes())


# ---------------------------------------------------------------------------------------------- 5. whole-genome coordinates
CHR1 = 248_956_422


def test_chr1_length_vcf_and_its_index(dec, tmp_path):
    """A VCF of more than SCAN_STEP blocks over three contigs as long as chr1, rows up to their ends: genome.write_vcf_gz on
    the device and on the host give the same .vcf.gz and .tbi, and the index finds exactly the rows that overlap random
    windows past 2^26."""
    rng = np.random.default_rng(909)
    contigs = ("chr1", "chr2", "chrX")
    rows, pos_all = [], []
    for ctg in contigs:
        ref_len = rng.choice([1, 2, 7, 40, 20000], 450000, p=[0.6, 0.2, 0.15, 0.0498, 0.0002])
        pos = rng.integers(1, CHR1 - ref_len + 2)
        ref_len[:2] = 20000, 1                                          # rows that end at the contig's last base
        pos[:2] = CHR1 - 20000 + 1, CHR1
        order = np.argsort(pos, kind="stable")
        pos, ref_len = pos[order], ref_len[order]
        gq = rng.integers(0, 99, len(pos))
        for p, r, q in zip(pos.tolist(), ref_len.tolist(), gq.tolist()):
            rows.append("%s\t%d\t.\t%s\tA\t%d.5\tPASS\tP\tGT:GQ\t0/1:%d\n" % (ctg, p, "ACGT"[p & 3] * r, q, q))
        pos_all.append((ctg, pos, ref_len))
    head = "".join("##contig=<ID=%s,length=%d>\n" % (c, CHR1) for c in contigs)
    text = "##fileformat=VCFv4.2\n" + head + "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tS\n" + "".join(rows)
    assert len(text) > SCAN_STEP * P
    dev_p, host_p = str(tmp_path / "dev.vcf.gz"), str(tmp_path / "host.vcf.gz")
    genome.write_vcf_gz(dev_p, text, decoder=dec)
    genome.write_vcf_gz(host_p, text)
    for suffix in ("", ".tbi"):
        with open(dev_p + suffix, "rb") as f1, open(host_p + suffix, "rb") as f2:
            assert f1.read() == f2.read(), suffix
    tbi = bam_io.read_tbi(dev_p + ".tbi")
    assert tbi["names"] == list(contigs) and [r["mapped"] for r in tbi["refs"]] == [len(p) for _, p, _ in pos_all]
    with open(dev_p, "rb") as f:
        raw = f.read()
    data = gzip.decompress(raw).decode()
    assert data == text
    starts, u = {}, 0
    for o, _, isize in bam_io.bgzf_blocks(raw):
        starts[o] = u
        u += isize
    uoff = lambda v: starts[v >> 16] + (v & 0xFFFF)  # noqa: E731
    for i in range(300):
        ctg, pos, ref_len = pos_all[i % len(contigs)]
        a = int(rng.integers(1 << 26, CHR1))
        b = min(a + int(rng.integers(1, 200000)), CHR1) if i % 10 else CHR1
        sel = (pos - 1 < b) & (pos - 1 + ref_len > a)
        want = {(int(p), int(r)) for p, r in zip(pos[sel], ref_len[sel])}
        got = set()
        for c0, c1 in bam_io.tbi_chunks(tbi, ctg, a, b):
            for row in data[uoff(c0):uoff(c1)].splitlines():
                c = row.split("\t")
                if row[0] != "#" and c[0] == ctg and int(c[1]) - 1 < b and int(c[1]) - 1 + len(c[3]) > a:
                    got.add((int(c[1]), len(c[3])))
        assert got == want, (ctg, a, b)
