"""A bgzip-compressed reference FASTA on the GPU: ``BamDecoder.fetch_fasta`` against the host's ``bam_io.fetch_fasta`` on the
cases of tests/test_fasta_bgzf_cpu.py and one 5,002,001-base window (a default chunk plus ``FETCH_EXPAND`` either side);
corrupt blocks reported by number and reason; and the genome route (``genome.call_genome`` and the CLI) on a seeded genome
with the FASTA bgzipped, against the same run on the plain FASTA.  ``--keep_iupac_bases`` on a reference with IUPAC codes at
candidate sites against the host route's rows."""
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bam_craft as bc  # noqa: E402
import bgzf_fasta as bf  # noqa: E402
import deflate_craft as dc  # noqa: E402
from clair3_b200 import bam_io, cascade, decode, genome, synth, synth_reads as sr, targets  # noqa: E402
from clair3_b200._ffi import C3BError  # noqa: E402
from clair3_b200.bam_decode import BamDecoder  # noqa: E402
from clair3_b200.model import Clair3_F, Clair3_P  # noqa: E402
from clair3_b200.pileup_counts import FETCH_EXPAND  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def dec():
    d = BamDecoder(0)
    yield d
    d.close()


def _host(t):
    return t.cpu().numpy().tobytes().decode()


# ---------------------------------------------------------------------------------------------- the window's bytes
@pytest.mark.parametrize("case", bf.CASES, ids=[c[0] for c in bf.CASES])
def test_fetch_matches_host(tmp_path, dec, case):
    plain, gz, starts, seqs = bf.make_case(str(tmp_path), case)
    rng = np.random.default_rng(len(case[0]))
    rows = {r[0]: r for r in bam_io.read_fai(gz + ".fai")}
    n = 0
    for name, seq in seqs:
        for a, b in bf.windows(rows[name], starts, rng):
            got = dec.fetch_fasta(gz, name, a, b)
            assert got.device == DEV and got.dtype == torch.uint8
            assert _host(got) == bam_io.fetch_fasta(gz, name, a, b) == seq[a:b], (name, a, b)
            n += 1
    assert n > 50


def test_chunk_window(tmp_path, dec):
    n = 5_000_000 + 2 * FETCH_EXPAND + 1
    assert n == 5_002_001
    rng = np.random.default_rng(3)
    seqs = [("chrA", bf.random_sequence(3001, rng)), ("chrB", bf.random_sequence(n + 4321, rng))]
    plain = bf.write_fasta(str(tmp_path / "big.fa"), seqs, width=60)
    gz = plain + ".gz"
    starts = bf.bgzip(plain, gz)
    assert len(starts) > 70
    for a in (0, 1234, 4321):
        got = dec.fetch_fasta(gz, "chrB", a, a + n)
        ms, launches = dec.last_ms()
        assert got.numel() == n and launches == 2 and ms > 0
        assert _host(got) == bam_io.fetch_fasta(gz, "chrB", a, a + n) == seqs[1][1][a:a + n]


def test_corrupt_blocks_raise(tmp_path, dec):
    plain, gz, starts, seqs = bf.make_case(str(tmp_path), bf.CASES[0])
    data = open(plain, "rb").read()
    name, seq = seqs[1]
    row = {r[0]: r for r in bam_io.read_fai(plain + ".fai")}[name]
    payload_cut = [u for _, u in starts]
    k = int(np.searchsorted(payload_cut, row[2] + 200, side="right")) - 1    # the block holding the sequence's 200th byte

    def rewrite(encode):
        out, at = str(tmp_path / "bad.fa.gz"), []
        with open(out, "wb") as f:
            for i, (a, b) in enumerate(zip(payload_cut, payload_cut[1:] + [len(data)])):
                at.append((f.tell(), a))
                f.write(encode(data[a:b]) if i == k else bc.bgzf(data[a:b]))
            f.write(bam_io._EOF)
        bf.write_gzi(out + ".gzi", at)
        with open(plain + ".fai", "rb") as src, open(out + ".fai", "wb") as dst:
            dst.write(src.read())
        return out

    bad_crc = lambda p: bc.bgzf(p)[:-8] + bytes(4) + bc.bgzf(p)[-4:]                                # noqa: E731
    good = bc.bgzf(data[payload_cut[k]:payload_cut[k + 1]])
    stored = dc.encode_mode(data[payload_cut[k]:payload_cut[k + 1]], "stored")
    bad_len = lambda p: bc.bgzf(p, stored[:3] + bytes([stored[3] ^ 1]) + stored[4:])                  # noqa: E731
    bad_header = lambda p: b"\x1f\x8b\x08\x00" + good[4:]                                             # noqa: E731
    for encode, match in ((bad_crc, "CRC32 mismatch"), (bad_len, "stored block length"),
                          (bad_header, "not a BGZF block")):
        path = rewrite(encode)
        with pytest.raises(C3BError, match=match):
            dec.fetch_fasta(path, name, 150, 400)
        # the next fetch on the same decoder is whole
        assert _host(dec.fetch_fasta(gz, name, 150, 400)) == seq[150:400]
    # a window that runs past the blocks it was given
    a, b, c0, c1, u0 = bam_io.fasta_span(row, 0, 400, bam_io.read_gzi(gz + ".gzi"))
    raw = open(gz, "rb").read()
    first = raw[c0:c0 + bam_io.bgzf_block(raw, c0)[0]]
    with pytest.raises(C3BError, match="past"):
        dec.fetch_fasta_bytes(first, u0, 0, row[3], row[4], 400 + 64 * 1024)


# ---------------------------------------------------------------------------------------------- the genome route
CHUNK, SPLIT, MIN_SIZE = 4000, 12, 1500
LAYOUT = [("chr1", 9000, 800, 11), ("chr2", 7000, 800, 12), ("chrUn_a", 5000, 800, 13), ("chr3", None, 0, 14), ("chr5", 300, 100, 15)]


def _models(dev=DEV):
    p = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    p.to(dev)
    p.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()})
    f = Clair3_F(add_indel_length=True, predict=True, input_channels=8)
    f.to(dev)
    f.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=8, seed=1).items()})
    return p, f


def make_genome(d, iupac=0):
    """(bam path, plain FASTA path, bgzipped FASTA path, {contig: bases}) of the seeded genome of tests/test_gpu_genome.py,
    indexed; the BGZF copy's blocks cut every 3,000 bytes.  ``iupac``: that many bases of each contig with reads replaced by
    IUPAC codes, inside the reads' region."""
    seqs, parts = [], []
    rng = np.random.default_rng(77)
    for tid, (name, region, read_len, seed) in enumerate(LAYOUT):
        if region is None:
            seqs.append((name, sr.random_reference(6000, seed=seed)))
            continue
        rec, ref, rs = sr.random_alignment(region, depth=20, read_len=read_len, seed=seed, origin=0)
        assert rs == 0
        if iupac:
            b = bytearray(ref.encode())
            for p in rng.choice(np.arange(50, region - 50), iupac, replace=False):
                b[p] = b"RYKMSWBDHV"[int(rng.integers(0, 10))]
            ref = b.decode()
        rec["tid"] = np.full(len(rec["pos"]), tid, np.int32)
        seqs.append((name, ref))
        parts.append(rec)
    rec = {}
    for k in parts[0]:
        if k.endswith("_off"):
            arrs, base = [parts[0][k][:1]], 0
            for r in parts:
                arrs.append(r[k][1:] + base)
                base += r[k][-1]
            rec[k] = np.concatenate(arrs)
        else:
            rec[k] = np.concatenate([r[k] for r in parts])
    bam, fa = os.path.join(d, "g.bam"), os.path.join(d, "g.fa")
    bam_io.write_bam(bam, rec, [(n, len(s)) for n, s in seqs])
    bam_io.write_bai(bam)
    bam_io.write_fasta(fa, seqs)
    bam_io.write_fai(fa)
    size = os.path.getsize(fa)
    bf.bgzip(fa, fa + ".gz", cuts=list(range(3000, size, 3000)))
    return bam, fa, fa + ".gz", dict(seqs)


@pytest.fixture(scope="module")
def genome_files(tmp_path_factory):
    return make_genome(str(tmp_path_factory.mktemp("genome")))


@pytest.fixture(scope="module")
def models():
    return _models()


@pytest.fixture(scope="module")
def ws():
    w = cascade.Workspaces(0)
    yield w
    w.close()


def _read_outputs(d):
    out = {}
    for n in ("pileup", "full_alignment", "merge_output"):
        p = os.path.join(d, n + ".vcf.gz")
        if os.path.exists(p):
            out[n] = gzip.open(p, "rt").read()
    return out


def _without_reference_line(text):
    return [x for x in text.split("\n") if not x.startswith("##reference=")]


def _bed(seqs):
    rng = np.random.default_rng(7)
    return targets.read_bed("".join("%s\t%d\t%d\n" % (c, a, a + 400) for c in ("chr1", "chrUn_a") for a in rng.integers(0, 4000, 5)))


CASES = {"ont": {}, "bed": {"bed_fn": "bed"}, "long_indel": {"enable_long_indel": True}}


@pytest.mark.parametrize("name", sorted(CASES))
def test_call_genome_bgzf_equals_plain(ws, models, genome_files, name, tmp_path):
    bam, fa, gz, seqs = genome_files
    kw = dict(CASES[name])
    if "bed_fn" in kw:
        kw["bed_fn"] = _bed(seqs)
    got = {}
    for label, ref in (("plain", fa), ("bgzf", gz)):
        res = genome.call_genome(bam, ref, models[0], models[1], str(tmp_path / label), cmdline="run --x", include_all_ctgs=True,
                                 min_contig_size=MIN_SIZE, chunk_size=CHUNK, split_bed_size=SPLIT, workspaces=ws, **kw)
        got[label] = _read_outputs(str(tmp_path / label))
        assert got[label] == res["texts"]
    assert sorted(got["bgzf"]) == sorted(got["plain"]) == ["full_alignment", "merge_output", "pileup"]
    assert genome.has_records(got["plain"]["pileup"])
    for n, text in got["plain"].items():
        assert "##reference=%s" % gz in got["bgzf"][n]
        assert _without_reference_line(got["bgzf"][n]) == _without_reference_line(text), n


def test_cli_with_bgzf_reference(ws, models, genome_files, tmp_path):
    bam, fa, gz, _ = genome_files
    mdir = tmp_path / "model"
    mdir.mkdir()
    torch.save({"state_dict": {k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()}},
               mdir / "pileup.pt")
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=8, seed=1).items()},
               mdir / "full_alignment.pt")
    out = tmp_path / "cli"
    cmd = [sys.executable, "-m", "clair3_b200.run_clair3", "--bam_fn", bam, "--ref_fn", gz, "--model_path", str(mdir),
           "--platform", "ont", "--output", str(out), "--include_all_ctgs", "True", "--min_contig_size", str(MIN_SIZE),
           "--chunk_size", str(CHUNK), "--no_phasing_for_fa", "True"]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = _read_outputs(str(out))
    genome.call_genome(bam, gz, models[0], models[1], str(tmp_path / "api"), include_all_ctgs=True, min_contig_size=MIN_SIZE,
                       chunk_size=CHUNK, workspaces=ws)
    want = _read_outputs(str(tmp_path / "api"))
    assert sorted(got) == sorted(want) == ["full_alignment", "merge_output", "pileup"]
    for n in want:
        assert [x for x in got[n].split("\n") if not x.startswith("##cmdline=")] == want[n].split("\n")


# ---------------------------------------------------------------------------------------------- --keep_iupac_bases
def _ref_letters(text):
    """The REF column's letters of a VCF text's rows."""
    return {c for row in text.split("\n") if row and row[0] != "#" for c in row.split("\t")[3]}


def test_keep_iupac_bases(ws, models, tmp_path):
    """Each contig's reference carries IUPAC codes inside its reads: the pileup rows equal the host route's (host records and
    the host FASTA -> count -> call -> ``decode.call_row`` with the config's ``keep_iupac_bases``), and a REF keeps an IUPAC
    letter only with the flag."""
    bam, fa, gz, seqs = make_genome(str(tmp_path), iupac=40)
    big = 10 ** 6                                   # one pileup chunk per contig: no row repeated between chunks
    texts = {}
    for keep in (False, True):
        res = genome.call_genome(bam, gz, models[0], models[1], str(tmp_path / str(keep)), include_all_ctgs=True,
                                 min_contig_size=MIN_SIZE, chunk_size=big, split_bed_size=SPLIT, workspaces=ws,
                                 keep_iupac_bases=keep)
        texts[keep] = res["texts"]
        cfg_p, _ = genome.output_configs(False, keep)
        contigs, chunks = genome.plan(bam, fa, include_all_ctgs=True, min_contig_size=MIN_SIZE, chunk_size=big)
        lengths, rows = dict(contigs), []
        _, _, snp, indel = genome.resolve_options("ont")
        for ctg, cid, n in chunks:
            (s, e), _ = genome.pileup_chunk_region(ctg, lengths[ctg], cid, n)
            r0, r1 = max(0, s - FETCH_EXPAND), min(lengths[ctg], e + FETCH_EXPAND + 1)
            rec, _ = bam_io.read_bam(bam, ctg, s, e)
            call = ws.counter.count(rec, s, e, bam_io.read_fasta(fa, ctg, r0, r1), r0, min_depth=2, min_snp_af=snp,
                                    min_indel_af=indel, min_mq=5, call_snp_only=False, call_ht=False, alt_info=True,
                                    max_indel_length=decode.MAX_INFER_LENGTH).call(models[0], cfg_p, ctg)
            rows += [decode.call_row(call, i, cfg_p) for i in cascade.row_indices(call)]
        body = genome.sort_rows(rows, [c for c, _ in contigs])
        assert [x for x in texts[keep]["pileup"].split("\n") if x and x[0] != "#"] == body.rstrip("\n").split("\n")
    iupac = set("RYKMSWBDHV")
    assert _ref_letters(texts[True]["pileup"]) & iupac
    for text in texts[False].values():
        assert not _ref_letters(text) & iupac
