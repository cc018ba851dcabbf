"""Read-based phasing on the GPU (clair3_b200/phase_gpu.py, csrc/phase.cu) against the statement (clair3_b200/phasing.py): the
observations, blocks, haplotypes, costs and rows must be exactly equal.  Then the true phase of a synthetic diploid contig, and
``call_genome(enable_phasing=True)`` / ``--enable_phasing`` on the genome route."""
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from clair3_b200 import bam_io, genome, phase_gpu, phasing
from clair3_b200.bam_decode import BamDecoder
from phase_cases import diploid_contig, random_fragments
from test_gpu_genome import CHUNK, MIN_SIZE, ROOT, SPLIT, _free_port, _models, make_genome

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def decoder():
    d = BamDecoder(0)
    yield d
    d.close()


def _write_contig(d, rec, ref, ctg="chr1"):
    bam, fa = os.path.join(d, "p.bam"), os.path.join(d, "p.fa")
    bam_io.write_bam(bam, rec, [(ctg, len(ref))])
    bam_io.write_bai(bam)
    bam_io.write_fasta(fa, [(ctg, ref)])
    bam_io.write_fai(fa)
    return bam


def _same(a, b):
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and np.array_equal(x, y)


def _check_against_host(decoder, bam, rec, rows, length, span):
    got = phase_gpu.phase_contig(decoder, bam, "chr1", length, rows, span)
    want = phasing.phase_contig(rows, bam_io.read_bam(bam, "chr1", fa_fields=True)[0])
    out, v, frag, lay, hap, cost = got
    assert out == want[0]
    _same(frag, want[2])
    _same(lay, want[3])
    assert np.array_equal(hap, want[4]) and np.array_equal(cost, want[5])
    return got


# (seed, contig length, depth, read length, het rate, span)
CASES = {
    "short": (1, 60000, 30, 250, 3e-3, 20000),
    "8kb": (2, 300000, 30, 8000, 2e-3, 70000),
    "sparse": (3, 120000, 8, 3000, 1e-3, 1 << 30),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_gpu_equals_host(decoder, tmp_path, name):
    seed, length, depth, read_len, het, span = CASES[name]
    rec, ref, rows, _ = diploid_contig(seed, length, depth, read_len, het_rate=het)
    bam = _write_contig(str(tmp_path), rec, ref)
    out, v, frag, lay, hap, cost = _check_against_host(decoder, bam, rec, rows, length, span)
    assert lay.n_blocks > 0 and any(o != r for o, r in zip(out, rows))
    if name == "8kb":
        assert np.diff(lay.blk_col_off).max() > 2 * phase_gpu.SEGMENT       # blocks of several backtrace segments
        assert lay.blk_kmax.max() == phasing.MAX_COVERAGE                     # columns with 15 active reads
    if span < length:                                                        # reads that cross a span edge are counted once
        ops, lens = rec["cigar"] & 15, (rec["cigar"] >> 4).astype(np.int64)
        ref_len = np.where(np.isin(ops, [0, 2, 3, 7, 8]), lens, 0)
        ends = rec["pos"] + np.add.reduceat(ref_len, rec["cigar_off"][:-1])
        assert any(((rec["pos"] < e) & (ends > e)).any() for e in range(span, length, span))


def test_contig_without_het_snp(decoder, tmp_path):
    rec, ref, rows, _ = diploid_contig(4, 20000, 10, 1000)
    rows = [r.replace("\t0/1:", "\t1/1:") for r in rows]
    bam = _write_contig(str(tmp_path), rec, ref)
    out, v, frag, lay, hap, cost = _check_against_host(decoder, bam, rec, rows, 20000, 5000)
    assert out == rows and len(v.pos) == 0 and lay.n_blocks == 0


@pytest.mark.parametrize("seed", range(40))
def test_dp_on_random_fragments(seed):
    """The DP alone, on the enumeration-sized instances the CPU test holds to brute force and on wider ones, with one CTA
    taking every block in turn and with one per block."""
    rng = np.random.default_rng(seed)
    if seed < 20:
        frag = random_fragments(seed, int(rng.integers(2, 11)), int(rng.integers(2, 9)), max_span=int(rng.integers(2, 9)))
    else:
        frag = random_fragments(seed, 400, 700, max_span=int(rng.integers(3, 40)))
    n_var = int(frag.var.max()) + 1 if len(frag.var) else 0
    lay = phasing.layout(frag, n_var)
    want = phasing.solve(lay)
    for n_ctas in (1, None):
        hap, cost = phase_gpu.solve(lay, DEV, n_ctas=n_ctas)
        assert np.array_equal(hap, want[0]) and np.array_equal(cost, want[1])


@pytest.mark.parametrize("seed", range(3))
def test_known_phase(decoder, tmp_path, seed):
    """Two haplotypes of het SNPs, reads drawn from each with 3 % errors at depth 30: every variant that admitted reads link is
    phased, with no switch error against the truth."""
    rec, ref, rows, truth = diploid_contig(40 + seed, 200000, 30, 8000 if seed else 2000, err=0.03)
    bam = _write_contig(str(tmp_path), rec, ref)
    out, v, frag, lay, hap, cost = phase_gpu.phase_contig(decoder, bam, "chr1", 200000, rows, 60000)
    linked = np.unique(frag.var[np.isin(frag.read, lay.read_id)])
    assert np.array_equal(np.sort(lay.col_var), linked) and len(linked) >= 0.95 * len(v.pos)
    for b in range(lay.n_blocks):
        cols = lay.col_var[lay.blk_col_off[b]:lay.blk_col_off[b + 1]]
        h, t = hap[lay.blk_col_off[b]:lay.blk_col_off[b + 1]], truth[cols]
        assert np.array_equal(h, t) or np.array_equal(h, 1 - t), "switch error in block %d" % b


def test_records_are_checked(decoder, tmp_path):
    rec, ref, rows, _ = diploid_contig(5, 20000, 10, 1000)
    bam = _write_contig(str(tmp_path), rec, ref)
    d = decoder.decode(bam, "chr1", 0, None, fa_fields=True)
    v = phasing.het_snvs(rows)
    d.t["cigar_off"] = d.t["cigar_off"].clone()
    d.t["cigar_off"][3] += 1000000
    with pytest.raises(Exception, match="cigar_off"):
        phase_gpu.fragments(d, phase_gpu.device_variants(v, DEV), 0, 1 << 62, 0)


# ---------------------------------------------------------------------------------------------- the route
@pytest.fixture(scope="module")
def genome_files(tmp_path_factory):
    return make_genome(str(tmp_path_factory.mktemp("genome")))


@pytest.fixture(scope="module")
def models():
    return _models()


def _read_outputs(d):
    """{name: text} of every ``.vcf.gz`` in d; each ``.tbi`` must name the file's contigs."""
    out = {}
    for f in sorted(os.listdir(d)):
        if f.endswith(".vcf.gz"):
            n = f[:-len(".vcf.gz")]
            out[n] = gzip.open(os.path.join(d, f), "rt").read()
            tbi = bam_io.read_tbi(os.path.join(d, f + ".tbi"))
            assert tbi["names"] == list(dict.fromkeys(r.split("\t")[0] for r in out[n].split("\n") if r and r[0] != "#"))
    return out


def _host_phased(bam, merged_text):
    head, _, body = merged_text.partition("\n#CHROM")
    head = head + "\n#CHROM" + body.split("\n", 1)[0]
    body = merged_text[len(head) + 1:]
    out = []
    for ctg, rows in phasing.split_contigs(body).items():
        out.extend(phasing.phase_contig(rows, bam_io.read_bam(bam, ctg, fa_fields=True)[0])[0])
    return phasing.phase_header(head) + "\n" + "".join(out)


KW = dict(cmdline="run --x", include_all_ctgs=True, min_contig_size=MIN_SIZE, chunk_size=CHUNK, split_bed_size=SPLIT)


def test_route_writes_the_phased_file(models, genome_files, tmp_path):
    bam, fa, _ = genome_files
    plain, phased = tmp_path / "plain", tmp_path / "phased"
    genome.call_genome(bam, fa, models[0], models[1], str(plain), **KW)
    res = genome.call_genome(bam, fa, models[0], models[1], str(phased), enable_phasing=True, **KW)
    a, b = _read_outputs(str(plain)), _read_outputs(str(phased))
    assert sorted(b) == ["full_alignment", "merge_output", "phased_merge_output", "pileup"]
    for n in a:
        assert (plain / (n + ".vcf.gz")).read_bytes() == (phased / (n + ".vcf.gz")).read_bytes(), n
        assert (plain / (n + ".vcf.gz.tbi")).read_bytes() == (phased / (n + ".vcf.gz.tbi")).read_bytes(), n
    assert b["phased_merge_output"] == _host_phased(bam, b["merge_output"])
    assert "|" in b["phased_merge_output"] and ":PS\t" in b["phased_merge_output"]
    assert res["rows"]["phased_merge_output"] == res["rows"]["merge_output"] and "phase" in res["stages"]
    assert os.path.exists(res["files"]["phased_merge_output"] + ".tbi")


def test_route_early_exits_write_no_phased_file(models, genome_files, tmp_path):
    bam, fa, _ = genome_files
    for i, kw in enumerate(({"pileup_only": True}, {"ctg_name": "chr3", "include_all_ctgs": False})):
        d = tmp_path / str(i)
        args = dict(KW, **kw)
        genome.call_genome(bam, fa, models[0], models[1], str(d), enable_phasing=True, **args)
        assert not any(n.startswith("phased") for n in os.listdir(d))


def _rank_worker(rank, world, port, bam, fa, out_dir, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        m_p, m_f = _models(dev)
        res = genome.call_genome(bam, fa, m_p, m_f, out_dir, device=dev, group=dist.group.WORLD, enable_phasing=True, **KW)
        q.put((rank, res is None))
    finally:
        dist.destroy_process_group()


def test_world_two_writes_the_same_bytes(models, genome_files, tmp_path):
    bam, fa, _ = genome_files
    one, two = tmp_path / "one", tmp_path / "two"
    genome.call_genome(bam, fa, models[0], models[1], str(one), enable_phasing=True, **KW)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, bam, fa, str(two), q)) for r in range(2)]
    for p in procs:
        p.start()
    got = sorted(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert got == [(0, False), (1, True)]
    names = sorted(os.listdir(one))
    assert names == sorted(os.listdir(two)) and len(names) == 8
    for n in names:
        assert (one / n).read_bytes() == (two / n).read_bytes(), n


def test_cli_enable_phasing(models, genome_files, tmp_path):
    bam, fa, _ = genome_files
    mdir = tmp_path / "model"
    mdir.mkdir()
    from clair3_b200 import synth
    torch.save({"state_dict": {k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()}},
               mdir / "pileup.pt")
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=8, seed=1).items()},
               mdir / "full_alignment.pt")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    api = tmp_path / "api"
    genome.call_genome(bam, fa, models[0], models[1], str(api), include_all_ctgs=True, min_contig_size=MIN_SIZE, chunk_size=CHUNK,
                       enable_phasing=True)
    want = _read_outputs(str(api))["phased_merge_output"].split("\n")
    for flag in ("--enable_phasing", "--use_whatshap_for_final_output_phasing"):
        out = tmp_path / flag.strip("-")
        cmd = [sys.executable, "-m", "clair3_b200.run_clair3", "--bam_fn", bam, "--ref_fn", fa, "--model_path", str(mdir),
               "--platform", "ont", "--output", str(out), "--include_all_ctgs", "True", "--min_contig_size", str(MIN_SIZE),
               "--chunk_size", str(CHUNK), "--no_phasing_for_fa", "True", flag, "True"]
        r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        assert "phased_merge_output" in r.stdout
        got = _read_outputs(str(out))["phased_merge_output"].split("\n")
        assert [x for x in got if not x.startswith("##cmdline=")] == want
