"""The genome route's host layer (clair3_b200/genome.py and the file I/O of bam_io.py) on the CPU: CheckEnvs (``plan``), the
VCF header, SortVcf (``sort_rows`` / ``vcf_text`` / ``postprocess_pileup``) and SelectQual + SelectCandidates over
overlapping chunks (``exchange``) against tests/golden/genome_cases.npz, minted from the reference's own Python
(tests/golden/make_genome_golden.py); the files' early exits (``file_texts``) on synthetic rows; the ``.fai`` fetch,
``idxstats``, BGZF and tabix against what was written; and the two-rank exchange (gloo) against the single-process one."""
import gzip
import json
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from clair3_b200 import bam_io, cascade, genome, synth_reads as sr

import cascade_cases as cc

G = json.loads(str(np.load(os.path.join(os.path.dirname(__file__), "golden", "genome_cases.npz"))["cases"]))


def _inputs(tmp_path):
    """The case's FASTA (placeholder bases), ``.fai``, BED, VCF and an (empty) BAM with its ``.bai``, as the maker wrote them."""
    ref = tmp_path / "ref.fa"
    ref.write_text("".join(">%s\n%s\n" % (n, "A" * L) for n, L in G["fai"]))
    bam_io.write_fai(str(ref))
    for p in ("in.bam", "in.bam.bai"):
        (tmp_path / p).write_bytes(b"")
    (tmp_path / "t.bed").write_text(G["bed"])
    (tmp_path / "k.vcf").write_text(G["vcf"])
    return str(ref), str(tmp_path / "in.bam")


@pytest.mark.parametrize("name", sorted(G["checkenvs"]))
def test_plan_matches_checkenvs(name, tmp_path):
    case = G["checkenvs"][name]
    opt = case["options"]
    ref, bam = _inputs(tmp_path)
    stats = [(n, L, G["mapped"][n], 0) for n, L in G["fai"]]
    contigs, chunks = genome.plan(bam, ref, ctg_name=opt.get("ctg_name"), include_all_ctgs=opt.get("include_all_ctgs", False),
                                  min_contig_size=opt.get("min_contig_size", 0), chunk_size=opt.get("chunk_size", 5000000),
                                  bed=str(tmp_path / "t.bed") if opt.get("bed") else None,
                                  known_sites=str(tmp_path / "k.vcf") if opt.get("vcf") else None, idxstats=stats)
    # the major contigs in their order; the others follow the .fai here and a set's iteration order (which changes from
    # run to run) in the reference, so they are compared as a set
    want = case["contigs"].split("\n") if case["contigs"] else []
    got = [c for c, _ in contigs]
    major = [c for c in want if c in cascade.MAJOR_CONTIGS]
    assert got[:len(major)] == major and sorted(got[len(major):]) == sorted(want[len(major):])
    assert got[len(major):] == [n for n, _ in G["fai"] if n in want[len(major):]]
    if contigs:
        rows = case["chunk_list"].splitlines(keepends=True)
        assert "".join("%s %d %d\n" % c for c in chunks) == "".join(r for c in got for r in rows if r.split()[0] == c)
    else:
        assert chunks == [] and case["header_only_merge"] == genome.header(G["ref_fn"], fai=ref + ".fai")


def test_plan_refusals(tmp_path):
    ref, bam = _inputs(tmp_path)
    with pytest.raises(ValueError, match="not both"):
        genome.plan(bam, ref, bed=str(tmp_path / "t.bed"), known_sites=str(tmp_path / "k.vcf"), idxstats=[])
    os.remove(bam + ".bai")
    with pytest.raises(FileNotFoundError, match="bai"):
        genome.plan(bam, ref, idxstats=[])
    (tmp_path / "in.csi").write_bytes(b"")
    with pytest.raises(NotImplementedError, match="CSI"):
        genome.plan(bam, ref, idxstats=[])
    with pytest.raises(NotImplementedError, match="CRAM"):
        genome.plan(str(tmp_path / "in.cram"), ref, idxstats=[])
    (tmp_path / "in.bam.bai").write_bytes(b"")
    os.remove(ref + ".fai")
    with pytest.raises(FileNotFoundError, match="fai"):
        genome.plan(bam, ref, idxstats=[])


@pytest.mark.parametrize("name", sorted(G["header"]))
def test_header_matches_get_header(name, tmp_path):
    case = G["header"][name]
    ref, _ = _inputs(tmp_path)
    assert genome.header(G["ref_fn"], case["sample"], case["cmd"], fai=ref + ".fai") == case["text"]


def _rows(files):
    return [r for _, text in files for r in text.splitlines(keepends=True) if r[0] != "#"]


@pytest.mark.parametrize("name", sorted(G["sortvcf"]))
def test_sort_matches_sortvcf(name, tmp_path):
    case = G["sortvcf"][name]
    ref, _ = _inputs(tmp_path)
    rows = _rows(case["files"])
    body = genome.sort_rows(rows, case["contigs"])
    if case["pileup_only"]:
        body = genome.postprocess_pileup(body, case["qual"], case["print_ref"])
    file_cmd = G["header"]["cmd"]["cmd"]
    head = genome.header(G["ref_fn"], "SAMPLE", file_cmd if rows else case["cmd"], fai=ref + ".fai")
    assert genome.vcf_text(head, body, bool(rows)) == case["out"]


def test_select_over_overlapping_chunks():
    """SelectQual's cut-offs and SelectCandidates' bed files from three pileup chunks that share rows at their edges."""
    case = G["select"]
    platform, pres, _ = cc.case("hifi")
    pres = dict(pres, chromosome=["chr1"] * len(pres["position"]))
    chunk_rows, idx = [], cascade.row_indices(pres)              # the fixture's chunks cut the VCF rows
    for a, b in case["chunks"]:
        pos, prob, flags, _ = cascade.row_summary(cascade.take_calls(pres, idx[a:b]))
        chunk_rows.append(("chr1", pos, prob, flags))
    keep, cuts, beds = genome.exchange(chunk_rows, [("chr1", 10 ** 6)], platform, split_bed_size=case["split_bed_size"])
    assert sum(int(k.sum()) for k in keep) == len(set(np.concatenate([r[1] for r in chunk_rows]).tolist()))
    assert "%.2f %.2f" % cuts == case["qual"].split("\n")[0].strip()
    assert [cascade.bed_text(c, p) for c, p in beds] == case["beds"]
    # the same as the region layer on the rows each once
    assert cuts == cascade.qual_cutoffs([pres], platform)
    want, chunks = cascade.select(pres, *cuts, split_bed_size=case["split_bed_size"])
    assert [p.tolist() for _, p in beds] == [want[a:b].tolist() for a, b in chunks]


# ---------------------------------------------------------------------------------------------- the files' early exits
HEAD = "##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE"
CONTIGS = ["chr1", "chr2"]


def _row(ctg, pos, alt="C"):
    filt, gt = ("RefCall", "0/0") if alt == "." else ("PASS", "0/1")
    return "%s\t%d\t.\tA\t%s\t12.00\t%s\tP\tGT:GQ:DP:AF\t%s:12:30:0.5000\n" % (ctg, pos, alt, filt, gt)


def _chunk(ctg, positions, alt="C"):
    """One pileup chunk's or bed file's rows as ``file_texts`` takes them: (contig, 1-based positions, row texts)."""
    return ctg, np.array(positions, np.int64), [_row(ctg, p, alt) for p in positions]


def test_file_texts_without_contig():
    assert genome.file_texts(HEAD, [], [], []) == {"merge_output": HEAD}


def test_file_texts_without_pileup_row():
    assert genome.file_texts(HEAD, CONTIGS, [_chunk("chr1", []), _chunk("chr2", [])], []) == {"pileup": HEAD, "merge_output": HEAD}


def test_file_texts_pileup_only():
    chunks = [_chunk("chr2", [30, 10]), _chunk("chr1", [50])]
    got = genome.file_texts(HEAD, CONTIGS, chunks, [], pileup_only=True)
    assert got == {"pileup": HEAD + "\n" + _row("chr1", 50) + _row("chr2", 10) + _row("chr2", 30)}
    # only reference rows, not printed: the pileup file holds no row, and merge_output is a copy of it
    got = genome.file_texts(HEAD, CONTIGS, [_chunk("chr1", [5, 7], alt=".")], [], pileup_only=True)
    assert sorted(got) == ["merge_output", "pileup"] and not genome.has_records(got["pileup"])
    assert got["merge_output"] == got["pileup"] == HEAD + "\n"


def test_file_texts_without_bed_file():
    got = genome.file_texts(HEAD, CONTIGS, [_chunk("chr2", [30]), _chunk("chr1", [50, 20], alt=".")], [])
    assert sorted(got) == ["merge_output", "pileup"]
    assert got["merge_output"] == got["pileup"] == HEAD + "\n" + _row("chr1", 20, ".") + _row("chr1", 50, ".") + _row("chr2", 30)


def test_file_texts_without_full_alignment_row():
    pileup = [_chunk("chr1", [50]), _chunk("chr2", [30])]
    got = genome.file_texts(HEAD, CONTIGS, pileup, [_chunk("chr1", []), _chunk("chr2", [])])
    assert sorted(got) == ["full_alignment", "merge_output", "pileup"] and got["full_alignment"] == HEAD
    assert got["merge_output"] == got["pileup"] == HEAD + "\n" + _row("chr1", 50) + _row("chr2", 30)


def test_fai_fetch_matches_read_fasta(tmp_path):
    rng = np.random.default_rng(5)
    seqs = [("c%d" % i, sr.random_reference(int(rng.integers(1, 3000)), seed=i)) for i in range(4)]
    for width in (60, 7):
        path = str(tmp_path / ("r%d.fa" % width))
        bam_io.write_fasta(path, seqs, width=width)
        bam_io.write_fai(path)
        assert [r[:2] for r in bam_io.read_fai(path + ".fai")] == [(n, len(s)) for n, s in seqs]
        for name, s in seqs:
            for _ in range(20):
                a = int(rng.integers(0, len(s) + 5))
                b = int(rng.integers(a, len(s) + 10))
                assert bam_io.fetch_fasta(path, name, a, b) == bam_io.read_fasta(path, name, a, b)
    gz = tmp_path / "r.fa.gz"
    gz.write_bytes(gzip.compress(open(path, "rb").read()))
    (tmp_path / "r.fa.gz.fai").write_text(open(path + ".fai").read())
    with pytest.raises(ValueError, match="compressed FASTA"):
        bam_io.fetch_fasta(str(gz), "c0", 0, 10)


def test_idxstats_counts_records(tmp_path):
    parts, refs = [], [("a", 9000), ("b", 5000), ("c", 7000)]
    for tid, seed in ((0, 1), (2, 2)):
        rec, ref, rs = sr.random_alignment(3000, depth=6, read_len=500, seed=seed, origin=0)
        rec["tid"] = np.full(len(rec["pos"]), tid, np.int32)
        parts.append(rec)
    rec = {k: np.concatenate([parts[0][k], parts[1][k] + (parts[0][k][-1] if k.endswith("_off") else 0)])
           if not k.endswith("_off") else np.concatenate([parts[0][k], parts[1][k][1:] + parts[0][k][-1]]) for k in parts[0]}
    path = str(tmp_path / "m.bam")
    bam_io.write_bam(path, rec, refs)
    bam_io.write_bai(path)
    got = bam_io.idxstats(path)
    for tid, (name, length, mapped, unmapped) in enumerate(got):
        m = rec["tid"] == tid
        assert (name, length) == refs[tid]
        assert mapped == int((m & (rec["flag"] & 4 == 0)).sum()) and unmapped == int((m & (rec["flag"] & 4 != 0)).sum())
    assert got[1][2] == 0 and got[0][2] > 0


def test_bgzf_round_trip(tmp_path):
    rng = np.random.default_rng(3)
    text = "".join("line %d %s\n" % (i, "x" * int(rng.integers(0, 200))) for i in range(3000))
    path = str(tmp_path / "t.gz")
    voff = bam_io.write_bgzf(path, text)
    raw = open(path, "rb").read()
    assert gzip.decompress(raw).decode() == text and raw.endswith(bam_io._EOF)
    blocks = bam_io.bgzf_blocks(raw)
    assert len(blocks) == (len(text) + 0xFEFF) // 0xFF00 + 1 and blocks[-1][2] == 0
    assert voff(0) == 0 and voff(0xFF00 + 5) == (blocks[1][0] << 16 | 5)


def _uoffsets(raw):
    """virtual offset -> uncompressed offset over a BGZF file's blocks."""
    starts, u = {}, 0
    for off, _, isize in bam_io.bgzf_blocks(raw):
        starts[off] = u
        u += isize
    return lambda v: starts[v >> 16] + (v & 0xFFFF)


def test_tbi_covers_overlapping_rows(tmp_path):
    rng = np.random.default_rng(9)
    rows = []
    for ctg, n, span in (("chr2", 4000, 2_000_000), ("chrUn", 50, 70_000), ("chr1", 2500, 300_000)):
        for p in np.sort(rng.integers(1, span, n)):
            ref = "ACGT"[int(rng.integers(0, 4))] * int(rng.choice([1, 1, 2, 40, 20000]))
            rows.append("%s\t%d\t.\t%s\tA\t5\tPASS\t.\tGT\t0/1\n" % (ctg, p, ref))
    text = "##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tS\n" + "".join(rows)
    path = genome.write_vcf_gz(str(tmp_path / "t.vcf.gz"), text)
    assert gzip.open(path, "rt").read() == text
    tbi = bam_io.read_tbi(path + ".tbi")
    assert tbi["header"] == (2, 1, 2, 0, ord("#"), 0) and tbi["names"] == ["chr2", "chrUn", "chr1"]
    assert [r["mapped"] for r in tbi["refs"]] == [4000, 50, 2500]
    raw = open(path, "rb").read()
    data = gzip.decompress(raw).decode()
    u = _uoffsets(raw)
    for _ in range(200):
        ctg = ["chr2", "chrUn", "chr1"][int(rng.integers(0, 3))]
        a = int(rng.integers(0, 2_100_000))
        b = a + int(rng.integers(1, 100_000))
        want = {r for r in rows if r.split("\t")[0] == ctg and int(r.split("\t")[1]) - 1 < b
                and int(r.split("\t")[1]) - 1 + len(r.split("\t")[3]) > a}
        got = set()
        for c0, c1 in bam_io.tbi_chunks(tbi, ctg, a, b):
            got.update(r for r in data[u(c0):u(c1)].splitlines(keepends=True) if r[0] != "#")
        assert want <= got
        assert {r for r in got if r.split("\t")[0] == ctg and int(r.split("\t")[1]) - 1 < b
                and int(r.split("\t")[1]) - 1 + len(r.split("\t")[3]) > a} == want


# ---------------------------------------------------------------------------------------------- two ranks (gloo)
def _synthetic_chunks():
    """Nine pileup chunks over three contigs from tests/cascade_cases.py's rows, neighbours sharing 15 rows."""
    out, contigs = [], []
    for ctg, name in (("chr1", "ont"), ("chr2", "hifi"), ("chrUn", "zero_ref")):
        _, pres, _ = cc.case(name)
        pres = dict(pres, chromosome=[ctg] * len(pres["position"]))
        n = len(pres["position"])
        contigs.append((ctg, int(pres["position"].max()) + 10))
        for a, b in ((0, n // 3 + 15), (n // 3, 2 * n // 3 + 15), (2 * n // 3, n)):
            pos, prob, flags, _ = cascade.row_summary(cascade.take_calls(pres, np.arange(a, b)))
            out.append((ctg, pos, prob, flags))
    return out, contigs


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from clair3_b200 import genome as gm
        from clair3_b200.sharding import site_range
        chunks, contigs = _synthetic_chunks()
        lo, hi = site_range(len(chunks), rank, world)
        keep, cuts, beds = gm.decisions([(g,) + chunks[g] for g in range(lo, hi)], contigs, "ont", split_bed_size=100,
                                        group=dist.group.WORLD)
        q.put((rank, [k.tolist() for k in keep], cuts, [(c, p.tolist()) for c, p in beds]))
    finally:
        dist.destroy_process_group()


def test_two_rank_exchange_matches_single_process():
    chunks, contigs = _synthetic_chunks()
    keep, cuts, beds = genome.decisions([(g,) + c for g, c in enumerate(chunks)], contigs, "ont", split_bed_size=100)
    assert len(beds) > 3 and cuts[0] > 0
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for _, k, c, b in got:
        assert k == [m.tolist() for m in keep] and c == cuts and b == [(x, p.tolist()) for x, p in beds]


# ---------------------------------------------------------------------------------------------- options and index names
# run_clair3.py:303-321 (0 means the platform's value) and :393-395 (a known-sites VCF sets both allele frequencies to 0)
RUN_CLAIR3_DEFAULTS = {"ont": (0.7, 0.1, 0.08, 0.15), "hifi": (0.3, 0.3, 0.08, 0.08)}


@pytest.mark.parametrize("platform", sorted(RUN_CLAIR3_DEFAULTS))
def test_options_follow_run_clair3(platform):
    assert genome.resolve_options(platform) == RUN_CLAIR3_DEFAULTS[platform]
    assert genome.resolve_options(platform, 0, 0, 0, 0) == RUN_CLAIR3_DEFAULTS[platform]
    assert genome.resolve_options(platform, 0.5, 0.2, 0.1, 0.2) == (0.5, 0.2, 0.1, 0.2)
    assert genome.resolve_options(platform, genotyping=True) == RUN_CLAIR3_DEFAULTS[platform][:2] + (0.0, 0.0)
    with pytest.raises(NotImplementedError):
        genome.resolve_options("ilmn")


def test_output_configs_follow_call_variants():
    """CallVariantsFromCffi as the pipeline runs it: ``--showRef`` True and ``--qual`` 2 by default (neither is passed),
    ``--add_indel_length`` for full alignment only, ``--enable_long_indel`` raising the inferred-length limit."""
    prm = G["params"]
    for long_indel in (False, True):
        cfg_p, cfg_f = genome.output_configs(long_indel)
        for cfg, pileup in ((cfg_p, True), (cfg_f, False)):
            assert cfg.is_show_reference and cfg.quality_score_for_pass == 2 and cfg.pileup == pileup
            assert cfg.add_indel_length == (not pileup) and cfg.enable_long_indel == long_indel
            assert not (cfg.gvcf or cfg.is_haploid_precise_mode_enabled or cfg.is_haploid_sensitive_mode_enabled)
            want = prm[("p" if pileup else "f") + "_max_indel" + ("_long" if long_indel else "")]
            assert cfg.maximum_variant_length_that_need_infer == want
        assert genome.LONG_INDEL == prm["p_max_indel_long"] == prm["f_max_indel_long"]
    from clair3_b200.fa_tensor import MATRIX_DEPTH
    assert {k: MATRIX_DEPTH[k] for k in ("ont", "hifi")} == {k: prm["matrix_depth"][k] for k in ("ont", "hifi")}


def test_plan_accepts_bai_without_bam_suffix(tmp_path):
    """run_clair3.py and the pipeline also take ``sample.bai`` for ``sample.bam``."""
    ref, bam = _inputs(tmp_path)
    os.remove(bam + ".bai")
    (tmp_path / "in.bai").write_bytes(b"")
    assert genome.bam_index(bam) == str(tmp_path / "in.bai")
    stats = [(n, L, G["mapped"][n], 0) for n, L in G["fai"]]
    contigs, _ = genome.plan(bam, ref, idxstats=stats, chunk_size=5000)
    assert "\n".join(c for c, _ in contigs) == G["checkenvs"]["default"]["contigs"]
