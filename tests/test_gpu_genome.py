"""The genome route on the GPU (clair3_b200/genome.py, run_clair3.py) on a seeded synthetic genome: two major contigs with
reads, an unplaced one, one without reads and one below ``--min_contig_size``, in one indexed BAM and an indexed FASTA, with
small chunks and bed files so every called contig has several of each.  Each written VCF must equal the text of a host route
assembled here from already-pinned pieces only: per chunk ``bam_io.read_bam`` -> count -> ``call``; ``cascade.qual_cutoffs``
over every chunk; per contig ``cascade.select``, then per bed file ``read_bam`` of its span -> host-candidate build ->
``call``; ``cascade.merge``; and the header / sort that tests/test_genome_cpu.py holds to the reference's SortVcf."""
import gzip
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from clair3_b200 import bam_io, cascade, genome, synth, synth_reads as sr, targets
from clair3_b200.fa_tensor import MATRIX_DEPTH
from clair3_b200.model import Clair3_F, Clair3_P
from clair3_b200.pileup_counts import FETCH_EXPAND, bed_chunk_region, chunk_region, counting_region, known_sites_chunk

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda:0")
CHUNK, SPLIT, MIN_SIZE = 4000, 12, 1500
# (name, region length for reads or None, read length, seed): chr3 has no reads, chr5 is below MIN_SIZE
LAYOUT = [("chr1", 9000, 800, 11), ("chr2", 7000, 800, 12), ("chrUn_a", 5000, 800, 13), ("chr3", None, 0, 14), ("chr5", 300, 100, 15)]


def _models(dev=DEV, fa_channels=8):
    p = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    p.to(dev)
    p.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()})
    f = Clair3_F(add_indel_length=True, predict=True, input_channels=fa_channels)
    f.to(dev)
    f.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=fa_channels, seed=1).items()})
    return p, f


def _concat_records(parts):
    out = {}
    for k in parts[0][0]:
        if k.endswith("_off"):
            arrs, base = [parts[0][0][k][:1]], 0
            for rec, _ in parts:
                arrs.append(rec[k][1:] + base)
                base += rec[k][-1]
            out[k] = np.concatenate(arrs)
        else:
            out[k] = np.concatenate([rec[k] for rec, _ in parts])
    out["tid"] = np.concatenate([np.full(len(rec["pos"]), tid, np.int32) for rec, tid in parts])
    return out


def _move_tables(rec, seed):
    """Seeded ``mv`` move tables (stride element, then one sample per base start) for every read but a few."""
    rng = np.random.default_rng(seed + 4243)
    mv, off = [], [0]
    for lq in rec["l_qseq"].tolist():
        if rng.random() < 0.1:                           # a read without a move table
            off.append(off[-1])
            continue
        runs = rng.geometric(0.3, lq + int(rng.integers(-3, 4)))
        m = np.zeros(1 + int(runs.sum()), np.int32)
        m[0] = 5
        m[1 + np.concatenate([[0], np.cumsum(runs)[:-1]])] = 1
        mv.append(m)
        off.append(off[-1] + len(m))
    rec["mv"] = np.concatenate(mv) if mv else np.zeros(0, np.int32)
    rec["mv_off"] = np.array(off, np.int64)


def make_genome(d, dwell=False, bai_without_bam=False):
    """(bam path, FASTA path, {contig: bases}) of the seeded genome, indexed.  ``dwell``: the reads carry ``mv`` tags;
    ``bai_without_bam``: the index is ``g.bai`` rather than ``g.bam.bai``."""
    seqs, parts = [], []
    for tid, (name, region, read_len, seed) in enumerate(LAYOUT):
        if region is None:
            seqs.append((name, sr.random_reference(6000, seed=seed)))
            continue
        rec, ref, rs = sr.random_alignment(region, depth=20, read_len=read_len, seed=seed, origin=0)
        assert rs == 0
        if dwell:
            _move_tables(rec, seed)
        seqs.append((name, ref))
        parts.append((rec, tid))
    bam, fa = os.path.join(d, "g.bam"), os.path.join(d, "g.fa")
    bam_io.write_bam(bam, _concat_records(parts), [(n, len(s)) for n, s in seqs])
    bam_io.write_bai(bam, os.path.join(d, "g.bai") if bai_without_bam else None)
    bam_io.write_fasta(fa, seqs)
    bam_io.write_fai(fa)
    return bam, fa, dict(seqs)


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


def _concat_results(results):
    """One contig's pileup ``call`` results as one (the text / ad pools placed one after another)."""
    out = {"chromosome": [], "position": [], "calls": [], "text": [], "ad": [], "start": [], "cand_ok": []}
    base = 0
    for r in results:
        n = max(len(r["text"]), len(r["ad"]))
        out["chromosome"] += list(r["chromosome"])
        for k in ("position", "calls", "cand_ok"):
            out[k].append(np.asarray(r[k]))
        out["text"].append(np.pad(np.asarray(r["text"]), (0, n - len(r["text"]))))
        out["ad"].append(np.pad(np.asarray(r["ad"]), (0, n - len(r["ad"]))))
        out["start"].append(np.asarray(r["start"]) + base)
        base += n
    return {k: (np.concatenate(v) if k != "chromosome" else v) for k, v in out.items()}


def host_route(ws, m_p, m_f, bam, fa, out_cmd=None, tgt=None, platform="ont", qual=2, print_ref=False, pileup_only=False,
               var_pct=None, ref_pct=None, include_all=True, ctg_name=None, chunk_size=CHUNK, split_bed_size=SPLIT,
               min_contig_size=MIN_SIZE, min_mq=5, min_coverage=2, call_snp_only=False, long_indel=False, call_ht=False,
               dwell=False, stats=None):
    """The texts of the files the run writes, through host records and host candidates.  ``stats``: a dict that receives
    ``repeated``, the number of (contig, position) rows that overlapping chunks repeat, and ``differing``, how many of them
    differ.  Without head / tail calling each must be byte-identical, which is what makes SortVcf's keep-one-of-them (in the
    reference: whichever file ``os.listdir`` lists last) well defined; with it, a position near a chunk's edge can get a
    padded window in one chunk and a whole one in the next, and the route keeps the last chunk's row (DESIGN.md 5g)."""
    genotyping = tgt is not None and tgt.kind == "vcf"
    var_pct, ref_pct, snp, indel = genome.resolve_options(platform, var_pct, ref_pct, None, None, genotyping)
    cfg_p, cfg_f = genome.output_configs(long_indel)
    max_indel = 100000 if long_indel else 50             # shared/param_{p,f}.py maximum_variant_length_that_need_infer(_include_long_indel)
    contigs, chunks = genome.plan(bam, fa, ctg_name=ctg_name, include_all_ctgs=include_all, min_contig_size=min_contig_size,
                                  chunk_size=chunk_size, bed=tgt if tgt is not None and not genotyping else None,
                                  known_sites=tgt if genotyping else None)
    head = genome.header(fa, "SAMPLE", out_cmd)
    names = [c for c, _ in contigs]
    if not contigs:
        return {"merge_output": head}
    L = dict(contigs)
    per = []
    for ctg, cid, n in chunks:
        ct = None
        if tgt is None:
            a, b = chunk_region(L[ctg], cid, n)
        elif not genotyping:
            ct = tgt.contig(ctg)
            a, b = bed_chunk_region(*ct.bed_region(), cid, n)
        else:
            c = known_sites_chunk(tgt.sites[ctg], cid, n)
            if c is None:
                continue
            a, b, ct = c[0], c[1], tgt.contig(ctg, chunk=(cid, n))
        s, e = counting_region(a, b)
        r0, r1 = max(0, s - FETCH_EXPAND), min(L[ctg], e + FETCH_EXPAND + 1)
        rec, _ = bam_io.read_bam(bam, ctg, s, e)
        res = ws.counter.count(rec, s, e, bam_io.read_fasta(fa, ctg, r0, r1), r0, min_depth=min_coverage, min_snp_af=snp,
                               min_indel_af=indel, min_mq=min_mq, call_snp_only=call_snp_only, call_ht=call_ht, alt_info=True,
                               max_indel_length=max_indel).call(m_p, cfg_p, ctg)
        res = cascade.take_calls(res, cascade.row_indices(res))
        if ct is not None:
            res = cascade.take_calls(res, np.nonzero(ct.keep(res["position"]))[0])
        per.append((ctg, res))
    first, repeated, differing = {}, 0, 0
    for ctg, res in per:
        for p, row in zip(*cascade.row_texts(res, cfg_p)):
            if (ctg, int(p)) in first:
                repeated += 1
                differing += first[(ctg, int(p))] != row
                assert call_ht or first[(ctg, int(p))] == row, "overlapping chunks print different rows at %s:%d" % (ctg, p)
            first.setdefault((ctg, int(p)), row)
    if stats is not None:
        stats.update(repeated=repeated, differing=differing)
    seen = set()                                   # SortVcf: of a repeated (contig, position) the last chunk's row
    for j in range(len(per) - 1, -1, -1):
        ctg, res = per[j]
        keep = [i for i, p in enumerate(res["position"].tolist()) if (ctg, p) not in seen]
        seen.update((ctg, p) for p in res["position"].tolist())
        per[j] = (ctg, cascade.take_calls(res, keep))
    rows = [r for _, res in per for r in cascade.row_texts(res, cfg_p)[1]]
    texts = {}
    if not rows:
        return {"pileup": head, "merge_output": head}
    body = genome.sort_rows(rows, names)
    if pileup_only:
        texts["pileup"] = genome.vcf_text(head, genome.postprocess_pileup(body, qual, print_ref), True)
        if not genome.has_records(texts["pileup"]):
            texts["merge_output"] = texts["pileup"]
        return texts
    texts["pileup"] = genome.vcf_text(head, body, True)
    cuts = cascade.qual_cutoffs([res for _, res in per], platform, var_pct, ref_pct, genotyping=genotyping)
    f_rows, merged, any_bed = [], [], False
    for ctg in names:
        res = _concat_results([r for c, r in per if c == ctg])
        pos, beds = cascade.select(res, *cuts, split_bed_size=split_bed_size)
        fres = []
        for a, b in beds:
            any_bed = True
            cand = pos[a:b]
            s, e = max(int(cand[0]) - 16, 0), int(cand[-1]) + 19
            r0, r1 = max(0, s - FETCH_EXPAND), min(L[ctg], e + FETCH_EXPAND + 1)
            rec, _ = bam_io.read_bam(bam, ctg, s, e, fa_fields=True)
            fres.append(ws.builder.build(rec, cand, bam_io.read_fasta(fa, ctg, r0, r1), r0, matrix_depth=MATRIX_DEPTH[platform],
                                         need_haplotagging=False, min_mq=min_mq, max_indel_length=max_indel, dwell=dwell,
                                         rand_seed=1, rand_skip=0).call(m_f, cfg_f, ctg))
            f_rows += cascade.row_texts(fres[-1], cfg_f)[1]
        merged.append(cascade.merge(res, fres, cfg_p, cfg_f, qual=qual, print_ref=print_ref))
    if not any_bed:
        texts["merge_output"] = texts["pileup"]
        return texts
    f_body = genome.sort_rows(f_rows, names)
    texts["full_alignment"] = genome.vcf_text(head, f_body)
    if not f_body:
        texts["merge_output"] = texts["pileup"]
        return texts
    m_body = genome.sort_rows("".join(merged).splitlines(keepends=True), names)
    texts["merge_output"] = genome.vcf_text(head, m_body)
    if genotyping and m_body:
        texts["merge_output"] = head + "\n" + cascade.add_back_missing(m_body, tgt)
    return texts


def _read_outputs(d):
    out = {}
    for n in ("pileup", "full_alignment", "merge_output"):
        p = os.path.join(d, n + ".vcf.gz")
        if os.path.exists(p):
            out[n] = gzip.open(p, "rt").read()
            tbi = bam_io.read_tbi(p + ".tbi")
            assert tbi["header"] == bam_io.TBI_VCF
            assert tbi["names"] == list(dict.fromkeys(r.split("\t")[0] for r in out[n].split("\n") if r and r[0] != "#"))
    return out


def _targets(kind, seqs):
    rng = np.random.default_rng(7)
    if kind == "bed":
        text = "".join("%s\t%d\t%d\n" % (c, a, a + 400) for c in ("chr1", "chrUn_a") for a in rng.integers(0, 4000, 5))
        return targets.read_bed(text)
    rows = []
    for c in ("chr2", "chr1"):
        for p in np.sort(rng.choice(np.arange(100, 5000), 40, replace=False)):
            rows.append("%s\t%d\t.\t%s\tC\t.\t.\t.\tGT\t0/1\n" % (c, p, seqs[c][p - 1].upper()))
    return targets.read_vcf("".join(rows) + "chr3\t200\t.\tA\tC\t.\t.\t.\tGT\t0/1\n")


CASES = {
    "ont": {},
    "hifi_print_ref": {"platform": "hifi", "print_ref": True},
    "bed": {"tgt": "bed"},
    "known_sites": {"tgt": "vcf"},
    "pileup_only": {"pileup_only": True},
    "pileup_only_print_ref": {"pileup_only": True, "print_ref": True, "qual": 0},
    "no_candidates": {"var_pct": 1e-9, "ref_pct": 1e-9},
    "no_contig": {"ctg_name": "chr3,chr5"},
    "read_filters": {"min_mq": 20, "min_coverage": 4, "call_snp_only": True},
    "long_indel_head_tail": {"long_indel": True, "call_ht": True},
}


def _call_kw(opt):
    return {"platform": opt.get("platform", "ont"), "qual": opt.get("qual", 2), "print_ref_calls": opt.get("print_ref", False),
            "pileup_only": opt.get("pileup_only", False), "var_pct_full": opt.get("var_pct"), "ref_pct_full": opt.get("ref_pct"),
            "ctg_name": opt.get("ctg_name"), "min_mq": opt.get("min_mq", 5), "min_coverage": opt.get("min_coverage", 2),
            "call_snp_only": opt.get("call_snp_only", False), "enable_long_indel": opt.get("long_indel", False),
            "enable_variant_calling_at_sequence_head_and_tail": opt.get("call_ht", False),
            "enable_dwell_time": opt.get("dwell", False)}


@pytest.mark.parametrize("name", sorted(CASES))
def test_call_genome_matches_host_route(ws, models, genome_files, name, tmp_path):
    bam, fa, seqs = genome_files
    opt = dict(CASES[name])
    tgt = _targets(opt.pop("tgt"), seqs) if "tgt" in opt else None
    stats = {}
    want = host_route(ws, models[0], models[1], bam, fa, out_cmd="run --x", tgt=tgt, stats=stats, **opt)
    kw = _call_kw(opt)
    if tgt is not None:
        kw["bed_fn" if tgt.kind == "bed" else "vcf_fn"] = tgt
    res = genome.call_genome(bam, fa, models[0], models[1], str(tmp_path), cmdline="run --x", include_all_ctgs=True,
                             min_contig_size=MIN_SIZE, chunk_size=CHUNK, split_bed_size=SPLIT, workspaces=ws, **kw)
    got = _read_outputs(str(tmp_path))
    assert sorted(got) == sorted(want)
    for n in want:
        assert got[n] == want[n], n
    assert got == res["texts"]
    if name in ("ont", "hifi_print_ref"):
        assert [c for c, _ in res["contigs"]] == ["chr1", "chr2", "chrUn_a"] and len(res["chunks"]) == 10
    if name == "ont":                                 # several bed files per contig, every stage run
        assert res["beds"] >= 6 and stats["repeated"] > 0
        assert res["rows"]["full_alignment"] > 0 and res["rows"]["merge_output"] > 0
        assert {"decode", "pileup", "fa build and call", "merge and format", "write"} <= set(res["stages"])
    if name == "no_candidates":
        assert "full_alignment" not in got and got["merge_output"] == got["pileup"] and res["beds"] == 0
    if name == "no_contig":
        assert list(got) == ["merge_output"] and not genome.has_records(got["merge_output"])


def test_dwell_genome_matches_host_route(ws, tmp_path):
    """ont with ``--enable_dwell_time``: reads with ``mv`` tags, a 9-channel Clair3_F, every bed file's build with the dwell
    channel; the BAM indexed as ``g.bai`` (the name the reference also accepts)."""
    (tmp_path / "in").mkdir()
    bam, fa, _ = make_genome(str(tmp_path / "in"), dwell=True, bai_without_bam=True)
    assert not os.path.exists(bam + ".bai") and os.path.exists(str(tmp_path / "in" / "g.bai"))
    m_p, m_f = _models(fa_channels=9)
    opt = {"dwell": True}
    stats = {}
    want = host_route(ws, m_p, m_f, bam, fa, out_cmd="run --x", stats=stats, **opt)
    res = genome.call_genome(bam, fa, m_p, m_f, str(tmp_path / "out"), cmdline="run --x", include_all_ctgs=True,
                             min_contig_size=MIN_SIZE, chunk_size=CHUNK, split_bed_size=SPLIT, workspaces=ws, **_call_kw(opt))
    got = _read_outputs(str(tmp_path / "out"))
    assert sorted(got) == sorted(want) == ["full_alignment", "merge_output", "pileup"]
    for n in want:
        assert got[n] == want[n], n
    assert res["beds"] >= 6 and res["rows"]["full_alignment"] > 0


def test_refusals(ws, models, genome_files, tmp_path):
    bam, fa, _ = genome_files
    for kw in ({"no_phasing_for_fa": False}, {"gvcf": True}, {"haploid_precise": True}, {"platform": "ilmn"}):
        with pytest.raises(NotImplementedError):
            genome.call_genome(bam, fa, models[0], models[1], str(tmp_path), workspaces=ws, **kw)
    with pytest.raises(ValueError, match="dwell"):
        genome.call_genome(bam, fa, models[0], models[1], str(tmp_path), workspaces=ws, platform="hifi", enable_dwell_time=True)


# ---------------------------------------------------------------------------------------------- world 2
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_worker(rank, world, port, bam, fa, out_dir, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        m_p, m_f = _models(dev)
        res = genome.call_genome(bam, fa, m_p, m_f, out_dir, cmdline="run --x", include_all_ctgs=True, min_contig_size=MIN_SIZE,
                                 chunk_size=CHUNK, split_bed_size=SPLIT, device=dev, group=dist.group.WORLD)
        q.put((rank, res is None))
    finally:
        dist.destroy_process_group()


def test_world_two_writes_the_same_bytes(ws, models, genome_files, tmp_path):
    """Two ranks (two devices when present, otherwise both on device 0 over gloo) write the same files as one."""
    bam, fa, _ = genome_files
    one, two = tmp_path / "one", tmp_path / "two"
    genome.call_genome(bam, fa, models[0], models[1], str(one), cmdline="run --x", include_all_ctgs=True, min_contig_size=MIN_SIZE,
                       chunk_size=CHUNK, split_bed_size=SPLIT, workspaces=ws)
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
    assert names == sorted(os.listdir(two)) and len(names) == 6
    for n in names:
        assert (one / n).read_bytes() == (two / n).read_bytes(), n


# ---------------------------------------------------------------------------------------------- the CLI
def test_cli_writes_what_the_api_writes(ws, models, genome_files, tmp_path):
    bam, fa, _ = genome_files
    mdir = tmp_path / "model"
    mdir.mkdir()
    torch.save({"state_dict": {k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()}},
               mdir / "pileup.pt")
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=8, seed=1).items()},
               mdir / "full_alignment.pt")
    out = tmp_path / "cli"
    cmd = [sys.executable, "-m", "clair3_b200.run_clair3", "--bam_fn", bam, "--ref_fn", fa, "--model_path", str(mdir),
           "--platform", "ont", "--output", str(out), "--threads", "4", "--include_all_ctgs", "True", "--min_contig_size",
           str(MIN_SIZE), "--chunk_size", str(CHUNK), "--no_phasing_for_fa", "True"]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = _read_outputs(str(out))
    api = tmp_path / "api"
    genome.call_genome(bam, fa, models[0], models[1], str(api), include_all_ctgs=True, min_contig_size=MIN_SIZE, chunk_size=CHUNK,
                       workspaces=ws)
    want = _read_outputs(str(api))
    assert sorted(got) == sorted(want) == ["full_alignment", "merge_output", "pileup"]
    for n in want:
        cli_lines = got[n].split("\n")
        cmdline = [x for x in cli_lines if x.startswith("##cmdline=")]
        assert len(cmdline) == 1 and "--no_phasing_for_fa True" in cmdline[0]
        assert [x for x in cli_lines if not x.startswith("##cmdline=")] == want[n].split("\n")
