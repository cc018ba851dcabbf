"""Clair3's whole-genome run, from an indexed BAM and an indexed FASTA to ``pileup.vcf.gz``, ``full_alignment.vcf.gz`` and
``merge_output.vcf.gz`` (DESIGN.md 5g).

The reference's ``run_clair3.py`` runs ``scripts/clair3_c_impl_pipeline.py``; with ``--no_phasing_for_fa True`` that is
CheckEnvs, one pileup call per CHUNK_LIST row, SortVcf, SelectQual, SelectCandidates per contig, one full-alignment call per
bed file, SortVcf, MergeVcf per contig, SortVcf and, with ``--vcf_fn``, AddBackMissingVariantsInGenotyping.  Here:

* ``plan`` is CheckEnvs: the contigs to call and the CHUNK_LIST;
* ``header``, ``sort_rows`` and ``vcf_text`` are SortVcf's file text, ``write_vcf_gz`` its ``bgzip`` and ``tabix -p vcf``;
* ``exchange`` takes every pileup chunk's rows to the genome-wide decisions: the duplicate rows of overlapping chunks dropped
  as SortVcf drops them, SelectQual's cut-offs (``qual_cutoffs_from``) and SelectCandidates' bed files (``candidates_from``);
* ``call_genome`` runs it all on one ``cascade.Workspaces``, on one GPU or, with a ``torch.distributed`` group, one process per
  GPU: contiguous runs of pileup chunks and of bed files per rank, with only the rows' (position, probability, flags) sent to
  every rank and the row texts sent to rank 0, which writes the files.

Each bed file's build starts a fresh ``rand()`` stream, as each of the reference's full-alignment calls is a process of its
own, and a site's network output does not depend on the sites it is batched with (DESIGN.md 8): the files do not depend on
the number of ranks.

Not implemented: phasing (``no_phasing_for_fa`` must be True: WhatsHap / LongPhase are not part of this project), gVCF, the
haploid modes and ``platform="ilmn"`` (``NotImplementedError``); CRAM input and CSI indexes (``NotImplementedError``).
"""
from __future__ import annotations

import os
import time

import numpy as np
import torch

from . import bam_io, cascade, decode
from .fa_tensor import MATRIX_DEPTH
from .pileup_counts import FETCH_EXPAND, bed_chunk_region, chunk_region, counting_region, known_sites_chunk
from .sharding import site_range

CHUNK_SIZE = 5_000_000                # CheckEnvs --chunk_size
CLAIR3_VERSION = "2.0.2"              # shared/version.py: the ##clair3_version line of the reference this project restates
LONG_INDEL = 100000                   # shared/param_{p,f}.py maximum_variant_length_that_need_infer_include_long_indel

_FLAG_GT00, _FLAG_REF = 1, 2          # per pileup row: GT prints 0/0 (SelectQual's split), ALT is "." or REF (SelectCandidates')


# ------------------------------------------------------------------------------------------------ options
def resolve_options(platform="ont", var_pct_full=None, ref_pct_full=None, snp_min_af=None, indel_min_af=None, genotyping=False):
    """run_clair3.py's per-platform defaults (:303-321, :393-395): (var_pct_full, ref_pct_full, snp_min_af, indel_min_af), where
    None or 0 means the platform's value, and a known-sites VCF sets both allele-frequency thresholds to 0."""
    cascade._check_platform(platform)
    var = var_pct_full or cascade.PCT_FULL[platform][0]
    ref = ref_pct_full or cascade.PCT_FULL[platform][1]
    snp = snp_min_af or 0.08
    indel = indel_min_af or (0.15 if platform == "ont" else 0.08)
    if genotyping:
        snp = indel = 0.0
    return var, ref, snp, indel


def output_configs(enable_long_indel=False):
    """The two decoders' OutputConfig as the pipeline's CallVariantsFromCffi runs them: showRef on, ``--qual`` at its default 2
    (the pipeline passes none), ``--add_indel_length`` for full alignment only, and the long-indel limit."""
    out = []
    for pileup in (True, False):
        cfg = decode.replay_config(pileup=pileup, add_indel_length=not pileup)._replace(is_show_reference=True)
        if enable_long_indel:
            cfg = cfg._replace(enable_long_indel=True, maximum_variant_length_that_need_infer=LONG_INDEL)
        out.append(cfg)
    return tuple(out)


# ------------------------------------------------------------------------------------------------ CheckEnvs
def _targets(bed=None, known_sites=None):
    from . import targets as tg
    if bed is not None and known_sites is not None:
        raise ValueError("genome: give either a BED or a known-sites VCF, not both (CheckEnvs refuses --bed_fn with --vcf_fn)")
    if bed is not None:
        return bed if isinstance(bed, tg.Targets) else tg.read_bed(bed)
    if known_sites is not None:
        return known_sites if isinstance(known_sites, tg.Targets) else tg.read_vcf(known_sites)
    return None


def bam_index(bam_fn):
    """The ``.bai`` of a BAM as run_clair3.py and the pipeline look for it (clair3_c_impl_pipeline.py:366-382):
    ``<bam>.bai``, else ``<bam without its extension>.bai``; None when neither exists."""
    for p in (str(bam_fn) + ".bai", os.path.splitext(str(bam_fn))[0] + ".bai"):
        if os.path.exists(p):
            return p
    return None


def check_inputs(bam_fn, ref_fn):
    """The files CheckEnvs and run_clair3.py require: the BAM with a ``.bai`` (``bam_index``) and the FASTA with a ``.fai``.
    CRAM input and a BAM indexed only by a ``.csi`` are not supported here (NotImplementedError).  Returns the ``.bai`` path."""
    bam_fn, ref_fn = str(bam_fn), str(ref_fn)
    if bam_fn.endswith(".cram"):
        raise NotImplementedError("genome: CRAM input is not supported; give a BAM")
    for p in (bam_fn, ref_fn):
        if not os.path.exists(p):
            raise FileNotFoundError("genome: %s not found" % p)
    if not os.path.exists(ref_fn + ".fai"):
        raise FileNotFoundError("genome: reference index %s.fai not found (samtools faidx the FASTA first)" % ref_fn)
    bai = bam_index(bam_fn)
    if bai is None:
        if os.path.exists(bam_fn + ".csi") or os.path.exists(os.path.splitext(bam_fn)[0] + ".csi"):
            raise NotImplementedError("genome: CSI indexes are not supported; index the BAM with a .bai")
        raise FileNotFoundError("genome: BAM index %s.bai not found (samtools index the BAM first)" % bam_fn)
    with open(ref_fn, "rb") as f:
        if f.read(2) == b"\x1f\x8b":
            raise ValueError("genome: compressed FASTA is not supported; decompress %s and index it" % ref_fn)
    return bai


def plan(bam_fn, ref_fn, ctg_name=None, include_all_ctgs=False, min_contig_size=0, chunk_size=CHUNK_SIZE, bed=None,
         known_sites=None, idxstats=None):
    """CheckEnvs (preprocess/CheckEnvs.py:180-389): returns (contigs [(name, length)], CHUNK_LIST [(name, chunk_id,
    chunk_num)]).  The contigs come from the FASTA's ``.fai``; without ``include_all_ctgs``, ``ctg_name`` (comma-separated),
    a BED or a known-sites VCF only chr1..22,X,Y / 1..22,X,Y are kept; ``ctg_name`` intersects with the BED's or VCF's contigs,
    without it the run takes their union; contigs shorter than ``min_contig_size`` and contigs without mapped reads (the
    ``.bai`` pseudo-bin, ``samtools idxstats``) are dropped; ``chunk_num = ceil(length / chunk_size)``, at least 1.  The major
    contigs come first in their order, the others in ``.fai`` order (the reference takes a set's iteration order there, which
    changes from run to run).  A contig named by ``ctg_name``, the BED or the VCF but absent from the ``.fai`` is dropped
    (the reference keeps it and then fails writing the CHUNK_LIST).  ``idxstats``: ``bam_io.idxstats``' rows, read from the
    BAM's index (``bam_index``) by default."""
    bai = check_inputs(bam_fn, ref_fn)
    tgt = _targets(bed, known_sites)
    names = [n for n in (ctg_name.split(",") if ctg_name and ctg_name != "EMPTY" else []) if n]
    given = bool(names)
    wanted = set(names)
    if tgt is not None:
        tc = set(tgt.intervals)              # CheckEnvs: the BED tree's contigs / the contigs split_extend_vcf wrote
        wanted = wanted & tc if given else wanted | tc
    restricted = given or tgt is not None
    kept = []
    for name, length, *_ in bam_io.read_fai(str(ref_fn) + ".fai"):
        if not include_all_ctgs and not restricted and name not in cascade.MAJOR_CONTIGS:
            continue
        if restricted and name not in wanted:
            continue
        if min_contig_size > 0 and length < min_contig_size:
            continue
        kept.append((name, length))
    mapped = {r[0]: r[2] for r in (idxstats if idxstats is not None else bam_io.idxstats(bam_fn, bai))}
    kept = [c for c in kept if mapped.get(c[0], 0) > 0]
    major = [c for m in cascade.MAJOR_CONTIGS for c in kept if c[0] == m]
    contigs = major + [c for c in kept if c[0] not in cascade.MAJOR_CONTIGS]
    chunks = []
    for name, length in contigs:
        n = max(length // chunk_size + (1 if length % chunk_size else 0), 1)
        chunks.extend((name, i, n) for i in range(1, n + 1))
    return contigs, chunks


# ------------------------------------------------------------------------------------------------ SortVcf and the files
_HEADER = """##fileformat=VCFv4.2
##source=Clair3
##clair3_version={}
##FILTER=<ID=PASS,Description="All filters passed">
##FILTER=<ID=LowQual,Description="Low quality variant">
##FILTER=<ID=RefCall,Description="Reference call">
##INFO=<ID=P,Number=0,Type=Flag,Description="Result from pileup calling">
##INFO=<ID=F,Number=0,Type=Flag,Description="Result from full-alignment calling">
##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">
##FORMAT=<ID=GQ,Number=1,Type=Integer,Description="Genotype Quality">
##FORMAT=<ID=DP,Number=1,Type=Integer,Description="Approximate read depth (reads 1. with MQ below 5 or an user-specified threshold, or 2. selected by 'samtools view -F 2316', are filtered)">
##FORMAT=<ID=AD,Number=R,Type=Integer,Description="Allelic depths for the ref and alt alleles in the order listed">
##FORMAT=<ID=PL,Number=G,Type=Integer,Description="Normalized, Phred-scaled likelihoods for genotypes as defined in the VCF specification">
##FORMAT=<ID=AF,Number=A,Type=Float,Description="Observed allele frequency in reads, for each ALT allele, in the same order as listed, or the REF allele for a RefCall">"""


def header(ref_fn, sample_name="SAMPLE", cmdline=None, fai=None):
    """``shared/utils.py:get_header`` (no gVCF): the fixed lines, ``##reference=<ref_fn as given>`` and ``##cmdline=`` (when
    ``cmdline`` is not empty, trailing white space removed) inserted at index 3, one ``##contig`` line per ``.fai`` row
    (default ``ref_fn + ".fai"``) and the ``#CHROM`` line, without a final newline."""
    lines = _HEADER.format(CLAIR3_VERSION).split("\n")
    lines.insert(3, "##reference=%s" % ref_fn)
    cmd = (cmdline or "").rstrip()
    if cmd:
        lines.insert(3, "##cmdline=%s" % cmd)
    text = "\n".join(lines) + "\n"
    with open(fai or str(ref_fn) + ".fai") as f:
        for row in f:
            c = row.strip().split("\t")
            text += "##contig=<ID=%s,length=%s>\n" % (c[0], c[1])
    return text + "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\t%s" % sample_name


def sort_rows(rows, contigs):
    """SortVcf's body (preprocess/SortVcf.py:sort_vcf_from): rows keyed by (contig, position), the last of a duplicate key
    kept; the contigs of ``contigs`` (the CONTIGS list) in its order with the major contigs first, positions ascending; rows of
    other contigs are left out."""
    by = {}
    for row in rows:
        c = row.strip().split(maxsplit=3)
        by.setdefault(c[0], {})[int(c[1])] = row
    names = list(contigs)
    order = sorted(names, key=(cascade.MAJOR_CONTIGS + names).index)
    return "".join(by[c][p] for c in order if c in by for p in sorted(by[c]))


def vcf_text(head, body, had_rows=None):
    """A VCF file's text as SortVcf leaves it: the header of the per-chunk files and the body, or - when its inputs held no
    row at all (``had_rows`` False; default: the body is empty) - ``output_header``'s header alone, without a final newline."""
    had_rows = bool(body) if had_rows is None else had_rows
    return head + "\n" + body if had_rows else head


def _records(text):
    return sum(1 for line in text.split("\n") if line and line[0] != "#")


def has_records(text):
    """``vcf_has_records``: some line does not start with ``#``."""
    return _records(text) > 0


def write_vcf_gz(path, text):
    """``bgzip -f`` and ``tabix -p vcf``: ``path`` (ending in ``.vcf.gz``) and ``path.tbi``."""
    voff = bam_io.write_bgzf(path, text)
    bam_io.write_tbi(path, text, voff)
    return path


# ------------------------------------------------------------------------------------------------ the genome-wide decisions
def qual_cutoffs_from(prob, gt00, platform="ont", var_pct_full=None, ref_pct_full=None, genotyping=False):
    """``cascade.qual_cutoffs`` on the (probability, GT is 0/0) pairs of every pileup row of the genome."""
    cascade._check_platform(platform)
    var_pct = cascade.PCT_FULL[platform][0] if var_pct_full is None else var_pct_full
    ref_pct = cascade.PCT_FULL[platform][1] if ref_pct_full is None else ref_pct_full
    if not genotyping:
        ref_pct = ref_pct if ref_pct else var_pct
    prob, gt00 = np.asarray(prob, np.float32), np.asarray(gt00, bool)
    return cascade._kth_qual([prob[~gt00]], var_pct), cascade._kth_qual([prob[gt00]], ref_pct)


def candidates_from(pos, prob, is_ref, var_qual, ref_qual):
    """``cascade.select``'s positions on one contig's pileup rows (1-based positions, probabilities, ALT is "." or REF): 0-based,
    sorted and unique."""
    bits = np.asarray(prob, np.float32).view(np.uint32).astype(np.int64)
    t = np.where(np.asarray(is_ref, bool), cascade.prob_threshold(ref_qual), cascade.prob_threshold(var_qual))
    return np.unique(np.asarray(pos, np.int64)[bits < t] - 1).astype(np.int64)


def row_summary(res):
    """(1-based positions, probabilities, flags, row indices) of a pileup ``call`` result's VCF rows: what the other ranks need
    of them."""
    idx = cascade._rows(res)
    c = res["calls"][idx]
    flags = np.where(c["genotype"] == 0, _FLAG_GT00, 0) | np.where(cascade._is_reference(res, idx), _FLAG_REF, 0)
    return np.asarray(res["position"])[idx].astype(np.int64), c["prob"].astype(np.float32), flags.astype(np.uint8), idx


def exchange(chunk_rows, contigs, platform="ont", var_pct_full=None, ref_pct_full=None, genotyping=False,
             split_bed_size=cascade.SPLIT_BED_SIZE):
    """The genome-wide decisions from every pileup chunk's rows.  ``chunk_rows``: per CHUNK_LIST row, in its order, (contig,
    positions, probabilities, flags) as ``row_summary`` gives them.  Returns (keep: per chunk a bool mask of its rows that
    pileup.vcf keeps - of a position repeated by overlapping chunks the last chunk's row, as SortVcf keeps it -, (var_qual,
    ref_qual), beds: [(contig, 0-based candidate positions)] per bed file, in contig order).  The rows a position repeats are
    identical except under head / tail calling, where a candidate near a chunk's edge gets a padded window in one chunk and a
    whole one in the next; the reference then keeps whichever file ``os.listdir`` lists last, which has no fixed order, and
    this route keeps the last chunk's row."""
    keep = [np.zeros(len(r[1]), bool) for r in chunk_rows]
    for ctg in {r[0] for r in chunk_rows}:
        gs = [g for g, r in enumerate(chunk_rows) if r[0] == ctg]
        pos = np.concatenate([np.asarray(chunk_rows[g][1], np.int64) for g in gs])
        src = np.concatenate([np.full(len(chunk_rows[g][1]), j, np.int64) for j, g in enumerate(gs)])
        row = np.concatenate([np.arange(len(chunk_rows[g][1])) for g in gs])
        order = np.lexsort((src, pos))                       # by position, then chunk: the last of each position wins
        last = np.ones(len(order), bool)
        last[:-1] = pos[order][1:] != pos[order][:-1]
        for j, g in enumerate(gs):
            hit = order[last & (src[order] == j)]
            keep[g][row[hit]] = True
    cat = lambda k: np.concatenate([np.asarray(r[k])[m] for r, m in zip(chunk_rows, keep)]) if chunk_rows else np.zeros(0)  # noqa: E731
    prob, flags = cat(2).astype(np.float32), cat(3).astype(np.uint8)
    cuts = qual_cutoffs_from(prob, flags & _FLAG_GT00, platform, var_pct_full, ref_pct_full, genotyping)
    beds = []
    for ctg in [c for c, _ in contigs]:
        sel = [(np.asarray(r[1])[m], np.asarray(r[2])[m], np.asarray(r[3])[m]) for r, m in zip(chunk_rows, keep) if r[0] == ctg]
        if not sel:
            continue
        pos = candidates_from(np.concatenate([s[0] for s in sel]), np.concatenate([s[1] for s in sel]).astype(np.float32),
                              np.concatenate([s[2] for s in sel]) & _FLAG_REF, *cuts)
        beds.extend((ctg, pos[a:b]) for a, b in cascade._chunks(len(pos), split_bed_size))
    return keep, cuts, beds


def decisions(mine, contigs, platform="ont", var_pct_full=None, ref_pct_full=None, genotyping=False,
              split_bed_size=cascade.SPLIT_BED_SIZE, group=None):
    """``exchange`` across the ranks of ``group`` (None: this process alone): ``mine`` holds this rank's pileup chunks as
    (CHUNK_LIST index, contig, positions, probabilities, flags); every rank gathers every chunk's arrays - no row text - and
    takes the same decisions.  Returns ``exchange``'s (keep per CHUNK_LIST row, cut-offs, bed files)."""
    world = _rank(group)[1]
    every = sorted((m for part in _all_gather(list(mine), group, world) for m in part), key=lambda m: m[0])
    return exchange([m[1:] for m in every], contigs, platform, var_pct_full, ref_pct_full, genotyping, split_bed_size)


def postprocess_pileup(body, qual=2, print_ref=False):
    """SortVcf's ``--pileup_only`` post-processing of a sorted pileup body: MarkLowQual on the variant rows, the reference rows
    (ALT "." or REF) only with ``print_ref`` (``cascade.merge_rows`` without full-alignment rows)."""
    by = {}
    for row in body.splitlines(keepends=True):
        by.setdefault(row.split("\t", 1)[0], []).append(row)
    return "".join(cascade.merge_rows([int(r.split("\t", 2)[1]) for r in rows], rows, [], [], qual=qual, print_ref=print_ref)
                   for rows in by.values())


def bed_span(positions):
    """The 0-based [start, end) the reference's full-alignment call reads for one bed file
    (preprocess/CreateTensorFullAlignmentFromCffi.py:60-115): its rows ``max(p - 16, 0) p + 18`` give the 1-based
    ``ctg_start = min(start) + 1`` and ``ctg_end = max(end) + 1``, and the region string ``ctg:ctg_start-ctg_end`` is
    [ctg_start - 1, ctg_end)."""
    p = np.asarray(positions, np.int64)
    return max(int(p.min()) - cascade.FLANK, 0), int(p.max()) + cascade.FLANK + 3


def pileup_chunk_region(ctg, length, chunk_id, chunk_num, tgt=None):
    """(counting [start, end), ContigTargets or None) of one CHUNK_LIST row, or None when the reference skips it (an empty
    known-sites slice): ``chunk_region`` without targets, ``bed_chunk_region`` over the extended BED's span with a BED, and the
    known-sites slice (``known_sites_chunk``) in genotyping mode."""
    if tgt is None:
        return counting_region(*chunk_region(length, chunk_id, chunk_num)), None
    if tgt.kind == "bed":
        ct = tgt.contig(ctg)
        if ct.bed_region() is None:
            return None
        return counting_region(*bed_chunk_region(*ct.bed_region(), chunk_id, chunk_num)), ct
    c = known_sites_chunk(tgt.sites.get(ctg, np.zeros(0, np.int64)), chunk_id, chunk_num)
    if c is None:
        return None
    return counting_region(c[0], c[1]), tgt.contig(ctg, chunk=(chunk_id, chunk_num))


# ------------------------------------------------------------------------------------------------ the route
class _StageClock:
    """``cascade._Stages`` summed per stage name over a whole run."""

    def __init__(self, device):
        self.st = cascade._Stages(device)
        self.t0 = time.perf_counter()

    def mark(self, name):
        self.st.mark(name)

    def report(self):
        out = {}
        for r in self.st.report():
            s = out.setdefault(r["stage"], {"wall_ms": 0.0, "device_ms": 0.0, "count": 0})
            s["wall_ms"] += r["wall_ms"]
            s["device_ms"] += r["device_ms"]
            s["count"] += 1
        out["total"] = {"wall_ms": 1e3 * (time.perf_counter() - self.t0)}
        return out


def _rank(group):
    if group is None:
        return 0, 1
    import torch.distributed as dist
    return dist.get_rank(group), dist.get_world_size(group)


def _all_gather(obj, group, world):
    if world == 1:
        return [obj]
    import torch.distributed as dist
    out = [None] * world
    dist.all_gather_object(out, obj, group=group)
    return out


def _gather0(obj, group, world, rank):
    if world == 1:
        return [obj]
    import torch.distributed as dist
    out = [None] * world if rank == 0 else None
    dist.gather_object(obj, out, dst=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    return out


def call_genome(bam_fn, ref_fn, model_p, model_f, out_dir, platform="ont", sample_name="SAMPLE", cmdline=None, ctg_name=None,
                include_all_ctgs=False, min_contig_size=0, chunk_size=CHUNK_SIZE, bed_fn=None, vcf_fn=None, qual=2,
                var_pct_full=None, ref_pct_full=None, snp_min_af=None, indel_min_af=None, min_mq=5, min_coverage=2,
                call_snp_only=False, enable_long_indel=False, enable_variant_calling_at_sequence_head_and_tail=False,
                print_ref_calls=False, pileup_only=False, no_phasing_for_fa=True, enable_dwell_time=False, gvcf=False,
                haploid_precise=False, haploid_sensitive=False, split_bed_size=cascade.SPLIT_BED_SIZE, workspaces=None,
                device=None, group=None, k=16):
    """Clair3's pipeline (scripts/clair3_c_impl_pipeline.py with ``--no_phasing_for_fa True``) over the genome: writes
    ``pileup.vcf.gz``, ``full_alignment.vcf.gz`` and ``merge_output.vcf.gz`` with their ``.tbi`` into ``out_dir``, as the
    reference does with its early exits (no contig: a header-only ``merge_output``; no pileup row, no full-alignment
    candidate or no full-alignment row: ``merge_output`` is a copy of ``pileup.vcf.gz``; ``pileup_only``: ``pileup.vcf.gz``
    alone).  Options as run_clair3.py names them (None / 0 percentages and allele frequencies: the platform's defaults, see
    ``resolve_options``); ``bed_fn`` / ``vcf_fn`` also take ``targets.read_bed`` / ``read_vcf`` results.  ``cmdline``: the
    ``##cmdline=`` header line (None: none).  ``chunk_size`` / ``split_bed_size``: CheckEnvs' and SelectCandidates' sizes.
    ``group``: a ``torch.distributed`` process group (one process per GPU, each on its own ``device``); every rank must call
    with the same arguments.  ``model_p`` / ``model_f``: Clair3_P and Clair3_F on this rank's device.

    Returns, on rank 0, a dict: ``files`` {name: path}, ``texts`` {name: decompressed text}, ``contigs``, ``chunks``,
    ``qual_cutoffs``, ``beds`` (number of bed files), ``rows`` {name: row count}, ``stages`` (wall and device ms per stage,
    this rank's); None on the other ranks."""
    if no_phasing_for_fa is not True:
        raise NotImplementedError("genome: phasing for full alignment (WhatsHap / LongPhase) is not implemented; "
                                  "run with no_phasing_for_fa=True")
    if gvcf:
        raise NotImplementedError("genome: gVCF output is not implemented")
    if haploid_precise or haploid_sensitive:
        raise NotImplementedError("genome: the haploid modes are not implemented")
    cascade._check_platform(platform)
    if enable_dwell_time and platform != "ont":
        raise ValueError("genome: dwell time is only supported for platform 'ont' (run_clair3.py refuses it too)")
    tgt = _targets(bed_fn, vcf_fn)
    genotyping = tgt is not None and tgt.kind == "vcf"
    var_pct, ref_pct, snp_af, indel_af = resolve_options(platform, var_pct_full, ref_pct_full, snp_min_af, indel_min_af, genotyping)
    cfg_p, cfg_f = output_configs(enable_long_indel)
    max_indel = LONG_INDEL if enable_long_indel else decode.MAX_INFER_LENGTH
    rank, world = _rank(group)
    contigs, chunks = plan(bam_fn, ref_fn, ctg_name, include_all_ctgs, min_contig_size, chunk_size,
                           bed=tgt if tgt is not None and tgt.kind == "bed" else None, known_sites=tgt if genotyping else None)
    out_dir = str(out_dir)
    paths = {n: os.path.join(out_dir, n + ".vcf.gz") for n in ("pileup", "full_alignment", "merge_output")}
    head = header(ref_fn, sample_name, cmdline)
    texts = {}

    def finish(stages=None):
        if rank != 0:
            return None
        os.makedirs(out_dir, exist_ok=True)
        for name, text in texts.items():
            write_vcf_gz(paths[name], text)
        return {"files": {n: paths[n] for n in texts}, "texts": dict(texts), "contigs": contigs, "chunks": chunks,
                "qual_cutoffs": cuts, "beds": len(beds), "rows": {n: _records(t) for n, t in texts.items()},
                "stages": stages}

    cuts, beds = None, []
    if not contigs:
        texts["merge_output"] = head
        return finish()
    own = workspaces is None
    if device is None:
        device = workspaces.counter._device if workspaces is not None else torch.cuda.current_device()
    ws = workspaces or cascade.Workspaces(device)
    dev = ws.counter._device
    lengths = dict(contigs)
    index = bam_io.read_bai(bam_index(bam_fn))          # parsed once; the decoder reads each region's byte range through it
    try:
        clock = _StageClock(dev)
        # ---- pileup: a contiguous run of CHUNK_LIST rows per rank
        lo, hi = site_range(len(chunks), rank, world)
        mine = []
        for g in range(lo, hi):
            ctg, cid, n = chunks[g]
            region = pileup_chunk_region(ctg, lengths[ctg], cid, n, tgt)
            if region is None:
                mine.append((g, ctg, np.zeros(0, np.int64), np.zeros(0, np.float32), np.zeros(0, np.uint8), []))
                continue
            (start, end), ct = region
            r0, r1 = max(0, start - FETCH_EXPAND), min(lengths[ctg], end + FETCH_EXPAND + 1)
            ref = bam_io.fetch_fasta(ref_fn, ctg, r0, r1)
            rec = ws.decoder.decode(bam_fn, ctg, start, end, fa_fields=False, index=index,
                                    ref_seq=torch.from_numpy(np.frombuffer(ref.encode(), np.uint8).copy()).to(dev))
            clock.mark("decode")
            res = ws.counter.count(rec, start, end, None, r0, min_depth=min_coverage, min_snp_af=snp_af, min_indel_af=indel_af,
                                   min_mq=min_mq, call_snp_only=call_snp_only,
                                   call_ht=enable_variant_calling_at_sequence_head_and_tail, alt_info=True,
                                   max_indel_length=max_indel, targets=ct).call(model_p, cfg_p, ctg, k=k)
            clock.mark("pileup")
            pos, prob, flags, idx = row_summary(res)
            rows = [decode.call_row(res, s, cfg_p) for s in idx]
            mine.append((g, ctg, pos, prob, flags, rows))
            del rec, res
            clock.mark("pileup format")
        # ---- every rank: the rows' positions, probabilities and flags -> duplicates, cut-offs, bed files
        keep, cuts, beds = decisions([m[:5] for m in mine], contigs, platform, var_pct, ref_pct, genotyping, split_bed_size, group)
        clock.mark("cutoffs and select")
        n_rows = sum(int(m.sum()) for m in keep)
        # ---- full alignment: a contiguous run of bed files per rank
        fa_rows = []
        if n_rows and not pileup_only:
            b0, b1 = site_range(len(beds), rank, world)
            fa = {"matrix_depth": MATRIX_DEPTH[platform], "need_haplotagging": False, "min_mq": min_mq,
                  "max_indel_length": max_indel, "dwell": bool(enable_dwell_time), "rand_seed": 1, "rand_skip": 0}
            for b in range(b0, b1):
                ctg, cand = beds[b]
                s, e = bed_span(cand)
                r0, r1 = max(0, s - FETCH_EXPAND), min(lengths[ctg], e + FETCH_EXPAND + 1)
                ref = bam_io.fetch_fasta(ref_fn, ctg, r0, r1)
                rec = ws.decoder.decode(bam_fn, ctg, s, e, fa_fields=True, index=index,
                                        ref_seq=torch.from_numpy(np.frombuffer(ref.encode(), np.uint8).copy()).to(dev))
                clock.mark("fa decode")
                res = ws.builder.build(rec, cand, None, r0, **fa).call(model_f, cfg_f, ctg, k=k)
                clock.mark("fa build and call")
                pos, rows = cascade._vcf(res, cfg_f)
                fa_rows.append((b, ctg, pos, rows))
                del rec, res
                clock.mark("fa format")
        # ---- rank 0: the row texts
        kept = [(g, ctg, pos[keep[g]], [r for r, k_ in zip(rows, keep[g]) if k_]) for g, ctg, pos, _, _, rows in mine]
        parts = _gather0((kept, fa_rows), group, world, rank)
        clock.mark("gather")
        if rank != 0:
            return None
        p_chunks = sorted((c for part in parts for c in part[0]), key=lambda c: c[0])
        f_beds = sorted((c for part in parts for c in part[1]), key=lambda c: c[0])
        names = [c for c, _ in contigs]
        p_body = sort_rows((r for c in p_chunks for r in c[3]), names)
        if not n_rows:
            texts["pileup"] = texts["merge_output"] = head                   # SortVcf: no variant found
        elif pileup_only:
            texts["pileup"] = vcf_text(head, postprocess_pileup(p_body, qual, print_ref_calls), True)
            if not has_records(texts["pileup"]):
                texts["merge_output"] = texts["pileup"]
        else:
            texts["pileup"] = vcf_text(head, p_body, True)
            if beds:
                f_body = sort_rows((r for c in f_beds for r in c[3]), names)
                texts["full_alignment"] = vcf_text(head, f_body, bool(f_body))
            if not beds or not has_records(texts["full_alignment"]):
                texts["merge_output"] = texts["pileup"]                      # ensure_merge_output
            else:
                merged = sort_rows("".join(_merge_contig(p_chunks, f_beds, ctg, qual, print_ref_calls) for ctg in names)
                                   .splitlines(keepends=True), names)
                texts["merge_output"] = vcf_text(head, merged, bool(merged))
                if genotyping and merged:
                    texts["merge_output"] = head + "\n" + cascade.add_back_missing(merged, tgt)
        clock.mark("merge and format")
        out = finish()
        clock.mark("write")
        out["stages"] = clock.report()
        return out
    finally:
        if own:
            ws.close()


def _merge_contig(p_chunks, f_beds, ctg, qual, print_ref):
    """MergeVcf of one contig on row text: its pileup rows (as pileup.vcf holds them: unique, by position) and its bed files'
    full-alignment rows."""
    p = {}
    for c in p_chunks:
        if c[1] == ctg:
            p.update(zip(np.asarray(c[2]).tolist(), c[3]))
    p_pos = sorted(p)
    f_pos, f_rows = [], []
    for c in f_beds:
        if c[1] == ctg:
            f_pos.extend(np.asarray(c[2]).tolist())
            f_rows.extend(c[3])
    return cascade.merge_rows(p_pos, [p[x] for x in p_pos], f_pos, f_rows, qual=qual, print_ref=print_ref)
