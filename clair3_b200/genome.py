"""Clair3's whole-genome run, from an indexed BAM and an indexed FASTA to ``pileup.vcf.gz``, ``full_alignment.vcf.gz`` and
``merge_output.vcf.gz`` (DESIGN.md 5g).

The reference's ``run_clair3.py`` runs ``scripts/clair3_c_impl_pipeline.py``; with ``--no_phasing_for_fa True`` that is
CheckEnvs, one pileup call per CHUNK_LIST row, SortVcf, SelectQual, SelectCandidates per contig, one full-alignment call per
bed file, SortVcf, MergeVcf per contig, SortVcf and, with ``--vcf_fn``, AddBackMissingVariantsInGenotyping.  Here:

* ``plan`` is CheckEnvs: the contigs to call and the CHUNK_LIST;
* ``header``, ``sort_rows`` and ``vcf_text`` are SortVcf's file text, ``write_vcf_gz`` its ``bgzip`` and ``tabix -p vcf``;
* ``exchange`` takes every pileup chunk's rows to the genome-wide decisions: the duplicate rows of overlapping chunks dropped
  as SortVcf drops them, SelectQual's cut-offs (``cascade.qual_cutoffs_from``) and SelectCandidates' bed files
  (``cascade.candidates_from``);
* ``file_texts`` turns the rows of the whole run into the files' texts: SortVcf, MergeVcf, the add-back and the early exits;
* ``call_genome`` runs it all on one ``cascade.Workspaces``, on one GPU or, with a ``torch.distributed`` group, one process per
  GPU: contiguous runs of pileup chunks and of bed files per rank, with only the rows' (position, probability, flags) sent to
  every rank and the row texts sent to rank 0, which writes the files.

Each bed file's build starts a fresh ``rand()`` stream, as each of the reference's full-alignment calls is a process of its
own, and a site's network output does not depend on the sites it is batched with (DESIGN.md 8): the files do not depend on
the number of ranks.

With ``enable_phasing`` the merged calls are phased on the GPU after MergeVcf (``clair3_b200.phasing``, DESIGN.md 5g.3) into
``phased_merge_output.vcf.gz``: the phase sets come from WhatsHap's model (all-heterozygous wMEC, coverage cap 15), but the
file is not WhatsHap's byte for byte.

Not implemented: phasing for full alignment (``no_phasing_for_fa`` must be True: WhatsHap / LongPhase are not part of this
project), gVCF, the haploid modes and ``platform="ilmn"`` (``NotImplementedError``); CRAM input and CSI indexes
(``NotImplementedError``).  The reference FASTA may be bgzip-compressed with its ``.gzi`` (DESIGN.md 5g.1): each window is then
inflated on the GPU.
"""
from __future__ import annotations

import functools
import os

import numpy as np
import torch

from . import bam_io, cascade, decode, phasing, targets
from .fa_tensor import MATRIX_DEPTH
from .pileup_counts import FETCH_EXPAND, bed_chunk_region, chunk_region, counting_region, known_sites_chunk
from .sharding import site_range

CHUNK_SIZE = 5_000_000                # CheckEnvs --chunk_size
CLAIR3_VERSION = "2.0.2"              # shared/version.py: the ##clair3_version line of the reference this project restates
LONG_INDEL = 100000                   # shared/param_{p,f}.py maximum_variant_length_that_need_infer_include_long_indel

row_summary = cascade.row_summary     # where earlier callers find it


# ------------------------------------------------------------------------------------------------ options
def resolve_options(platform="ont", var_pct_full=None, ref_pct_full=None, snp_min_af=None, indel_min_af=None, genotyping=False):
    """run_clair3.py's per-platform defaults (:303-321, :393-395): (var_pct_full, ref_pct_full, snp_min_af, indel_min_af), where
    None or 0 means the platform's value, and a known-sites VCF sets both allele-frequency thresholds to 0."""
    cascade.check_platform(platform)
    var = var_pct_full or cascade.PCT_FULL[platform][0]
    ref = ref_pct_full or cascade.PCT_FULL[platform][1]
    snp = snp_min_af or 0.08
    indel = indel_min_af or (0.15 if platform == "ont" else 0.08)
    if genotyping:
        snp = indel = 0.0
    return var, ref, snp, indel


def output_configs(enable_long_indel=False, keep_iupac_bases=False):
    """The two decoders' OutputConfig as the pipeline's CallVariantsFromCffi runs them: showRef on, ``--qual`` at its default 2
    (the pipeline passes none), ``--add_indel_length`` for full alignment only, the long-indel limit and
    ``--keep_iupac_bases``, which both calls take."""
    out = []
    for pileup in (True, False):
        cfg = decode.replay_config(pileup=pileup, add_indel_length=not pileup)._replace(is_show_reference=True,
                                                                                        keep_iupac_bases=bool(keep_iupac_bases))
        if enable_long_indel:
            cfg = cfg._replace(enable_long_indel=True, maximum_variant_length_that_need_infer=LONG_INDEL)
        out.append(cfg)
    return tuple(out)


# ------------------------------------------------------------------------------------------------ CheckEnvs
def bam_index(bam_fn):
    """The ``.bai`` of a BAM as run_clair3.py and the pipeline look for it (clair3_c_impl_pipeline.py:366-382):
    ``<bam>.bai``, else ``<bam without its extension>.bai``; None when neither exists."""
    for p in (str(bam_fn) + ".bai", os.path.splitext(str(bam_fn))[0] + ".bai"):
        if os.path.exists(p):
            return p
    return None


def check_inputs(bam_fn, ref_fn):
    """The files CheckEnvs and run_clair3.py require: the BAM with a ``.bai`` (``bam_index``) and the FASTA with a ``.fai`` -
    plain, or bgzip-compressed with its ``.gzi`` too, as ``samtools faidx`` indexes it.  CRAM input and a BAM indexed only by a
    ``.csi`` are not supported here (NotImplementedError); a gzip FASTA that is not BGZF is refused (ValueError).  Returns the
    ``.bai`` path."""
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
    try:
        bam_io.fasta_bgzf_gzi(ref_fn)
    except ValueError:
        raise ValueError("genome: compressed FASTA is not supported unless bgzip-compressed; decompress %s and index it, or "
                         "recompress it with bgzip and samtools faidx it" % ref_fn) from None
    except FileNotFoundError:
        raise FileNotFoundError("genome: BGZF index %s.gzi not found (samtools faidx the FASTA first)" % ref_fn) from None
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
    tgt = targets.resolve(bed, known_sites)
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


def write_vcf_gz(path, text, decoder=None, stages=None):
    """``bgzip -f`` and ``tabix -p vcf``: ``path`` (ending in ``.vcf.gz``) and ``path.tbi``.  With ``decoder`` (a
    ``BamDecoder``) both files are compressed on its GPU (``BamDecoder.write_bgzf``), otherwise on the host
    (``bam_io.write_bgzf``); the bytes are the same.  ``stages``: a ``cascade.Stages`` that marks the compression and the
    file writes ("compress") apart from building the index ("write")."""
    write = decoder.write_bgzf if decoder is not None else bam_io.write_bgzf
    mark = stages.mark if stages is not None else (lambda name: None)
    voff = write(path, text)
    mark("compress")
    index = bam_io.tbi_bytes(text, voff)
    mark("write")
    write(str(path) + ".tbi", index)
    mark("compress")
    return path


# ------------------------------------------------------------------------------------------------ the genome-wide decisions
def exchange(chunk_rows, contigs, platform="ont", var_pct_full=None, ref_pct_full=None, genotyping=False,
             split_bed_size=cascade.SPLIT_BED_SIZE):
    """The genome-wide decisions from every pileup chunk's rows.  ``chunk_rows``: per CHUNK_LIST row, in its order, (contig,
    positions, probabilities, flags) as ``cascade.row_summary`` gives them.  Returns (keep: per chunk a bool mask of its rows
    that pileup.vcf keeps - of a position repeated by overlapping chunks the last chunk's row, as SortVcf keeps it -,
    (var_qual, ref_qual), beds: [(contig, 0-based candidate positions)] per bed file, in contig order).  The rows a position
    repeats are identical except under head / tail calling, where a candidate near a chunk's edge gets a padded window in one
    chunk and a whole one in the next; the reference then keeps whichever file ``os.listdir`` lists last, which has no fixed
    order, and this route keeps the last chunk's row."""
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
    cuts = cascade.qual_cutoffs_from(prob, flags & cascade.FLAG_GT00, platform, var_pct_full, ref_pct_full, genotyping)
    beds = []
    for ctg in [c for c, _ in contigs]:
        sel = [(np.asarray(r[1])[m], np.asarray(r[2])[m], np.asarray(r[3])[m]) for r, m in zip(chunk_rows, keep) if r[0] == ctg]
        if not sel:
            continue
        pos = cascade.candidates_from(np.concatenate([s[0] for s in sel]), np.concatenate([s[1] for s in sel]),
                                      np.concatenate([s[2] for s in sel]) & cascade.FLAG_REF, *cuts)
        beds.extend((ctg, pos[a:b]) for a, b in cascade.bed_chunks(len(pos), split_bed_size))
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
                haploid_precise=False, haploid_sensitive=False, keep_iupac_bases=False, split_bed_size=cascade.SPLIT_BED_SIZE,
                workspaces=None, device=None, group=None, k=16, enable_phasing=False):
    """Clair3's pipeline (scripts/clair3_c_impl_pipeline.py with ``--no_phasing_for_fa True``) over the genome: writes
    ``pileup.vcf.gz``, ``full_alignment.vcf.gz`` and ``merge_output.vcf.gz`` with their ``.tbi`` into ``out_dir``, as the
    reference does with its early exits (``file_texts``).  Options as run_clair3.py names them (None / 0 percentages and allele frequencies: the platform's defaults, see
    ``resolve_options``); ``bed_fn`` / ``vcf_fn`` also take ``targets.read_bed`` / ``read_vcf`` results.  ``cmdline``: the
    ``##cmdline=`` header line (None: none).  ``chunk_size`` / ``split_bed_size``: CheckEnvs' and SelectCandidates' sizes.
    ``group``: a ``torch.distributed`` process group (one process per GPU, each on its own ``device``); every rank must call
    with the same arguments.  ``model_p`` / ``model_f``: Clair3_P and Clair3_F on this rank's device.

    Returns, on rank 0, a dict: ``files`` {name: path}, ``texts`` {name: decompressed text}, ``contigs``, ``chunks``,
    ``qual_cutoffs``, ``beds`` (number of bed files), ``rows`` {name: row count}, ``stages`` (wall and device ms per stage,
    this rank's); None on the other ranks.

    ``enable_phasing`` (run_clair3.py's ``--enable_phasing``): when the run reaches MergeVcf and ``merge_output`` has a record,
    each contig's merged rows are phased (``_phase``; rank r takes a contiguous run of the contigs) and
    ``phased_merge_output.vcf.gz`` is written with its ``.tbi`` too.  The phase sets follow WhatsHap's model
    (``clair3_b200.phasing``); the file is not WhatsHap's byte for byte."""
    if no_phasing_for_fa is not True:
        raise NotImplementedError("genome: phasing for full alignment (WhatsHap / LongPhase) is not implemented; "
                                  "run with no_phasing_for_fa=True")
    if gvcf:
        raise NotImplementedError("genome: gVCF output is not implemented")
    if haploid_precise or haploid_sensitive:
        raise NotImplementedError("genome: the haploid modes are not implemented")
    cascade.check_platform(platform)
    if enable_dwell_time and platform != "ont":
        raise ValueError("genome: dwell time is only supported for platform 'ont' (run_clair3.py refuses it too)")
    tgt = targets.resolve(bed_fn, vcf_fn)
    genotyping = tgt is not None and tgt.kind == "vcf"
    var_pct, ref_pct, snp_af, indel_af = resolve_options(platform, var_pct_full, ref_pct_full, snp_min_af, indel_min_af, genotyping)
    cfg_p, cfg_f = output_configs(enable_long_indel, keep_iupac_bases)
    max_indel = LONG_INDEL if enable_long_indel else decode.MAX_INFER_LENGTH
    rank, world = _rank(group)
    contigs, chunks = plan(bam_fn, ref_fn, ctg_name, include_all_ctgs, min_contig_size, chunk_size,
                           bed=None if genotyping else tgt, known_sites=tgt if genotyping else None)
    head = header(ref_fn, sample_name, cmdline)
    names = [c for c, _ in contigs]
    out = {"contigs": contigs, "chunks": chunks, "qual_cutoffs": None, "beds": 0, "stages": None}
    if not contigs:
        return _write(out_dir, file_texts(head, names, [], []), out) if rank == 0 else None
    lengths = dict(contigs)
    index = bam_io.read_bai(bam_index(bam_fn))          # parsed once; the decoder reads each region's byte range through it
    own = workspaces is None
    if device is None:
        device = workspaces.counter._device if workspaces is not None else torch.cuda.current_device()
    ws = workspaces or cascade.Workspaces(device)
    try:
        st = cascade.Stages(ws.counter._device)
        read = functools.partial(_read_span, ws.decoder, bam_fn, ref_fn, bam_io.is_bgzf(ref_fn), index, lengths)
        count = {"min_depth": min_coverage, "min_snp_af": snp_af, "min_indel_af": indel_af, "min_mq": min_mq,
                 "call_snp_only": call_snp_only, "call_ht": enable_variant_calling_at_sequence_head_and_tail,
                 "max_indel_length": max_indel}
        mine = _pileup_chunks(ws.counter, st, read, lengths, chunks, range(*site_range(len(chunks), rank, world)), tgt,
                              model_p, cfg_p, k, count)
        # every rank: the rows' positions, probabilities and flags -> duplicates, cut-offs, bed files
        keep, cuts, beds = decisions([m[:5] for m in mine], contigs, platform, var_pct, ref_pct, genotyping, split_bed_size, group)
        st.mark("cutoffs and select")
        fa_rows = []
        if not pileup_only:
            fa = {"matrix_depth": MATRIX_DEPTH[platform], "need_haplotagging": False, "min_mq": min_mq,
                  "max_indel_length": max_indel, "dwell": bool(enable_dwell_time), "rand_seed": 1, "rand_skip": 0}
            fa_rows = _bed_files(ws.builder, st, read, beds, range(*site_range(len(beds), rank, world)), model_f, cfg_f, k, fa)
        # rank 0: the row texts
        kept = [(g, ctg, pos[keep[g]], [r for r, k_ in zip(rows, keep[g]) if k_]) for g, ctg, pos, _, _, rows in mine]
        parts = _gather0((kept, fa_rows), group, world, rank)
        st.mark("gather")
        merged = None
        if rank == 0:
            texts, merged = _file_texts(head, names,
                                        [c[1:] for c in sorted((c for part in parts for c in part[0]), key=lambda c: c[0])],
                                        [c[1:] for c in sorted((c for part in parts for c in part[1]), key=lambda c: c[0])],
                                        qual, print_ref_calls, pileup_only, tgt if genotyping else None)
            st.mark("merge and format")
        phased = None
        if enable_phasing:
            phased = _phase(ws.decoder, st, bam_fn, index, lengths, merged, chunk_size, group, world, rank)
        if rank != 0:
            return None
        if phased is not None:
            texts["phased_merge_output"] = vcf_text(phasing.phase_header(head), phased)
        out.update(qual_cutoffs=cuts, beds=len(beds))
        _write(out_dir, texts, out, ws.decoder, st)
        st.mark("write")
        out["stages"] = st.summed()
        return out
    finally:
        if own:
            ws.close()


def _read_span(decoder, bam_fn, ref_fn, bgzf, index, lengths, ctg, start, end, fa_fields):
    """The records of the 0-based [start, end) of contig ``ctg``, decoded with the FASTA window the counter and the builder
    read around it (``FETCH_EXPAND`` bases either side, clipped to the contig): (records, the window's start).  A plain
    FASTA's window is read on the host; a bgzip-compressed one's is inflated on the device, and its status is read after the
    decode's own wait."""
    r0, r1 = max(0, start - FETCH_EXPAND), min(lengths[ctg], end + FETCH_EXPAND + 1)
    if not bgzf:
        ref = bam_io.fetch_fasta(ref_fn, ctg, r0, r1)
        return decoder.decode(bam_fn, ctg, start, end, fa_fields=fa_fields, index=index, ref_seq=ref), r0
    ref = decoder.fetch_fasta(ref_fn, ctg, r0, r1, wait=False)
    rec = decoder.decode(bam_fn, ctg, start, end, fa_fields=fa_fields, index=index, ref_seq=ref)
    decoder.fasta_status()
    return rec, r0


def _pileup_chunks(counter, st, read, lengths, chunks, mine, tgt, model_p, cfg_p, k, count):
    """The pileup calls of the CHUNK_LIST rows ``mine`` (indices into ``chunks``): per row (index, contig, positions,
    probabilities, flags, row texts) of its VCF rows (``cascade.row_summary``), none for a row the reference skips.
    ``count``: ``PileupCounter.count``'s thresholds and read filters."""
    out = []
    for g in mine:
        ctg, cid, n = chunks[g]
        region = pileup_chunk_region(ctg, lengths[ctg], cid, n, tgt)
        if region is None:
            out.append((g, ctg, np.zeros(0, np.int64), np.zeros(0, np.float32), np.zeros(0, np.uint8), []))
            continue
        (start, end), ct = region
        rec, r0 = read(ctg, start, end, False)
        st.mark("decode")
        res = counter.count(rec, start, end, None, r0, alt_info=True, targets=ct, **count).call(model_p, cfg_p, ctg, k=k)
        st.mark("pileup")
        pos, prob, flags, idx = cascade.row_summary(res)
        out.append((g, ctg, pos, prob, flags, [decode.call_row(res, s, cfg_p) for s in idx]))
        del rec, res
        st.mark("pileup format")
    return out


def _bed_files(builder, st, read, beds, mine, model_f, cfg_f, k, fa):
    """The full-alignment calls of the bed files ``mine`` (indices into ``beds``), each over its ``bed_span``: per bed file
    (index, contig, 1-based positions, row texts) of its VCF rows.  ``fa``: ``FullAlignmentBuilder.build``'s arguments."""
    out = []
    for b in mine:
        ctg, cand = beds[b]
        rec, r0 = read(ctg, *bed_span(cand), True)
        st.mark("fa decode")
        res = builder.build(rec, cand, None, r0, **fa).call(model_f, cfg_f, ctg, k=k)
        st.mark("fa build and call")
        pos, rows = cascade.row_texts(res, cfg_f)
        out.append((b, ctg, pos, rows))
        del rec, res
        st.mark("fa format")
    return out


def file_texts(head, contigs, pileup_chunks, fa_beds, qual=2, print_ref=False, pileup_only=False, known=None):
    """``_file_texts``' texts alone."""
    return _file_texts(head, contigs, pileup_chunks, fa_beds, qual, print_ref, pileup_only, known)[0]


def _file_texts(head, contigs, pileup_chunks, fa_beds, qual=2, print_ref=False, pileup_only=False, known=None):
    """(texts, merged): the files' texts, {name: text}, from the rows of the whole run: SortVcf, MergeVcf per contig and, with ``known`` (the
    known-sites ``Targets``), AddBackMissingVariantsInGenotyping.  ``head``: ``header``'s text; ``contigs``: the contig names
    in CONTIGS order; ``pileup_chunks`` / ``fa_beds``: per pileup chunk (the rows pileup.vcf keeps) / per bed file, in order,
    (contig, 1-based positions, row texts).  The reference's early exits: no contig - a header-only ``merge_output`` alone; no
    pileup row - header-only ``pileup`` and ``merge_output``; ``pileup_only`` - ``pileup`` alone, and ``merge_output`` a copy
    of it when it holds no row; no bed file or no full-alignment row - ``merge_output`` a copy of ``pileup``.  ``merged``: the
    sorted MergeVcf body before the add-back, which ``--enable_phasing`` phases; None on every early exit, and when it holds no
    row (the pipeline's exit in variant merging)."""
    if not contigs:
        return {"merge_output": head}, None
    p_body = sort_rows((r for c in pileup_chunks for r in c[2]), contigs)
    if not p_body:
        return {"pileup": head, "merge_output": head}, None              # SortVcf: no variant found
    if pileup_only:
        pileup = vcf_text(head, postprocess_pileup(p_body, qual, print_ref), True)
        return ({"pileup": pileup} if has_records(pileup) else {"pileup": pileup, "merge_output": pileup}), None
    texts = {"pileup": vcf_text(head, p_body, True)}
    if fa_beds:
        texts["full_alignment"] = vcf_text(head, sort_rows((r for c in fa_beds for r in c[2]), contigs))
    if not fa_beds or not has_records(texts["full_alignment"]):
        texts["merge_output"] = texts["pileup"]                         # ensure_merge_output
        return texts, None
    merged = sort_rows("".join(_merge_contig(pileup_chunks, fa_beds, ctg, qual, print_ref) for ctg in contigs)
                       .splitlines(keepends=True), contigs)
    texts["merge_output"] = vcf_text(head, merged)
    if known is not None and merged:
        texts["merge_output"] = head + "\n" + cascade.add_back_missing(merged, known)
    return texts, (merged if has_records(merged) else None)


def _broadcast0(obj, group, world):
    if world == 1:
        return obj
    import torch.distributed as dist
    box = [obj]
    dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    return box[0]


def _phase(decoder, st, bam_fn, index, lengths, merged, span, group, world, rank):
    """``--enable_phasing``: the phased body of ``merged`` (rank 0's MergeVcf body; None: the run left early, and nothing is
    phased) on every rank's GPU - rank r the contigs ``site_range`` gives it, in the body's order, each decoded in spans of
    ``span`` bases (``phase_gpu.phase_contig``) - gathered on rank 0.  Returns the body on rank 0, None elsewhere."""
    from . import phase_gpu
    merged = _broadcast0(merged, group, world)
    if merged is None:
        return None
    by = phasing.split_contigs(merged)
    ctgs = list(by)
    mine = {}
    for ctg in ctgs[slice(*site_range(len(ctgs), rank, world))]:
        mine[ctg] = phase_gpu.phase_contig(decoder, bam_fn, ctg, lengths[ctg], by[ctg], span, index)[0]
    st.mark("phase")
    parts = _gather0(mine, group, world, rank)
    if rank != 0:
        return None
    done = {k: v for part in parts for k, v in part.items()}
    return "".join("".join(done[c]) for c in ctgs)


def _merge_contig(p_chunks, f_beds, ctg, qual, print_ref):
    """MergeVcf of one contig on row text: its pileup rows (as pileup.vcf holds them: unique, by position) and its bed files'
    full-alignment rows."""
    p = {}
    for c in p_chunks:
        if c[0] == ctg:
            p.update(zip(np.asarray(c[1]).tolist(), c[2]))
    p_pos = sorted(p)
    f_pos, f_rows = [], []
    for c in f_beds:
        if c[0] == ctg:
            f_pos.extend(np.asarray(c[1]).tolist())
            f_rows.extend(c[2])
    return cascade.merge_rows(p_pos, [p[x] for x in p_pos], f_pos, f_rows, qual=qual, print_ref=print_ref)


def _write(out_dir, texts, out, decoder=None, stages=None):
    """Writes each of ``texts`` as ``<name>.vcf.gz`` with its ``.tbi`` into ``out_dir`` (``write_vcf_gz`` with ``decoder`` and
    ``stages``), and adds ``files``, ``texts`` and ``rows`` (the row count per file) to the result ``out``."""
    out_dir = str(out_dir)
    os.makedirs(out_dir, exist_ok=True)
    out.update(files={n: write_vcf_gz(os.path.join(out_dir, n + ".vcf.gz"), t, decoder, stages) for n, t in texts.items()},
               texts=texts,
               rows={n: _records(t) for n, t in texts.items()})
    return out
