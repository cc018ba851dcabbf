"""Clair3's pileup -> full-alignment cascade for one region, from BAM bytes to the merged VCF rows (DESIGN.md 5e).

The reference joins its two networks with three pypy scripts over VCF text (HKU-BAL/Clair3, as
``scripts/clair3_c_impl_pipeline.py`` runs them in its steps 5-7): ``SelectQual`` picks QUAL cut-offs from the genome-wide
pileup VCF, ``SelectCandidates`` writes bed files of full-alignment candidates, one ``CallVariantsFromCffi`` process per bed
file re-calls them with Clair3_F, and ``MergeVcf`` merges the two VCFs.  Here the same decisions are taken from the call
records, in three layers each usable on its own:

* ``qual_cutoffs`` (``SelectQual``), ``prob_threshold``, ``select`` / ``bed_text`` (``SelectCandidates``) and ``merge``
  (``MergeVcf``) on host call results (``PileupCounter.call`` / ``FullAlignmentBuilder.call``);
* ``select_device``: the same selection on the device (``c3b_cascade_select``), whose candidates a full-alignment build takes
  where they are (``FullAlignmentBuilder.build(..., cand_count=...)``);
* ``call_region``: the whole route on one stream, and ``call_region_host``, the same calls with host records and host
  candidates, which is what the device route is tested against.

Both routes take the reference's two ways of restricting a run (DESIGN.md 5f): a BED (``--bed_fn``) and a known-sites VCF
(``--vcf_fn``, genotyping mode, which ``add_back_missing`` finishes as AddBackMissingVariantsInGenotyping does).  The device
route drops the other candidates inside the counter, the host route drops them from the host call results.

Not implemented (``NotImplementedError``): ``platform="ilmn"`` (``MergeVcf_illumina`` and another bed geometry), the haploid
modes and gVCF output.
"""
from __future__ import annotations

import time

import numpy as np
import torch

from . import decode
from ._ffi import C3BError, check, ffi, lib
from .fa_tensor import MATRIX_DEPTH

# run_clair3.py:302-313: --var_pct_full / --ref_pct_full default to 0, which means these
PCT_FULL = {"ont": (0.7, 0.1), "hifi": (0.3, 0.3)}          # (var_pct_full, ref_pct_full)
SPLIT_BED_SIZE = 10000                                       # SelectCandidates --split_bed_size
FLANK = 16                                                   # shared/param_f.py flankingBaseNum
_ONE = 0x3F800000                                            # float32 1.0: QUAL is undefined above it (log of a negative)


def _check_platform(platform):
    if platform == "ilmn":
        raise NotImplementedError("cascade: platform 'ilmn' (MergeVcf_illumina and its bed geometry) is not implemented")
    if platform not in PCT_FULL:
        raise ValueError("cascade: platform must be 'ont' or 'hifi', got %r" % (platform,))


def _check_config(cfg):
    decode._check_config(cfg)
    for name in ("is_haploid_precise_mode_enabled", "is_haploid_sensitive_mode_enabled"):
        if getattr(cfg, name, False):
            raise NotImplementedError("cascade: the haploid modes are not implemented")


# ------------------------------------------------------------------------------------------------ rows of a call result
def _rows(res):
    """Indices of the calls that are rows of the VCF: printed, and for pileup calls ``cand_ok``."""
    m = res["calls"]["printed"] != 0
    if "cand_ok" in res:
        m &= np.asarray(res["cand_ok"]) != 0
    return np.nonzero(m)[0]


def _is_reference(res, idx):
    """SelectCandidates' and MergeVcf's test on the row text: ALT is "." or ALT == REF (not the genotype)."""
    calls, text, start = res["calls"], res["text"], res["start"]
    out = np.zeros(len(idx), bool)
    for j, s in enumerate(idx):
        o, rl, al = int(start[s]), int(calls["ref_len"][s]), int(calls["alt_len"][s])
        alt = text[o + rl:o + rl + al]
        out[j] = (al == 1 and alt[0] == ord(".")) or (rl == al and np.array_equal(text[o:o + rl], alt))
    return out


# ------------------------------------------------------------------------------------------------ SelectQual
def _kth_qual(probs, pct):
    """The last of the lowest ``int(pct * n)`` QUALs, or 0.0 when that is none.  QUAL is monotone non-decreasing in the
    float32 probability (``prob_threshold``), so it is the QUAL of the k-th lowest probability: one host call, not one per row."""
    p = np.concatenate(probs) if probs else np.zeros(0, np.float32)
    k = int(pct * len(p))
    if k == 0:
        return 0.0
    return decode.quality_score_from(np.partition(p, k - 1)[k - 1])


def qual_cutoffs(results, platform="ont", var_pct_full=None, ref_pct_full=None, genotyping=False):
    """``SelectQual`` without ``--phase`` (preprocess/SelectQual.py:select_qual_from_stdin) over any number of pileup ``call``
    results (every region of a genome for the genome-wide cut-offs): returns (var_qual, ref_qual).  Rows whose GT prints as
    ``0/0`` give the reference cut-off, all others the variant cut-off; ``ref_pct_full`` 0 means ``var_pct_full``, as there,
    except in genotyping mode (``--vcf_fn``, ``genotyping=True``), where ``ref_pct_full`` is used as given (:97).  The
    percentages default to run_clair3.py's for the platform."""
    _check_platform(platform)
    var_pct = PCT_FULL[platform][0] if var_pct_full is None else var_pct_full
    ref_pct = PCT_FULL[platform][1] if ref_pct_full is None else ref_pct_full
    if not genotyping:
        ref_pct = ref_pct if ref_pct else var_pct
    ref_p, var_p = [], []
    for res in results:
        c = res["calls"][_rows(res)]
        gt00 = c["genotype"] == 0                       # decode.GENOTYPES: 0 prints "0/0"
        ref_p.append(c["prob"][gt00])
        var_p.append(c["prob"][~gt00])
    return _kth_qual(var_p, var_pct), _kth_qual(ref_p, ref_pct)


def _qual_of_bits(bits):
    return decode.quality_score_from(np.array(bits, np.uint32).view(np.float32)[()])


def prob_threshold(cut):
    """The smallest float32 bit pattern t in [0, 1.0] with ``quality_score_from(t) >= cut`` (1.0's pattern + 1 when there is
    none).  QUAL is monotone non-decreasing in the probability and a non-negative float32's bit pattern orders as its value,
    so for a probability p in [0, 1] ``quality_score_from(p) < cut`` exactly when ``bits(p) < t``: the device compares bits."""
    lo, hi = 0, _ONE + 1
    while lo < hi:
        mid = (lo + hi) // 2
        if _qual_of_bits(mid) >= cut:
            hi = mid
        else:
            lo = mid + 1
    return lo


# ------------------------------------------------------------------------------------------------ SelectCandidates
def _chunks(n, split_bed_size):
    return [(i, min(i + split_bed_size, n)) for i in range(0, n, split_bed_size)]


def select(pileup_result, var_qual, ref_qual, split_bed_size=SPLIT_BED_SIZE):
    """``SelectCandidates`` (preprocess/SelectCandidates.py:187-270, ``--phasing_info_in_bam`` at its default) on one region's
    pileup ``call`` result: reference rows (by ALT text) with QUAL < ``ref_qual`` and the other rows with QUAL < ``var_qual``.
    Returns (0-based positions int64, sorted and unique; [(lo, hi)] index ranges of the bed files, ``split_bed_size`` each)."""
    idx = _rows(pileup_result)
    bits = pileup_result["calls"]["prob"][idx].view(np.uint32)
    t = np.where(_is_reference(pileup_result, idx), prob_threshold(ref_qual), prob_threshold(var_qual)).astype(np.int64)
    pos = np.unique(np.asarray(pileup_result["position"])[idx][bits.astype(np.int64) < t] - 1).astype(np.int64)
    return pos, _chunks(len(pos), split_bed_size)


def bed_text(ctg, positions):
    """One bed file of SelectCandidates (:262-267) for the 0-based ``positions`` of a chunk: ``ctg max(p - 16, 0) p + 18``
    per candidate, which ``fa_tensor.candidates_from_bed`` turns back into the candidates."""
    return "".join("%s\t%d\t%d\n" % (ctg, max(int(p) - FLANK, 0), int(p) + FLANK + 2) for p in positions) if len(positions) else "\n"


def select_device(pileup_result, var_qual, ref_qual):
    """``select``'s positions on the device, stream-ordered with no host wait (``c3b_cascade_select``), from the records
    ``call`` left there (``pileup_result["device"]``, so before the counter's next count).  Returns (int64 [max(n_calls, 1)] whose
    first ``count`` entries are the candidates, int64 [1] ``count``), both on the device: ``FullAlignmentBuilder.build(records,
    selected, ..., cand_count=count)`` takes them where they are."""
    d = pileup_result["device"]
    n = int(d["calls"].shape[0])
    dev = d["calls"].device
    scratch = torch.empty(max(2 * n, 1), dtype=torch.int64, device=dev)
    selected = torch.empty(max(n, 1), dtype=torch.int64, device=dev)        # never a null pointer, even without calls
    count = torch.empty(1, dtype=torch.int64, device=dev)
    ok = d.get("cand_ok")
    c = ffi.cast
    check(lib().c3b_cascade_select(c("const c3b_call *", d["calls"].data_ptr()), c("const char *", d["text"].data_ptr()),
                                   c("const int64_t *", d["decoder_off"].data_ptr()), c("const int64_t *", d["position"].data_ptr()),
                                   c("const uint8_t *", ok.data_ptr()) if ok is not None else ffi.NULL, n,
                                   prob_threshold(var_qual), prob_threshold(ref_qual), c("int64_t *", scratch.data_ptr()),
                                   c("int64_t *", selected.data_ptr()), c("int64_t *", count.data_ptr()),
                                   c("void *", torch.cuda.current_stream(dev).cuda_stream)))
    return selected, count


# ------------------------------------------------------------------------------------------------ MergeVcf
def _vcf(res, cfg):
    """(1-based positions, row texts) of a call result's VCF rows."""
    idx = _rows(res)
    return np.asarray(res["position"])[idx].astype(np.int64), [decode.call_row(res, s, cfg) for s in idx]


def merge(pileup_result, fa_results, output_config_p, output_config_f, qual=2, print_ref=False):
    """``MergeVcf`` (preprocess/MergeVcf.py, the non-ilmn ``MergeVcf``) of one region: the merged VCF body, byte for byte
    what it writes after the header.  A full-alignment row of any kind drops the pileup row at its position; reference rows
    (by ALT text) are kept only with ``print_ref``; the others are re-marked LowQual when ``qual`` is set and QUAL <= ``qual``;
    the rows come out in position order.  ``fa_results``: the full-alignment ``call`` results of the region's bed files, in
    order."""
    for cfg in (output_config_p, output_config_f):
        _check_config(cfg)
    p_pos, p_rows = _vcf(pileup_result, output_config_p)
    f_pos, f_rows = np.zeros(0, np.int64), []
    for res in fa_results:
        pos, rows = _vcf(res, output_config_f)
        f_pos, f_rows = np.concatenate([f_pos, pos]), f_rows + rows
    return merge_rows(p_pos, p_rows, f_pos, f_rows, qual=qual, print_ref=print_ref)


def merge_rows(p_pos, p_rows, f_pos, f_rows, qual=2, print_ref=False):
    """``merge`` on row text: one contig's pileup rows and full-alignment rows (1-based positions, ascending, and their row
    texts).  With no full-alignment rows this is SortVcf's ``--pileup_only`` post-processing (``postprocess_row_with_params``
    without the haploid modes)."""
    p_pos, f_pos = np.asarray(p_pos, np.int64), np.asarray(f_pos, np.int64)
    j = np.searchsorted(f_pos, p_pos)
    replaced = (j < len(f_pos)) & (f_pos[np.minimum(j, max(len(f_pos) - 1, 0))] == p_pos) if len(f_pos) else np.zeros(len(p_pos), bool)
    pos, rows = [], []
    for source_pos, source_rows, drop in ((f_pos, f_rows, None), (p_pos, p_rows, replaced)):
        for i, row in enumerate(source_rows):
            if drop is not None and drop[i]:
                continue
            cols = row.split("\t")
            if not (cols[4] == "." or cols[3] == cols[4]):
                if qual and float(cols[5]) <= qual:                  # MarkLowQual
                    cols[6] = "LowQual"
                    row = "\t".join(cols)
            elif not print_ref:
                continue
            pos.append(source_pos[i])
            rows.append(row)
    order = np.argsort(np.asarray(pos, np.int64), kind="stable")
    return "".join(rows[i] for i in order)


# ------------------------------------------------------------------------------------------------ targets
def contig_targets(ctg, bed=None, known_sites=None):
    """One contig's ``targets.ContigTargets`` from ``bed`` / ``known_sites``: a path (gzip or plain), a ``targets.Targets``
    (``read_bed`` / ``read_vcf``) or already a ``ContigTargets`` (``Targets.contig(ctg, chunk=...)``); None for neither.
    Giving both is a ValueError, as CheckEnvs refuses ``--bed_fn`` with ``--vcf_fn``."""
    from . import targets as tg
    if bed is not None and known_sites is not None:
        raise ValueError("cascade: give either bed or known_sites, not both (the reference refuses --bed_fn with --vcf_fn)")
    src, read = (bed, tg.read_bed) if bed is not None else (known_sites, tg.read_vcf)
    if src is None:
        return None
    if isinstance(src, tg.ContigTargets):
        t = src
    else:
        t = (src if isinstance(src, tg.Targets) else read(src)).contig(ctg)
    if (t.known is not None) != (known_sites is not None):
        raise ValueError("cascade: bed needs a BED's targets and known_sites a VCF's")
    return t


def take_calls(res, idx):
    """The call result ``res`` (``PileupCounter.call``) at the candidates ``idx`` only, as a targeted count gives it; the
    ``device`` views are left out."""
    idx = np.asarray(idx, np.int64)
    out = {k: v for k, v in res.items() if k != "device"}
    for k in ("position", "calls", "start", "cand_ok"):
        if k in res:
            out[k] = np.asarray(res[k])[idx]
    out["chromosome"] = [res["chromosome"][i] for i in idx]
    if "Y" in res:
        out["Y"] = res["Y"][torch.as_tensor(idx, device=res["Y"].device)]
    return out


# major_contigs_order of preprocess/CheckEnvs.py and postprocess/AddBackMissingVariantsInGenotyping.py
MAJOR_CONTIGS = ["chr%s" % a for a in list(range(1, 23)) + ["X", "Y"]] + [str(a) for a in list(range(1, 23)) + ["X", "Y"]]


def _known_rows(known_vcf):
    from . import targets as tg
    if isinstance(known_vcf, tg.ContigTargets):
        return {(known_vcf.ctg, p): r for p, r in known_vcf.rows.items()}
    return (known_vcf if isinstance(known_vcf, tg.Targets) else tg.read_vcf(known_vcf)).rows


def add_back_missing(merged_body, known_vcf, region=None):
    """AddBackMissingVariantsInGenotyping (postprocess/AddBackMissingVariantsInGenotyping.py:94-159, ``switch_genotype`` at
    its default) on a merged VCF body: one row per known site and nothing else - Clair3's row where it called the site, the
    known row otherwise, padded to 10 columns with REF cut to its first base (``.`` if empty), ALT / QUAL / FILTER / INFO
    ``.``, FORMAT ``GT`` and sample ``./.``.  The major contigs come first in their order, then the others in the order the
    known VCF first names them (the reference takes a set's order there, which changes from run to run); sites by position;
    of duplicate (contig, position) keys the last row wins.  ``known_vcf``: a path, ``targets.read_vcf``'s ``Targets`` or a
    ``ContigTargets`` (its known sites only).  ``region`` = (ctg, start, end): only the known sites inside the 0-based
    [start, end), which ``call_region`` is responsible for."""
    known = _known_rows(known_vcf)
    if region is not None:
        c, a, b = region
        known = {k: r for k, r in known.items() if k[0] == c and a < k[1] <= b}
    called = {}
    for row in merged_body.splitlines(keepends=True):
        cols = row.strip().split()
        if cols and cols[0][0] != "#":
            called[(cols[0], int(cols[1]))] = row
    by_ctg = {}
    for (ctg, pos), row in known.items():
        if (ctg, pos) in called:
            row = called[(ctg, pos)]
        else:
            cols = row.rstrip().split("\t")
            cols += ["."] * (10 - len(cols))
            cols[3] = cols[3][0] if len(cols[3]) > 0 else "."
            cols[4] = cols[5] = cols[6] = cols[7] = "."
            cols[8], cols[9] = "GT", "./."
            row = "\t".join(cols) + "\n"
        by_ctg.setdefault(ctg, []).append((pos, row))
    order = [c for c in MAJOR_CONTIGS if c in by_ctg] + [c for c in by_ctg if c not in MAJOR_CONTIGS]
    return "".join(r for c in order for _, r in sorted(by_ctg[c], key=lambda x: x[0]))


# ------------------------------------------------------------------------------------------------ the route
class Workspaces:
    """The BAM reader, the pileup counter and the full-alignment builder of a region route on one device."""

    def __init__(self, device=0):
        from .bam_decode import BamDecoder
        from .fa_tensor import FullAlignmentBuilder
        from .pileup_counts import PileupCounter
        self.decoder, self.counter, self.builder = BamDecoder(device), PileupCounter(device), FullAlignmentBuilder(device)

    def close(self):
        for w in (self.decoder, self.counter, self.builder):
            w.close()


class _Stages:
    """CUDA events and host clock at the stage boundaries of a route (no host wait: read after the route has waited)."""

    def __init__(self, device):
        self.device, self.marks = device, []
        self.mark("start")

    def mark(self, name):
        ev = torch.cuda.Event(enable_timing=True)
        ev.record(torch.cuda.current_stream(self.device))
        self.marks.append((name, ev, time.perf_counter()))

    def report(self):
        torch.cuda.current_stream(self.device).synchronize()
        return [{"stage": b[0], "wall_ms": 1e3 * (b[2] - a[2]), "device_ms": a[1].elapsed_time(b[1])}
                for a, b in zip(self.marks, self.marks[1:])]


def _route_args(platform, output_config_p, output_config_f, fa_params):
    _check_platform(platform)
    for cfg in (output_config_p, output_config_f):
        _check_config(cfg)
        if not cfg.is_show_reference:
            # CallVariantsFromCffi prints RefCall rows by default (showRef): SelectQual's reference list, SelectCandidates'
            # reference candidates and MergeVcf's replacement of pileup rows all read them
            raise ValueError("cascade: both output configs need is_show_reference=True, as the reference's pipeline runs")
    fa = {"matrix_depth": MATRIX_DEPTH[platform]}
    fa.update(fa_params or {})
    return fa


def _span(start, end):
    """The decoded span: the region and the 16-base flank of a full-alignment window at either end."""
    return max(0, int(start) - FLANK - 1), int(end) + FLANK + 1


def call_region(bam_path, ctg, start, end, ref_seq, ref_start, model_p, model_f, output_config_p, output_config_f, var_qual=None,
                ref_qual=None, phased_variants=None, platform="ont", print_ref=False, qual=2, split_bed_size=SPLIT_BED_SIZE,
                count_params=None, fa_params=None, index=None, workspaces=None, device=0, k=16, bed=None, known_sites=None):
    """Clair3's cascade for the 0-based region [start, end) of contig ``ctg``: one ``BamDecoder.decode`` (fa_fields) whose
    device records feed the counter and every full-alignment build, Clair3_P over the pileup candidates, the selection on the
    device, one full-alignment build per ``split_bed_size`` candidates with a fresh glibc ``rand()`` stream (each of the
    reference's bed files runs in a process of its own), Clair3_F, and the merge.  ``ref_seq``: the reference bases from
    ``ref_start`` (str / bytes), covering the region and 17 bases beyond it.  ``var_qual`` / ``ref_qual``: the cut-offs,
    default the region's own (``qual_cutoffs`` of its pileup calls: right for a one-region run; a genome-wide run takes
    ``qual_cutoffs`` over every region's pileup calls first).  ``phased_variants``: ``fa_tensor.phased_variants_from_vcf`` of
    the contig.  ``output_config_p`` / ``_f``: the two decoders' configs (the reference prints the pileup's RefCall rows:
    ``is_show_reference=True``).  ``count_params`` / ``fa_params``: extra keyword arguments of ``PileupCounter.count`` /
    ``FullAlignmentBuilder.build`` (the matrix depth defaults to the platform's).  ``bed`` / ``known_sites``: call only
    inside a BED's targets, or only at a VCF's known sites (``contig_targets``: a path, a ``targets.Targets`` or a
    ``ContigTargets``); the counter drops the other candidates on the device, and with known sites the cut-offs follow
    SelectQual's genotyping rule and ``add_back_missing`` finishes the body.

    Returns a dict: ``vcf`` (the merged body), ``pileup`` and ``full_alignment`` (the ``call`` results), ``qual_cutoffs``,
    ``candidates`` (int64 0-based, host), ``chunks`` and ``stages`` (wall and device ms per stage); with ``known_sites`` also
    ``genotyped``, the body after ``add_back_missing`` over the known sites inside the region."""
    fa = _route_args(platform, output_config_p, output_config_f, fa_params)
    tgt = contig_targets(ctg, bed, known_sites)
    genotyping = known_sites is not None
    own = workspaces is None
    ws = workspaces or Workspaces(device)
    dev = ws.counter._device
    try:
        st = _Stages(dev)
        lo, hi = _span(start, end)
        ref = torch.from_numpy(np.frombuffer(ref_seq.encode() if isinstance(ref_seq, str) else bytes(ref_seq), np.uint8).copy())
        rec = ws.decoder.decode(bam_path, ctg, lo, hi, fa_fields=True, ref_seq=ref.to(dev), index=index)
        st.mark("decode")
        pres = ws.counter.count(rec, start, end, None, ref_start, alt_info=True, targets=tgt,
                                **(count_params or {})).call(model_p, output_config_p, ctg, k=k)
        st.mark("pileup")
        if var_qual is None or ref_qual is None:
            own_var, own_ref = qual_cutoffs([pres], platform, genotyping=genotyping)
            var_qual = own_var if var_qual is None else var_qual
            ref_qual = own_ref if ref_qual is None else ref_qual
        selected, count = select_device(pres, var_qual, ref_qual)
        st.mark("select")
        fres, first, total = [], 0, None
        while total is None or first < total:
            ws.builder.build(rec, selected, None, ref_start, variants=phased_variants, rand_seed=1, rand_skip=0, cand_count=count,
                             cand_first=first, cand_max=split_bed_size, **fa)
            total = ws.builder.device_count()
            if total == 0:
                break
            fres.append(ws.builder.call(model_f, output_config_f, ctg, k=k))
            st.mark("full_alignment %d" % len(fres))
            first += split_bed_size
        vcf = merge(pres, fres, output_config_p, output_config_f, qual=qual, print_ref=print_ref)
        st.mark("merge")
        stages = st.report()
        out = {"vcf": vcf, "pileup": pres, "full_alignment": fres, "qual_cutoffs": (var_qual, ref_qual),
               "candidates": selected[:total].cpu().numpy(), "chunks": _chunks(total, split_bed_size), "stages": stages}
        if genotyping:
            out["genotyped"] = add_back_missing(vcf, tgt, region=(ctg, start, end))
        return out
    finally:
        if own:
            ws.close()


def call_region_host(bam_path, ctg, start, end, ref_seq, ref_start, model_p, model_f, output_config_p, output_config_f, var_qual=None,
                     ref_qual=None, phased_variants=None, platform="ont", print_ref=False, qual=2, split_bed_size=SPLIT_BED_SIZE,
                     count_params=None, fa_params=None, workspaces=None, device=0, k=16, bed=None, known_sites=None):
    """``call_region`` through host records and host candidates: ``bam_io.read_bam`` -> count -> call -> ``select`` on the
    host -> one host-candidate build per chunk -> call -> ``merge``.  Same arguments and result (without ``stages``); the
    count is untargeted and ``bed`` / ``known_sites`` drop the other candidates from its call results (``ContigTargets.keep``)."""
    from . import bam_io
    fa = _route_args(platform, output_config_p, output_config_f, fa_params)
    tgt = contig_targets(ctg, bed, known_sites)
    genotyping = known_sites is not None
    own = workspaces is None
    ws = workspaces or Workspaces(device)
    try:
        lo, hi = _span(start, end)
        rec, _ = bam_io.read_bam(bam_path, ctg, lo, hi, fa_fields=True)
        pres = ws.counter.count(rec, start, end, ref_seq, ref_start, alt_info=True, **(count_params or {})).call(model_p, output_config_p,
                                                                                                              ctg, k=k)
        if tgt is not None:
            pres = take_calls(pres, np.nonzero(tgt.keep(pres["position"]))[0])
        if var_qual is None or ref_qual is None:
            own_var, own_ref = qual_cutoffs([pres], platform, genotyping=genotyping)
            var_qual = own_var if var_qual is None else var_qual
            ref_qual = own_ref if ref_qual is None else ref_qual
        pos, chunks = select(pres, var_qual, ref_qual, split_bed_size)
        fres = [ws.builder.build(rec, pos[a:b], ref_seq, ref_start, variants=phased_variants, rand_seed=1, rand_skip=0, **fa)
                .call(model_f, output_config_f, ctg, k=k) for a, b in chunks]
        vcf = merge(pres, fres, output_config_p, output_config_f, qual=qual, print_ref=print_ref)
        out = {"vcf": vcf, "pileup": pres, "full_alignment": fres, "qual_cutoffs": (var_qual, ref_qual), "candidates": pos,
               "chunks": chunks}
        if genotyping:
            out["genotyped"] = add_back_missing(vcf, tgt, region=(ctg, start, end))
        return out
    finally:
        if own:
            ws.close()
