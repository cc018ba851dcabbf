"""Mints tests/golden/genome_cases.npz from the reference's own genome-level Python (needs the reference checkout:
CLAIR3_REFERENCE or a sibling directory; everything runs on the CPU under this Python).

* CheckEnvs (preprocess/CheckEnvs.py:CheckEnvs) on a crafted ``.fai`` with major, unplaced, short and read-less contigs,
  with ``--include_all_ctgs``, ``--ctg_name``, ``--min_contig_size``, a BED and a known-sites VCF: its CONTIGS and CHUNK_LIST.
  The tool-version checks are stubbed and ``samtools idxstats`` answers from the case's table.
* ``shared/utils.py:get_header`` for that ``.fai``, with and without a command line.
* SortVcf (preprocess/SortVcf.py:sort_vcf_from) over per-chunk pileup files (its ``--use_gpu`` branch, as the pipeline runs
  it for pileup.vcf and full_alignment.vcf), with ``--pileup_only`` post-processing, and over per-contig merge files (its
  per-contig branch, as for merge_output.vcf): duplicate keys, ``##commandline`` rows, contigs sharing a prefix, rows of a
  contig not in CONTIGS, and the header-only output of a run without rows.
* SelectQual and SelectCandidates over one contig whose rows come from three overlapping chunks and exceed
  ``--split_bed_size``.
* The indel-length limits and full-alignment depths of ``shared/param_p.py`` / ``shared/param_f.py``.

Everything is stored as one JSON document (``cases``).
    python tests/golden/make_genome_golden.py"""
import gzip
import io
import json
import os
import subprocess
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.fa_ref import reference_src  # noqa: E402

src = reference_src()
if src is None:
    sys.exit("the reference checkout is needed: set CLAIR3_REFERENCE")
REF = os.path.dirname(src)
sys.path.insert(0, REF)

import preprocess.CheckEnvs as ce  # noqa: E402
import preprocess.SortVcf as sv  # noqa: E402
from shared.utils import get_header  # noqa: E402

import cascade_cases as cc  # noqa: E402
from clair3_b200 import cascade  # noqa: E402

CLAIR3 = os.path.join(REF, "clair3.py")

FAI = [("chr1", 12000), ("chr2", 8000), ("chrUn_x", 5000), ("chr3", 6000), ("chr4", 500), ("chrM", 300), ("chr11", 4000)]
MAPPED = {"chr1": 500, "chr2": 300, "chrUn_x": 40, "chr3": 0, "chr4": 12, "chrM": 9, "chr11": 80}
BED = "chr1\t100\t900\nchrUn_x\t10\t50\nchrQ\t5\t10\nchr3\t1\t2\n"
VCF = ("##fileformat=VCFv4.2\nchr2\t500\t.\tA\tC\nchr2\t700\t.\tA\tG\nchr1\t10\t.\tA\tT\nchr4\t100\t.\tC\tA\n"
       "chrUn_x\t40\t.\tG\tT\n")
# (name, options): --ctg_name / --include_all_ctgs / --min_contig_size / --chunk_size / BED / VCF
CHECKENVS = [
    ("default", {"chunk_size": 5000}),
    ("all", {"include_all_ctgs": True, "chunk_size": 3000}),
    ("all_min_size", {"include_all_ctgs": True, "min_contig_size": 1000, "chunk_size": 4000}),
    ("ctg_name", {"ctg_name": "chr2,chrUn_x,chr3,chrZ", "chunk_size": 2500}),
    ("bed", {"bed": True, "chunk_size": 5000}),
    ("bed_ctg_name", {"bed": True, "ctg_name": "chr1,chr2", "chunk_size": 5000}),
    ("vcf", {"vcf": True, "chunk_size": 3000}),
    ("vcf_min_size", {"vcf": True, "min_contig_size": 1000, "chunk_size": 3000}),
    ("none", {"ctg_name": "chr3"}),
    ("exact_chunks", {"ctg_name": "chr1,chr2", "chunk_size": 4000}),
]


def idxstats_text():
    return "".join("%s\t%d\t%d\t0\n" % (n, L, MAPPED[n]) for n, L in FAI) + "*\t0\t0\t0\n"


def run_checkenvs(d, name, opt):
    out = os.path.join(d, "ce_" + name)
    bam = os.path.join(d, "in.bam")
    args = types.SimpleNamespace(
        bam_fn=bam, ref_fn=os.path.join(d, "ref.fa"), bed_fn=os.path.join(d, "t.bed") if opt.get("bed") else None,
        vcf_fn=os.path.join(d, "k.vcf") if opt.get("vcf") else None, output_fn_prefix=out, pypy="pypy3", samtools="samtools",
        whatshap="whatshap", parallel="parallel", qual=2, var_pct_full=0.7, ref_pct_full=0.1, snp_min_af=0.08, indel_min_af=0.15,
        min_contig_size=opt.get("min_contig_size", 0), sampleName="SAMPLE", cmd_fn=None, include_all_ctgs=opt.get("include_all_ctgs", False),
        ctg_name=opt.get("ctg_name", "EMPTY"), chunk_num=0, chunk_size=opt.get("chunk_size", 5000000), no_phasing_for_fa=True)
    real = ce.subprocess_popen

    def popen(cmd, *a, **k):
        if "idxstats" in cmd:
            return types.SimpleNamespace(stdout=io.StringIO(idxstats_text()))
        return real(cmd, *a, **k)
    ce.subprocess_popen, ce.check_tools_version = popen, lambda *a: None
    try:
        ce.CheckEnvs(args)
    finally:
        ce.subprocess_popen = real
    tmp = os.path.join(out, "tmp")
    read = lambda p: open(p).read() if os.path.exists(p) else None  # noqa: E731
    merge = os.path.join(out, "merge_output.vcf")
    return {"options": opt, "contigs": read(os.path.join(tmp, "CONTIGS")), "chunk_list": read(os.path.join(tmp, "CHUNK_LIST")),
            "header_only_merge": read(merge) if os.path.exists(merge) else (gzip.open(merge + ".gz", "rt").read()
                                                                           if os.path.exists(merge + ".gz") else None)}


def row(ctg, pos, ref="A", alt="C", qual="5.00", filt="PASS", gt="0/1"):
    return "%s\t%d\t.\t%s\t%s\t%s\t%s\tP\tGT:GQ:DP:AD:AF\t%s:5:20:10,10:0.5000\n" % (ctg, pos, ref, alt, qual, filt, gt)


def run_sortvcf(d, name, files, prefix, contigs, use_gpu, pileup_only=False, print_ref=False, qual=2, cmd=None):
    idir = os.path.join(d, "sv_" + name)
    os.makedirs(idir)
    for fn, text in files:
        with open(os.path.join(idir, fn), "w") as f:
            f.write(text)
    cfn = os.path.join(d, "contigs_" + name)
    with open(cfn, "w") as f:
        f.write("\n".join(contigs))
    cmd_fn = os.path.join(d, "cmd_" + name)
    if cmd:
        with open(cmd_fn, "w") as f:
            f.write(cmd)
    out = os.path.join(d, name + ".vcf")
    args = types.SimpleNamespace(output_fn=out, input_dir=idir, vcf_fn_prefix=prefix, vcf_fn_suffix=".vcf",
                                 ref_fn=os.path.join(d, "ref.fa"), sampleName="SAMPLE", contigs_fn=cfn, cmd_fn=cmd_fn,
                                 pileup_only=pileup_only, print_ref_calls=print_ref, check_malformed_records=True,
                                 haploid_precise=False, haploid_sensitive=False, qual=qual, output_all_contigs_in_gvcf_header=False,
                                 use_gpu=use_gpu)
    sv.sort_vcf_from(args)
    return {"files": files, "prefix": prefix, "contigs": contigs, "use_gpu": use_gpu, "pileup_only": pileup_only,
            "print_ref": print_ref, "qual": qual, "cmd": cmd, "out": open(out).read()}


out = {"fai": FAI, "mapped": MAPPED, "bed": BED, "vcf": VCF, "checkenvs": {}, "header": {}, "sortvcf": {}, "select": {}}
with tempfile.TemporaryDirectory() as d:
    with open(os.path.join(d, "ref.fa"), "w") as f:
        f.write("".join(">%s\n%s\n" % (n, "A" * L) for n, L in FAI))
    with open(os.path.join(d, "ref.fa.fai"), "w") as f:
        off = 0
        for n, L in FAI:
            off += len(n) + 2
            f.write("%s\t%d\t%d\t%d\t%d\n" % (n, L, off, L, L + 1))
            off += L + 1
    for p in ("in.bam", "in.bam.bai"):
        open(os.path.join(d, p), "w").close()
    with open(os.path.join(d, "t.bed"), "w") as f:
        f.write(BED)
    with open(os.path.join(d, "k.vcf"), "w") as f:
        f.write(VCF)
    for name, opt in CHECKENVS:
        out["checkenvs"][name] = run_checkenvs(d, name, opt)
        print("CheckEnvs %s: %r" % (name, out["checkenvs"][name]["contigs"]))

    ref_fn = os.path.join(d, "ref.fa")
    with open(os.path.join(d, "cmd"), "w") as f:
        f.write("run_clair3.py --bam_fn in.bam --ref_fn ref.fa  \n")
    for name, cmd in (("plain", None), ("cmd", os.path.join(d, "cmd"))):
        out["header"][name] = {"sample": "S1", "cmd": open(cmd).read() if cmd else None,
                               "text": get_header(reference_file_path=ref_fn, cmd_fn=cmd, sample_name="S1")}
    out["ref_fn"] = ref_fn

    head = get_header(reference_file_path=ref_fn, cmd_fn=os.path.join(d, "cmd"), sample_name="SAMPLE") + "\n"
    chunks = [
        ("pileup_chr1_1.vcf", head + row("chr1", 300) + row("chr1", 120, alt=".", filt="RefCall", gt="0/0", qual="3.00")
         + row("chr1", 500, qual="1.50") + row("chr1", 300, alt="G")),
        ("pileup_chr1_2.vcf", head + "##commandline=whatshap phase\n" + row("chr1", 900, qual="2.00") + row("chr1", 700)),
        ("pileup_chr11_1.vcf", head + row("chr11", 50) + row("chr11", 20, ref="C", alt="C", qual="9.00")),
        ("pileup_chrUn_x_1.vcf", head + row("chrUn_x", 30, qual="0.50")),
        ("pileup_chr2_1.vcf", head + row("chr2", 40, alt=".", filt="RefCall", gt="0/0", qual="12.00") + row("chr2", 41)),
        ("pileup_chrQ_1.vcf", head + row("chrQ", 5)),
        ("pileup_chr4_1.vcf", head),
    ]
    contigs = ["chr1", "chr2", "chr11", "chrUn_x"]
    out["sortvcf"]["chunks"] = run_sortvcf(d, "chunks", chunks, "pileup", contigs, True)
    for q, pr in ((2, False), (2, True), (0, False)):
        key = "pileup_only_q%d_ref%d" % (q, pr)
        out["sortvcf"][key] = run_sortvcf(d, key, chunks, "pileup", contigs, True, pileup_only=True, print_ref=pr, qual=q)
    out["sortvcf"]["empty"] = run_sortvcf(d, "empty", [("pileup_chr1_1.vcf", head), ("pileup_chr2_1.vcf", head)], "pileup",
                                          contigs, True, cmd="run_clair3.py --x 1\n")
    merges = [("merge_chr1.vcf", head + row("chr1", 120, alt=".", filt="RefCall", gt="0/0") + row("chr1", 300) + row("chr1", 700)),
              ("merge_chr11.vcf", head + row("chr11", 20) + row("chr11", 50)),
              ("merge_chrUn_x.vcf", head), ("merge_chr2.vcf", head + row("chr2", 41))]
    out["sortvcf"]["merge"] = run_sortvcf(d, "merge", merges, "merge", contigs, False)
    for k, v in out["sortvcf"].items():
        print("SortVcf %s: %d lines" % (k, v["out"].count("\n")))

    # SelectQual + SelectCandidates over one contig's rows from three overlapping chunks (tests/cascade_cases.py "hifi")
    platform, pres, _ = cc.case("hifi")
    rows = cascade.row_texts(pres, cc.CFG_P)[1]
    rows = [r.replace(cc.CTG + "\t", "chr1\t", 1) for r in rows]
    n = len(rows)
    cuts = [(0, n // 3 + 20), (n // 3, 2 * n // 3 + 20), (2 * n // 3, n)]       # overlapping: 20 rows appear twice
    sel_dir = os.path.join(d, "select")
    os.makedirs(sel_dir)
    pvcf = os.path.join(d, "sel_pileup.vcf")
    body = "".join(rows)                                                        # each row once, as pileup.vcf holds them
    with open(pvcf, "w") as f:
        f.write("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE\n" + body)
    var_pct, ref_pct = cascade.PCT_FULL[platform]
    for args, stdin in ((["SelectQual", "--output_fn", sel_dir, "--var_pct_full", str(var_pct), "--ref_pct_full", str(ref_pct),
                          "--platform", platform], open(pvcf).read()),
                        (["SelectCandidates", "--pileup_vcf_fn", pvcf, "--split_folder", sel_dir, "--var_pct_full", str(var_pct),
                          "--ref_pct_full", str(ref_pct), "--platform", platform, "--ctgName", "chr1", "--split_bed_size", "150"], None)):
        r = subprocess.run([sys.executable, CLAIR3] + args, input=stdin, capture_output=True, text=True)
        if r.returncode:
            sys.exit(r.stderr)
    listing = os.path.join(sel_dir, "FULL_ALN_FILE_chr1")
    beds = [open(p.strip()).read() for p in open(listing)] if os.path.exists(listing) else []
    out["select"] = {"platform": platform, "chunks": cuts, "split_bed_size": 150, "qual": open(os.path.join(sel_dir, "qual")).read(),
                     "beds": beds}
    print("SelectCandidates: %d bed files, qual %r" % (len(beds), out["select"]["qual"]))

# the limits and depths the route's options resolve to (shared/param_p.py, shared/param_f.py)
import shared.param_f as param_f  # noqa: E402
import shared.param_p as param_p  # noqa: E402
out["params"] = {"p_max_indel": param_p.maximum_variant_length_that_need_infer,
                 "p_max_indel_long": param_p.maximum_variant_length_that_need_infer_include_long_indel,
                 "f_max_indel": param_f.maximum_variant_length_that_need_infer,
                 "f_max_indel_long": param_f.maximum_variant_length_that_need_infer_include_long_indel,
                 "matrix_depth": param_f.matrix_depth_dict}

np.savez_compressed(os.path.join(ROOT, "tests", "golden", "genome_cases.npz"), cases=np.array(json.dumps(out)))
