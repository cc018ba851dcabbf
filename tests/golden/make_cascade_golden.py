"""Mints tests/golden/cascade.npz from the reference's own SelectQual, SelectCandidates and MergeVcf (needs the reference
checkout: CLAIR3_REFERENCE or a sibling directory; the scripts run on the CPU under this Python).

For every case of tests/cascade_cases.py (the call results are rebuilt from that module's code) it writes the pileup VCF those
calls print, and runs the scripts as scripts/clair3_c_impl_pipeline.py runs them in its steps 5 and 7: SelectQual with the
platform's --var_pct_full / --ref_pct_full, SelectCandidates without --phasing_info_in_bam (with the case's phased VCF as
--phased_vcf_fn where it has one: that option adds nothing on this path), and MergeVcf with --print_ref_calls False and True
over the full-alignment VCF of tests/cascade_cases.py:fa_results.  It stores, per case, ``<name>/qual`` (the qual file),
``<name>/beds`` (each bed file, in FULL_ALN_FILE order), ``<name>/merged`` (the two merged bodies, header removed).
    python tests/golden/make_cascade_golden.py"""
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from clair3_b200 import cascade  # noqa: E402
from oracle.fa_ref import reference_src  # noqa: E402
import cascade_cases as cases  # noqa: E402

src = reference_src()
if src is None:
    sys.exit("the reference checkout is needed: set CLAIR3_REFERENCE")
CLAIR3 = os.path.join(os.path.dirname(src), "clair3.py")


def run(args, stdin=None):
    r = subprocess.run([sys.executable, CLAIR3] + args, input=stdin, capture_output=True, text=True)
    if r.returncode:
        sys.exit("%s failed:\n%s\n%s" % (args[0], r.stdout, r.stderr))


out = {"names": np.array(cases.NAMES)}
for name in cases.NAMES:
    platform, pileup, phased = cases.case(name)
    var_pct, ref_pct = cascade.PCT_FULL[platform]
    with tempfile.TemporaryDirectory() as d:
        pvcf = os.path.join(d, "pileup.vcf")
        with open(pvcf, "w") as f:
            f.write(cases.vcf_text(pileup, cases.CFG_P))
        split = os.path.join(d, "split")
        os.makedirs(split)
        run(["SelectQual", "--output_fn", split, "--var_pct_full", str(var_pct), "--ref_pct_full", str(ref_pct), "--platform", platform],
            stdin=open(pvcf).read())
        extra = []
        if phased:
            with open(os.path.join(d, "phased.vcf"), "w") as f:
                f.write(phased)
            extra = ["--phased_vcf_fn", os.path.join(d, "phased.vcf")]
        run(["SelectCandidates", "--pileup_vcf_fn", pvcf, "--split_folder", split, "--var_pct_full", str(var_pct), "--ref_pct_full",
             str(ref_pct), "--platform", platform, "--ctgName", cases.CTG] + extra)
        qual = open(os.path.join(split, "qual")).read()
        listing = os.path.join(split, "FULL_ALN_FILE_" + cases.CTG)
        beds = [open(p.strip()).read() for p in open(listing)] if os.path.exists(listing) else []
        # the full-alignment calls at the candidates those bed files give (the reference's own bed files: candidates_from_bed)
        from clair3_b200.fa_tensor import candidates_from_bed
        positions, chunks = [], []
        for b in beds:
            with open(os.path.join(d, "b.bed"), "w") as f:
                f.write(b)
            c = candidates_from_bed(os.path.join(d, "b.bed"), cases.CTG)[0]
            chunks.append((len(positions), len(positions) + len(c)))
            positions += c
        fa = cases.fa_results(pileup, np.array(positions, np.int64), chunks, seed=len(name))
        fvcf = os.path.join(d, "full_alignment.vcf")
        with open(fvcf, "w") as f:
            f.write(cases.HEADER + "".join("".join(cascade.row_texts(r, cases.CFG_F)[1]) for r in fa))
        merged = []
        for print_ref in ("False", "True"):
            mo = os.path.join(d, "merge_%s.vcf" % print_ref)
            run(["MergeVcf", "--pileup_vcf_fn", pvcf, "--full_alignment_vcf_fn", fvcf, "--output_fn", mo, "--platform", platform,
                 "--print_ref_calls", print_ref, "--qual", "2", "--ctgName", cases.CTG, "--gvcf", "False",
                 "--haploid_precise", "False", "--haploid_sensitive", "False"])
            text = open(mo).read()
            assert text.startswith(cases.HEADER)
            merged.append(text[len(cases.HEADER):])
    out[name + "/qual"] = np.array(qual)
    out[name + "/beds"] = np.array(beds if beds else [""])[:len(beds)] if beds else np.zeros(0, "U1")
    out[name + "/merged"] = np.array(merged)
    print("%s: qual %r, %d bed files, %d candidates, merged %d / %d rows" % (name, qual, len(beds), len(positions),
                                                                          merged[0].count("\n"), merged[1].count("\n")))
np.savez_compressed(os.path.join(ROOT, "tests", "golden", "cascade.npz"), **out)
