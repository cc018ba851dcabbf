"""Mints tests/golden/targets_cases.npz from the reference's own BED / known-sites code (needs the reference checkout:
CLAIR3_REFERENCE or a sibling directory; everything runs on the CPU under this Python).

* BED cases: ``preprocess/CheckEnvs.py:split_extend_bed`` writes the per-contig extended BEDs, ``shared/interval_tree.py:
  bed_tree_from`` reads them back (with ``return_bed_region``) and ``is_region_in(tree, ctg, pos - 1, pos + 1)`` decides every
  probe position; the chunks are the arithmetic of ``preprocess/CreateTensorPileupFromCffi.py:295-298``.  A case whose BED the
  reference refuses is stored as refused.
* VCF cases: ``split_extend_vcf`` and ``shared/utils.py:vcf_candidates_from``, the chunk slices of :300-308 (empty ones
  included), and per chunk the two tests of :347-355.
* SelectQual with ``--vcf_fn`` over the pileup VCFs of tests/cascade_cases.py, at the platform's and at zero ``--ref_pct_full``.
* ``postprocess/AddBackMissingVariantsInGenotyping.py`` over known VCFs and Clair3 bodies.

Giving both ``--bed_fn`` and ``--vcf_fn`` is refused by CheckEnvs (:248) before it reads either; the test checks that
refusal on ``cascade.contig_targets`` directly.  Everything is stored as one JSON document (``cases``).
    python tests/golden/make_targets_golden.py"""
import gzip
import json
import os
import subprocess
import sys
import tempfile

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

from preprocess.CheckEnvs import split_extend_bed, split_extend_vcf  # noqa: E402
from shared.interval_tree import bed_tree_from, is_region_in  # noqa: E402
from shared.utils import vcf_candidates_from  # noqa: E402
import postprocess.AddBackMissingVariantsInGenotyping as addback  # noqa: E402

from clair3_b200 import cascade  # noqa: E402
import cascade_cases as cc  # noqa: E402


def write(d, name, text, gz):
    p = os.path.join(d, name + (".gz" if gz else ""))
    with (gzip.open(p, "wt") if gz else open(p, "w")) as f:
        f.write(text)
    return p


def refused(fn, *a):
    try:
        fn(*a)
    except (SystemExit, IndexError):      # split_extend_vcf's own message for pos 0 fails to format: refused all the same
        return True
    return False


BEDS = {
    # zero-length, overlapping, unsorted and duplicate rows, a row at 0, '#' lines, a second contig
    "mixed": ("# header\nctg1\t500\t500\nctg1\t300\t420\nctg1\t0\t10\nctg1\t350\t360\nctg1\t300\t420\nctg1\t900\t1000\n"
              "#ctg1\t2000\t2100\nctg2\t40\t41\n", False),
    "gzip": ("ctg1\t120\t130\textra\tcols\nctg1\t1200\t1300\nchr20\t10\t20\n", True),
    "far": ("ctg1\t5000\t5100\n", False),                           # nothing near the probed span
    "reversed": ("ctg1\t10\t20\nctg1\t300\t200\n", False),          # e < s: refused
    "negative": ("ctg1\t-5\t20\n", False),                          # refused
}
VCFS = {
    # sites at pos <= 33 (one kept through a neighbour's interval), duplicates, other contigs, '#' lines, gzip
    "mixed": ("##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE\n"
              "ctg1\t5\t.\tA\tC\t10\tPASS\t.\tGT\t0/1\nctg1\t30\t.\tG\tT\t.\t.\t.\tGT\t1/1\nctg1\t34\t.\tC\tG\t5\tPASS\t.\tGT\t0/1\n"
              "ctg1\t400\t.\tT\tA\t8\tPASS\t.\tGT\t0/1\nctg1\t400\t.\tT\tAA\t9\tPASS\t.\tGT\t1/1\nctg1\t420\t.\tA\tG\t7\tPASS\t.\tGT\t0/1\n"
              "ctg1\t900\t.\tG\tC\t6\tPASS\t.\tGT\t0/1\nchr2\t77\t.\tA\tT\t4\tPASS\t.\tGT\t0/1\nctg1\t1000\t.\tC\tA\t6\tPASS\t.\tGT\t0/1\n", True),
    "sparse": ("ctg1\t50\t.\tA\tC\nctg1\t60\t.\tA\tC\nctg1\t700\t.\tA\tC\n", False),
    "zero": ("ctg1\t0\t.\tA\tC\n", False),                           # pos - 1 < 0: refused
}
PROBE = 1400                       # 1-based positions 1 .. PROBE of every contig are probed
CHUNKS = (1, 2, 3, 7)

out = {"bed": {}, "vcf": {}, "qual": [], "addback": []}
with tempfile.TemporaryDirectory() as d:
    for name, (text, gz) in BEDS.items():
        path = write(d, "in_" + name + ".bed", text, gz)
        split = os.path.join(d, "split_bed_" + name)
        os.makedirs(split)
        case = {"text": text, "gzip": gz, "refused": refused(split_extend_bed, path, split), "contigs": {}}
        if not case["refused"]:
            for ctg in sorted(os.listdir(split)):
                rows = [r.split() for r in open(os.path.join(split, ctg)).read().split("\n") if r]
                tree, bs, be = bed_tree_from(os.path.join(split, ctg), contig_name=ctg, return_bed_region=True)
                keep = [is_region_in(tree, ctg, p - 1, p + 1) for p in range(1, PROBE + 1)]
                chunks = {}
                for n in CHUNKS:
                    for cid in range(n):
                        size = (be - bs) // n + 1 if (be - bs) % n else (be - bs) // n
                        s = bs + 1 + size * cid
                        chunks["%d/%d" % (cid + 1, n)] = [s, s + size]
                case["contigs"][ctg] = {"starts": [int(r[1]) for r in rows], "ends": [int(r[2]) for r in rows],
                                        "bed_region": [bs, be], "keep": np.packbits(keep).tobytes().hex(), "chunks": chunks}
        out["bed"][name] = case
        print("bed %s: refused %s, contigs %s" % (name, case["refused"], sorted(case["contigs"])))

    for name, (text, gz) in VCFS.items():
        path = write(d, "in_" + name + ".vcf", text, gz)
        split = os.path.join(d, "split_vcf_" + name)
        os.makedirs(split)
        case = {"text": text, "gzip": gz, "refused": refused(split_extend_vcf, path, split), "contigs": {}}
        if not case["refused"]:
            ctgs = sorted(set(os.listdir(split)) | {r.split()[0] for r in text.splitlines() if r and r[0] != "#"})
            for ctg in ctgs:
                bed = os.path.join(split, ctg)
                rows = [r.split() for r in open(bed).read().split("\n") if r] if os.path.exists(bed) else []
                tree = bed_tree_from(bed if rows else None, contig_name=ctg)
                known = vcf_candidates_from(path, contig_name=ctg)
                chunks = {}
                for n in CHUNKS:
                    for cid in range(n):
                        size = len(known) // n if len(known) % n == 0 else len(known) // n + 1
                        part = set(known[cid * size:cid * size + size])
                        keep = [is_region_in(tree, ctg, p - 1, p + 1) and p in part for p in range(1, PROBE + 1)]
                        chunks["%d/%d" % (cid + 1, n)] = {"range": [min(part), max(part)] if part else None,
                                                          "sites": sorted(part), "keep": np.packbits(keep).tobytes().hex()}
                case["contigs"][ctg] = {"starts": [int(r[1]) for r in rows], "ends": [int(r[2]) for r in rows],
                                        "known": known, "chunks": chunks}
        out["vcf"][name] = case
        print("vcf %s: refused %s, contigs %s" % (name, case["refused"], sorted(case["contigs"])))

    # SelectQual in genotyping mode: --vcf_fn makes --ref_pct_full count as given, 0 included
    clair3 = os.path.join(REF, "clair3.py")
    known = write(d, "known.vcf", VCFS["sparse"][0], False)
    for name in cc.NAMES:
        platform, pileup, _ = cc.case(name)
        var_pct, ref_pct = cascade.PCT_FULL[platform]
        for rp in (ref_pct, 0.0):
            q = os.path.join(d, "q_%s_%s" % (name, rp))
            os.makedirs(q)
            r = subprocess.run([sys.executable, clair3, "SelectQual", "--output_fn", q, "--var_pct_full", str(var_pct),
                                "--ref_pct_full", str(rp), "--platform", platform, "--vcf_fn", known],
                               input=cc.vcf_text(pileup, cc.CFG_P), capture_output=True, text=True)
            if r.returncode:
                sys.exit(r.stderr)
            qual = open(os.path.join(q, "qual")).read()
            out["qual"].append({"case": name, "var_pct": var_pct, "ref_pct": rp, "qual": qual})
            print("SelectQual %s ref_pct %s: %s" % (name, rp, qual))

    # AddBackMissingVariantsInGenotyping
    bodies = {
        "mixed": (VCFS["mixed"][0],
                  "ctg1\t34\t.\tC\tG\t12.5\tPASS\tP\tGT:GQ:DP:AD:AF\t0/1:12:30:15,15:0.5\n"
                  "ctg1\t77\t.\tA\tT\t3\tLowQual\tP\tGT:GQ:DP:AD:AF\t0/1:3:20:10,10:0.5\n"          # not a known site: dropped
                  "ctg1\t400\t.\tT\tA\t20\tPASS\tF\tGT:GQ:DP:AD:AF\t1/1:20:30:0,30:1.0\n"
                  "chr2\t77\t.\tA\t.\t9\tRefCall\tP\tGT:GQ:DP:AD:AF\t0/0:9:18:18:0\n"),
        "short_rows": ("chr1\t10\nchr1\t5\t.\t\t\nctg9\t3\t.\tACGT\tA\t50\tPASS\n2\t8\t.\tT\tC\n2\t8\t.\tTT\tC\nchrX\t1\t.\tG\n",
                       "chrX\t1\t.\tG\tA\t9\tPASS\tP\tGT\t1/1\n"),
    }
    for name, (kvcf, body) in bodies.items():
        kp = write(d, "ab_known_%s.vcf" % name, kvcf, False)
        cp = write(d, "ab_clair3_%s.vcf" % name, "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE\n" + body, False)
        op = os.path.join(d, "ab_out_%s.vcf" % name)
        args = type("A", (), {"vcf_fn": kp, "clair3_input_vcf_fn": cp, "output_fn": op, "switch_genotype": True})
        addback.genotype_vcf(args)
        res = gzip.open(op + ".gz", "rt").read() if os.path.exists(op + ".gz") else open(op).read()
        res = "".join(r for r in res.splitlines(keepends=True) if r[0] != "#")
        out["addback"].append({"name": name, "known": kvcf, "body": body, "out": res})
        print("addback %s: %d rows" % (name, res.count("\n")))

np.savez_compressed(os.path.join(ROOT, "tests", "golden", "targets_cases.npz"), cases=np.array(json.dumps(out)))
