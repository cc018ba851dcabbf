"""Mints tests/golden/pileup_counts.npz and tests/golden/pileup_ref_cases.npz from the reference's own calculate_clair3_pileup,
compiled by oracle/pileup_ref.py (needs the reference checkout: CLAIR3_REFERENCE or a sibling directory).

pileup_counts.npz: two small seeded record sets, INPUT RECORDS INCLUDED, so that the committed vectors pin both the C oracle and
(on a GPU) the CUDA counter against drift.  matrix, major, cand_cols, the all_alt_info strings and the gVCF arrays are the
reference's outputs; stats and cand_ok, which the reference does not have, come from oracle/pileup_oracle.c, and the script
refuses to write anything unless the oracle equals the reference on every shared output - cand_ok included: the positions it
keeps must be those the reference's own CreateTensorPileup keeps (oracle/pileup_tensor_ref.py) for the 1-based slice whose
counter region is the case's region.  These vectors are reference-confirmed.

pileup_ref_cases.npz: the reference's outputs on every targeted case of tests/plp_ref_cases.py (the inputs are rebuilt from that
module's code), so those cases pin the oracle even where oracle/_ref/ was not built.
    python tests/golden/make_pileup_counts_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from clair3_b200 import synth_reads as sr  # noqa: E402
from clair3_b200.pileup_counts import counting_region  # noqa: E402
from oracle import pileup_oracle as po, pileup_ref as pr, pileup_tensor_ref as ptr  # noqa: E402
import plp_ref_cases as cases  # noqa: E402
from test_pileup_reference_cpu import compare  # noqa: E402

if pr.build() is None or not ptr.available():
    sys.exit("the reference checkout is needed: set CLAIR3_REFERENCE")

out = {}
for tag, kw, cnt in (("a", dict(region_len=600, depth=25, read_len=300, seed=71, wild=True, indel_rate=0.08, n_rate=0.01), dict(gvcf=True)),
                     ("b", dict(region_len=900, depth=12, read_len=150, seed=72, gaps=[(1400, 1470)], origin=1000), dict(call_ht=True, max_indel_length=5))):
    rec, ref, rs = sr.random_alignment(**kw)
    start = kw.get("origin", 1000)
    end = start + kw["region_len"]
    want = pr.clair3_pileup(rec, start, end, ref, rs, **cnt)
    r = po.clair3_pileup(rec, start, end, ref, rs, alt_info=True, **cnt)
    compare("pileup_counts_%s" % tag, r, want, True)
    ctg_start, ctg_end = start + 35, end - 33
    assert counting_region(ctg_start, ctg_end) == (start, end)
    _, pos_info, _ = ptr.create_tensor_pileup(rec, ref, rs, ctg_start, ctg_end, call_ht=cnt.get("call_ht", False))
    kept = r["major"][r["cand_cols"][r["cand_ok"] == 1]] + 1
    if not np.array_equal(kept, ptr.kept_positions(pos_info)):
        sys.exit("pileup_counts_%s: the oracle's cand_ok keeps %s, the reference %s" % (tag, kept.tolist(), ptr.kept_positions(pos_info).tolist()))
    for k, v in rec.items():
        out["%s_rec_%s" % (tag, k)] = v
    out["%s_ref" % tag] = np.frombuffer(ref.encode(), dtype=np.uint8)
    out["%s_meta" % tag] = np.array([start, end, rs, int(cnt.get("gvcf", False)), int(cnt.get("call_ht", False)), cnt.get("max_indel_length", 50)], np.int64)
    for k in ("matrix", "major", "cand_cols", "pos_ref_count", "pos_total_count"):
        out["%s_%s" % (tag, k)] = want[k]
    for k in ("stats", "cand_ok"):
        out["%s_%s" % (tag, k)] = r[k]
    out["%s_alt_info" % tag] = np.array(want["alt_info"])
np.savez_compressed(os.path.join(ROOT, "tests", "golden", "pileup_counts.npz"), **out)
print({k: v.shape for k, v in out.items() if k.endswith(("matrix", "alt_info"))})

ref_cases = {"names": np.array([n for n, _ in cases.TARGETED])}
for name, build in cases.TARGETED:
    rec, ref, rs, start, end, kw = build()
    want = pr.clair3_pileup(rec, start, end, ref, rs, **kw)
    for k in ("matrix", "major", "cand_cols", "pos_ref_count", "pos_total_count"):
        ref_cases["%s/%s" % (name, k)] = want[k]
    ref_cases["%s/alt_info" % name] = np.array(want["alt_info"], dtype=str)
np.savez_compressed(os.path.join(ROOT, "tests", "golden", "pileup_ref_cases.npz"), **ref_cases)
print("%d targeted cases" % len(cases.TARGETED))
