"""The pileup feature counter's C oracle (oracle/pileup_oracle.c) against the reference's OWN ``calculate_clair3_pileup``
(src/clair3_pileup.c, compiled with src/medaka_bamiter.c and the reference's khash into oracle/_ref/libclair3_pileup_ref.so by
oracle/pileup_ref.py): bit-exact on the matrix, the column positions, the candidate columns, the all_alt_info strings byte for
byte and the gVCF arrays, on every case of tests/plp_ref_cases.py.  The GPU counter is held to the oracle by
tests/test_gpu_pileup_counts.py and to the reference directly by tests/test_gpu_pileup_reference.py.

tests/golden/pileup_ref_cases.npz keeps the reference's outputs of the targeted cases, so that they pin the oracle even where the
reference checkout (and with it oracle/_ref/) is absent."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import pileup_oracle as po  # noqa: E402
import plp_ref_cases as cases  # noqa: E402

KEYS = ("matrix", "major", "cand_cols")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pileup_ref_cases.npz")


def reference():
    from oracle import pileup_ref
    if not pileup_ref.available():
        pytest.skip("oracle/_ref/libclair3_pileup_ref.so is not built (needs the reference checkout at build time: CLAIR3_REFERENCE)")
    return pileup_ref


def compare(tag, got, want, gvcf):
    """Bit-exact comparison of a counter's outputs with the reference's; returns the number of compared cells and strings."""
    n = 0
    for k in KEYS + (("pos_ref_count", "pos_total_count") if gvcf else ()):
        assert got[k].shape == want[k].shape, "%s: %s shape %s, reference %s" % (tag, k, got[k].shape, want[k].shape)
        d = np.argwhere(got[k] != want[k])
        assert len(d) == 0, "%s: %s differs at %d places, first %s: %s vs reference %s" % (
            tag, k, len(d), d[0].tolist(), got[k][tuple(d[0])], want[k][tuple(d[0])])
        n += got[k].size
    assert len(got["alt_info"]) == len(want["alt_info"]), "%s: %d candidate strings, reference %d" % (tag, len(got["alt_info"]), len(want["alt_info"]))
    for a, b in zip(got["alt_info"], want["alt_info"]):
        assert a == b, "%s: all_alt_info %r, reference %r" % (tag, a, b)
    return n + len(want["alt_info"])


@pytest.mark.parametrize("name", cases.IDS)
def test_oracle_equals_reference(name):
    ref_lib = reference()
    rec, ref, rs, start, end, kw = cases.BUILD[name]()
    want = ref_lib.clair3_pileup(rec, start, end, ref, rs, **kw)
    got = po.clair3_pileup(rec, start, end, ref, rs, alt_info=True, **kw)
    compare(name, got, want, kw.get("gvcf", False))


def test_targeted_cases_are_aimed():
    """The targeted cases reach the lines they are written for (checked on the reference's own outputs)."""
    ref_lib = reference()
    out = {}
    for name in ("af_snp_2_of_25", "af_snp_1_of_25", "af_ins_3_of_20", "af_ins_2_of_20", "equal_majority_alt_G_ref_C",
                 "insertions_25_distinct_trailing_puts", "long_deletion_at_region_end", "region_start_0", "read_base_N",
                 "deletion_len_200"):
        if name not in cases.BUILD:
            continue
        rec, ref, rs, start, end, kw = cases.BUILD[name]()
        out[name] = ref_lib.clair3_pileup(rec, start, end, ref, rs, **kw)
    assert len(out["af_snp_2_of_25"]["alt_info"]) == 1 and len(out["af_snp_1_of_25"]["alt_info"]) == 0
    assert len(out["af_ins_3_of_20"]["alt_info"]) == 1 and len(out["af_ins_2_of_20"]["alt_info"]) == 0
    s = out["insertions_25_distinct_trailing_puts"]["alt_info"][0]
    assert s.count(" I") + s.count("-I") >= 20
    d = out["long_deletion_at_region_end"]["alt_info"][0]
    assert len(d.split(" ")[0].split("-D")[1]) == 1001               # clipped at end + 1000 inclusive
    assert (out["deletion_len_200"]["matrix"][:, [6, 15]].sum()) >= 3


def test_read_past_the_contig_end_is_a_documented_deviation():
    """A kept read that reaches past the contig end makes the reference read its reference sequence out of bounds, so the binding
    refuses it; the oracle (and the GPU counter, tests/test_gpu_pileup_reference.py) treat the missing bases as 'N': the columns
    are counted, their reference feature is A's (base2index of N) and none of them is a candidate."""
    ref_lib = reference()
    rec, ref, rs, start, end, kw = cases.past_contig_end()
    with pytest.raises(ValueError, match="past the contig end"):
        ref_lib.clair3_pileup(rec, start, end, ref, rs, **kw)
    got = po.clair3_pileup(rec, start, end, ref, rs, alt_info=True, **kw)
    beyond = got["major"] >= len(ref)
    assert beyond.sum() == 10 and (got["matrix"][beyond][:, 0] < 0).all()
    assert all(int(s.split("-")[0]) <= len(ref) for s in got["alt_info"])
    want = ref_lib.clair3_pileup(rec, start, end, ref + "N" * 10, rs, **kw)
    compare("past_contig_end_as_N", got, want, False)


def test_committed_reference_outputs():
    """tests/golden/pileup_ref_cases.npz (minted from the compiled reference by tests/golden/make_pileup_counts_golden.py) against
    the oracle, for every targeted case: runs without the reference checkout."""
    z = np.load(GOLDEN)
    names = [str(x) for x in z["names"]]
    assert len(names) == len(cases.TARGETED)
    for name in names:
        rec, ref, rs, start, end, kw = cases.BUILD[name]()
        got = po.clair3_pileup(rec, start, end, ref, rs, alt_info=True, **kw)
        want = {k: z["%s/%s" % (name, k)] for k in KEYS + ("pos_ref_count", "pos_total_count")}
        want["alt_info"] = [str(x) for x in z["%s/alt_info" % name]]
        compare(name, got, want, kw.get("gvcf", False))
