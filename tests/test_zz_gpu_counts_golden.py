"""The feature counter against the COMMITTED fixtures of tests/golden/pileup_counts.npz, through the C-ABI (counts, candidates, gVCF
arrays, all_alt_info).  Kept in its own module, collected last, after the counter's operation-by-operation tests in
tests/test_gpu_pileup_counts.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def counter():
    from clair3_b200 import pileup_counts as pc
    c = pc.PileupCounter(0)
    yield c
    c.close()


@pytest.mark.parametrize("tag", ["a", "b"])
def test_committed_golden_vectors(counter, tag):
    from test_pileup_oracle import load_counts_golden
    rec, ref, rs, start, end, kw, want = load_counts_golden(tag)
    got = counter.count(rec, start, end, ref, rs, alt_info=True, **kw).fetch()
    for k in ("major", "matrix", "stats", "cand_cols", "cand_ok") + (("pos_ref_count", "pos_total_count") if kw["gvcf"] else ()):
        assert got[k].shape == want[k].shape and np.array_equal(got[k], want[k]), k
    assert counter.alt_info_strings(got) == want["alt_info"]
