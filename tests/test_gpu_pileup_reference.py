"""The GPU pileup feature counter (clair3_b200/csrc/plp_counts.cu) against the reference's OWN ``calculate_clair3_pileup``
(compiled into oracle/_ref/libclair3_pileup_ref.so by oracle/pileup_ref.py at build time): every case of tests/plp_ref_cases.py,
bit-exact on the matrix, the column positions, the candidate columns, the all_alt_info strings and the gVCF arrays."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import plp_ref_cases as cases  # noqa: E402
from test_pileup_reference_cpu import compare  # noqa: E402

pytestmark = pytest.mark.gpu


def _reference():
    from oracle import pileup_ref
    if not pileup_ref.available():
        pytest.skip("oracle/_ref/libclair3_pileup_ref.so is not built (needs the reference checkout at build time: CLAIR3_REFERENCE)")
    return pileup_ref


@pytest.fixture(scope="module")
def counter():
    from clair3_b200 import pileup_counts as pc
    c = pc.PileupCounter(0)
    yield c
    c.close()


def _gpu(counter, rec, start, end, ref, rs, kw):
    got = counter.count(rec, start, end, ref, rs, alt_info=True, **kw).fetch()
    got["alt_info"] = counter.alt_info_strings(got)
    return got


@pytest.mark.parametrize("name", cases.IDS)
def test_gpu_equals_reference(counter, name):
    ref_lib = _reference()
    rec, ref, rs, start, end, kw = cases.BUILD[name]()
    want = ref_lib.clair3_pileup(rec, start, end, ref, rs, **kw)
    compare(name, _gpu(counter, rec, start, end, ref, rs, kw), want, kw.get("gvcf", False))


def test_device_resident_records_equal_reference(counter):
    """Records already in HBM (``BamRecords.to_device``) give the reference's counts and candidates."""
    import torch
    from clair3_b200 import pileup_counts as pc
    ref_lib = _reference()
    rec, ref, rs, start, end, kw = cases.BUILD["random_3"]()
    want = ref_lib.clair3_pileup(rec, start, end, ref, rs, **kw)
    drec = pc.BamRecords.from_dict(rec).to_device(torch.device("cuda:0"), ref)
    got = counter.count(drec, start, end, None, rs, **kw).fetch()
    got["alt_info"] = want["alt_info"]                   # the text is formatted from host records only
    compare("device_records", got, want, kw.get("gvcf", False))
    assert len(want["cand_cols"]) > 5


def test_read_past_the_contig_end_reads_as_N(counter):
    """The documented deviation (DESIGN.md, pileup counter): bases past the contig end are 'N' - the GPU gives what the reference
    gives on the contig padded with N, the input on which the reference is defined."""
    from oracle import pileup_oracle as po
    ref_lib = _reference()
    rec, ref, rs, start, end, kw = cases.past_contig_end()
    got = _gpu(counter, rec, start, end, ref, rs, kw)
    compare("past_contig_end", got, ref_lib.clair3_pileup(rec, start, end, ref + "N" * 10, rs, **kw), False)
    want = po.clair3_pileup(rec, start, end, ref, rs, **kw)
    assert np.array_equal(got["stats"], want["stats"]) and np.array_equal(got["cand_ok"], want["cand_ok"])
