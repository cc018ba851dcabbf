"""A BAM written by bam_io and read back with fa_fields=True builds the same full-alignment tensor and allele text as the
in-memory records it was written from."""
import numpy as np
import pytest

from clair3_b200 import bam_io
from clair3_b200 import synth_reads as sr
from clair3_b200.fa_tensor import FullAlignmentBuilder

pytestmark = pytest.mark.gpu


def test_bam_round_trip_builds_the_same_tensor(tmp_path):
    rec, ref, cand, var = sr.random_fa_case(81, depth=120, dwell=True, dup_frac=0.1)
    path = str(tmp_path / "fa.bam")
    bam_io.write_bam(path, rec, [("ctg", len(ref))])
    got, _ = bam_io.read_bam(path, "ctg", fa_fields=True)
    b = FullAlignmentBuilder(0)
    try:
        b.build(rec, cand, ref, 0, variants=var, dwell=True)
        want_m, want_alt, want_sizes = b.fetch(), b.alt_info_strings(), b.sizes()
        assert want_sizes[2] > 0
        b.build(got, cand, ref, 0, variants=var, dwell=True)
        assert np.array_equal(b.fetch(), want_m)
        assert b.alt_info_strings() == want_alt and b.sizes() == want_sizes
    finally:
        b.close()
