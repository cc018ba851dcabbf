"""``DeviceBamRecords.from_tensors`` against the record table (clair3_b200/records.py): the width and the length of every field it
is given are checked from tensor metadata alone, so CPU tensors show what device tensors get."""
import numpy as np
import pytest
import torch

from clair3_b200 import bam_io
from clair3_b200 import synth_reads as sr
from clair3_b200._ffi import C3BError
from clair3_b200.records import DeviceBamRecords


@pytest.fixture(scope="module")
def tensors(tmp_path_factory):
    """The records ``read_bam`` returns, with the full-alignment fields, as tensors of its own dtypes."""
    rec, _, _ = sr.random_alignment(500, depth=5, read_len=100, seed=8)
    path = str(tmp_path_factory.mktemp("records") / "r.bam")
    bam_io.write_bam(path, rec, [("c", 10000)])
    got, _ = bam_io.read_bam(path, "c", fa_fields=True)
    return {k: torch.from_numpy(v) for k, v in got.items() if k != "tid"}


def test_read_bam_records_are_accepted(tensors):
    d = DeviceBamRecords.from_tensors(tensors, "cpu")
    assert d.n_reads == len(tensors["pos"]) > 0
    h = d.host()
    assert sorted(h) == sorted(tensors)
    for k, v in h.items():
        assert np.array_equal(v, tensors[k].numpy()), k
    # the signed views a device decoder writes for the unsigned fields
    signed = dict(tensors, flag=tensors["flag"].view(torch.int16), cigar=tensors["cigar"].view(torch.int32))
    assert DeviceBamRecords.from_tensors(signed, "cpu").n_reads == d.n_reads


@pytest.mark.parametrize("field,bad,match", [
    ("pos", lambda t: t.to(torch.int32), "pos needs 8-byte integers"),
    ("cigar", lambda t: t.to(torch.int64), "cigar needs 4-byte integers"),
    ("mv", lambda t: t.to(torch.float32), "mv needs 4-byte integers"),
    ("cigar_off", lambda t: t[:-1], "cigar_off has"),
    ("qual_off", lambda t: t[:-1], "qual_off has"),
    ("l_qseq", lambda t: t[:-1], "l_qseq has"),
], ids=["pos_int32", "cigar_int64", "mv_float32", "cigar_off_short", "qual_off_short", "l_qseq_short"])
def test_wrong_width_or_length_is_refused(tensors, field, bad, match):
    with pytest.raises(C3BError, match=match):
        DeviceBamRecords.from_tensors(dict(tensors, **{field: bad(tensors[field])}), "cpu")


def test_optional_field_needs_its_offsets(tensors):
    with pytest.raises(C3BError, match="qname and qname_off go together"):
        DeviceBamRecords.from_tensors(dict(tensors, qname_off=None), "cpu")
