"""The GPU full-alignment tensor builder (clair3_b200/csrc/fa_tensor.cu + the host text formatter in clair3_b200/fa_tensor.py)
against the reference's own ``calculate_clair3_full_alignment`` on every case of tests/fa_ref_cases.py: bit-exact on the matrix,
the all_alt_info strings and the rand() draws.  The targeted cases are also held to the committed fixture
tests/golden/fa_ref_cases.npz, which needs no reference build; the live-reference comparisons skip where oracle/_ref/ is absent.

Further: the rand() jump is additive at high offset bits, a ref_start > 0 slice of the contig gives the same outputs, device-resident
records give the same matrix, the capacities are errors without a fault, and the inputs on which the reference is undefined give
the library's documented values (DESIGN.md 5b)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import fa_ref_cases as cases  # noqa: E402
from fa_golden import builder_kwargs  # noqa: E402
from test_fa_reference_cpu import TARGETED_IDS, compare, fixture, skip_large  # noqa: E402

pytestmark = pytest.mark.gpu


def _reference():
    from oracle import fa_ref
    if not fa_ref.available():
        pytest.skip("oracle/_ref/libclair3_fa_ref.so is not built (needs the reference checkout at build time: CLAIR3_REFERENCE)")
    return fa_ref


@pytest.fixture(scope="module")
def builder():
    from clair3_b200.fa_tensor import FullAlignmentBuilder
    b = FullAlignmentBuilder(0)
    yield b
    b.close()


def _gpu(builder, rec, ref, cand, var, p, ref_start=0):
    builder.build(rec, cand, ref, ref_start, variants=var, **builder_kwargs(p))
    return builder.fetch(), builder.alt_info_strings(), builder.sizes()[2]


@pytest.mark.parametrize("name", cases.IDS)
def test_gpu_equals_reference(builder, name):
    fa_ref = _reference()
    skip_large(name)
    rec, ref, cand, var, p = cases.BUILD[name]()
    compare(name, _gpu(builder, rec, ref, cand, var, p), fa_ref.full_alignment(rec, cand, ref, variants=var, **p))


@pytest.mark.parametrize("name", TARGETED_IDS)
def test_gpu_equals_fixture(builder, name):
    rec, ref, cand, var, p = cases.BUILD[name]()
    compare(name, _gpu(builder, rec, ref, cand, var, p), fixture(name))


def test_reverse_order_on_one_builder(builder):
    """Every targeted case again, last to first, on the builder that just ran them all: scratch reused after larger calls."""
    for name in reversed(TARGETED_IDS):
        rec, ref, cand, var, p = cases.BUILD[name]()
        compare(name, _gpu(builder, rec, ref, cand, var, p), fixture(name))


@pytest.mark.parametrize("S", [2 ** 33 + 7, 2 ** 40, 2 ** 62 - 10 ** 6])
def test_rand_jump_is_additive_at_high_bits(builder, S):
    """Candidate 1 of a call at rand_skip S is candidate 0 of a call at S + (candidate 0's draws).  Self-consistency only: the
    large-skip fixture cases pin the jump to glibc."""
    rec, ref, cand, var, p = cases.BUILD["ten_shuffling_candidates"]()
    cand = cand[:2]
    m, _, d = _gpu(builder, rec, ref, cand, var, dict(p, rand_skip=S))
    _, _, d0 = _gpu(builder, rec, ref, cand[:1], var, dict(p, rand_skip=S))
    assert 0 < d0 < d
    m1, _, _ = _gpu(builder, rec, ref, cand[1:], var, dict(p, rand_skip=S + d0))
    assert np.array_equal(m[1], m1[0])
    m2, _, _ = _gpu(builder, rec, ref, cand[1:], var, dict(p, rand_skip=S + d0 + 1))
    assert not np.array_equal(m[1], m2[0])


@pytest.mark.parametrize("name", ["deletion_len_50_max_50", "haplotag_two_phase_sets_gt_12", "cigar_deletion_then_insertion",
                                  "dwell_insertion_signal_wraps"])
def test_reference_slice_with_offset(builder, name):
    """ref_start > 0 with a slice that covers every read, variant context and deletion text gives the ref_start = 0 outputs."""
    rec, ref, cand, var, p = cases.BUILD[name]()
    rs = int(min([int(rec["pos"].min()), int(cand.min()) - 16] + [v[0] - 11 for v in var])) - 3
    assert rs > 0
    want = _gpu(builder, rec, ref, cand, var, p)
    compare(name + "@%d" % rs, _gpu(builder, rec, ref[rs:], cand, var, p, ref_start=rs), want)


@pytest.mark.parametrize("name", ["names_4096_distinct", "dwell_insertion_signal_wraps", "cigar_insertion_2I1I_shared_string"])
def test_device_resident_records(builder, name):
    import torch
    from clair3_b200.pileup_counts import BamRecords
    rec, ref, cand, var, p = cases.BUILD[name]()
    want_m, _, want_d = fixture(name)
    dev = BamRecords.from_dict(rec).to_device(torch.device("cuda:0"), ref)
    builder.build(dev, cand, None, 0, variants=var, **builder_kwargs(p))
    compare(name + "_device", (builder.fetch(), [], builder.sizes()[2]), (want_m, [], want_d))


def _still_usable(builder):
    name = "cigar_insertion_2I1I_shared_string"
    rec, ref, cand, var, p = cases.BUILD[name]()
    compare(name, _gpu(builder, rec, ref, cand, var, p), fixture(name))


def test_capacities_are_errors(builder):
    """1537 reads on one window (K11's shared memory holds 1536) and 65 phase sets on one read: a C3BError from sizes(), no
    fault, and the builder stays usable."""
    from clair3_b200._ffi import C3BError
    reads = [cases.match(cases.C - 16 + i % 20, 20) for i in range(1537)]
    r2, ref2, cand2, var2, p2 = cases.case(reads, [cases.C])
    builder.build(r2, cand2, ref2, 0, variants=var2, **builder_kwargs(p2))
    with pytest.raises(C3BError, match="overlap one candidate window"):
        builder.sizes()
    _still_usable(builder)
    C = cases.C
    var = [(C - 32 + i, cases.REF[C - 32 + i], cases.SNP[cases.REF[C - 32 + i]], 1, 100 + i) for i in range(65)]
    r3, ref3, cand3, var3, p3 = cases.case([cases.match(C - 32, 70), cases.match(C - 32, 70)], [C], variants=var, need_haplotagging=True)
    builder.build(r3, cand3, ref3, 0, variants=var3, **builder_kwargs(p3))
    with pytest.raises(C3BError, match="more than 64 phase sets"):
        builder.sizes()
    _still_usable(builder)


def test_inputs_the_reference_leaves_undefined(builder):
    """DESIGN.md 5b: a candidate below 16 gets no matrix rows (the reference's size_t start wraps) and draws nothing, though its
    counters see the reads; a column under a reference skip is uncovered on that read (all channels 0)."""
    C = cases.C
    reads = [cases.match(0, 40, subst={10: "A"} if i % 2 else None) for i in range(12)]
    r, ref, cand, var, p = cases.case(reads, [10])
    m, alt, d = _gpu(builder, r, ref, cand, var, p)
    assert not m.any() and d == 0
    assert alt[0].startswith("11-12-")
    skip = cases.read(C - 30, [("M", 25), ("N", 10), ("M", 25)], cases.REF[C - 30:C - 5] + cases.REF[C + 5:C + 30])
    r, ref, cand, var, p = cases.case([skip], [C])
    m, alt, d = _gpu(builder, r, ref, cand, var, p)
    row = m[0, (p["matrix_depth"] - 1) // 2]             # one read: the prefix padding is (depth - 1) >> 1 rows
    assert not row[16 - 5:16 + 5].any()
    assert row[:16 - 5, 0].all() and row[16 + 5:, 0].all()
    assert alt[0].startswith("301-0-")
