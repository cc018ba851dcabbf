"""The cascade's host layer (clair3_b200/cascade.py) against the reference's own SelectQual, SelectCandidates and MergeVcf
(tests/golden/cascade.npz, minted by tests/golden/make_cascade_golden.py from the call results of tests/cascade_cases.py), and
the probability threshold that makes the device selection exact."""
import os

import numpy as np
import pytest

import cascade_cases as cases
from clair3_b200 import cascade, decode
from clair3_b200.fa_tensor import candidates_from_bed

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "cascade.npz"))


def _qual(bits):
    return decode.quality_score_from(np.array(bits, np.uint32).view(np.float32)[()])


@pytest.fixture(scope="module", params=cases.NAMES)
def case(request):
    name = request.param
    platform, pileup, _ = cases.case(name)
    return name, platform, pileup


def test_qual_cutoffs(case):
    name, platform, pileup = case
    var_q, ref_q = cascade.qual_cutoffs([pileup], platform)
    assert str(var_q) + " " + str(ref_q) == str(GOLDEN[name + "/qual"])


def test_qual_cutoffs_over_several_results(case):
    """Genome-wide: the cut-offs of the rows of several results together (SelectQual reads the whole pileup VCF)."""
    name, platform, pileup = case
    n = len(pileup["calls"])
    halves = []
    for sl in (slice(0, n // 2), slice(n // 2, n)):
        h = {k: (v[sl] if k != "text" and k != "ad" else v) for k, v in pileup.items()}
        h["chromosome"] = pileup["chromosome"][sl]
        halves.append(h)
    assert cascade.qual_cutoffs(halves, platform) == cascade.qual_cutoffs([pileup], platform)


def test_select_and_bed_files(case, tmp_path):
    name, platform, pileup = case
    var_q, ref_q = (float(x) for x in str(GOLDEN[name + "/qual"]).split())
    pos, chunks = cascade.select(pileup, var_q, ref_q)
    beds = list(GOLDEN[name + "/beds"])
    assert len(chunks) == len(beds)
    if name == "two_chunks":
        assert len(chunks) == 2 and chunks[0] == (0, cascade.SPLIT_BED_SIZE)
    if name == "zero_ref":
        assert ref_q == 0.0
    for (lo, hi), bed in zip(chunks, beds):
        assert cascade.bed_text(cases.CTG, pos[lo:hi]) == bed
        path = tmp_path / "c.bed"
        path.write_text(bed)
        assert np.array_equal(candidates_from_bed(str(path), cases.CTG)[0], pos[lo:hi])
    if name in ("ont", "hifi"):
        assert pos[0] < 17, "the case must select candidates within 17 bases of the contig start"


def test_merge(case):
    name, platform, pileup = case
    var_q, ref_q = (float(x) for x in str(GOLDEN[name + "/qual"]).split())
    pos, chunks = cascade.select(pileup, var_q, ref_q)
    fa = cases.fa_results(pileup, pos, chunks, seed=len(name))
    for print_ref, want in zip((False, True), GOLDEN[name + "/merged"]):
        got = cascade.merge(pileup, fa, cases.CFG_P, cases.CFG_F, qual=2, print_ref=print_ref)
        assert got == str(want)
    if name == "ont":
        body = str(GOLDEN[name + "/merged"][0])
        assert "\t2.00\tLowQual\t" in body, "QUAL 2.00 flips to LowQual"


@pytest.mark.parametrize("cut", [0.0, 0.01, 2.0, 2.005, 9.48, 9.485, 17.06, 42.5, 109.99, 110.0, 110.01])
def test_prob_threshold_exhaustive_around(cut):
    """QUAL is monotone over the bit patterns around the threshold and the threshold splits them exactly: below it QUAL < cut,
    from it on QUAL >= cut (checked pattern by pattern over 4097 patterns each side)."""
    t = cascade.prob_threshold(cut)
    lo, hi = max(0, t - 4096), min(0x3F800000, t + 4096)
    quals = [_qual(b) for b in range(lo, hi + 1)]
    assert all(a <= b for a, b in zip(quals, quals[1:]))
    for b, q in zip(range(lo, hi + 1), quals):
        assert (q < cut) == (b < t), (cut, b, q, t)


def test_prob_threshold_rounding_boundaries():
    """Either side of a %.2f rounding boundary: the first pattern of each QUAL value is its threshold."""
    t = cascade.prob_threshold(2.0)
    for cut in (_qual(t - 1), _qual(t), _qual(t + 50000), _qual(t + 50001)):
        u = cascade.prob_threshold(cut)
        assert _qual(u) == cut and (u == 0 or _qual(u - 1) < cut)
        assert abs(round(cut, 2) - cut) < 1e-12
    assert cascade.prob_threshold(0.0) == 0
    assert cascade.prob_threshold(1e9) == 0x3F800001


def test_prob_threshold_monotone_sampled():
    rng = np.random.default_rng(7)
    bits = np.sort(rng.integers(0, 0x3F800001, 20000))
    quals = [_qual(b) for b in bits]
    assert all(a <= b for a, b in zip(quals, quals[1:]))


def test_out_of_scope():
    _, pileup, _ = cases.case("zero_ref")
    with pytest.raises(NotImplementedError):
        cascade.qual_cutoffs([pileup], "ilmn")
    with pytest.raises(NotImplementedError):
        cascade.merge(pileup, [], cases.CFG_P._replace(is_haploid_sensitive_mode_enabled=True), cases.CFG_F)
    with pytest.raises(NotImplementedError):
        cascade.merge(pileup, [], cases.CFG_P, cases.CFG_F._replace(gvcf=True))


@pytest.mark.parametrize("which", ["p", "f"])
def test_route_needs_reference_rows(which):
    """The reference's pipeline prints RefCall rows from both networks, and the cut-offs, the selection and the merge read
    them: a route without them is refused before any work."""
    cfg_p = cases.CFG_P._replace(is_show_reference=which != "p")
    cfg_f = cases.CFG_F._replace(is_show_reference=which != "f")
    for route in (cascade.call_region, cascade.call_region_host):
        with pytest.raises(ValueError, match="is_show_reference"):
            route("x.bam", cases.CTG, 0, 100, "A" * 200, 0, None, None, cfg_p, cfg_f)
