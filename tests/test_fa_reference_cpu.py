"""The full-alignment cases of tests/fa_ref_cases.py against the reference's own ``calculate_clair3_full_alignment`` (compiled into
oracle/_ref/libclair3_fa_ref.so by oracle/fa_ref.py), without a GPU: the committed fixture tests/golden/fa_ref_cases.npz (minted by
tests/golden/make_fa_ref_cases_golden.py) must equal a fresh reference run on every targeted case, hold exactly the targeted
cases, and show that each case reaches the reference line it is written for.  The GPU builder is held to the same fixture and to
the live reference by tests/test_gpu_fa_reference.py.

16 seeded and 122 targeted cases.  The four targeted cases with ``rand_skip`` >= 2^31 step glibc's rand() that many times before the
reference starts (about 17 ns a draw, 40 to 75 s a case); their fresh reference runs are opt-in: CLAIR3_FA_REF_LARGE_SKIP=1."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import fa_ref_cases as cases  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fa_ref_cases.npz")
LARGE_SKIP_ENV = "CLAIR3_FA_REF_LARGE_SKIP"
TARGETED_IDS = [n for n, _ in cases.TARGETED]


def reference():
    from oracle import fa_ref
    if not fa_ref.available():
        pytest.skip("oracle/_ref/libclair3_fa_ref.so is not built (needs the reference checkout at build time: CLAIR3_REFERENCE)")
    return fa_ref


def skip_large(name):
    if name in cases.LARGE_SKIP and not os.environ.get(LARGE_SKIP_ENV):
        pytest.skip("rand_skip >= 2^31: the reference steps rand() that often first (set %s=1)" % LARGE_SKIP_ENV)


def fixture(name):
    """(matrix, alt_info strings, draws) the reference gave on a targeted case."""
    z = _golden()
    return z["%s/matrix" % name], [str(s) for s in z["%s/alt_info" % name]], int(z["%s/draws" % name])


_Z = {}


def _golden():
    if "z" not in _Z:
        with np.load(GOLDEN) as z:
            _Z["z"] = {k: z[k] for k in z.files}
    return _Z["z"]


def compare(tag, got, want):
    """Bit-exact: matrix (first differing cell reported), all_alt_info strings, rand() draws."""
    (gm, ga, gd), (wm, wa, wd) = got, want
    assert gm.shape == wm.shape, "%s: matrix shape %s, reference %s" % (tag, gm.shape, wm.shape)
    bad = np.argwhere(gm != wm)
    assert len(bad) == 0, "%s: matrix differs at %d cells, first %s: got %d, reference %d" % (
        tag, len(bad), tuple(bad[0]), gm[tuple(bad[0])], wm[tuple(bad[0])])
    assert len(ga) == len(wa), "%s: %d strings, reference %d" % (tag, len(ga), len(wa))
    for i, (a, b) in enumerate(zip(ga, wa)):
        assert a == b, "%s: all_alt_info[%d] %r, reference %r" % (tag, i, a, b)
    assert gd == wd, "%s: %d rand() draws, reference %d" % (tag, gd, wd)


@pytest.mark.parametrize("name", TARGETED_IDS)
def test_fixture_equals_reference(name):
    fa_ref = reference()
    skip_large(name)
    rec, ref, cand, var, p = cases.BUILD[name]()
    compare(name, fixture(name), fa_ref.full_alignment(rec, cand, ref, variants=var, **p))


def test_fixture_holds_the_targeted_cases():
    z = _golden()
    assert [str(n) for n in z["names"]] == TARGETED_IDS
    keys = {k.rsplit("/", 1)[0] for k in z if "/" in k and not k.startswith("glibc_rand/")}
    assert keys == set(TARGETED_IDS)
    assert len(TARGETED_IDS) >= 100 and len(cases.SEEDED) >= 16
    for name in TARGETED_IDS:
        m = z["%s/matrix" % name]
        _, _, cand, _, p = cases.BUILD[name]()
        assert m.shape == (len(cand), p["matrix_depth"], 33, 9 if p["enable_dwell_time"] else 8)


def test_glibc_rand_restatement_at_large_skips():
    """clair3_b200.fa_tensor.glibc_rand (the jump-ahead the GPU builder shares) against the C library's rand() stepped 2^31 - 1 to
    2^32 + 12345 times, as recorded in the fixture."""
    from clair3_b200.fa_tensor import glibc_rand
    z = _golden()
    for skip in cases.LARGE_SKIPS:
        assert np.array_equal(glibc_rand(1, skip, 80), z["glibc_rand/%d" % skip]), skip


def _fields(s):
    """all_alt_info text -> (depth, [allele field tokens])."""
    head, rest = s.split("-", 3)[1], s.split("-", 3)[3]
    return int(head), rest.split(" ")[0::2][:-1] if rest else []


def test_targeted_cases_are_aimed():
    """The targeted cases reach the lines they are written for, on the reference's outputs (the fixture)."""
    def rows(name, ch, col=16):
        m, _, _ = fixture(name)
        return m[:, :, col, ch]

    # the shuffle draws n - 1 only above matrix_depth (:121-134); offsets add up over consecutive candidates
    assert fixture("reads_depth_plus_0")[2] == 0 and fixture("reads_depth_plus_1")[2] == 8
    assert fixture("reads_1536_on_one_window")[2] == 1535
    assert fixture("ten_shuffling_candidates")[2] == sum(8 + k for k in range(10))
    for name in cases.LARGE_SKIP:
        assert fixture(name)[2] == fixture("ten_shuffling_candidates")[2]
    seeds = [fixture(n)[0] for n in ("ten_shuffling_candidates", "rand_seed_0", "rand_seed_42", "rand_seed_4294967295")]
    assert not np.array_equal(seeds[0], seeds[2]) and not np.array_equal(seeds[2], seeds[3])
    assert np.array_equal(seeds[0], seeds[1])                    # glibc's srand(0) is srand(1)
    # 49 distinct insertion strings / deletion lengths are 49 allele fields
    for kind in ("insertions", "deletions"):
        for suffix in ("", "_repeat_after_last"):
            _, f = _fields(fixture("%s_49_distinct%s" % (kind, suffix))[1][0])
            assert sum(t[0] == kind[0].upper() for t in f) == 49
    # flags 512 and 1024 are not in 2316: those reads are kept, their SNP is in the matrix (alt channel) and the text
    for fl in (512, 1024):
        assert (rows("flag_%d_kept" % fl, 1) != 0).sum() == 3 and _fields(fixture("flag_%d_kept" % fl)[1][0])[0] == 6
    for fl in (4, 8, 256, 2048):
        assert (rows("flag_%d_dropped" % fl, 1) != 0).sum() == 0
    assert _fields(fixture("mapq_19_min_20")[1][0])[0] == 3 and _fields(fixture("mapq_20_min_20")[1][0])[0] == 6
    # a passing read claims its name even without overlapping a window; a filtered one does not
    assert _fields(fixture("name_first_without_overlap")[1][0])[0] == 2
    assert _fields(fixture("name_first_filtered")[1][0])[0] == 3
    # normalize_af(count / (float)depth) expands to 100 * count / (float)depth (.h:13): 53 and 59 at depth 100, where the
    # float32 product 100 * (count / depth) would round down to 52 and 58
    m, alt, _ = fixture("af_grid_depth_81_to_120")
    at100 = [i for i, s in enumerate(alt) if _fields(s)[0] == 100]
    af100 = set(m[at100][:, :, 16, 5].ravel().tolist())
    assert {53, 59} <= af100 and not {52, 58} & af100
    for c in (53, 59):
        assert int(np.float32(100) * (np.float32(c) / np.float32(100))) == c - 1
    # normalize_mq at every mapq (.h:11), min_mq 0
    assert set(rows("mapq_0_to_255", 3).ravel().tolist()) == {int(100 * q / 60.0) for q in range(60)} | {100}
    m, _, _ = fixture("base_quality_0_to_255")
    assert set(m[:, :, :, 4].ravel().tolist()) - {0} == {int(100 * q / 40.0) for q in range(1, 40)} | {100}
    assert set(fixture("base_quality_absent")[0][:, :, :, 4].ravel().tolist()) - {0} == {100}
    # haplotagging only from mapq 20 (:629); two phase sets with max == |min| give HAP_2 (90)
    for mq, want in ((19, {60}), (20, {30, 90})):
        hap, mqv = rows("haplotag_mapq_%d" % mq, 7), rows("haplotag_mapq_%d" % mq, 3)
        assert set(hap[mqv == int(100 * mq / 60.0)].tolist()) <= want | {60} and (mq == 19 or want & set(hap.ravel().tolist()))
    assert 90 in set(rows("haplotag_two_phase_sets_gt_12", 7).ravel().tolist())
    assert {30, 90} & set(rows("haplotag_64_phase_sets", 7).ravel().tolist())
    # the overwritten insertion of 2I1I / 1I1P1I is counted (:746-752)
    assert "IAGA 1" in fixture("cigar_insertion_2I1I_on_candidate")[1][0]
    assert "IAGA 3" in fixture("cigar_insertion_2I1I_shared_string")[1][0]
    # dwell: the signal channel wraps past 127 and the reverse strand flips the signal
    m, _, _ = fixture("dwell_insertion_signal_wraps")
    assert (m[:, :, :, 8] < 0).any()
    m, _, _ = fixture("dwell_reverse_strand")
    assert len({tuple(r) for r in m[0, :, :, 8].tolist() if any(r)}) == 2
