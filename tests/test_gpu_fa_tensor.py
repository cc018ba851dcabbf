"""The GPU full-alignment tensor builder (clair3_b200.fa_tensor) against the reference's own calculate_clair3_full_alignment:
the committed golden fixture, and - where oracle/_ref/libclair3_fa_ref.so has been built - seeded random regions run through the
compiled reference.  Bit-exact on the matrix, the all_alt_info strings and the number of rand() draws."""
import numpy as np
import pytest
import torch

from clair3_b200 import synth_reads as sr
from clair3_b200._ffi import C3BError
from clair3_b200.fa_tensor import FullAlignmentBuilder, create_tensor_full_alignment
from fa_golden import builder_kwargs, load_fa_golden
import fa_ref_cases

pytestmark = pytest.mark.gpu


def _oracle():
    from oracle import fa_ref
    if not fa_ref.available():
        pytest.skip("oracle/_ref/libclair3_fa_ref.so is not built (CLAIR3_REFERENCE at build time)")
    return fa_ref


@pytest.fixture(scope="module")
def builder():
    b = FullAlignmentBuilder(0)
    yield b
    b.close()


def _check(builder, rec, ref, cand, var, params, want_m, want_alt, want_draws):
    builder.build(rec, cand, ref, 0, variants=var, **builder_kwargs(params))
    got = builder.fetch()
    assert got.shape == want_m.shape
    bad = np.argwhere(got != want_m)
    assert len(bad) == 0, "matrix differs at %d cells, first %s: got %d want %d" % (
        len(bad), tuple(bad[0]), got[tuple(bad[0])], want_m[tuple(bad[0])])
    assert builder.alt_info_strings() == want_alt
    assert builder.sizes()[2] == want_draws


def test_golden_fixture(builder):
    rec, ref, cand, var, params, m, alt, draws = load_fa_golden()
    assert draws > 0
    _check(builder, rec, ref, cand, var, params, m, alt, draws)


CASES = [c for c in fa_ref_cases.GEN if not c[1].get("wild")]   # seed, generator arguments, parameters: one list, shared


@pytest.mark.parametrize("seed,gen,params", CASES, ids=[str(c[0]) for c in CASES])
def test_random_regions_vs_reference(builder, seed, gen, params):
    fa_ref = _oracle()
    rec, ref, cand, var = sr.random_fa_case(seed, **gen)
    m, alt, draws = fa_ref.full_alignment(rec, cand, ref, variants=var, **params)
    if gen.get("depth", 0) > 100:
        assert draws > 0                      # the shuffle ran
    _check(builder, rec, ref, cand, var, params, m, alt, draws)


def test_chained_calls(builder):
    """Two calls in one reference process = the second call seeded with the first call's draws."""
    fa_ref = _oracle()
    rec, ref, cand, var = sr.random_fa_case(31, depth=140)
    half = len(cand) // 2
    p = dict(need_haplotagging=True, matrix_depth=89, enable_dwell_time=False)
    m1, alt1, d1 = fa_ref.full_alignment(rec, cand[:half], ref, variants=var, **p)
    m2, alt2, d2 = fa_ref.full_alignment(rec, cand[half:], ref, variants=var, rand_skip=d1, **p)
    assert d1 > 0 and d2 > 0
    _check(builder, rec, ref, cand[:half], var, p, m1, alt1, d1)
    _check(builder, rec, ref, cand[half:], var, dict(p, rand_skip=d1), m2, alt2, d2)


def test_empty_inputs(builder):
    fa_ref = _oracle()
    rec, ref, cand, var = sr.random_fa_case(41, depth=10)
    p = dict(need_haplotagging=True, matrix_depth=89, enable_dwell_time=False)
    for c in (cand[:0], cand):
        empty = {k: (v[:1] * 0 if k.endswith("_off") else v[:0]) for k, v in rec.items()}
        for r in (rec, empty):
            m, alt, d = fa_ref.full_alignment(r, c, ref, variants=var, **p)
            _check(builder, r, ref, c, var, p, m, alt, d)


@pytest.mark.parametrize("channels", [8, 9])
def test_forward_from_device_matrix(builder, channels):
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_F
    rec, ref, cand, var = sr.random_fa_case(51, depth=40, dwell=channels == 9)
    sd = synth.fa_state_dict(True, channels=channels, seed=5)
    f = Clair3_F(add_indel_length=True, predict=True, input_channels=channels)
    f.to(torch.device("cuda:0"))
    f.eval()
    f.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    builder.build(rec, cand, ref, 0, variants=var, matrix_depth=89, dwell=channels == 9)
    y = builder.forward(f)
    want = f(torch.from_numpy(builder.fetch()))
    y, want = (y if isinstance(y, tuple) else (y,)), (want if isinstance(want, tuple) else (want,))
    for a, b in zip(y, want):
        assert torch.equal(a.cpu(), b.cpu())


def test_device_records_and_pipe_output(builder):
    rec, ref, cand, var = sr.random_fa_case(61, depth=30)
    from clair3_b200.pileup_counts import BamRecords
    builder.build(rec, cand, ref, 0, variants=var)
    want = builder.fetch()
    strings = builder.alt_info_strings()
    dev = BamRecords.from_dict(rec).to_device("cuda:0", ref)
    builder.build(dev, cand, None, 0, variants=var)
    assert np.array_equal(builder.fetch(), want)
    m, pos_info, alt_info = create_tensor_full_alignment(rec, "chr20", cand, ref, 0, variants=var, builder=builder)
    assert np.array_equal(m, want)
    assert [p.split(":")[1] for p in pos_info] == [s.split("-")[0] for s in strings]
    f = strings[0].rstrip().split("-")
    assert pos_info[0] == "chr20:%s:%s" % (f[0], f[2]) and alt_info[0] == f[1] + "-" + f[3]


def test_capacity_overflow_is_an_error(builder):
    """More reads on one window than the per-candidate kernel holds: an error message, no fault, and the builder stays usable."""
    n = 1700
    items = [(100, 0, 60, [("M", 50)], "A" * 50) for _ in range(n)]
    rec = sr.records_from_lists(items)
    ref = "C" * 400
    builder.build(rec, np.array([120]), ref, 0, matrix_depth=89)
    with pytest.raises(C3BError, match="overlap one candidate window"):
        builder.fetch()
    rec2, ref2, cand2, var2 = sr.random_fa_case(71, depth=10)
    builder.build(rec2, cand2, ref2, 0, variants=var2)
    assert builder.fetch().shape[0] == len(cand2)
