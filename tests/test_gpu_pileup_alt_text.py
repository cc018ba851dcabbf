"""The pileup counter's ``all_alt_info`` text formatted on the GPU (clair3_b200/csrc/plp_alt_text.cu, ``PileupCounter.alt_text``)
against the host formatter (``pileup_counts.format_alt_info`` + ``khash_iteration_order``), the reference's committed outputs
(tests/golden/pileup_ref_cases.npz) and, where oracle/_ref/ is built, the reference's own ``calculate_clair3_pileup`` - byte
for byte on every case of tests/plp_ref_cases.py; the decoder form, ``ref_base`` and ``position`` against ``alt_info_list``;
``PileupCounter.call`` against the route through host strings and ``decode.batch_calls``; misuse through its error returns."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import plp_ref_cases as cases  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pileup_ref_cases.npz")
CTG = "ctg"


@pytest.fixture(scope="module")
def counter():
    from clair3_b200 import pileup_counts as pc
    c = pc.PileupCounter(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def model():
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_P
    m = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    m.to(torch.device("cuda:0"))
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()})
    return m


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN)
    return {str(n): [str(x) for x in z["%s/alt_info" % n]] for n in z["names"]}


def config(**kw):
    from clair3_b200 import decode
    return decode.replay_config(pileup=True, add_indel_length=False)._replace(quality_score_for_pass=None)._replace(**kw)


def host_and_device(counter, case):
    """The host formatter's strings and the device's results for one count."""
    rec, ref, rs, start, end, kw = case
    counter.count(rec, start, end, ref, rs, alt_info=True, **kw)
    host = counter.alt_info_strings()
    return host, counter.alt_text().alt_text_fetch()


def check_decoder_fields(got, strings):
    from clair3_b200 import pileup_counts as pc
    want = pc.alt_info_list(strings, CTG)
    assert len(want) == len(strings) == len(got["decoder"])
    for j, (pos, chr_pos_ref, alt) in enumerate(want):
        assert got["decoder"][j] == alt, j
        assert int(got["position"][j]) == pos and CTG + ":%d:%s" % (pos, chr(got["ref_base"][j])) == chr_pos_ref, j


@pytest.mark.parametrize("name", cases.IDS)
def test_device_text_equals_host_formatter_and_golden(counter, golden, name):
    host, got = host_and_device(counter, cases.BUILD[name]())
    assert got["text"] == host
    if name in golden:
        assert got["text"] == golden[name]
    check_decoder_fields(got, host)


@pytest.mark.parametrize("name", cases.IDS)
def test_device_text_equals_reference(counter, name):
    from oracle import pileup_ref
    if not pileup_ref.available():
        pytest.skip("oracle/_ref/libclair3_pileup_ref.so is not built (needs the reference checkout at build time: CLAIR3_REFERENCE)")
    rec, ref, rs, start, end, kw = cases.BUILD[name]()
    want = pileup_ref.clair3_pileup(rec, start, end, ref, rs, **kw)["alt_info"]
    got = counter.count(rec, start, end, ref, rs, alt_info=True, **kw).alt_text().alt_text_fetch()["text"]
    assert got == want


def test_golden_covers_the_targeted_cases(golden):
    assert sorted(golden) == sorted(n for n, _ in cases.TARGETED)


def test_device_resident_records(counter):
    """Records that live in HBM: ``alt_info_strings()`` hands out the device's text, equal to the host formatter's on the host
    copy of the same records."""
    from clair3_b200 import pileup_counts as pc
    rec, ref, rs, start, end, kw = cases.BUILD["random_3"]()
    host = counter.count(rec, start, end, ref, rs, alt_info=True, **kw).alt_info_strings()
    assert len(host) > 5
    drec = pc.BamRecords.from_dict(rec).to_device(torch.device("cuda:0"), ref)
    counter.count(drec, start, end, None, rs, alt_info=True, **kw)
    assert counter.alt_info_strings() == host
    check_decoder_fields(counter.alt_text_fetch(), host)
    v = counter.alt_text_device()
    assert bytes(v["text"].cpu().numpy()).decode("latin-1") == "".join(host)
    assert v["text_off"].cpu().numpy().tolist() == np.concatenate([[0], np.cumsum([len(s) for s in host])]).tolist()


def _wide_insertion_column(n, trailing):
    """n distinct insertion strings on column P, a third of them on both strands: khash tables far beyond 64 buckets.
    trailing: reads after the last new string put present strings again."""
    strs = cases._insertion_strings(n, seed=n, long_len=12)
    first = [cases._ins_read(cases.REF, cases.P, s, flag=16 * (i & 1)) for i, s in enumerate(strs)]
    again = [cases._ins_read(cases.REF, cases.P, strs[i], flag=16 * ((i + 1) & 1)) for i in range(0, n, 3)]
    items = first + again if trailing else first[:-1] + again + first[-1:]
    items += [cases._match(cases.REF, cases.P - 40, 80) for _ in range(4)]
    return cases._case(items, cases.P - 40, cases.P + 40, call_ht=True, max_indel_length=10)


@pytest.mark.parametrize("trailing", [False, True], ids=["last_put_is_new", "trailing_puts"])
@pytest.mark.parametrize("n", [300, 799])
def test_hundreds_of_distinct_insertions(counter, n, trailing):
    host, got = host_and_device(counter, _wide_insertion_column(n, trailing))
    column = [s for s in host if s.startswith("%d-" % (cases.P + 1))]
    assert len(column) == 1 and column[0].count(" I") + column[0].count("-I") > 0.7 * n
    assert got["text"] == host
    check_decoder_fields(got, host)


def test_max_indel_length_at_and_below_an_alleles_length(counter):
    items = [cases._ins_read(cases.REF, cases.P, "ACGTAC", flag=16 * (i & 1)) for i in range(3)]
    items += [cases._del_read(cases.REF, cases.P, 6, flag=16 * (i & 1)) for i in range(3)]
    items += [cases._match(cases.REF, cases.P - 40, 80) for _ in range(4)]
    texts = {}
    for limit in (6, 5):
        host, got = host_and_device(counter, cases._case(items, cases.P - 40, cases.P + 40, call_ht=True, max_indel_length=limit))
        assert got["text"] == host
        texts[limit] = host
        other = 11 - limit                                    # the same count, formatted with the other limit
        texts["%d_as_%d" % (limit, other)] = counter.alt_text(max_indel_length=other).alt_text_fetch()["text"]
    assert sum(s.count("ACGTAC ") for s in texts[6]) == 1 and sum(s.count("ACGTAC ") for s in texts[5]) == 0
    assert texts["6_as_5"] == texts[5] and texts["5_as_6"] == texts[6]


def test_deletion_text_stops_at_the_supplied_reference_and_at_nul(counter):
    """A deletion that runs past the end of the supplied reference bases, and one across a NUL byte in them."""
    P, REF = cases.P, cases.REF
    items = [cases._del_read(REF, P, 15, flag=16 * (i & 1)) for i in range(3)] + [cases._match(REF, P - 40, 41) for _ in range(3)]
    short = REF[:P + 5]
    host, got = host_and_device(counter, cases._case(items, P - 40, P + 1, ref=short, call_ht=True))
    assert got["text"] == host and any("D%s " % REF[P + 1:P + 5] in s for s in host)
    nul = REF[:P + 3] + "\0" + REF[P + 4:]
    host, got = host_and_device(counter, cases._case(items, P - 40, P + 1, ref=nul, call_ht=True))
    assert got["text"] == host and any("D%s " % REF[P + 1:P + 3] in s for s in host)
    check_decoder_fields(got, host)


@pytest.mark.parametrize("cfg", [dict(is_haploid_precise_mode_enabled=True), dict(is_show_reference=True), {}],
                         ids=["haploid_precise", "show_ref", "default"])
def test_call_equals_the_route_through_host_strings(counter, model, cfg):
    from clair3_b200 import decode, pileup_counts as pc
    cfg = config(**cfg)
    rec, ref, rs, start, end, kw = cases.BUILD["alt_info_3"]()
    counter.count(rec, start, end, ref, rs, alt_info=True, **kw)
    strings = counter.alt_info_strings()
    Y, ok = counter.forward(model)
    tuples = pc.alt_info_list(strings, CTG)
    want = decode.batch_calls(model, [t[1] for t in tuples], [t[2] for t in tuples], Y, cfg)
    got = counter.call(model, cfg, CTG)
    assert len(strings) > 15 and ok.sum() > 10
    assert np.array_equal(got["cand_ok"], ok) and torch.equal(got["Y"], Y)
    assert np.array_equal(got["position"], want["position"]) and got["chromosome"] == want["chromosome"]
    assert np.array_equal(got["start"], want["start"])
    keep = np.nonzero(ok)[0]
    for name in want["calls"].dtype.names:
        if name != "pad":
            assert np.array_equal(got["calls"][name][keep].view(np.uint8), want["calls"][name][keep].view(np.uint8)), name
    assert want["calls"]["printed"][keep].sum() > 0
    for s in keep:
        o, c = int(want["start"][s]), want["calls"][s]
        n = int(c["ref_len"]) + int(c["alt_len"])
        assert got["text"][o:o + n].tobytes() == want["text"][o:o + n].tobytes(), s
        assert np.array_equal(got["ad"][o:o + int(c["n_ad"])], want["ad"][o:o + int(c["n_ad"])]), s
    text = decode.calls_text(got, cfg)
    assert text == decode.calls_text(want, cfg) and text.count("\n") > 0


def test_no_candidates_and_empty_region(counter, model):
    from clair3_b200 import decode
    P, REF = cases.P, cases.REF
    rec, ref, rs, start, end, kw = cases._case([cases._match(REF, P - 40, 80, flag=16 * (i & 1)) for i in range(6)], P - 40, P + 40)
    for s, e in ((start, end), (start, start)):
        got = counter.count(rec, s, e, ref, rs, alt_info=True, **kw).alt_text().alt_text_fetch()
        assert got["text"] == [] and got["decoder"] == [] and len(got["ref_base"]) == 0 and len(got["position"]) == 0
        assert counter.alt_text_sizes() == (0, 0) and counter.sizes()[1] == 0
        v = counter.alt_text_device()
        assert v["decoder"].numel() == 0 and v["decoder_off"].cpu().tolist() == [0]
        res = counter.count(rec, s, e, ref, rs, alt_info=True, **kw).call(model, config(), CTG)
        assert len(res["calls"]) == 0 and res["Y"].shape == (0, 24) and decode.calls_text(res, config()) == ""


def test_text_stage_needs_a_count_with_alt_info():
    from clair3_b200 import pileup_counts as pc
    from clair3_b200._ffi import C3BError, ffi, lib
    c = pc.PileupCounter(0)
    try:
        with pytest.raises(C3BError, match="count"):
            c.alt_text()
        assert lib().c3b_plp_alt_text(c._h, 50) != 0 and b"no c3b_plp_count" in ffi.string(lib().c3b_last_error())
        with pytest.raises(C3BError, match="no c3b_plp_alt_text"):
            c.alt_text_sizes()
        rec, ref, rs, start, end, kw = cases.BUILD["af_ins_3_of_20"]()
        c.count(rec, start, end, ref, rs, **kw)
        with pytest.raises(C3BError, match="alt_info"):
            c.alt_text()
        assert lib().c3b_plp_alt_text(c._h, 50) != 0 and b"without params.alt_info" in ffi.string(lib().c3b_last_error())
        with pytest.raises(C3BError):
            c.alt_text_fetch()
        # and the stage's own timing, read apart from the count's
        c.count(rec, start, end, ref, rs, alt_info=True, **kw).alt_text()
        assert len(c.alt_text_fetch()["text"]) == 1
        ms, launches = c.alt_text_last_ms()
        assert ms > 0 and launches == 4 and c.last_ms()[1] == 8
    finally:
        c.close()


class _Spy:
    """The library with every entry point's name and arguments logged."""

    def __init__(self, real, log):
        self._real, self._log = real, log

    def __getattr__(self, name):
        f = getattr(self._real, name)

        def logged(*args):
            self._log.append((name, args))
            return f(*args)
        return logged


def test_call_waits_once_before_the_results_are_copied(counter, model, monkeypatch):
    """Between ``count`` and the decoder's launch ``call()`` enters exactly one C entry point that waits for the stream
    (``c3b_plp_sizes``, the only ``cudaStreamSynchronize`` on the path), and it does so before Clair3_P is enqueued: the
    network and the decoder are queued back to back."""
    import clair3_b200.model as model_mod
    from clair3_b200 import pileup_counts as pc
    from clair3_b200._ffi import ffi, lib
    log = []
    spy = _Spy(lib(), log)
    monkeypatch.setattr(pc, "lib", lambda: spy)
    monkeypatch.setattr(model_mod, "lib", lambda: spy)
    rec, ref, rs, start, end, kw = cases.BUILD["alt_info_3"]()
    res = counter.count(rec, start, end, ref, rs, alt_info=True, **kw).call(model, config(), CTG)
    assert len(res["calls"]) > 15
    names = [n for n, _ in log]
    first, last = names.index("c3b_plp_count"), names.index("c3b_decode_calls")
    waits = {"c3b_plp_sizes", "c3b_plp_fetch", "c3b_plp_fetch_alleles", "c3b_plp_fetch_alt_text", "c3b_plp_last_ms",
             "c3b_plp_alt_text_last_ms"}
    waited = [n for n, a in log[first:last] if n in waits or (n == "c3b_plp_window_bounds" and a[1] != ffi.NULL)]
    assert waited == ["c3b_plp_sizes"]
    order = [names.index(n) for n in ("c3b_plp_count", "c3b_plp_alt_text", "c3b_plp_sizes", "c3b_plp_alt_text_sizes",
                                      "c3b_forward_windows_bounded", "c3b_decode_calls")]
    assert order == sorted(order)               # alt_text_sizes after sizes reads the totals that wait brought; it does not wait
