"""The full-alignment builder's ``all_alt_info`` text formatted on the GPU (clair3_b200/csrc/fa_alt_text.cu,
``FullAlignmentBuilder.alt_text``) against the host formatter (``fa_tensor.format_alt_info`` + ``khash_iteration_order``), the
reference's committed outputs (tests/golden/fa_ref_cases.npz) and, where oracle/_ref/ is built, the reference's own
``calculate_clair3_full_alignment`` - byte for byte on every case of tests/fa_ref_cases.py; the decoder form, ``ref_base`` and
``position`` against ``create_tensor_full_alignment``'s split; khash tables of hundreds of keys; ``FullAlignmentBuilder.call``
against the route through host strings and ``decode.batch_calls``; misuse through its error returns."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import fa_ref_cases as cases  # noqa: E402
from fa_golden import builder_kwargs  # noqa: E402
from test_fa_reference_cpu import TARGETED_IDS, fixture, skip_large  # noqa: E402

pytestmark = pytest.mark.gpu

CTG = "ctg"
C = cases.C


@pytest.fixture(scope="module")
def builder():
    from clair3_b200.fa_tensor import FullAlignmentBuilder
    b = FullAlignmentBuilder(0)
    yield b
    b.close()


@pytest.fixture(scope="module")
def model():
    from clair3_b200 import synth
    from clair3_b200.model import Clair3_F
    m = Clair3_F(add_indel_length=True, predict=True, input_channels=8)
    m.to(torch.device("cuda:0"))
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=8, seed=1).items()})
    return m


def config(**kw):
    from clair3_b200 import decode
    return decode.replay_config(pileup=False, add_indel_length=True)._replace(quality_score_for_pass=None)._replace(**kw)


def build(builder, case, ref_start=0):
    rec, ref, cand, var, p = case
    return builder.build(rec, cand, ref[ref_start:], ref_start, variants=var, **builder_kwargs(p))


def host_and_device(builder, case, ref_start=0):
    """The host formatter's strings and the device's results for one build."""
    build(builder, case, ref_start)
    host = builder.alt_info_strings()
    return host, builder.alt_text().alt_text_fetch()


def split(strings):
    """``create_tensor_full_alignment``'s (all_position_info, all_alt_info) of the strings."""
    pos_info, alt_info = [], []
    for s in strings:
        pos, depth, center_ref_base, alt = s.rstrip().split("-")[:4]
        pos_info.append(CTG + ":" + pos + ":" + center_ref_base)
        alt_info.append(depth + "-" + alt)
    return pos_info, alt_info


def check_decoder_fields(got, strings):
    pos_info, alt_info = split(strings)
    assert len(strings) == len(got["decoder"]) == len(got["ref_base"]) == len(got["position"])
    for j, (pi, alt) in enumerate(zip(pos_info, alt_info)):
        assert got["decoder"][j] == alt, j
        assert CTG + ":%d:%s" % (got["position"][j], chr(got["ref_base"][j])) == pi, j


@pytest.mark.parametrize("name", cases.IDS)
def test_device_text_equals_host_formatter_and_fixture(builder, name):
    host, got = host_and_device(builder, cases.BUILD[name]())
    assert got["text"] == host
    if name in TARGETED_IDS:
        assert got["text"] == fixture(name)[1]
    check_decoder_fields(got, host)


@pytest.mark.parametrize("name", cases.IDS)
def test_device_text_equals_reference(builder, name):
    from oracle import fa_ref
    if not fa_ref.available():
        pytest.skip("oracle/_ref/libclair3_fa_ref.so is not built (needs the reference checkout at build time: CLAIR3_REFERENCE)")
    skip_large(name)
    rec, ref, cand, var, p = cases.BUILD[name]()
    want = fa_ref.full_alignment(rec, cand, ref, variants=var, **p)[1]
    assert build(builder, cases.BUILD[name]()).alt_text().alt_text_fetch()["text"] == want


def test_the_cases_cover_dwell_and_depth_55():
    ps = [cases.BUILD[n]()[4] for n in cases.IDS if n.startswith(("seeded", "wild"))]
    assert any(p["enable_dwell_time"] for p in ps) and any(p["matrix_depth"] == 55 for p in ps)


def _many_alleles(kind, n, trailing):
    """One candidate with n distinct insertion strings or deletion lengths, each first shown by its own read.  trailing: reads
    after the last new allele show earlier ones again; otherwise one repeat comes before the last new allele."""
    ref = cases.sr.random_reference(n + 400, seed=17, lower_frac=0.1, n_frac=0.0)
    if kind == "ins":
        strs = cases._insertion_strings(n, seed=n)
        new = [cases.ins_read(C, s, ref=ref) for s in strs]
        rep = [cases.ins_read(C, strs[i], ref=ref) for i in range(0, n, 97)]
    else:
        new = [cases.del_read(C, 1 + i, ref=ref, right=10) for i in range(n)]
        rep = [cases.del_read(C, 1 + i, ref=ref, right=10) for i in range(0, n, 97)]
    reads = new + rep if trailing else new[:-1] + rep + new[-1:]
    return cases.case(reads + cases.cover(3, ref=ref), [C], ref=ref, max_indel_length=n + 10)


@pytest.mark.parametrize("trailing", [False, True], ids=["last_put_is_new", "repeat_after_last_new"])
@pytest.mark.parametrize("kind,n", [("ins", 300), ("ins", 700), ("del", 300)])
def test_hundreds_of_distinct_alleles(builder, kind, n, trailing):
    host, got = host_and_device(builder, _many_alleles(kind, n, trailing))
    fields = host[0].split(" ")[::2]
    assert sum(f.startswith(kind[0].upper(), f.rfind("-") + 1) for f in fields) == n
    assert got["text"] == host
    check_decoder_fields(got, host)


def test_max_indel_length_at_and_below_an_alleles_length(builder):
    items = [cases.ins_read(C, "ACGTAC", flag=16 * (i & 1)) for i in range(3)] + [cases.del_read(C, 6) for _ in range(2)]
    items += cases.cover(3)
    texts = {}
    for limit in (6, 5):
        host, got = host_and_device(builder, cases.case(items, [C], max_indel_length=limit))
        assert got["text"] == host
        check_decoder_fields(got, host)
        texts[limit] = host
        other = 11 - limit                                    # the same build, formatted with the other limit
        texts["%d_as_%d" % (limit, other)] = builder.alt_text(max_indel_length=other).alt_text_fetch()["text"]
    assert "I%sACGTAC 3 " % cases.REF[C] in texts[6][0] and "D%s 2 " % cases.REF[C + 1:C + 7] in texts[6][0]
    assert "ACGTAC" not in texts[5][0] and " D" not in texts[5][0]
    assert texts["6_as_5"] == texts[5] and texts["5_as_6"] == texts[6]


def test_deletion_text_stops_at_the_supplied_reference_and_at_nul(builder):
    """A deletion that runs past the end of the supplied reference bases, and one across a NUL byte in them."""
    REF = cases.REF
    items = [cases.del_read(C, 15) for _ in range(3)] + [cases.match(C - 20, 21) for _ in range(2)]
    host, got = host_and_device(builder, cases.case(items, [C], ref=REF[:C + 5]))
    assert got["text"] == host and "D%s 3 " % REF[C + 1:C + 5] in host[0]
    nul = REF[:C + 3] + "\0" + REF[C + 4:]
    host, got = host_and_device(builder, cases.case(items, [C], ref=nul))
    assert got["text"] == host and "D%s 3 " % REF[C + 1:C + 3] in host[0]
    check_decoder_fields(got, host)


@pytest.mark.parametrize("name", ["deletion_len_50_max_50", "deletions_49_distinct_repeat_after_last", "deletion_text_to_contig_end",
                                  "seeded_9", "seeded_12"])
def test_reference_slice_with_offset(builder, name):
    """ref_start > 0 with a slice that covers every read, variant context and deletion text gives the ref_start = 0 strings."""
    case = cases.BUILD[name]()
    rec, _, cand, var, _ = case
    rs = int(min([int(rec["pos"].min()), int(cand.min()) - 16] + [v[0] - 11 for v in var])) - 3
    assert rs > 0
    host, want = host_and_device(builder, case)
    got = build(builder, case, ref_start=rs).alt_text().alt_text_fetch()
    assert got["text"] == want["text"] == host
    assert builder.alt_info_strings() == host
    check_decoder_fields(got, host)


@pytest.mark.parametrize("name", ["seeded_9", "cigar_insertion_2I1I_shared_string", "insertions_49_distinct_repeat_after_last",
                                  "dwell_insertion_signal_wraps"])
def test_device_resident_records(builder, name):
    """Records that live in HBM: ``alt_info_strings()`` hands out the device's text, equal to the host formatter's on the host
    copy of the same records."""
    from clair3_b200.pileup_counts import BamRecords
    rec, ref, cand, var, p = cases.BUILD[name]()
    host = build(builder, (rec, ref, cand, var, p)).alt_info_strings()
    dev = BamRecords.from_dict(rec).to_device(torch.device("cuda:0"), ref)
    builder.build(dev, cand, None, 0, variants=var, **builder_kwargs(p))
    assert builder.alt_info_strings() == host
    check_decoder_fields(builder.alt_text_fetch(), host)
    v = builder.alt_text_device()
    assert bytes(v["text"].cpu().numpy()).decode("latin-1") == "".join(host)
    assert v["text_off"].cpu().numpy().tolist() == np.concatenate([[0], np.cumsum([len(s) for s in host])]).tolist()


@pytest.mark.parametrize("cfg", [dict(is_haploid_precise_mode_enabled=True), dict(is_show_reference=True), {}],
                         ids=["haploid_precise", "show_ref", "default"])
def test_call_equals_the_route_through_host_strings(builder, model, cfg):
    from clair3_b200 import decode
    cfg = config(**cfg)
    case = cases.BUILD["seeded_7"]()                          # depth 90 on matrix_depth 55: the candidates shuffle
    build(builder, case)
    assert builder.sizes()[2] > 0
    builder.fetch()
    pos_info, alt_info = split(builder.alt_info_strings())
    Y = builder.forward(model)
    want = decode.batch_calls(model, pos_info, alt_info, Y, cfg)
    got = build(builder, case).call(model, cfg, CTG)
    assert len(pos_info) > 30 and torch.equal(got["Y"], Y)
    assert np.array_equal(got["position"], want["position"]) and got["chromosome"] == want["chromosome"]
    assert np.array_equal(got["start"], want["start"])
    for name in want["calls"].dtype.names:
        if name != "pad":
            g, w = (np.ascontiguousarray(r["calls"][name]).view(np.uint8) for r in (got, want))
            assert np.array_equal(g, w), name
    # haploid precise mode prints homozygous calls only, and the seeded weights make none on this region; every field above
    # is compared all the same
    assert want["calls"]["printed"].sum() > 0 or cfg.is_haploid_precise_mode_enabled
    for s in range(len(pos_info)):
        o, c = int(want["start"][s]), want["calls"][s]
        n = int(c["ref_len"]) + int(c["alt_len"])
        assert got["text"][o:o + n].tobytes() == want["text"][o:o + n].tobytes(), s
        assert np.array_equal(got["ad"][o:o + int(c["n_ad"])], want["ad"][o:o + int(c["n_ad"])]), s
    text = decode.calls_text(got, cfg)
    assert text == decode.calls_text(want, cfg) and (text.count("\n") > 0 or cfg.is_haploid_precise_mode_enabled)


def test_no_candidates_and_no_reads(builder, model):
    from clair3_b200 import decode
    rec, ref, _, var, p = cases.case(cases.cover(4), [C])
    got = builder.build(rec, [], ref, 0, **builder_kwargs(p)).alt_text().alt_text_fetch()
    assert got["text"] == [] and got["decoder"] == [] and len(got["ref_base"]) == 0 and len(got["position"]) == 0
    assert builder.alt_text_sizes() == (0, 0)
    v = builder.alt_text_device()
    assert v["decoder"].numel() == 0 and v["decoder_off"].cpu().tolist() == [0] and v["text_off"].cpu().tolist() == [0]
    res = builder.build(rec, [], ref, 0, **builder_kwargs(p)).call(model, config(), CTG)
    assert len(res["calls"]) == 0 and res["Y"].shape == (0, 90) and decode.calls_text(res, config()) == ""
    # no reads: every candidate still has its string, with depth 0
    empty = cases.case([], [C, C + 40])
    host, got = host_and_device(builder, empty)
    assert host == ["%d-0-%s-" % (c + 1, cases.REF[c]) for c in (C, C + 40)] and got["text"] == host
    check_decoder_fields(got, host)


def test_text_stage_needs_a_build():
    from clair3_b200._ffi import C3BError, ffi, lib
    from clair3_b200.fa_tensor import FullAlignmentBuilder
    b = FullAlignmentBuilder(0)
    try:
        with pytest.raises(C3BError, match="build"):
            b.alt_text()
        assert lib().c3b_fa_alt_text(b._h, 50) != 0 and b"no c3b_fa_build has been issued" in ffi.string(lib().c3b_last_error())
        with pytest.raises(C3BError, match="no c3b_fa_alt_text has been issued"):
            b.alt_text_sizes()
        build(b, cases.BUILD["cigar_insertion_2I1I_shared_string"]())
        for f in (b.alt_text_sizes, b.alt_text_fetch, b.alt_text_device, b.alt_text_last_ms):
            with pytest.raises(C3BError, match="no c3b_fa_alt_text has been issued"):
                f()
        n = ffi.NULL
        assert lib().c3b_fa_fetch_alt_text(b._h, n, n, n, n, n, n) != 0
        assert b"no c3b_fa_alt_text has been issued" in ffi.string(lib().c3b_last_error())
        # and the stage's own timing, read apart from the build's
        build_launches = b.last_ms()[1]
        assert len(b.alt_text().alt_text_fetch()["text"]) == 1
        ms, launches = b.alt_text_last_ms()
        assert ms > 0 and launches == 4 and b.last_ms()[1] == build_launches
        # a new build drops the text
        build(b, cases.BUILD["cigar_insertion_2I1I_shared_string"]())
        with pytest.raises(C3BError, match="no c3b_fa_alt_text has been issued"):
            b.alt_text_fetch()
    finally:
        b.close()


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


def test_call_waits_once_before_the_network_is_queued(builder, model, monkeypatch):
    """Between the text stage and the decoder's launch ``call()`` enters exactly one C entry point that waits for the stream
    (``c3b_fa_sizes``), and it does so before Clair3_F is enqueued: the network and the decoder are queued back to back."""
    import clair3_b200.model as model_mod
    from clair3_b200 import fa_tensor
    from clair3_b200._ffi import lib
    log = []
    spy = _Spy(lib(), log)
    monkeypatch.setattr(fa_tensor, "lib", lambda: spy)
    monkeypatch.setattr(model_mod, "lib", lambda: spy)
    res = build(builder, cases.BUILD["seeded_7"]()).call(model, config(), CTG)
    assert len(res["calls"]) > 30
    names = [n for n, _ in log]
    first, last = names.index("c3b_fa_alt_text"), names.index("c3b_decode_calls")
    waits = {"c3b_fa_sizes", "c3b_fa_fetch", "c3b_fa_fetch_alleles", "c3b_fa_fetch_alt_text", "c3b_fa_last_ms",
             "c3b_fa_alt_text_last_ms"}
    assert [n for n in names[first:last] if n in waits] == ["c3b_fa_sizes"]
    order = [names.index(n) for n in ("c3b_fa_build", "c3b_fa_alt_text", "c3b_fa_sizes", "c3b_fa_alt_text_sizes", "c3b_forward",
                                      "c3b_decode_calls")]
    assert order == sorted(order)               # alt_text_sizes after sizes reads the totals that wait brought; it does not wait
