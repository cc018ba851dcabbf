"""Decoder records without a GPU: the record oracle (``oracle/decode_calls_oracle.py``) formatted through
``decode.batch_output``'s records route reproduces the reference's ``batch_output`` text and ``output_from`` results in
``tests/golden/decode_stage2.npz``; malformed alt_info gives the host path's exceptions."""
import os

import numpy as np
import pytest

from clair3_b200 import decode
from oracle import decode_calls_oracle as dco

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "decode_stage2.npz")
CONFIG_NAMES = ("default", "show_ref", "haploid_precise", "haploid_sensitive", "long_indel", "qual_iupac")


def make_config(out_dim, name):
    kw = dict(is_show_reference=False, is_debug=False, is_haploid_precise_mode_enabled=False,
              is_haploid_sensitive_mode_enabled=False, is_output_for_ensemble=False, quality_score_for_pass=None, tensor_fn="PIPE",
              input_probabilities=True, add_indel_length=(out_dim == 90), gvcf=False, pileup=(out_dim == 24),
              enable_long_indel=False, maximum_variant_length_that_need_infer=50, keep_iupac_bases=False)
    kw.update({"default": {}, "show_ref": {"is_show_reference": True},
               "haploid_precise": {"is_haploid_precise_mode_enabled": True},
               "haploid_sensitive": {"is_haploid_sensitive_mode_enabled": True},
               "long_indel": {"enable_long_indel": True, "is_show_reference": True,
                              "maximum_variant_length_that_need_infer": 100000},
               "qual_iupac": {"quality_score_for_pass": 12.0, "keep_iupac_bases": True}}[name])
    return decode.OutputConfig(**kw)


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


@pytest.mark.parametrize("name", CONFIG_NAMES)
@pytest.mark.parametrize("out_dim", [24, 90])
def test_oracle_records_format_to_reference_text(z, out_dim, name):
    pre = "real%d_" % out_dim
    text = decode.batch_output(dco.OracleCalls(out_dim), list(z[pre + "pos"]), list(z[pre + "alt"]), z[pre + "y"],
                               make_config(out_dim, name))
    assert text == z[pre + "text_" + name].item()


@pytest.mark.parametrize("out_dim,tag", [(24, ""), (24, "_long"), (90, ""), (90, "_long")])
def test_oracle_records_hold_reference_output_from(z, out_dim, tag):
    """Flags, probability and (with showRef, so every row prints) REF / ALT of each record equal the reference's output_from."""
    pre = "real%d_" % out_dim
    cfg = make_config(out_dim, "long_indel" if tag else "show_ref")._replace(keep_iupac_bases=True)
    res = decode.batch_calls(dco.OracleCalls(out_dim), list(z[pre + "pos"]), list(z[pre + "alt"]), z[pre + "y"], cfg)
    calls, text, start = res["calls"], res["text"], res["start"]
    for i in range(len(calls)):
        flags = z[pre + "of_flags" + tag][i]
        assert calls["flags"][i] == sum(int(f) << b for b, f in enumerate(flags)), i
        assert calls["prob"][i].view(np.uint32) == z[pre + "of_prob" + tag][i].view(np.uint32), i
        o, rl, al = int(start[i]), int(calls["ref_len"][i]), int(calls["alt_len"][i])
        ref, alt = text[o:o + rl].tobytes().decode(), text[o + rl:o + rl + al].tobytes().decode()
        want_ref, want_alt = str(z[pre + "of_ref" + tag][i]), str(z[pre + "of_alt" + tag][i])
        if calls["printed"][i]:
            assert ref == want_ref and alt == ("." if flags[0] else want_alt), i


# alt_info strings the host path rejects, with its exception
MALFORMED = [("x-XA 3", ValueError), ("30-XA three", ValueError), ("30-XA 3 XC", None), ("30-XA 3  XC 4", ValueError),
             ("30-XA 1_0 R 2_", ValueError), ("30- 5", IndexError), ("30-X 5 XA 9", IndexError), ("3_0-XA +7 R \t4\t ", None),
             ("30-XA 3-XC 4", None), ("30", None), ("30-", None), ("30-XA 3 XA 9 R 1", None)]


@pytest.mark.parametrize("alt,exc", MALFORMED)
def test_malformed_alt_info_raises_as_the_host_path(alt, exc):
    y = np.zeros((1, 24), np.float32)
    y[0, 22] = y[0, 4] = np.float32(0.9)                 # homo-variant C: the walk tries SNPs first
    pos = ["chr1:100:" + "A" * 16 + "A" + "A" * 16]
    cfg = make_config(24, "show_ref")
    host = calls = None
    try:
        host = decode.batch_output(_StagesOnly(), pos, [alt], y, cfg)
    except Exception as e:                                # noqa: BLE001
        host = e
    try:
        calls = decode.batch_output(dco.OracleCalls(24), pos, [alt], y, cfg)
    except Exception as e:                                # noqa: BLE001
        calls = e
    if exc is None:
        assert isinstance(host, str) and calls == host
    else:
        assert isinstance(host, exc) and isinstance(calls, exc)


class _StagesOnly:
    def decode_stage1(self, y, g):
        from oracle import decode_oracle as dec1
        return dec1.decode_stage1(y, g)

    def decode_stage2(self, y, g, sites=None, n_sites=None, k=16):
        from oracle import decode_stage2_oracle as dec2
        return dec2.decode_stage2(y, g, sites, n_sites, k)


def test_empty_batch_and_out_of_scope_configs():
    res = decode.batch_calls(dco.OracleCalls(90), [], [], np.zeros((0, 90), np.float32), make_config(90, "default"))
    assert len(res["calls"]) == 0 and decode.calls_text(res, make_config(90, "default")) == ""
    for field in ("gvcf", "is_debug", "is_output_for_ensemble"):
        with pytest.raises(NotImplementedError, match=field):
            decode.batch_calls(dco.OracleCalls(24), ["chr1:1:A"], ["3-XA 1"], np.zeros((1, 24), np.float32),
                               make_config(24, "default")._replace(**{field: True}))


# ------------------------------------------------------------------------------------------------ the targeted fixture
CALLS_GOLDEN = os.path.join(HERE, "golden", "decode_calls.npz")


@pytest.fixture(scope="module")
def zc():
    return np.load(CALLS_GOLDEN)


def _single(model, pos, alt, y, cfg):
    try:
        return decode.batch_output(model, [pos], [alt], y[None], cfg), ""
    except Exception as e:                                   # noqa: BLE001
        return "", type(e).__name__


@pytest.mark.parametrize("name", CONFIG_NAMES)
@pytest.mark.parametrize("out_dim", [24, 90])
def test_targeted_cases_records_and_host_walk_match_reference(zc, out_dim, name):
    """Every targeted row, alone in its batch: the oracle's records formatted, and the host walk, give the reference's row or
    raise the reference's exception."""
    pre = "c%d_" % out_dim
    y, pos, alts = zc[pre + "y"], [str(p) for p in zc[pre + "pos"]], [str(a) for a in zc[pre + "alt"]]
    cfg = make_config(out_dim, name)
    texts, excs = zc[pre + "text_" + name], zc[pre + "exc_" + name]
    for i in range(len(y)):
        want = (str(texts[i]), str(excs[i]))
        assert _single(dco.OracleCalls(out_dim), pos[i], alts[i], y[i], cfg) == want, (i, alts[i])
        assert _single(_StagesOnly(), pos[i], alts[i], y[i], cfg) == want, (i, alts[i])


@pytest.mark.parametrize("out_dim,tag", [(24, ""), (24, "_long"), (90, ""), (90, "_long")])
def test_targeted_cases_records_hold_reference_output_from(zc, out_dim, tag):
    pre = "c%d_" % out_dim
    y, pos, alts = zc[pre + "y"], [str(p) for p in zc[pre + "pos"]], [str(a) for a in zc[pre + "alt"]]
    ok = (zc[pre + "of_exc" + tag] == "") & (zc[pre + "exc_" + ("long_indel" if tag else "show_ref")] == "")
    cfg = make_config(out_dim, "long_indel" if tag else "show_ref")._replace(keep_iupac_bases=True)
    for i in np.nonzero(ok)[0]:
        res = decode.batch_calls(dco.OracleCalls(out_dim), [pos[i]], [alts[i]], y[i:i + 1], cfg)
        c = res["calls"][0]
        assert c["flags"] == sum(int(f) << b for b, f in enumerate(zc[pre + "of_flags" + tag][i])), i
        assert c["prob"].view(np.uint32) == zc[pre + "of_prob" + tag][i].view(np.uint32), i
        if c["printed"] and not (c["flags"] & 1):
            o = int(res["start"][0])
            ref = res["text"][o:o + c["ref_len"]].tobytes().decode()
            alt = res["text"][o + c["ref_len"]:o + c["ref_len"] + c["alt_len"]].tobytes().decode()
            assert (ref, alt) == (str(zc[pre + "of_ref" + tag][i]), str(zc[pre + "of_alt" + tag][i])), i


def test_targeted_cases_cover_their_rules(zc):
    exc = set(str(e) for e in zc["c90_exc_default"])
    assert {"ValueError", "IndexError", "ZeroDivisionError"} <= exc
    alts = [str(a) for a in zc["c90_alt"]]
    assert max(len(a) for a in alts) > 500 and any(a.count(" I") >= 59 for a in alts)
    y = zc["c90_y"]
    gt = np.array([decode.GT21_OF_BASE[decode.BASE2ACGT[str(p).split(":")[-1][16]]] for p in zc["c90_pos"]], np.uint8)
    from oracle import decode_stage2_oracle as dec2
    assert dec2.decode_stage2(y, gt, k=1024)["count"].max() > 16       # walks that pass 16 entries


@pytest.mark.skipif(not os.environ.get("CLAIR3_REFERENCE"), reason="needs a Clair3 checkout named by CLAIR3_REFERENCE")
def test_fresh_reference_runs_equal_the_fixture(zc):
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_decode_calls_golden",
                                                  os.path.join(HERE, "golden", "make_decode_calls_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    fresh = mk.mint(os.environ["CLAIR3_REFERENCE"])
    assert sorted(fresh) == sorted(zc.files)
    for k, v in fresh.items():
        w = zc[k]
        if v.dtype.kind == "f":
            assert np.array_equal(v.view(np.uint32), w.view(np.uint32)), k
        else:
            assert np.array_equal(v, w), k
