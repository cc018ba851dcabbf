"""Without a device: the text stage's C-ABI (include/clair3_b200_pileup.h) parses through the cffi binding and resolves in the
built library, and ``PileupCounter.alt_text`` / ``call`` reject bad arguments before they reach it."""
import pytest

from clair3_b200 import _ffi, decode, pileup_counts as pc

NEW = ("c3b_plp_alt_text", "c3b_plp_alt_text_sizes", "c3b_plp_fetch_alt_text", "c3b_plp_alt_text_device", "c3b_plp_alt_text_last_ms")


def test_declarations_parse_and_resolve():
    for name in NEW:
        assert name in _ffi.DECLARED_FUNCTIONS
        assert _ffi.ffi.typeof(getattr(_ffi.lib(), name)).kind == "function"
    t = _ffi.ffi.typeof(_ffi.lib().c3b_plp_fetch_alt_text)
    assert [a.cname for a in t.args] == ["c3b_plp *", "char *", "int64_t *", "char *", "int64_t *", "uint8_t *", "int64_t *"]
    assert _ffi.ffi.sizeof("c3b_plp_params") == 40            # the existing struct keeps its layout


def test_null_workspace_is_an_error_with_a_message():
    L, N = _ffi.lib(), _ffi.ffi.NULL
    assert L.c3b_plp_alt_text(N, 50) != 0 and b"c3b_plp_alt_text" in _ffi.ffi.string(L.c3b_last_error())
    assert L.c3b_plp_alt_text_sizes(N, N, N) != 0
    assert L.c3b_plp_fetch_alt_text(N, N, N, N, N, N, N) != 0
    assert L.c3b_plp_alt_text_device(N, N, N, N, N, N, N) != 0
    assert L.c3b_plp_alt_text_last_ms(N, N, N) != 0


def _counter(alt):
    c = object.__new__(pc.PileupCounter)                     # no device here: only the checks made before the library call
    c._h, c._alt = None, alt
    return c


def test_alt_text_argument_checks():
    with pytest.raises(_ffi.C3BError, match="count"):
        _counter(None).alt_text()
    with pytest.raises(_ffi.C3BError, match="without alt_info"):
        _counter((False, 0, 10, 0, 50)).alt_text()
    for bad in (1.5, "50", True):
        with pytest.raises(_ffi.C3BError, match="max_indel_length"):
            _counter((True, 0, 10, 0, 50)).alt_text(max_indel_length=bad)
    with pytest.raises(_ffi.C3BError, match="count"):
        _counter(None).alt_info_strings()


def test_call_argument_checks():
    cfg = decode.replay_config(pileup=True, add_indel_length=False)
    with pytest.raises(NotImplementedError, match="gvcf"):
        _counter((True, 0, 10, 0, 50)).call(object(), cfg._replace(gvcf=True), "ctg")
    with pytest.raises(_ffi.C3BError, match="call: the model has no device"):
        _counter((True, 0, 10, 0, 50)).call(object(), cfg, "ctg")
