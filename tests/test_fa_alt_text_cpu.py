"""Without a device: the full-alignment text stage's C-ABI (include/clair3_b200_fa.h) parses through the cffi binding and resolves
in the built library, and ``FullAlignmentBuilder.alt_text`` / ``call`` reject bad arguments before they reach it."""
import pytest

from clair3_b200 import _ffi, decode, fa_tensor

NEW = ("c3b_fa_alt_text", "c3b_fa_alt_text_sizes", "c3b_fa_fetch_alt_text", "c3b_fa_alt_text_device", "c3b_fa_alt_text_last_ms")


def test_declarations_parse_and_resolve():
    for name in NEW:
        assert name in _ffi.DECLARED_FUNCTIONS
        assert _ffi.ffi.typeof(getattr(_ffi.lib(), name)).kind == "function"
    t = _ffi.ffi.typeof(_ffi.lib().c3b_fa_fetch_alt_text)
    assert [a.cname for a in t.args] == ["c3b_fa *", "char *", "int64_t *", "char *", "int64_t *", "uint8_t *", "int64_t *"]
    t = _ffi.ffi.typeof(_ffi.lib().c3b_fa_alt_text_device)
    assert [a.cname for a in t.args] == ["c3b_fa *", "char * *", "int64_t * *", "char * *", "int64_t * *", "uint8_t * *",
                                         "int64_t * *"]


def test_null_workspace_is_an_error_with_a_message():
    L, N = _ffi.lib(), _ffi.ffi.NULL
    assert L.c3b_fa_alt_text(N, 50) != 0 and b"no c3b_fa_build has been issued" in _ffi.ffi.string(L.c3b_last_error())
    for rc in (L.c3b_fa_alt_text_sizes(N, N, N), L.c3b_fa_fetch_alt_text(N, N, N, N, N, N, N),
               L.c3b_fa_alt_text_device(N, N, N, N, N, N, N), L.c3b_fa_alt_text_last_ms(N, N, N)):
        assert rc != 0 and b"no c3b_fa_alt_text has been issued" in _ffi.ffi.string(L.c3b_last_error())


def _builder(alt, shape=(3, 89, 8)):
    b = object.__new__(fa_tensor.FullAlignmentBuilder)      # no device here: only the checks made before the library call
    b._h, b._alt, b._shape, b._keep = None, alt, shape, None
    return b


def test_alt_text_argument_checks():
    with pytest.raises(_ffi.C3BError, match="build"):
        _builder(None).alt_text()
    with pytest.raises(_ffi.C3BError, match="build"):
        _builder(None).alt_info_strings()
    for bad in (1.5, "50", True):
        with pytest.raises(_ffi.C3BError, match="max_indel_length"):
            _builder((b"ACGT", 0, 50)).alt_text(max_indel_length=bad)


def test_call_argument_checks():
    cfg = decode.replay_config(pileup=False, add_indel_length=True)
    with pytest.raises(NotImplementedError, match="gvcf"):
        _builder((b"ACGT", 0, 50)).call(object(), cfg._replace(gvcf=True), "ctg")
    with pytest.raises(_ffi.C3BError, match="call: the model has no device"):
        _builder((b"ACGT", 0, 50)).call(object(), cfg, "ctg")
