"""cffi (ABI-mode) binding of libclair3b200.so.

The reference binds its native library the same way (cffi, declarations taken from the C headers with the
preprocessor lines stripped: ``build.py:44-79`` of HKU-BAL/Clair3); here the declarations come from
``include/clair3_b200.h``.  There is no Python/CPU fallback: if the shared object is missing it is built
with nvcc, and if that fails the import raises.
"""
from __future__ import annotations

import os
import re

import cffi

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(_HERE), "include", "clair3_b200.h")
DEBUG_HEADER = os.path.join(os.path.dirname(_HERE), "include", "clair3_b200_debug.h")     # taps / probes, not the drop-in surface
PILEUP_HEADER = os.path.join(os.path.dirname(_HERE), "include", "clair3_b200_pileup.h")   # pileup feature counter (SURVEY 8f N4)
FA_HEADER = os.path.join(os.path.dirname(_HERE), "include", "clair3_b200_fa.h")           # full-alignment tensor builder (N4)
LIB_PATH = os.path.join(_HERE, "libclair3b200.so")

ffi = cffi.FFI()


def _cdef_source(path):
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    consts = {m.group(1): m.group(2) for m in re.finditer(r"^#define\s+(C3B_\w+)\s+(\d+)\s*$", src, flags=re.M)}
    body = "\n".join(l for l in src.splitlines() if not l.lstrip().startswith("#")
                     and 'extern "C"' not in l and l.strip() not in ("}",))
    return body, {k: int(v) for k, v in consts.items()}


_body, CONSTANTS = _cdef_source(HEADER)
_dbg_body, _ = _cdef_source(DEBUG_HEADER)
_plp_body, _ = _cdef_source(PILEUP_HEADER)
_fa_body, _ = _cdef_source(FA_HEADER)
ffi.cdef(_body)
ffi.cdef(_dbg_body)
ffi.cdef(_plp_body)
ffi.cdef(_fa_body)
DECLARED_FUNCTIONS = sorted(set(re.findall(r"\b(c3b_\w+)\s*\(", _body + _dbg_body + _plp_body + _fa_body)))

_lib = None


def lib():
    """dlopen the library (building it first if the .so is absent)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            from . import build
            build.build_library()
        _lib = ffi.dlopen(LIB_PATH)
    return _lib


class C3BError(RuntimeError):
    pass


def check(rc):
    if rc != 0:
        raise C3BError(ffi.string(lib().c3b_last_error()).decode())
