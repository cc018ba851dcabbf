"""CPU-side checks: the C-ABI library builds, loads and exports every symbol include/clair3_b200.h declares; the
product path fails loudly (no CPU fallback) when no H100 is present."""
import ctypes
import os

import pytest

from clair3_b200 import _ffi


def test_library_exports_every_declared_symbol():
    path = _ffi.LIB_PATH
    _ffi.lib()
    assert os.path.exists(path)
    dll = ctypes.CDLL(path)
    assert len(_ffi.DECLARED_FUNCTIONS) >= 13
    for name in _ffi.DECLARED_FUNCTIONS:
        assert hasattr(dll, name), name


def test_header_has_no_torch_types():
    import re
    for path in (_ffi.HEADER, _ffi.PILEUP_HEADER, _ffi.DEBUG_HEADER):
        src = open(path).read()
        code = re.sub(r"/\*.*?\*/", "", src, flags=re.S)          # declarations only, comments stripped
        assert "torch" not in code.lower() and "at::" not in code and "std::" not in code, path
        assert 'extern "C"' in code, path


def test_headers_are_plain_c_and_a_c_caller_links(tmp_path):
    """The drop-in boundary is a C ABI: every header compiles as C99 on its own, and a C translation unit that calls the entry points
    a maintainer would bind (network forward + pileup feature counter) links against the shared object."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    inc = os.path.join(root, "include")
    for h in ("clair3_b200.h", "clair3_b200_pileup.h", "clair3_b200_debug.h"):
        r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-x", "c", os.path.join(inc, h)], capture_output=True, text=True)
        assert r.returncode == 0, (h, r.stderr)
    src = tmp_path / "caller.c"
    src.write_text(r"""
#include <stdio.h>
#include "clair3_b200.h"
#include "clair3_b200_pileup.h"
int main(void) {
    c3b_model *m = NULL;
    c3b_plp *w = NULL;
    c3b_bam_records recs = {0};
    c3b_plp_params prm = {2, 0.08f, 0.15f, 5, 0, 0, 0, 0};
    int64_t n_cols = 0, n_cand = 0;
    if (c3b_create(&m, C3B_PILEUP, 18, 0, 0) != 0 || c3b_plp_create(&w, 0) != 0) {      /* no GPU here: fails loudly, no fallback */
        printf("%s\n", c3b_last_error());
        return 3;
    }
    if (c3b_plp_count(w, &recs, 0, 0, 0, "", 0, 0, &prm, NULL) || c3b_plp_sizes(w, &n_cols, &n_cand)) return 4;
    c3b_plp_destroy(w);
    c3b_destroy(m);
    return 0;
}
""")
    exe = tmp_path / "caller"
    libdir = os.path.dirname(_ffi.LIB_PATH)
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-I", inc, str(src), "-o", str(exe), "-L", libdir, "-lclair3b200",
                        "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    import torch
    if not torch.cuda.is_available():
        run = subprocess.run([str(exe)], capture_output=True, text=True)
        assert run.returncode == 3 and "no CUDA device" in run.stdout


def test_version_and_error_strings():
    L = _ffi.lib()
    assert b"sm_90a" in _ffi.ffi.string(L.c3b_version())
    assert L.c3b_out_dim(_ffi.ffi.NULL) == -1


def test_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from clair3_b200.model import Clair3_P
    m = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    with pytest.raises(_ffi.C3BError):
        m.to(torch.device("cpu"))
    with pytest.raises(_ffi.C3BError, match="no CUDA device|no CPU"):
        m.load_state_dict({})
    out = _ffi.ffi.new("c3b_model **")
    assert _ffi.lib().c3b_create(out, 0, 18, 0, 0) != 0
    assert b"no CPU fallback" in _ffi.ffi.string(_ffi.lib().c3b_last_error())


def test_product_path_never_imports_oracle():
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "clair3_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), f
