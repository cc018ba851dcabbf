"""TEST INFRASTRUCTURE ONLY: the reference's own full-alignment tensor builder, compiled, as a checker.

``calculate_clair3_full_alignment`` (HKU-BAL/Clair3 ``src/clair3_full_alignment_dwell.c:437-1054``) needs only a small slice of
htslib.  ``build()`` compiles the reference's C (that file, ``levenshtein.c``, ``medaka_khcounter.c``, ``medaka_common.c``) against
the in-memory stand-in under ``oracle/hts_stub/`` into ``oracle/_ref/libclair3_fa_ref.so`` (git-ignored).  The reference tree is
found through the ``CLAIR3_REFERENCE`` environment variable or next to this repository (``reference_src``); it is read at build
time only.  Without it an earlier build is kept.

``full_alignment()`` registers the records and the contig with the stand-in, seeds libc's ``rand()`` (the reference shuffles with
the process-global generator, ``:117-134``) and calls the function exactly as ``preprocess/CreateTensorFullAlignmentFromCffi.py``
does.  Only tests/, ``__graft_entry__.smoke()`` and tools/ may import this module; the product (clair3_b200/) never does.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
STUB = os.path.join(HERE, "hts_stub")
OUT_DIR = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT_DIR, "libclair3_fa_ref.so")
SKIP_SRC = os.path.join(HERE, "rand_skip.c")
SKIP_LIB = os.path.join(HERE, "_build", "librand_skip.so")
REF_SOURCES = ("clair3_full_alignment_dwell.c", "levenshtein.c", "medaka_khcounter.c", "medaka_common.c")
CONTIG = "ctg"


SIBLING_NAMES = ("Clair3", "clair3", "reference")


def reference_src():
    """The reference checkout's ``src/`` directory, or None when none is available: ``CLAIR3_REFERENCE`` if it is set, otherwise a
    checkout named Clair3 / clair3 / reference next to this repository or next to one of its parent directories."""
    roots = [os.environ["CLAIR3_REFERENCE"]] if os.environ.get("CLAIR3_REFERENCE") else []
    d = os.path.dirname(HERE)
    for _ in range(3):
        parent = os.path.dirname(d)
        roots += [os.path.join(parent, n) for n in SIBLING_NAMES]
        if parent == d:
            break
        d = parent
    for root in roots:
        src = os.path.join(root, "src")
        if all(os.access(os.path.join(src, f), os.R_OK) for f in REF_SOURCES):
            return src
    return None


def available():
    return os.path.exists(LIB)


def build_rand_skip(out=SKIP_LIB):
    """gcc -O2 -shared oracle/rand_skip.c -> oracle/_build/librand_skip.so (git-ignored).  Project source only, so it is built
    whether or not a reference checkout is found; an ``oracle/_ref/`` kept from an earlier build never lacks it."""
    if not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(SKIP_SRC):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        tmp = out + ".tmp%d" % os.getpid()
        subprocess.run(["gcc", "-O2", "-shared", "-fPIC", "-o", tmp, SKIP_SRC], check=True)
        os.replace(tmp, out)
    return out


def build(force=False):
    """Compile the oracle when the reference sources are available; otherwise keep an earlier build (or do nothing).  Returns the
    library path or None."""
    src = reference_src()
    if src is None:
        return LIB if os.path.exists(LIB) else None
    stub_files = [os.path.join(STUB, f) for f in ("hts_stub.c", "fa_ref_shim.h", "htslib/sam.h", "htslib/faidx.h")]
    deps = [os.path.join(src, f) for f in REF_SOURCES] + stub_files
    if force or not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(OUT_DIR, exist_ok=True)
        tmp = LIB + ".tmp%d" % os.getpid()
        # the stand-in's include directory comes first, so "htslib/sam.h" resolves to it and never to a vendored copy
        cmd = (["gcc", "-O2", "-shared", "-fPIC", "-w", "-I", STUB, "-I", src, "-include", os.path.join(STUB, "fa_ref_shim.h"),
                "-o", tmp] + [os.path.join(src, f) for f in REF_SOURCES] + [os.path.join(STUB, "hts_stub.c"), "-lm"])
        subprocess.run(cmd, check=True)
        os.replace(tmp, LIB)
    return LIB


class Variant(ctypes.Structure):
    """``struct Variant`` (src/clair3_full_alignment_dwell.h:111-118)."""
    _fields_ = [("position", ctypes.c_int), ("ref_base", ctypes.c_char), ("alt_base", ctypes.c_char),
                ("genotype", ctypes.c_int), ("phase_set", ctypes.c_int)]


class _FaData(ctypes.Structure):
    _fields_ = [("matrix", ctypes.POINTER(ctypes.c_int8)), ("all_alt_info", ctypes.POINTER(ctypes.c_char_p)),
                ("candidates_num", ctypes.c_size_t)]


_lib = None
_libc = None
_skip = None


def _load_rand_skip():
    try:
        path = build_rand_skip()
    except (OSError, subprocess.CalledProcessError):          # a read-only tree: build it in a temporary directory
        import tempfile
        path = build_rand_skip(os.path.join(tempfile.mkdtemp(prefix="clair3_fa_ref_"), "librand_skip.so"))
    S = ctypes.CDLL(path)
    S.fa_ref_skip_rand.argtypes = [ctypes.c_uint64]
    return S


def _load():
    global _lib, _libc, _skip
    if _lib is None:
        path = build()
        if path is None:
            raise FileNotFoundError("oracle/_ref/libclair3_fa_ref.so is not built (no reference checkout found: set CLAIR3_REFERENCE)")
        L = ctypes.CDLL(path)
        L.calculate_clair3_full_alignment.restype = ctypes.POINTER(_FaData)
        L.calculate_clair3_full_alignment.argtypes = [
            ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(ctypes.POINTER(Variant)), ctypes.c_size_t,
            ctypes.POINTER(ctypes.c_size_t), ctypes.c_size_t, ctypes.c_bool, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t,
            ctypes.c_size_t, ctypes.c_bool]
        L.destroy_fa_data.argtypes = [ctypes.POINTER(_FaData)]
        L.fa_ref_set_contig.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int64]
        L.fa_ref_set_records.argtypes = [ctypes.c_int64] + [ctypes.c_void_p] * 14
        L.fa_ref_rand_draws.restype = ctypes.c_longlong
        _skip = _load_rand_skip()
        _lib = L
        _libc = ctypes.CDLL(None)
    return _lib


def libc_rand(seed, n, skip=0):
    """``n`` values of glibc ``rand()`` after ``srand(seed)`` and ``skip`` draws (the generator the reference shuffles with)."""
    _load()
    _libc.srand(ctypes.c_uint(seed))
    _skip.fa_ref_skip_rand(int(skip))
    return np.array([_libc.rand() for _ in range(n)], dtype=np.int64)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def full_alignment(rec, candidates, ref_seq, variants=(), need_haplotagging=False, min_mq=5, matrix_depth=89,
                   max_indel_length=50, enable_dwell_time=False, rand_seed=1, rand_skip=0):
    """The reference function on in-memory records.  ``rec``: dict with the ``BamRecords`` arrays, optionally ``qual`` /
    ``qual_off``, ``qname`` / ``qname_off`` (bytes, concatenated names without NULs) and ``mv`` / ``mv_off``.  ``ref_seq``: the
    WHOLE contig from position 0.  ``variants``: (position, ref_base, alt_base, genotype, phase_set) tuples, sorted by position.
    Returns (matrix int8 [n_cand, depth, 33, 8|9], alt_info strings, rand draws consumed)."""
    L = _load()
    ref = ref_seq.encode() if isinstance(ref_seq, str) else bytes(ref_seq)
    n = int(len(rec["pos"]))
    arr = {k: np.ascontiguousarray(rec[k], dtype=dt) for k, dt in
           (("pos", np.int64), ("flag", np.uint16), ("mapq", np.uint8), ("cigar_off", np.int64), ("cigar", np.uint32),
            ("seq_off", np.int64), ("seq", np.uint8), ("l_qseq", np.int32))}
    for k, dt in (("qual_off", np.int64), ("qual", np.uint8), ("qname_off", np.int64), ("mv_off", np.int64), ("mv", np.int32)):
        arr[k] = np.ascontiguousarray(rec[k], dtype=dt) if rec.get(k) is not None else None
    qname = rec.get("qname")
    arr["qname"] = None if qname is None else np.frombuffer(bytes(qname) + b"\0", dtype=np.uint8).copy()
    if arr["qual"] is not None and len(arr["qual"]) == 0:
        arr["qual"] = np.zeros(1, np.uint8)
    if arr["mv"] is not None and len(arr["mv"]) == 0:
        arr["mv"] = np.zeros(1, np.int32)
    if arr["qname_off"] is None:
        arr["qname"] = None
    L.fa_ref_set_contig(CONTIG.encode(), ref, len(ref))
    L.fa_ref_set_records(n, *[_ptr(arr[k]) for k in ("pos", "flag", "mapq", "cigar_off", "cigar", "seq_off", "seq", "l_qseq",
                                                     "qual_off", "qual", "qname_off", "qname", "mv_off", "mv")])
    cands = np.ascontiguousarray(candidates, dtype=np.uint64)
    nv = len(variants)
    vs = (Variant * max(nv, 1))()
    vp = (ctypes.POINTER(Variant) * max(nv, 1))()
    for i, (p, rb, ab, gt, ps) in enumerate(variants):
        vs[i] = Variant(int(p), rb.encode() if isinstance(rb, str) else bytes([rb]), ab.encode() if isinstance(ab, str) else bytes([ab]),
                        int(gt), int(ps))
        vp[i] = ctypes.pointer(vs[i])
    _libc.srand(ctypes.c_uint(rand_seed))
    _skip.fa_ref_skip_rand(int(rand_skip))  # a C loop: about 2^32 draws take tens of seconds
    L.fa_ref_reset_rand_draws()
    region = ("%s:1-%d" % (CONTIG, len(ref))).encode()
    d = L.calculate_clair3_full_alignment(region, b"in-memory.bam", b"in-memory.fa", vp, nv,
                                          cands.ctypes.data_as(ctypes.POINTER(ctypes.c_size_t)), len(cands),
                                          bool(need_haplotagging), int(min_mq), 0, int(matrix_depth), int(max_indel_length),
                                          bool(enable_dwell_time))
    draws = int(L.fa_ref_rand_draws())
    C = 9 if enable_dwell_time else 8
    total = len(cands) * matrix_depth * 33 * C
    m = np.ctypeslib.as_array(d.contents.matrix, shape=(total,)).copy() if total else np.zeros(0, np.int8)
    alt = [d.contents.all_alt_info[i].decode("latin-1") for i in range(len(cands))]
    L.destroy_fa_data(d)
    return m.reshape(len(cands), matrix_depth, 33, C), alt, draws
