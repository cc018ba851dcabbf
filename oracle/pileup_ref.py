"""TEST INFRASTRUCTURE ONLY: the reference's own pileup feature counter, compiled, as a checker.

``calculate_clair3_pileup`` (HKU-BAL/Clair3 ``src/clair3_pileup.c:142-476``) reads its records through ``src/medaka_bamiter.c``'s
``read_bam`` and htslib's pileup engine.  ``build()`` compiles the reference's C (those two files, ``medaka_khcounter.c`` with the
reference's own ``khash.h``, ``medaka_common.c``) against the in-memory stand-in under ``oracle/hts_stub/`` - which restates the
pileup engine, see ``hts_stub.c`` - into ``oracle/_ref/libclair3_pileup_ref.so`` (git-ignored).  It is a library of its own, next
to the full-alignment one, so the two never share symbols.  ``fa_ref_shim.h`` is force-included here too: its guarded allocator
absorbs the reference's ``matrix[-1]`` write when the first emitted column holds a non-A/C/G/T read base (``:286`` with feature
index -1).  The reference tree is found as for ``oracle/fa_ref.py`` (``reference_src``) and read at build time only; without it an
earlier build is kept.

``clair3_pileup()`` takes the signature and defaults of ``oracle.pileup_oracle.clair3_pileup`` so the two compare directly.  Only
tests/ and tools/ may import this module; the product (clair3_b200/) never does.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from oracle.fa_ref import CONTIG, OUT_DIR, STUB, reference_src

LIB = os.path.join(OUT_DIR, "libclair3_pileup_ref.so")
REF_SOURCES = ("clair3_pileup.c", "medaka_bamiter.c", "medaka_khcounter.c", "medaka_common.c")
FEATURES = 18
UNMAP, SECONDARY, QCFAIL, DUP, SUPPLEMENTARY = 4, 256, 512, 1024, 2048


def available():
    return os.path.exists(LIB)


def build(force=False):
    """Compile the checker when the reference sources are available; otherwise keep an earlier build (or do nothing).  Returns
    the library path or None."""
    src = reference_src()
    if src is None or not all(os.access(os.path.join(src, f), os.R_OK) for f in REF_SOURCES + ("khash.h",)):
        return LIB if os.path.exists(LIB) else None
    stub_files = [os.path.join(STUB, f) for f in ("hts_stub.c", "fa_ref_shim.h", "htslib/sam.h", "htslib/faidx.h")]
    deps = [os.path.join(src, f) for f in REF_SOURCES] + stub_files + [os.path.abspath(__file__)]
    if force or not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(OUT_DIR, exist_ok=True)
        tmp = LIB + ".tmp%d" % os.getpid()
        # the stand-in's include directory comes first, so "htslib/sam.h" resolves to it and never to the reference's src/sam.h
        cmd = (["gcc", "-O2", "-shared", "-fPIC", "-w", "-I", STUB, "-I", src, "-include", os.path.join(STUB, "fa_ref_shim.h"),
                "-o", tmp] + [os.path.join(src, f) for f in REF_SOURCES] + [os.path.join(STUB, "hts_stub.c"), "-lm"])
        subprocess.run(cmd, check=True)
        os.replace(tmp, LIB)
    return LIB


class _PlpData(ctypes.Structure):
    """``struct _plp_data`` (src/clair3_pileup.h:5-17)."""
    _fields_ = [("buffer_cols", ctypes.c_size_t), ("num_dtypes", ctypes.c_size_t), ("num_homop", ctypes.c_size_t),
                ("n_cols", ctypes.c_size_t), ("matrix", ctypes.POINTER(ctypes.c_int64)), ("major", ctypes.POINTER(ctypes.c_int64)),
                ("minor", ctypes.POINTER(ctypes.c_int64)), ("all_alt_info", ctypes.POINTER(ctypes.c_char_p)),
                ("candidates_num", ctypes.c_size_t), ("pos_ref_count", ctypes.POINTER(ctypes.c_int64)),
                ("pos_total_count", ctypes.POINTER(ctypes.c_int64))]


_lib = None


def _load():
    global _lib
    if _lib is None:
        path = build()
        if path is None:
            raise FileNotFoundError("oracle/_ref/libclair3_pileup_ref.so is not built (no reference checkout found: set CLAIR3_REFERENCE)")
        L = ctypes.CDLL(path)
        L.calculate_clair3_pileup.restype = ctypes.POINTER(_PlpData)
        L.calculate_clair3_pileup.argtypes = [
            ctypes.c_char_p, ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_float, ctypes.c_float, ctypes.c_size_t,
            ctypes.c_size_t, ctypes.c_bool, ctypes.c_size_t, ctypes.c_bool, ctypes.c_bool]
        L.destroy_plp_data.argtypes = [ctypes.POINTER(_PlpData), ctypes.c_bool]
        L.create_bam_fset.restype = ctypes.c_void_p
        L.create_bam_fset.argtypes = [ctypes.c_char_p, ctypes.c_char_p]
        L.destroy_bam_fset.argtypes = [ctypes.c_void_p]
        L.fa_ref_set_contig.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int64]
        L.fa_ref_set_records.argtypes = [ctypes.c_int64] + [ctypes.c_void_p] * 14
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def kept_reads(rec, min_mq):
    """Indices of the records the reference's reader keeps (src/medaka_bamiter.c:20-22) and their reference ends."""
    ops = rec["cigar"] & 15
    refl = np.where(np.isin(ops, (0, 2, 3, 7, 8)), (rec["cigar"] >> 4).astype(np.int64), 0)
    csum = np.concatenate([[0], np.cumsum(refl)])
    rend = rec["pos"].astype(np.int64) + csum[rec["cigar_off"][1:]] - csum[rec["cigar_off"][:-1]]
    keep = ((rec["flag"] & (UNMAP | SECONDARY | QCFAIL | DUP | SUPPLEMENTARY)) == 0) & (rec["mapq"].astype(np.int64) >= min_mq)
    return np.nonzero(keep)[0], rend


def register(reads, ref_seq, ref_start, min_mq):
    """Registers the records and the contig ``'N' * ref_start + ref_seq`` (named ``CONTIG``) with the stand-in, for the next
    ``calculate_clair3_pileup``.  Returns (the record arrays, the contig bytes): the stand-in keeps pointers into them, so the
    caller holds on to them until its calls are done.  Raises ValueError when a read the reference keeps reaches past the contig
    end: the reference would read the reference sequence out of bounds there (see DESIGN.md, the pileup counter's deviations)."""
    L = _load()
    ref = ref_seq.encode() if isinstance(ref_seq, str) else bytes(ref_seq)
    contig = b"N" * int(ref_start) + ref
    arr = {k: np.ascontiguousarray(reads[k], dtype=dt) for k, dt in
           (("pos", np.int64), ("flag", np.uint16), ("mapq", np.uint8), ("cigar_off", np.int64), ("cigar", np.uint32),
            ("seq_off", np.int64), ("seq", np.uint8), ("l_qseq", np.int32))}
    n = int(len(arr["pos"]))
    idx, rend = kept_reads(arr, int(min_mq))
    if len(idx) and int(rend[idx].max()) > len(contig):
        raise ValueError("a kept read reaches position %d, past the contig end %d: the reference would read out of bounds"
                         % (int(rend[idx].max()), len(contig)))
    for k in ("cigar", "seq"):
        if len(arr[k]) == 0:
            arr[k] = np.zeros(1, arr[k].dtype)
    L.fa_ref_set_contig(CONTIG.encode(), contig, len(contig))
    L.fa_ref_set_records(n, *[_ptr(arr[k]) for k in ("pos", "flag", "mapq", "cigar_off", "cigar", "seq_off", "seq", "l_qseq")],
                         None, None, None, None, None, None)
    return arr, contig


def clair3_pileup(reads, start, end, ref_seq, ref_start, min_depth=2, min_snp_af=0.08, min_indel_af=0.15, min_mq=5,
                  call_snp_only=False, call_ht=False, gvcf=False, max_indel_length=50, alt_info=True):
    """The reference function on in-memory records, with the arguments of ``oracle.pileup_oracle.clair3_pileup``: records as
    ``clair3_b200.pileup_counts.BamRecords`` arrays, region [start, end) 0-based, reference bases [ref_start, ref_start +
    len(ref_seq)).  The contig is registered as ``'N' * ref_start + ref_seq`` and queried as ``ctg:{start+1}-{end}``.  Returns a
    dict: matrix [n_cols, 18] int64, major [n_cols] int64, alt_info (the candidates' strings), cand_cols (the column of each
    candidate, from its string), pos_ref_count / pos_total_count [end - start] (with ``gvcf``; zeros otherwise).  ``alt_info`` is
    accepted for signature parity; the strings are always returned.

    Raises ValueError when a read the reference keeps reaches past the contig end: the reference would read the reference
    sequence out of bounds there (see DESIGN.md, the pileup counter's deviations)."""
    L = _load()
    keep = register(reads, ref_seq, ref_start, min_mq)     # noqa: F841 - the stand-in reads these arrays during the call
    fset = L.create_bam_fset(b"in-memory.bam", b"in-memory.fa")
    region = ("%s:%d-%d" % (CONTIG, int(start) + 1, int(end))).encode()
    try:
        d = L.calculate_clair3_pileup(region, fset, b"in-memory.fa", int(min_depth), float(min_snp_af), float(min_indel_af),
                                      int(min_mq), int(max_indel_length), bool(call_snp_only), 0, bool(gvcf), bool(call_ht))
    finally:
        L.destroy_bam_fset(fset)
    c = d.contents
    nc, nk, W = int(c.n_cols), int(c.candidates_num), max(int(end) - int(start), 0)
    matrix = np.ctypeslib.as_array(c.matrix, shape=(nc * FEATURES,)).reshape(nc, FEATURES).copy() if nc else np.zeros((0, FEATURES), np.int64)
    major = np.ctypeslib.as_array(c.major, shape=(nc,)).copy() if nc else np.zeros(0, np.int64)
    alt = [c.all_alt_info[i].decode("latin-1") for i in range(nk)]
    prc, ptc = np.zeros(W, np.int64), np.zeros(W, np.int64)
    if gvcf and W:
        prc = np.ctypeslib.as_array(c.pos_ref_count, shape=(W,)).copy()
        ptc = np.ctypeslib.as_array(c.pos_total_count, shape=(W,)).copy()
    L.destroy_plp_data(d, bool(gvcf))
    cand_pos = np.array([int(s.split("-", 1)[0]) - 1 for s in alt], dtype=np.int64)
    cand_cols = np.searchsorted(major, cand_pos).astype(np.int64)
    assert (cand_cols < nc).all() and np.array_equal(major[cand_cols] if nk else cand_pos, cand_pos)
    return {"matrix": matrix, "major": major, "alt_info": alt, "cand_cols": cand_cols, "pos_ref_count": prc, "pos_total_count": ptc}
