"""TEST INFRASTRUCTURE ONLY: ctypes binding of oracle/pileup_oracle.c (the plain-C restatement of the reference's
``calculate_clair3_pileup``, src/clair3_pileup.c:142-476).  Only tests/, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU
baseline leg may import this module; the product (clair3_b200/) never does.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "pileup_oracle.c")
OUT_DIR = os.path.join(HERE, "_build")
LIB = os.path.join(OUT_DIR, "libpileup_oracle.so")


def build(force=False):
    """gcc -O2 -shared oracle/pileup_oracle.c -> oracle/_build/libpileup_oracle.so (a git-ignored build product)."""
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        os.makedirs(OUT_DIR, exist_ok=True)
        subprocess.run(["gcc", "-O2", "-shared", "-fPIC", "-o", LIB, SRC], check=True)
    return LIB


class _Params(ctypes.Structure):
    _fields_ = [("min_depth", ctypes.c_int64), ("min_snp_af", ctypes.c_float), ("min_indel_af", ctypes.c_float),
                ("min_mq", ctypes.c_int32), ("call_snp_only", ctypes.c_int32), ("call_ht", ctypes.c_int32),
                ("gvcf", ctypes.c_int32), ("max_indel_length", ctypes.c_int64)]


_lib = None


def _load():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
        _lib.oracle_clair3_pileup.restype = ctypes.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def clair3_pileup(reads, start, end, ref_seq, ref_start, min_depth=2, min_snp_af=0.08, min_indel_af=0.15, min_mq=5,
                  call_snp_only=False, call_ht=False, gvcf=False, max_indel_length=50, alt_info=False):
    """reads: dict of numpy arrays with the keys of ``clair3_b200.pileup_counts.BamRecords`` (pos, flag, mapq, cigar_off, cigar,
    seq_off, seq, l_qseq).  Returns a dict: matrix [n_cols,18] int64, major [n_cols] int64, stats [n_cols,6] int32, cand_cols,
    cand_ok, pos_ref_count, pos_total_count, window_bounds [n_cand,2] int64 (the rows [lo, hi) of each candidate's window that
    lie in its contiguous run; the reference reads the others as zero) (+ alt_info: the all_alt_info strings of the candidates,
    with ``alt_info=True``)."""
    L = _load()
    n = int(len(reads["pos"]))
    W = max(int(end - start), 0)
    pos = np.ascontiguousarray(reads["pos"], dtype=np.int64)
    flag = np.ascontiguousarray(reads["flag"], dtype=np.uint16)
    mapq = np.ascontiguousarray(reads["mapq"], dtype=np.uint8)
    cigar_off = np.ascontiguousarray(reads["cigar_off"], dtype=np.int64)
    cigar = np.ascontiguousarray(reads["cigar"], dtype=np.uint32)
    seq_off = np.ascontiguousarray(reads["seq_off"], dtype=np.int64)
    seq = np.ascontiguousarray(reads["seq"], dtype=np.uint8)
    l_qseq = np.ascontiguousarray(reads["l_qseq"], dtype=np.int32)
    ref = np.frombuffer(ref_seq.encode() if isinstance(ref_seq, str) else bytes(ref_seq), dtype=np.uint8).copy()
    prm = _Params(int(min_depth), float(min_snp_af), float(min_indel_af), int(min_mq), int(bool(call_snp_only)),
                  int(bool(call_ht)), int(bool(gvcf)), int(max_indel_length))
    matrix = np.zeros((W, 18), dtype=np.int64)
    major = np.zeros(W, dtype=np.int64)
    stats = np.zeros((W, 6), dtype=np.int32)
    cand = np.zeros(W, dtype=np.int64)
    ok = np.zeros(W, dtype=np.uint8)
    prc = np.zeros(W, dtype=np.int64)
    ptc = np.zeros(W, dtype=np.int64)
    n_cols = ctypes.c_int64(0)
    n_cand = ctypes.c_int64(0)
    alt_cap = 64 * 1024 * 1024 if alt_info else 0
    alt_buf = ctypes.create_string_buffer(alt_cap) if alt_info else None
    alt_len = ctypes.c_int64(0)
    bounds = np.zeros((W, 2), dtype=np.int64)
    rc = L.oracle_clair3_pileup(ctypes.c_int64(n), _p(pos), _p(flag), _p(mapq), _p(cigar_off), _p(cigar), _p(seq_off), _p(seq),
                                _p(l_qseq), ctypes.c_int64(int(start)), ctypes.c_int64(int(end)), _p(ref),
                                ctypes.c_int64(int(ref_start)), ctypes.c_int64(len(ref)), ctypes.byref(prm),
                                ctypes.byref(n_cols), _p(matrix), _p(major), _p(stats), _p(cand), _p(ok), ctypes.byref(n_cand),
                                _p(prc), _p(ptc), alt_buf, ctypes.c_int64(alt_cap), ctypes.byref(alt_len), _p(bounds))
    if rc != 0:
        raise MemoryError("oracle_clair3_pileup failed")
    nc, nk = n_cols.value, n_cand.value
    extra = {}
    if alt_info:
        if alt_len.value > alt_cap:
            raise MemoryError("alt_info text buffer too small")
        extra["alt_info"] = alt_buf.raw[:alt_len.value].decode().split("\n")[:-1]
    return {**extra, "matrix": matrix[:nc].copy(), "major": major[:nc].copy(), "stats": stats[:nc].copy(), "cand_cols": cand[:nk].copy(),
            "cand_ok": ok[:nk].copy(), "pos_ref_count": prc, "pos_total_count": ptc, "window_bounds": bounds[:nk].copy()}


def _reads_overlapping(rec, lo, hi):
    """The records an indexed fetch of [lo, hi) would return (what sam_itr_querys hands the reference for its region string)."""
    ops = rec["cigar"] & 15
    lens = (rec["cigar"] >> 4).astype(np.int64)
    refl = np.where(np.isin(ops, (0, 2, 3, 7, 8)), lens, 0)
    csum = np.concatenate([[0], np.cumsum(refl)])
    span = csum[rec["cigar_off"][1:]] - csum[rec["cigar_off"][:-1]]
    keep = np.nonzero((rec["pos"] < hi) & (rec["pos"] + span > lo))[0]
    if len(keep) == 0:
        return None
    a, b = int(keep[0]), int(keep[-1]) + 1            # sorted by pos: a contiguous run is a superset and keeps the order
    c0, s0 = int(rec["cigar_off"][a]), int(rec["seq_off"][a])
    return {"pos": rec["pos"][a:b], "flag": rec["flag"][a:b], "mapq": rec["mapq"][a:b], "l_qseq": rec["l_qseq"][a:b],
            "cigar_off": rec["cigar_off"][a:b + 1] - c0, "cigar": rec["cigar"][c0:int(rec["cigar_off"][b])],
            "seq_off": rec["seq_off"][a:b + 1] - s0, "seq": rec["seq"][s0:int(rec["seq_off"][b])]}


def _worker_main(argv):
    """python -m oracle.pileup_oracle <records.npz> <start> <end> <min seconds>: one single-threaded worker of the CPU baseline (the
    reference runs one such process per chunk under GNU parallel, scripts/clair3_c_impl.sh): counts its region repeatedly for at
    least <min seconds> and prints {"bases": ..., "seconds": ...} - bases = sum of the per-column depths, as bench.py counts them."""
    import json
    import time
    path, start, end, min_s = argv[0], int(argv[1]), int(argv[2]), float(argv[3])
    z = np.load(path)
    rec = {k: z[k] for k in ("pos", "flag", "mapq", "cigar_off", "cigar", "seq_off", "seq", "l_qseq")}
    ref, rs = z["ref"].tobytes(), int(z["ref_start"])
    sub = _reads_overlapping(rec, start, end)
    bases, reps, t0 = 0, 0, time.perf_counter()
    while sub is not None:
        r = clair3_pileup(sub, start, end, ref, rs)
        bases += int(r["stats"][:, 0].sum())
        reps += 1
        if time.perf_counter() - t0 >= min_s:
            break
    print(json.dumps({"bases": bases, "seconds": time.perf_counter() - t0, "reps": reps}))


if __name__ == "__main__":
    import sys
    _worker_main(sys.argv[1:])
