"""The record check every consumer's intake makes (``clair3_b200/csrc/records_check.cuh``) built for the host with AddressSanitizer
and UBSan, against ``BamRecords``: on valid records and on thousands of seeded single mutations of them, the check must fail
exactly when ``BamRecords`` raises, with the reason ``BamRecords`` names and at the first read that breaks it, and must never read
outside the n_reads per-read entries and n_reads + 1 offsets it is given.  The header is ``__host__ __device__``: the same code
runs as the device check of records that arrive as device tensors, and on the host for host records."""
import os
import shutil
import struct
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import deflate_craft as dc  # noqa: E402
import fa_ref_cases as frc  # noqa: E402
from test_bam_cg_cpu import ultra_long_case  # noqa: E402

from clair3_b200 import synth_reads as sr  # noqa: E402
from clair3_b200._ffi import C3BError  # noqa: E402
from clair3_b200.records import FIELDS, BamRecords, records_struct  # noqa: E402

OFFSETS = ("cigar", "seq", "qual", "qname", "mv")          # the check's field order
# records_check.cuh's reasons, as the part of BamRecords' message that names each
REASONS = {1: "span cigar / seq", 2: "span cigar / seq", 3: "must not decrease", 4: "must not decrease", 5: "sorted by pos",
           6: "shorter than (l_qseq + 1) / 2", 7: "qual and qual_off go together", 8: "qual_off must be",
           9: "l_qseq base qualities", 10: "qname and qname_off go together", 11: "qname_off must be",
           12: "mv and mv_off go together", 13: "mv_off must be"}
PAIR = {"qual": 7, "qname": 10, "mv": 12}
SPAN = {"cigar": 1, "seq": 2, "qual": 8, "qname": 11, "mv": 13}
DEC = {"cigar": 3, "seq": 4, "qual": 8, "qname": 11, "mv": 13}


def build_driver(out_dir):
    """Compiles tests/records_check_host.cpp with AddressSanitizer and UBSan into ``out_dir``; its path, or None without g++."""
    cxx = shutil.which("g++")
    if cxx is None:
        return None
    exe = os.path.join(out_dir, "records_check_host")
    r = subprocess.run([cxx, "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-fno-omit-frame-pointer", "-Wall", "-Werror", "-I", os.path.join(os.path.dirname(HERE), "clair3_b200", "csrc"),
                        os.path.join(HERE, "records_check_host.cpp"), "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def encode(a):
    """One case of the driver's input (records_check_host.cpp) from record arrays as ``BamRecords`` takes them."""
    n = len(a["pos"])
    present, lens, offs = 0, [], b""
    for f, k in enumerate(OFFSETS):
        o, v = a.get(k + "_off"), a.get(k)
        present |= (o is not None) << f | (v is not None) << (8 + f)
        lens.append(0 if v is None else len(v))
        if o is not None:
            assert len(o) == n + 1
            offs += np.ascontiguousarray(o, np.int64).tobytes()
    return (struct.pack("<qII5q", n, present, 0, *lens) + np.ascontiguousarray(a["pos"], np.int64).tobytes()
            + np.ascontiguousarray(a["l_qseq"], np.int32).tobytes() + offs)


def run_check(exe, cases):
    """(reason, read) per case, 0 for records the check passes; fails on any sanitizer report."""
    out = dc.run_host(exe, "", b"".join(encode(a) for a in cases)).decode().split("\n")[:-1]
    assert len(out) == len(cases)
    return [tuple(int(x) for x in line.split()) for line in out]


def host_verdict(a):
    """BamRecords' message for the arrays, None when it takes them."""
    try:
        BamRecords(**a)
    except C3BError as e:
        return str(e)
    return None


def fault(a):
    """(reason, first read that breaks it) of records_check.cuh, stated plainly over the arrays; (0, 0) for none."""
    n = len(a["pos"])
    found = [(PAIR[k], 0) for k in PAIR if (a.get(k) is None) != (a.get(k + "_off") is None)]
    for k in OFFSETS:
        o = a.get(k + "_off")
        if o is None or (k in ("cigar", "seq") and n == 0):
            continue
        length = 0 if a.get(k) is None else len(a[k])
        if o[0] != 0:
            found.append((SPAN[k], 0))
        if o[n] != length:
            found.append((SPAN[k], max(n - 1, 0)))
        down = np.nonzero(o[1:] < o[:-1])[0]
        if len(down):
            found.append((DEC[k], int(down[0])))
    if n:
        lq = np.asarray(a["l_qseq"], np.int64)
        for reason, bad, at in ((5, a["pos"][1:] < a["pos"][:-1], 1), (6, (lq + 1) // 2 > np.diff(a["seq_off"]), 0),
                                (9, np.diff(a["qual_off"]) != lq if a.get("qual_off") is not None else np.zeros(0, bool), 0)):
            if bad.any():
                found.append((reason, int(np.argmax(bad)) + at))
    return min(found, default=(0, 0))


# ---------------------------------------------------------------------------------------------------------------- the records
def _core(rec):
    return {f.name: np.asarray(rec[f.name]) for f in FIELDS if rec.get(f.name) is not None}


def bases():
    """Valid runs of records: synthetic reads, the ultra-long CIGAR case with qualities, names and mv tables, and
    full-alignment cases with qualities, names and dwell mv tags."""
    out = []
    rec, _, _ = sr.random_alignment(20000, depth=6, read_len=1500, seed=7, wild=True)
    out.append(("synth", _core(rec)))
    rec, _, _, _ = ultra_long_case(n_cycles=3000)
    out.append(("ultra_long", _core(rec)))
    for name in ("dwell_insertion_signal_wraps", "dwell_more_moves_than_bases"):
        out.append((name, _core(frc.BUILD[name]()[0])))
    return out


BIG = (2 ** 62, 2 ** 63 - 1, -1, -2, -(2 ** 62), -(2 ** 63))


def _with(a, **changes):
    b = dict(a)
    for k, v in changes.items():
        if v is None:
            b.pop(k, None)
        else:
            b[k] = v
    return b


def mutate(a, kind, rng):
    """One seeded single mutation of the arrays, or None where the kind does not apply to them."""
    n = len(a["pos"])
    fields = [k for k in OFFSETS if a.get(k + "_off") is not None]
    k = fields[rng.integers(len(fields))]
    o = a[k + "_off"].copy()
    if kind == "first_offset":
        o[0] = rng.choice([1, -1, int(rng.integers(2, 1000))])
    elif kind == "last_offset":
        o[n] += rng.choice([-1, 1])
    elif kind == "decrease":
        i = int(rng.integers(1, n + 1))
        o[i] = o[i - 1] - int(rng.integers(1, 4))
    elif kind == "huge":
        o[int(rng.integers(0, n + 1))] = rng.choice(BIG)
    elif kind == "wrapped":
        # a step down past -2^63 and a step back up that each fit 64 bits: np.diff sees two steps up
        if n < 3:
            return None
        i = int(rng.integers(1, n - 1))
        o[i], o[i + 1] = -(2 ** 63) + int(rng.integers(0, 8)), -int(rng.integers(1, 8))
    elif kind == "pos":
        if n < 2:
            return None
        i = int(rng.integers(1, n))
        p = a["pos"].copy()
        p[i] = p[i - 1] - int(rng.integers(1, 5))
        return _with(a, pos=p)
    elif kind == "l_qseq":
        i = int(rng.integers(0, n))
        lq = a["l_qseq"].copy()
        lq[i] = 2 * (a["seq_off"][i + 1] - a["seq_off"][i]) + 1          # one base more than the packed bytes hold
        return _with(a, l_qseq=lq)
    elif kind == "qual_span":
        if a.get("qual_off") is None or n < 2:
            return None
        o = a["qual_off"].copy()
        o[int(rng.integers(1, n))] += rng.choice([-1, 1])
        return _with(a, qual_off=o)
    elif kind == "unpaired":
        opt = [f for f in ("qual", "qname", "mv") if a.get(f) is not None]
        if not opt:
            return None
        f = opt[rng.integers(len(opt))]
        return _with(a, **{f + "_off" if rng.random() < 0.5 else f: None})
    else:
        raise AssertionError(kind)
    return _with(a, **{k + "_off": o})


KINDS = ("first_offset", "last_offset", "decrease", "huge", "wrapped", "pos", "l_qseq", "qual_span", "unpaired")


def edge_cases():
    """0 reads, 1 read, and empty value arrays (the non-null placeholder records_struct passes for them)."""
    e64, e8 = np.zeros(0, np.int64), np.zeros(0, np.uint8)
    zero = dict(pos=e64, flag=np.zeros(0, np.uint16), mapq=e8, l_qseq=np.zeros(0, np.int32), cigar_off=np.zeros(1, np.int64),
                cigar=np.zeros(0, np.uint32), seq_off=np.zeros(1, np.int64), seq=e8)
    one = dict(pos=np.array([100], np.int64), flag=np.zeros(1, np.uint16), mapq=np.array([60], np.uint8),
               l_qseq=np.array([5], np.int32), cigar_off=np.array([0, 1], np.int64), cigar=np.array([5 << 4], np.uint32),
               seq_off=np.array([0, 3], np.int64), seq=np.array([0x12, 0x48, 0x10], np.uint8))
    empty = dict(pos=np.array([5, 5], np.int64), flag=np.zeros(2, np.uint16), mapq=np.zeros(2, np.uint8),
                 l_qseq=np.zeros(2, np.int32), cigar_off=np.zeros(3, np.int64), cigar=np.zeros(0, np.uint32),
                 seq_off=np.zeros(3, np.int64), seq=e8, qual_off=np.zeros(3, np.int64), qual=e8, qname_off=np.zeros(3, np.int64),
                 qname=e8, mv_off=np.zeros(3, np.int64), mv=np.zeros(0, np.int32))
    one_q = dict(one, qual_off=np.array([0, 5], np.int64), qual=np.arange(5, dtype=np.uint8))
    return [
        ("0 reads", zero),
        ("0 reads, core offsets not read", dict(zero, cigar_off=np.array([3], np.int64))),
        ("0 reads, optional offsets at 0", dict(zero, qual_off=np.zeros(1, np.int64), qual=e8, mv_off=np.zeros(1, np.int64),
                                               mv=np.zeros(0, np.int32))),
        ("0 reads, qual_off past qual", dict(zero, qual_off=np.ones(1, np.int64), qual=e8)),
        ("0 reads, qname without offsets", dict(zero, qname=e8)),
        ("1 read", one),
        ("1 read with qual", one_q),
        ("1 read, seq one byte short", dict(one, l_qseq=np.array([7], np.int32))),
        ("1 read, cigar_off past cigar", dict(one, cigar_off=np.array([0, 2], np.int64))),
        ("1 read, qual one short", dict(one_q, qual_off=np.array([0, 4], np.int64), qual=np.arange(4, dtype=np.uint8))),
        ("empty value arrays", empty),
        ("empty seq, one base", dict(empty, l_qseq=np.array([0, 1], np.int32))),
        ("empty qual, one base", dict(empty, l_qseq=np.array([0, 1], np.int32), seq_off=np.array([0, 0, 1], np.int64),
                                      seq=np.zeros(1, np.uint8))),
        ("empty mv, offset 1", dict(empty, mv_off=np.array([0, 0, 1], np.int64))),
    ]


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = build_driver(str(tmp_path_factory.mktemp("records_check_host")))
    if exe is None:
        pytest.skip("needs g++ for the sanitized host build")
    return exe


def _agree(exe, named):
    got = run_check(exe, [a for _, a in named])
    verdicts = {}
    for (name, a), (reason, read) in zip(named, got):
        msg = host_verdict(a)
        assert (reason, read) == fault(a), name
        if msg is None:
            assert reason == 0, (name, reason, read)
        else:
            assert reason in REASONS and REASONS[reason] in msg, (name, reason, msg)
        verdicts[reason] = verdicts.get(reason, 0) + 1
    return verdicts


def test_valid_records_pass(driver):
    assert run_check(driver, [a for _, a in bases()]) == [(0, 0)] * len(bases())


def test_edge_cases_match_bam_records(driver):
    _agree(driver, edge_cases())


def test_seeded_mutations_match_bam_records(driver):
    rng = np.random.default_rng(20261018)
    named = []
    for base, a in bases():
        for kind in KINDS:
            for j in range(80):
                m = mutate(a, kind, rng)
                if m is not None:
                    named.append(("%s %s %d" % (base, kind, j), m))
    assert len(named) >= 2500
    verdicts = _agree(driver, named)
    assert set(verdicts) >= set(range(1, 14)) - {7}, verdicts      # every reason met; a qual pair break needs qual present
    assert verdicts[7] > 0 and verdicts.get(0, 0) < len(named) // 10, verdicts


def test_offsets_that_wrap_np_diff_are_rejected():
    """An offset near -2^63 between two small ones is two steps up to np.diff; BamRecords compares steps instead."""
    a = dict(edge_cases()[-1][1])
    a["cigar_off"] = np.array([0, -(2 ** 63) + 1, 0], np.int64)
    with pytest.raises(C3BError, match="must not decrease"):
        BamRecords(**a)


def test_records_struct_passes_each_value_arrays_length():
    rec = _core(frc.BUILD["dwell_insertion_signal_wraps"]()[0])
    host = BamRecords(**rec)
    s = records_struct(host, optional=True)
    assert (s.core.n_cigar, s.core.n_seq, s.n_qual, s.n_qname, s.n_mv) == tuple(len(rec[k]) for k in OFFSETS)
    assert records_struct(host).n_seq == len(rec["seq"])
