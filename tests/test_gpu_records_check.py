"""Records that arrive as device tensors are checked on the device before any kernel indexes through their offsets
(``clair3_b200/csrc/records_check.cuh``): every consumer (the pileup count, the targeted count, the count behind the pileup
all_alt_info text, the full-alignment build behind its text, ``cascade.call_region``) must reject each kind of malformed run
that ``BamRecords`` rejects on the host, with a ``C3BError`` naming the field and the first read that breaks it, and must then
compute on the same workspace exactly what a fresh workspace computes.  Valid device records, including views at a storage
offset and tensors written on another stream, must give the host route's outputs bit for bit.  The host build of the same
check is held to ``BamRecords`` on thousands of mutations in test_records_check_cpu.py; every case here is one of those kinds,
rejected by a kernel that reads only the per-read entries and offsets whose sizes the call is given."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import fa_ref_cases as frc  # noqa: E402
from test_records_check_cpu import KINDS, fault, host_verdict, mutate  # noqa: E402

from clair3_b200 import bam_io, cascade, decode, synth, synth_reads as sr, targets  # noqa: E402
from clair3_b200._ffi import C3BError  # noqa: E402
from clair3_b200.fa_tensor import FullAlignmentBuilder  # noqa: E402
from clair3_b200.model import Clair3_F, Clair3_P  # noqa: E402
from clair3_b200.pileup_counts import PileupCounter  # noqa: E402
from clair3_b200.records import CORE, FIELDS, BamRecords, DeviceBamRecords  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
# the field each reason of records_check.cuh names in the error
NAMES = {1: "cigar_off", 2: "seq_off", 3: "cigar_off", 4: "seq_off", 5: "pos", 6: "seq holds", 7: "qual and qual_off",
         8: "qual_off", 9: "qual holds", 10: "qname and qname_off", 11: "qname_off", 12: "mv and mv_off", 13: "mv_off"}
CFG_P = decode.replay_config(pileup=True, add_indel_length=False)._replace(is_show_reference=True)
CFG_F = decode.replay_config(pileup=False, add_indel_length=True)._replace(is_show_reference=True)


def _tensors(a, stream=None):
    """Device tensors of record arrays (torch's signed views of the unsigned fields), written on ``stream`` if given."""
    out = {}
    with torch.cuda.stream(stream or torch.cuda.current_stream(DEV)):
        for f in FIELDS:
            v = a.get(f.name)
            out[f.name] = None if v is None else torch.from_numpy(np.ascontiguousarray(v, f.dtype).view(f.view)).to(DEV)
    if stream is not None:
        torch.cuda.current_stream(DEV).wait_stream(stream)
    return out


def _device(a, ref, stream=None):
    return DeviceBamRecords.from_tensors(_tensors(a, stream), DEV, ref)


@pytest.fixture(scope="module")
def pileup_case():
    rec, ref, rs = sr.random_alignment(6000, depth=16, read_len=900, seed=29, wild=True)
    a = {f.name: np.asarray(rec[f.name]) for f in CORE}
    return a, ref, rs, rs + 1000, rs + 5000


@pytest.fixture(scope="module")
def fa_case():
    rec, ref, cands, _, _ = frc.BUILD["dwell_insertion_signal_wraps"]()
    a = {f.name: np.asarray(rec[f.name]) for f in FIELDS if rec.get(f.name) is not None}
    return a, ref, cands


def _cases(a, seed, per_kind=3):
    """Seeded single mutations of ``a`` that BamRecords rejects, each with the reason and read the device must name."""
    rng = np.random.default_rng(seed)
    out = []
    for kind in KINDS:
        for _ in range(per_kind):
            m = mutate(a, kind, rng)
            if m is None or host_verdict(m) is None:
                continue
            reason, read = fault(m)
            assert reason
            out.append((kind, m, reason, read))
    return out


def _rejects(call, reason, read):
    with pytest.raises(C3BError) as e:
        call()
    assert "records: read %d: %s" % (read, NAMES[reason]) in str(e.value), (reason, read, str(e.value))


def _count(counter, rec, case, **kw):
    a, ref, rs, start, end = case
    out = counter.count(rec, start, end, ref if isinstance(rec, dict) else None, rs, alt_info=True, **kw).fetch()
    out["text"] = counter.alt_text().alt_text_fetch()["text"]
    return out


def _same(x, y):
    assert x.keys() == y.keys()
    for k in x:
        if isinstance(x[k], np.ndarray):
            assert x[k].dtype == y[k].dtype and np.array_equal(x[k], y[k]), k
        else:
            assert x[k] == y[k], k


def test_pileup_consumers_reject_malformed_device_records(pileup_case):
    a, ref, rs, start, end = pileup_case
    dref = torch.from_numpy(np.frombuffer(ref.encode(), np.uint8).copy()).to(DEV)
    every = targets.ContigTargets("ctg", [0], [end + 100])
    counter = PileupCounter(0)
    good = _device(a, dref)
    _count(counter, good, pileup_case)                       # a text stage could follow this count, but not a rejected one
    cases = _cases(a, 1)
    assert {k for k, *_ in cases} >= {"first_offset", "last_offset", "decrease", "huge", "wrapped", "pos", "l_qseq"}
    for kind, m, reason, read in cases:
        rec = _device(m, dref)
        _rejects(lambda: counter.count(rec, start, end, None, rs), reason, read)
        _rejects(lambda: counter.count(rec, start, end, None, rs, targets=every), reason, read)
        _rejects(lambda: counter.count(rec, start, end, None, rs, alt_info=True), reason, read)
        with pytest.raises(C3BError, match="no c3b_plp_count"):
            counter.alt_text()
    got = _count(counter, good, pileup_case)
    fresh = PileupCounter(0)
    _same(got, _count(fresh, good, pileup_case))
    _same(got, _count(fresh, dict(a), pileup_case))
    counter.close()
    fresh.close()


def _build(builder, rec, case, ref=None):
    a, href, cands = case
    b = builder.build(rec, cands, href if ref is None else ref, 0, matrix_depth=8, need_haplotagging=False, dwell=True)
    return {"matrix": b.fetch(), "sizes": b.sizes(), "text": b.alt_text().alt_text_fetch()["text"]}


def test_fa_consumers_reject_malformed_device_records(fa_case):
    a, ref, cands = fa_case
    dref = torch.from_numpy(np.frombuffer(ref.encode(), np.uint8).copy()).to(DEV)
    builder = FullAlignmentBuilder(0)
    good = _device(a, dref)
    _build(builder, good, fa_case, dref)
    cases = _cases(a, 2, per_kind=4)
    assert {r for *_, r, _ in cases} & {8, 9, 11, 13}          # the optional fields' offsets are checked too
    for kind, m, reason, read in cases:
        if kind == "unpaired":                                  # from_tensors takes no field without its offsets
            with pytest.raises(C3BError, match="go together"):
                _device(m, dref)
            continue
        rec = _device(m, dref)
        _rejects(lambda: builder.build(rec, cands, None, 0, matrix_depth=8, need_haplotagging=False, dwell=True), reason, read)
        with pytest.raises(C3BError, match="no c3b_fa_build"):
            builder.alt_text()
    got = _build(builder, good, fa_case, dref)
    fresh = FullAlignmentBuilder(0)
    want = _build(fresh, good, fa_case, dref)
    assert np.array_equal(got["matrix"], want["matrix"]) and got["sizes"] == want["sizes"] and got["text"] == want["text"]
    host = _build(fresh, dict(a), fa_case)
    assert np.array_equal(got["matrix"], host["matrix"]) and got["sizes"] == host["sizes"] and got["text"] == host["text"]
    builder.close()
    fresh.close()


def test_valid_device_records_match_the_host_route(pileup_case, fa_case):
    """Records at a storage offset inside larger tensors, and records written on another stream, count and build as host
    records do."""
    a, ref, rs, start, end = pileup_case
    dref = torch.from_numpy(np.frombuffer(ref.encode(), np.uint8).copy()).to(DEV)
    counter = PileupCounter(0)
    want = _count(counter, dict(a), pileup_case)
    t = _tensors(a)
    shifted = {k: None for k in t}
    for k, v in ((k, v) for k, v in t.items() if v is not None):
        big = torch.zeros(v.numel() + 7, dtype=v.dtype, device=DEV)
        big[3:3 + v.numel()] = v
        shifted[k] = big[3:3 + v.numel()]
        assert shifted[k].storage_offset() == 3 and shifted[k].is_contiguous()
    side = torch.cuda.Stream(DEV)
    for rec in (DeviceBamRecords.from_tensors(shifted, DEV, dref), _device(a, dref, side),
                BamRecords(**a).to_device(DEV, ref)):
        _same(_count(counter, rec, pileup_case), want)
    fa, fref, cands = fa_case
    builder = FullAlignmentBuilder(0)
    fwant = _build(builder, dict(fa), fa_case)
    fdref = torch.from_numpy(np.frombuffer(fref.encode(), np.uint8).copy()).to(DEV)
    for rec in (_device(fa, fdref, side), BamRecords(**fa).to_device(DEV, fref)):
        got = _build(builder, rec, fa_case, rec.ref)
        assert np.array_equal(got["matrix"], fwant["matrix"]) and got["sizes"] == fwant["sizes"] and got["text"] == fwant["text"]
    counter.close()
    builder.close()


@pytest.fixture(scope="module")
def models():
    p = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    p.to(DEV)
    p.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()})
    f = Clair3_F(add_indel_length=True, predict=True, input_channels=8)
    f.to(DEV)
    f.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=8, seed=1).items()})
    return p, f


def test_call_region_rejects_malformed_device_records(models, tmp_path):
    """call_region hands the decoder's device records to the counter and every build: records broken after the decode are
    rejected there, and the same workspaces then call the region as fresh ones do."""
    rec, ref, rs = sr.random_alignment(8000, depth=20, read_len=1500, seed=71, origin=3000)
    path = str(tmp_path / "r.bam")
    bam_io.write_bam(path, rec, [("ctg", rs + len(ref))])
    bam_io.write_bai(path)
    start, end = 3000, 11000
    ws = cascade.Workspaces(0)
    decode_bam = ws.decoder.decode
    broken = []

    def decode_and_break(*args, **kw):
        d = decode_bam(*args, **kw)
        if not broken:
            return d
        tensors = dict(d.t)
        tensors.update(_tensors(broken[0]))
        return DeviceBamRecords.from_tensors(tensors, DEV, d.ref)

    ws.decoder.decode = decode_and_break
    try:
        want = cascade.call_region(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F)
        lo, hi = cascade._span(start, end)
        h = decode_bam(path, "ctg", lo, hi, fa_fields=True, ref_seq=ref).host()
        a = {f.name: h[f.name] for f in CORE}
        cases = _cases(a, 3, per_kind=1)
        for kind, m, reason, read in cases:
            broken[:] = [m]
            _rejects(lambda: cascade.call_region(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F,
                                                 workspaces=ws), reason, read)
        broken.clear()
        got = cascade.call_region(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F, workspaces=ws)
        assert len(want["candidates"]) and np.array_equal(got["candidates"], want["candidates"])
        assert got["vcf"] == want["vcf"]
    finally:
        ws.close()
