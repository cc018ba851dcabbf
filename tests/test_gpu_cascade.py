"""The pileup -> full-alignment cascade on the GPU (clair3_b200/cascade.py, csrc/cascade.cu): the device selection against
the host ``select`` on the same call records, a build from device candidates against a build from host candidates, and
``call_region`` against the same calls assembled through host records and host candidates (``call_region_host``)."""
import numpy as np
import pytest
import torch

from clair3_b200 import bam_io, cascade, decode, synth, synth_reads as sr
from clair3_b200._ffi import C3BError
from clair3_b200.model import Clair3_F, Clair3_P

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
CFG_P = decode.replay_config(pileup=True, add_indel_length=False)._replace(is_show_reference=True)
CFG_F = decode.replay_config(pileup=False, add_indel_length=True)._replace(is_show_reference=True)


@pytest.fixture(scope="module")
def models():
    p = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    p.to(DEV)
    p.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()})
    f = Clair3_F(add_indel_length=True, predict=True, input_channels=8)
    f.to(DEV)
    f.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=8, seed=1).items()})
    return p, f


@pytest.fixture(scope="module")
def ws():
    w = cascade.Workspaces(0)
    yield w
    w.close()


@pytest.fixture(scope="module")
def region(tmp_path_factory):
    """A 12 kb region at depth 24 with 2 kb reads, written as an indexed BAM."""
    rec, ref, rs = sr.random_alignment(12000, depth=24, read_len=2000, seed=61, origin=3000)
    path = str(tmp_path_factory.mktemp("cascade") / "r.bam")
    bam_io.write_bam(path, rec, [("ctg", rs + len(ref))])
    bam_io.write_bai(path)
    return path, ref, rs, 3000, 15000


def _phased(ref, rs, start, end, step=900, seed=3):
    rng = np.random.default_rng(seed)
    out = []
    for p in range(start + 50, end, step):
        b = ref[p - rs].upper()
        alt = "ACGT"[("ACGT".index(b) + 1 + int(rng.integers(0, 3))) % 4] if b in "ACGT" else "A"
        out.append((p, b, alt, int(rng.integers(1, 3)), start))
    return out


def _pileup(ws, models, region):
    path, ref, rs, start, end = region
    lo, hi = cascade._span(start, end)
    rec = ws.decoder.decode(path, "ctg", lo, hi, fa_fields=True,
                            ref_seq=torch.from_numpy(np.frombuffer(ref.encode(), np.uint8).copy()).to(DEV))
    res = ws.counter.count(rec, start, end, None, rs, alt_info=True).call(models[0], CFG_P, "ctg")
    return rec, res


@pytest.mark.parametrize("cuts", ["none", "own", "all", "references", "variants"])
def test_device_selection_matches_host(ws, models, region, cuts):
    rec, res = _pileup(ws, models, region)
    var_q, ref_q = {"none": (0.0, 0.0), "own": cascade.qual_cutoffs([res], "ont"), "all": (1000.0, 1000.0),
                    "references": (0.0, 1000.0), "variants": (1000.0, 0.0)}[cuts]
    want, _ = cascade.select(res, var_q, ref_q)
    sel, count = cascade.select_device(res, var_q, ref_q)
    n = int(count.item())
    assert np.array_equal(sel[:n].cpu().numpy(), want)
    rows = cascade.row_indices(res)
    is_ref = cascade.is_reference(res, rows)
    # the reference / variant split by ALT text: (0, 1000) keeps exactly the reference rows, (1000, 0) exactly the others
    expect = {"none": 0, "all": len(rows), "references": int(is_ref.sum()), "variants": int((~is_ref).sum())}
    if cuts in expect:
        assert n == expect[cuts]
    if cuts != "none":
        assert n > 0


def test_device_candidate_build_matches_host(ws, models, region):
    path, ref, rs, start, end = region
    rec, res = _pileup(ws, models, region)
    sel, count = cascade.select_device(res, 1000.0, 1000.0)
    n = int(count.item())
    host = sel[:n].cpu().numpy()
    var = _phased(ref, rs, start, end)
    split = n // 2 + 1
    draws = 0
    for first in (0, split):
        kw = dict(variants=var, matrix_depth=12, rand_seed=1, rand_skip=0)
        b = ws.builder.build(rec, host[first:first + split], None, rs, **kw)
        mh, kh, sh = b.fetch(), b.kept_reads(), b.sizes()
        th = b.alt_text().alt_text_fetch()["text"]
        d = ws.builder.build(rec, sel, None, rs, cand_count=count, cand_first=first, cand_max=split, **kw)
        assert d.device_count() == n
        md, kd, sd = d.fetch(), d.kept_reads(), d.sizes()
        td = d.alt_text().alt_text_fetch()["text"]
        assert sd == sh and sd[0] == len(host[first:first + split])
        assert np.array_equal(md, mh) and all(np.array_equal(x, y) for x, y in zip(kd, kh)) and td == th
        draws += sd[2]
    assert draws > 0, "the case must shuffle some candidates"


def test_device_candidate_checks(ws, models, region):
    path, ref, rs, start, end = region
    rec, _ = _pileup(ws, models, region)
    bad = torch.tensor([start + 10, start + 10, start + 40], dtype=torch.int64, device=DEV)
    with pytest.raises(C3BError, match="strictly ascending"):
        ws.builder.build(rec, bad, None, rs, matrix_depth=12)
    neg = torch.tensor([-1, start + 40], dtype=torch.int64, device=DEV)
    with pytest.raises(C3BError, match="strictly ascending"):
        ws.builder.build(rec, neg, None, rs, matrix_depth=12)
    # past the device count: an empty build, no error
    ok = torch.tensor([start + 10, start + 40], dtype=torch.int64, device=DEV)
    b = ws.builder.build(rec, ok, None, rs, cand_count=torch.tensor([2], device=DEV), cand_first=5, matrix_depth=12)
    assert b.sizes()[0] == 0 and b.device_count() == 2


@pytest.mark.parametrize("phased", [False, True])
@pytest.mark.parametrize("chunks", [0, 1, 2])
def test_call_region_matches_host_route(ws, models, region, phased, chunks):
    path, ref, rs, start, end = region
    _, res = _pileup(ws, models, region)
    own = cascade.qual_cutoffs([res], "ont")
    cuts = {0: (0.0, 0.0), 1: own, 2: own}[chunks]
    n_own = len(cascade.select(res, *own)[0])
    split = {0: 10000, 1: max(n_own, 1), 2: max(1, (n_own + 1) // 2)}[chunks]
    kw = dict(var_qual=cuts[0], ref_qual=cuts[1], phased_variants=_phased(ref, rs, start, end) if phased else None,
              split_bed_size=split, workspaces=ws)
    for print_ref in (False, True):
        got = cascade.call_region(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F, print_ref=print_ref, **kw)
        want = cascade.call_region_host(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F, print_ref=print_ref, **kw)
        assert len(got["chunks"]) == chunks == len(want["chunks"])
        assert np.array_equal(got["candidates"], want["candidates"])
        assert np.array_equal(got["pileup"]["calls"], want["pileup"]["calls"])
        for a, b in zip(got["full_alignment"], want["full_alignment"]):
            assert np.array_equal(a["calls"], b["calls"]) and np.array_equal(a["position"], b["position"])
        assert got["vcf"] == want["vcf"] and len(got["vcf"]) > 0


def test_region_without_candidates(ws, models, tmp_path):
    """A region no read covers: no pileup calls, no full-alignment build, an empty merged body on both routes."""
    rec, ref, rs = sr.random_alignment(14000, depth=12, read_len=1000, seed=71, origin=2000, gaps=((8000, 11000),))
    path = str(tmp_path / "gap.bam")
    bam_io.write_bam(path, rec, [("ctg", rs + len(ref))])
    bam_io.write_bai(path)
    start, end = 8600, 10400
    for phased in (None, [(9000, "A", "C", 1, 8600)]):
        got = cascade.call_region(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F, phased_variants=phased,
                                  workspaces=ws)
        want = cascade.call_region_host(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F,
                                        phased_variants=phased, workspaces=ws)
        assert len(got["pileup"]["calls"]) == 0 == len(want["pileup"]["calls"])
        assert got["vcf"] == want["vcf"] == "" and got["chunks"] == want["chunks"] == [] and len(got["candidates"]) == 0
        assert got["full_alignment"] == want["full_alignment"] == []


def test_out_of_scope(models, region):
    path, ref, rs, start, end = region
    with pytest.raises(NotImplementedError):
        cascade.call_region(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F, platform="ilmn")
    with pytest.raises(NotImplementedError):
        cascade.call_region(path, "ctg", start, end, ref, rs, models[0], models[1],
                            CFG_P._replace(is_haploid_precise_mode_enabled=True), CFG_F)
    with pytest.raises(NotImplementedError):
        cascade.call_region(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F._replace(gvcf=True))
