"""The BED / known-sites filter inside the pileup counter (``c3b_plp_count_targeted``, ``PileupCounter.count(targets=...)``)
against the untargeted count filtered on the host by ``ContigTargets.keep``, and ``cascade.call_region(bed=, known_sites=)``
against ``call_region_host``: everything keyed by candidate must be the untargeted count's at the kept candidates, everything
else must not change, and the call records must be equal (per-site bit invariance, DESIGN.md 8, makes that exact)."""
import numpy as np
import pytest
import torch

from clair3_b200 import bam_io, cascade, decode, synth, synth_reads as sr, targets
from clair3_b200._ffi import C3BError, ffi
from clair3_b200.model import Clair3_F, Clair3_P
from clair3_b200.pileup_counts import PileupCounter

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
def counter():
    c = PileupCounter(0)
    yield c
    c.close()


def _region(seed, width=9000, origin=2000):
    rec, ref, rs = sr.random_alignment(width, depth=22, read_len=1200, seed=seed, origin=origin, wild=seed % 2 == 1)
    return rec, ref, rs, origin, origin + width


def _random_bed(rng, start, end, n, lo=1, hi=400):
    s = rng.integers(start - 200, end, n)
    e = s + rng.integers(0, hi, n)
    rows = "".join("ctg\t%d\t%d\n" % (a, b) for a, b in zip(np.maximum(s, 0), e))
    return targets.read_bed(rows).contig("ctg")


def _random_sites(rng, start, end, cand_pos, n):
    pick = rng.choice(cand_pos, min(n, len(cand_pos)), replace=False) if len(cand_pos) else np.zeros(0, np.int64)
    extra = rng.integers(start, end, n)
    rows = "".join("ctg\t%d\t.\tA\tC\n" % p for p in np.concatenate([pick, extra]))
    return targets.read_vcf(rows).contig("ctg")


def _count(counter, region, tg, **kw):
    rec, ref, rs, start, end = region
    counter.count(rec, start, end, ref, rs, alt_info=True, targets=tg, **kw)
    r = counter.fetch()
    r["bounds"] = counter.window_bounds()
    r["text"] = counter.alt_text().alt_text_fetch()["text"]
    return r


def _assert_filtered(got, full, keep):
    for k in ("matrix", "major", "stats"):
        assert np.array_equal(got[k], full[k]), k
    assert np.array_equal(got["cand_cols"], full["cand_cols"][keep])
    assert np.array_equal(got["cand_ok"], full["cand_ok"][keep])
    assert np.array_equal(got["bounds"], full["bounds"][keep])
    assert got["text"] == [t for t, k in zip(full["text"], keep) if k]


@pytest.mark.parametrize("seed", [3, 4, 5])
@pytest.mark.parametrize("kind", ["bed_sparse", "bed_dense", "known_sites"])
def test_targeted_count_is_the_filtered_count(counter, seed, kind):
    region = _region(seed)
    start, end = region[3], region[4]
    full = _count(counter, region, None)
    pos1 = full["major"][full["cand_cols"]] + 1
    rng = np.random.default_rng(seed * 7 + len(kind))
    tg = {"bed_sparse": lambda: _random_bed(rng, start, end, 12, hi=150),
          "bed_dense": lambda: _random_bed(rng, start, end, 60, hi=600),
          "known_sites": lambda: _random_sites(rng, start, end, pos1, 40)}[kind]()
    keep = tg.keep(pos1)
    assert 0 < keep.sum() < len(keep), "the case must keep some candidates and drop others"
    got = _count(counter, region, tg)
    assert counter.sizes()[1] == int(keep.sum())
    _assert_filtered(got, full, keep)


@pytest.mark.parametrize("call_ht", [False, True])
def test_targeted_call_records(counter, models, call_ht):
    region = _region(8)
    rec, ref, rs, start, end = region
    full = counter.count(rec, start, end, ref, rs, alt_info=True, call_ht=call_ht).call(models[0], CFG_P, "ctg")
    tg = _random_bed(np.random.default_rng(1), start, end, 20, hi=300)
    keep = tg.keep(full["position"])
    assert 0 < keep.sum() < len(keep)
    got = counter.count(rec, start, end, ref, rs, alt_info=True, call_ht=call_ht, targets=tg).call(models[0], CFG_P, "ctg")
    idx = np.nonzero(keep)[0]
    assert np.array_equal(got["position"], full["position"][idx])
    assert np.array_equal(got["calls"], full["calls"][idx])
    assert np.array_equal(got["cand_ok"], full["cand_ok"][idx])
    assert torch.equal(got["Y"], full["Y"][torch.as_tensor(idx, device=DEV)])
    want = cascade.take_calls(full, idx)
    assert [decode.call_row(got, s, CFG_P) for s in range(len(idx))] == [decode.call_row(want, s, CFG_P) for s in range(len(idx))]


def test_empty_and_covering_targets(counter, models):
    region = _region(9)
    rec, ref, rs, start, end = region
    full = _count(counter, region, None)
    yf = counter.count(rec, start, end, ref, rs, alt_info=True).call(models[0], CFG_P, "ctg")
    # no interval at all: no candidate, an empty call
    for empty in (targets.ContigTargets("ctg", [], []), targets.ContigTargets("ctg", [], [], known=[])):
        got = _count(counter, region, empty)
        _assert_filtered(got, full, np.zeros(len(full["cand_cols"]), bool))
        res = counter.count(rec, start, end, ref, rs, alt_info=True, targets=empty).call(models[0], CFG_P, "ctg")
        assert len(res["calls"]) == 0 and res["Y"].shape[0] == 0
    # known sites without an interval around them keep nothing either
    sites = targets.ContigTargets("ctg", [], [], known=full["major"][full["cand_cols"]] + 1)
    assert counter.count(rec, start, end, ref, rs, targets=sites).sizes()[1] == 0
    # one interval over the whole region: the untargeted count, bit for bit
    every = targets.ContigTargets("ctg", [0], [end + 100])
    got = _count(counter, region, every)
    _assert_filtered(got, full, np.ones(len(full["cand_cols"]), bool))
    res = counter.count(rec, start, end, ref, rs, alt_info=True, targets=every).call(models[0], CFG_P, "ctg")
    assert np.array_equal(res["calls"], yf["calls"]) and torch.equal(res["Y"], yf["Y"])


class _Raw:
    """Target arrays handed over as given: device tensors (checked on the stream) or host arrays (checked at the call)."""

    def __init__(self, starts, ends, end_max, sites=None, on_device=True):
        self.a = [np.asarray(x, np.int64) for x in (starts, ends, end_max)] + [None if sites is None else np.asarray(sites, np.int64)]
        self.on_device = on_device

    def struct(self, device):
        if self.on_device:
            t = [None if x is None else torch.from_numpy(x).to(device) for x in self.a]
            return targets.device_struct(*t)
        st = targets.device_struct(*[torch.from_numpy(x) if x is not None else None for x in self.a])[0]
        st.on_device = 0
        p = lambda x: ffi.cast("const int64_t *", x.ctypes.data) if x is not None and len(x) else ffi.NULL  # noqa: E731
        st.starts, st.ends, st.end_max, st.sites = p(self.a[0]), p(self.a[1]), p(self.a[2]), p(self.a[3])
        return st, self.a


def test_target_arrays_are_checked(counter):
    region = _region(10)
    rec, ref, rs, start, end = region
    full = _count(counter, region, None)
    ct = _random_bed(np.random.default_rng(2), start, end, 15)
    good = (ct.starts, ct.ends, ct.end_max)
    # host arrays: the same result as the device copies
    got = _count(counter, region, _Raw(*good, on_device=False))
    _assert_filtered(got, full, ct.keep(full["major"][full["cand_cols"]] + 1))
    bad = {"unsorted": (ct.starts[::-1].copy(), ct.ends[::-1].copy(), np.maximum.accumulate(ct.ends[::-1])),
           "end_before_start": (ct.starts, ct.starts - 1, np.maximum.accumulate(ct.starts - 1)),
           "not_running_max": (ct.starts, ct.ends, ct.ends.copy() * 0 + int(ct.ends.min()))}
    for name, arrs in bad.items():
        with pytest.raises(C3BError, match="c3b_plp_count_targeted"):
            counter.count(rec, start, end, ref, rs, targets=_Raw(*arrs, on_device=False))
        # device arrays: queued without a wait, reported by the count's own wait
        counter.count(rec, start, end, ref, rs, targets=_Raw(*arrs))
        with pytest.raises(C3BError, match="out of order"):
            counter.sizes()
    for sites in ([5, 5], [9, 3]):
        counter.count(rec, start, end, ref, rs, targets=_Raw(*good, sites=sites))
        with pytest.raises(C3BError, match="out of order"):
            counter.sizes()
    # the workspace is whole again after a failed check
    _assert_filtered(_count(counter, region, ct), full, ct.keep(full["major"][full["cand_cols"]] + 1))


@pytest.fixture(scope="module")
def ws():
    w = cascade.Workspaces(0)
    yield w
    w.close()


@pytest.fixture(scope="module")
def bam(tmp_path_factory):
    rec, ref, rs = sr.random_alignment(12000, depth=24, read_len=2000, seed=61, origin=3000)
    path = str(tmp_path_factory.mktemp("targets") / "r.bam")
    bam_io.write_bam(path, rec, [("ctg", rs + len(ref))])
    bam_io.write_bai(path)
    return path, ref, rs, 3000, 15000


@pytest.mark.parametrize("mode", ["bed", "bed_file", "known_sites", "known_sites_chunk"])
def test_call_region_targeted_matches_host_route(ws, models, bam, mode, tmp_path):
    path, ref, rs, start, end = bam
    rng = np.random.default_rng(11)
    full = cascade.call_region_host(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F, workspaces=ws)
    pos = full["pileup"]["position"]
    kw = {}
    if mode.startswith("bed"):
        s = rng.integers(start, end, 25)
        text = "".join("ctg\t%d\t%d\n" % (a, a + b) for a, b in zip(s, rng.integers(0, 300, 25)))
        if mode == "bed_file":
            (tmp_path / "t.bed").write_text(text)
            kw["bed"] = str(tmp_path / "t.bed")
        else:
            kw["bed"] = targets.read_bed(text)
    else:
        sites = np.sort(np.concatenate([rng.choice(pos, 60, replace=False), rng.integers(start, end, 30)]))
        text = "".join("ctg\t%d\t.\t%s\tC\t.\t.\t.\tGT\t0/1\n" % (p, ref[p - 1 - rs]) for p in sites)
        known = targets.read_vcf(text)
        kw["known_sites"] = known.contig("ctg", chunk=(2, 3)) if mode == "known_sites_chunk" else known
    for print_ref in (False, True):
        got = cascade.call_region(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F, print_ref=print_ref,
                                  workspaces=ws, **kw)
        want = cascade.call_region_host(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F, print_ref=print_ref,
                                        workspaces=ws, **kw)
        assert 0 < len(got["pileup"]["calls"]) < len(full["pileup"]["calls"])
        assert np.array_equal(got["pileup"]["calls"], want["pileup"]["calls"])
        assert np.array_equal(got["pileup"]["position"], want["pileup"]["position"])
        assert got["qual_cutoffs"] == want["qual_cutoffs"]
        assert np.array_equal(got["candidates"], want["candidates"])
        assert got["vcf"] == want["vcf"]
        if mode.startswith("known"):
            assert got["genotyped"] == want["genotyped"] and len(got["genotyped"]) > 0
            known = cascade.contig_targets("ctg", known_sites=kw["known_sites"]).known
            n_known = int(((known > start) & (known <= end)).sum())
            assert got["genotyped"].count("\n") == n_known
        else:
            assert "genotyped" not in got
    with pytest.raises(ValueError, match="either bed or known_sites"):
        cascade.call_region(path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F, workspaces=ws,
                            bed=targets.read_bed("ctg\t1\t2\n"), known_sites=targets.read_vcf("ctg\t5\t.\tA\tC\n"))
