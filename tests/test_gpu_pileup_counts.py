"""GPU parity of the pileup feature counter (clair3_b200/csrc/plp_counts.cu through the C-ABI of include/clair3_b200_pileup.h)
against oracle/pileup_oracle.c - integer work, so the bar is BIT-EXACT on every output array."""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

KEYS = ("major", "matrix", "stats", "cand_cols", "cand_ok")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_STATS = {}


def _dump():
    out = os.environ.get("C3B_REPORT_DIR")           # optional: where to keep the parity statistics of the run
    if not out:
        return
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "plp_parity.json"), "w") as f:
        json.dump(_STATS, f, indent=1, sort_keys=True)


def _compare(tag, got, want, gvcf=False):
    keys = KEYS + (("pos_ref_count", "pos_total_count") if gvcf else ())
    for k in keys:
        assert got[k].shape == want[k].shape, "%s: %s shape %s vs oracle %s" % (tag, k, got[k].shape, want[k].shape)
        if not np.array_equal(got[k], want[k]):
            d = np.argwhere(got[k] != want[k])
            raise AssertionError("%s: %s differs at %d places, first %s: gpu %s oracle %s" % (
                tag, k, len(d), d[0].tolist(), got[k][tuple(d[0])], want[k][tuple(d[0])]))
    _STATS[tag] = {"n_cols": int(len(want["major"])), "n_candidates": int(len(want["cand_cols"])),
                   "complete_windows": int(want["cand_ok"].sum()), "bit_exact": True}
    _dump()


@pytest.fixture(scope="module")
def counter():
    from clair3_b200 import pileup_counts as pc
    c = pc.PileupCounter(0)
    yield c
    c.close()


def test_known_answer_cases(counter):
    from oracle import pileup_oracle as po
    from test_pileup_oracle import case_indels, case_quirks
    rec, ref, matrix, major, stats5, cand = case_indels()
    r = counter.count(rec, 0, 20, ref, 0, call_ht=True).fetch()
    assert np.array_equal(r["major"], major) and np.array_equal(r["matrix"], matrix)
    assert np.array_equal(r["stats"][:, :5], stats5) and np.array_equal(r["cand_cols"], cand)
    _compare("known_indels", r, po.clair3_pileup(rec, 0, 20, ref, 0, call_ht=True))
    rec, ref, matrix, major, stats5, zero_rows = case_quirks()
    r = counter.count(rec, 0, 12, ref, 0, call_ht=True, min_depth=1).fetch()
    assert np.array_equal(r["major"], major) and np.array_equal(r["matrix"], matrix)
    assert np.array_equal((r["stats"][:, 5] & 2) != 0, zero_rows)
    _compare("known_quirks", r, po.clair3_pileup(rec, 0, 12, ref, 0, call_ht=True, min_depth=1))


@pytest.mark.parametrize("seed", range(12))
def test_random_alignments_bit_exact(counter, seed):
    from clair3_b200 import synth_reads as sr
    from oracle import pileup_oracle as po
    wild = seed % 2 == 0
    origin = [1000, 0, 5, 300][seed % 4]
    width = [700, 256, 1025, 513][seed % 4]                 # ragged last tile, exactly one tile, one column into a fifth tile
    gaps = [(origin + 100, origin + 190)] if seed % 3 == 0 else ()
    rec, ref, rs = sr.random_alignment(width, depth=[4, 12, 35][seed % 3], read_len=[60, 150, 400][seed % 3], seed=100 + seed,
                                       wild=wild, origin=origin, gaps=gaps, indel_rate=0.08, n_rate=0.01)
    kw = dict(min_depth=[2, 4][seed % 2], min_mq=[5, 20][seed % 2], call_snp_only=seed % 5 == 0, call_ht=seed % 7 == 0,
              gvcf=seed % 2 == 1)
    got = counter.count(rec, origin, origin + width, ref, rs, **kw).fetch()
    _compare("random_%d" % seed, got, po.clair3_pileup(rec, origin, origin + width, ref, rs, **kw), gvcf=kw["gvcf"])


def test_long_reads_large_region(counter):
    from clair3_b200 import synth_reads as sr
    from oracle import pileup_oracle as po
    rec, ref, rs = sr.random_alignment(40000, depth=30, read_len=5000, seed=7, indel_rate=0.05)
    got = counter.count(rec, 1000, 41000, ref, rs, gvcf=True).fetch()
    want = po.clair3_pileup(rec, 1000, 41000, ref, rs, gvcf=True)
    _compare("long_reads_40k", got, want, gvcf=True)
    pinned = counter.fetch(pinned=True)              # the page-locked staging path returns the same arrays
    for k in got:
        assert np.array_equal(pinned[k], got[k]), k
    ms, launches = counter.last_ms()
    assert launches == 8 and ms > 0
    _STATS["long_reads_40k"]["device_ms"] = ms
    _STATS["long_reads_40k"]["aligned_bases"] = int(want["stats"][:, 0].sum())
    _dump()


def test_deep_indel_rich_tile_spills_to_the_global_pool(counter):
    """More distinct indel alleles in one 256-column tile than its shared-memory pool holds (704 nodes)."""
    from clair3_b200 import synth_reads as sr
    from oracle import pileup_oracle as po
    rec, ref, rs = sr.random_alignment(600, depth=300, read_len=300, seed=9, indel_rate=0.12, wild=False)
    got = counter.count(rec, 1000, 1600, ref, rs).fetch()
    want = po.clair3_pileup(rec, 1000, 1600, ref, rs)
    distinct = int((want["matrix"][:, [4, 13, 6, 15]] > 0).sum())
    _compare("deep_indel_rich", got, want)
    _STATS["deep_indel_rich"]["columns_with_indels_x4"] = distinct
    _dump()


def test_empty_and_filtered_inputs(counter):
    from clair3_b200 import synth_reads as sr
    from oracle import pileup_oracle as po
    rec, ref, rs = sr.random_alignment(300, depth=5, read_len=100, seed=3)
    empty = {k: v[:0] if k not in ("cigar_off", "seq_off") else np.zeros(1, np.int64) for k, v in rec.items()}
    r = counter.count(empty, 1000, 1300, ref, rs).fetch()
    assert r["matrix"].shape == (0, 18) and len(r["cand_cols"]) == 0
    r = counter.count(rec, 1000, 1000, ref, rs).fetch()              # zero-width region
    assert r["matrix"].shape == (0, 18)
    allbad = dict(rec)
    allbad["mapq"] = np.zeros_like(rec["mapq"])
    r = counter.count(allbad, 1000, 1300, ref, rs, min_mq=5).fetch()
    assert r["matrix"].shape == (0, 18)
    far = counter.count(rec, 500000, 500300, ref, rs).fetch()        # region nobody covers
    assert far["matrix"].shape == (0, 18)
    _compare("after_empty_calls", counter.count(rec, 1000, 1300, ref, rs).fetch(), po.clair3_pileup(rec, 1000, 1300, ref, rs))


def test_device_resident_records_and_chained_forward(counter):
    """Records already in HBM (on_device = 1) give the same counts, and Clair3_P over the candidates' windows straight from the
    device-resident matrix equals the forward over host-sliced [33, 18] tensors of the oracle's matrix
    (preprocess/CreateTensorPileupFromCffi.py:357-369)."""
    import torch
    from clair3_b200 import pileup_counts as pc, synth, synth_reads as sr
    from clair3_b200.model import Clair3_P
    from oracle import pileup_oracle as po
    rec, ref, rs = sr.random_alignment(3000, depth=25, read_len=800, seed=21)
    want = po.clair3_pileup(rec, 1000, 4000, ref, rs)
    dev = torch.device("cuda:0")
    drec = pc.BamRecords.from_dict(rec).to_device(dev, ref)
    got = counter.count(drec, 1000, 4000, None, rs).fetch()
    _compare("device_records", got, want)
    sd = synth.pileup_state_dict(False, seed=3)
    m = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    m.to(dev)
    m.eval()
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    y, ok = counter.forward(m)
    torch.cuda.synchronize()
    y = y.cpu().numpy()
    assert np.array_equal(ok, want["cand_ok"]) and ok.sum() > 5
    sel = np.nonzero(ok)[0]
    x = np.stack([want["matrix"][c - 16:c + 17] for c in want["cand_cols"][sel]]).astype(np.int32)
    yref = m(torch.from_numpy(x).to(dev)).cpu().numpy()
    assert float(np.abs(y[sel] - yref).max()) < 1e-5            # same kernels, same per-site arithmetic (cf. test_forward_windows_equals_host_sliced_tensors)
    _STATS["chained_forward"] = {"candidates": int(len(ok)), "complete_windows": int(ok.sum()), "identical_to_host_sliced_forward": True}
    _dump()


def test_additivity_at_bench_size(counter):
    """The bench region (1,048,576 columns, depth 40) is too large for the oracle to be the comparison of record in a test, so the
    full size is checked through a size-independent property: linearity of the counts in the set of reads (see
    tests/test_pileup_oracle.py::check_additivity), plus the oracle itself on a 32,768-column window of the same call."""
    from clair3_b200 import synth_reads as sr
    from oracle import pileup_oracle as po
    from test_pileup_oracle import check_additivity
    region, origin = 1 << 20, 10000
    rec, ref, rs = sr.random_alignment(region, depth=40, read_len=8000, seed=5, indel_rate=0.04, origin=origin, n_rate=0.0,
                                       filtered_frac=0.0)
    rec["mapq"][:] = 60
    n = check_additivity(lambda r: counter.count(r, origin, origin + region, ref, rs).fetch(), rec, origin, origin + region, ref, rs)
    whole = counter.count(rec, origin, origin + region, ref, rs).fetch()
    want = po.clair3_pileup(rec, origin, origin + 32768, ref, rs)
    k = len(want["major"]) - 40            # the window's last columns see no right-hand neighbours in the oracle's shorter region
    assert np.array_equal(whole["major"][:k], want["major"][:k]) and np.array_equal(whole["matrix"][:k], want["matrix"][:k])
    assert np.array_equal(whole["stats"][:k, :5], want["stats"][:k, :5])
    _STATS["additivity_1M"] = {"columns_compared": n, "linear_features_additive": True, "oracle_window_columns": int(k)}
    _dump()


@pytest.mark.parametrize("seed", range(4))
def test_all_alt_info_text(counter, seed):
    """calculate_clair3_pileup's all_alt_info strings (src/clair3_pileup.c:391-450): allele lists exported by the count kernel,
    text formatted on the host - byte for byte the oracle's text, insertion alleles in khash bucket order."""
    from clair3_b200 import synth_reads as sr
    from oracle import pileup_oracle as po
    rec, ref, rs = sr.random_alignment([700, 3000, 513, 20000][seed], depth=[15, 40, 300, 30][seed], read_len=[100, 600, 300, 3000][seed],
                                       seed=60 + seed, wild=seed == 0, indel_rate=[0.08, 0.06, 0.12, 0.05][seed], n_rate=0.01)
    width = [700, 3000, 513, 20000][seed]
    max_indel = [50, 5, 50, 50][seed]
    kw = dict(call_ht=seed == 0, gvcf=seed == 1)
    want = po.clair3_pileup(rec, 1000, 1000 + width, ref, rs, alt_info=True, max_indel_length=max_indel, **kw)
    got = counter.count(rec, 1000, 1000 + width, ref, rs, alt_info=True, max_indel_length=max_indel, **kw).fetch()
    _compare("alt_info_%d" % seed, got, want, gvcf=kw["gvcf"])
    text = counter.alt_info_strings(got)
    assert len(text) == len(want["alt_info"]) == len(want["cand_cols"])
    for a, b in zip(text, want["alt_info"]):
        assert a == b, (a, b)
    _STATS["alt_info_%d" % seed]["alt_info_strings_identical"] = len(text)
    _dump()


def test_pileup_counts_clair3_shape_of_the_reference_caller(counter):
    """pileup_counts_clair3 (preprocess/CreateTensorPileupFromCffi.py:30-85): contiguous chunks, candidate tuples, gVCF arrays."""
    from clair3_b200 import pileup_counts as pc, synth_reads as sr
    from oracle import pileup_oracle as po
    rec, ref, rs = sr.random_alignment(900, depth=8, read_len=120, seed=17, gaps=[(1300, 1420), (1700, 1760)])
    want = po.clair3_pileup(rec, 1000, 1900, ref, rs, alt_info=True, gvcf=True)
    chunks, tuples, gv = pc.pileup_counts_clair3(rec, "chr20", 1000, 1900, ref, rs, counter=counter, gvcf=True)
    assert np.array_equal(np.concatenate([c for c, _ in chunks]), want["matrix"])
    assert np.array_equal(np.concatenate([p["major"] for _, p in chunks]), want["major"]) and len(chunks) >= 3
    assert tuples == pc.alt_info_list(want["alt_info"], "chr20") and len(tuples) > 0
    assert np.array_equal(gv[0], want["pos_ref_count"]) and np.array_equal(gv[1], want["pos_total_count"])

