"""The BED / known-sites layer on the host (clair3_b200/targets.py, the chunk helpers of pileup_counts.py, cascade's
``qual_cutoffs(genotyping=True)``, ``add_back_missing`` and ``contig_targets``) against tests/golden/targets_cases.npz, minted
from the reference's own CheckEnvs, interval tree, chunk arithmetic, SelectQual and AddBackMissingVariantsInGenotyping
(tests/golden/make_targets_golden.py)."""
import gzip
import json
import os

import numpy as np
import pytest

from clair3_b200 import cascade, targets
from clair3_b200._ffi import C3BError
from clair3_b200.pileup_counts import bed_chunk_region, known_sites_chunk

import cascade_cases as cc

G = json.loads(str(np.load(os.path.join(os.path.dirname(__file__), "golden", "targets_cases.npz"))["cases"]))
PROBE = np.arange(1, 1401)


def _source(case, tmp_path, name):
    """The case's file, written the way the golden maker handed it to the reference (gzip or plain)."""
    p = tmp_path / (name + (".gz" if case["gzip"] else ""))
    p.write_bytes(gzip.compress(case["text"].encode()) if case["gzip"] else case["text"].encode())
    return str(p)


def _bits(hexstr):
    return np.unpackbits(np.frombuffer(bytes.fromhex(hexstr), np.uint8))[:len(PROBE)].astype(bool)


@pytest.mark.parametrize("name", sorted(G["bed"]))
def test_bed_cases(name, tmp_path):
    case = G["bed"][name]
    path = _source(case, tmp_path, name + ".bed")
    if case["refused"]:
        with pytest.raises(ValueError, match="invalid BED"):
            targets.read_bed(path)
        return
    t = targets.read_bed(path)
    assert sorted(t.contigs()) == sorted(case["contigs"])
    for ctg, want in case["contigs"].items():
        s, e = t.intervals[ctg]
        assert s.tolist() == want["starts"] and e.tolist() == want["ends"]
        ct = t.contig(ctg)
        assert list(ct.bed_region()) == want["bed_region"]
        assert np.array_equal(ct.keep(PROBE), _bits(want["keep"]))
        for key, region in want["chunks"].items():
            cid, n = (int(x) for x in key.split("/"))
            assert list(bed_chunk_region(*ct.bed_region(), cid, n)) == region
    # the arrays the device test reads: sorted by start, running maximum of the ends
    ct = t.contig(sorted(case["contigs"])[0])
    assert np.all(np.diff(ct.starts) >= 0) and np.array_equal(ct.end_max, np.maximum.accumulate(ct.ends))


@pytest.mark.parametrize("name", sorted(G["vcf"]))
def test_vcf_cases(name, tmp_path):
    case = G["vcf"][name]
    path = _source(case, tmp_path, name + ".vcf")
    if case["refused"]:
        with pytest.raises(ValueError, match="invalid VCF"):
            targets.read_vcf(path)
        return
    t = targets.read_vcf(path)
    assert sorted(t.contigs()) == sorted(case["contigs"])
    kept_by_neighbour = 0
    for ctg, want in case["contigs"].items():
        s, e = t.intervals.get(ctg, (np.zeros(0, np.int64),) * 2)
        assert s.tolist() == want["starts"] and e.tolist() == want["ends"]
        assert t.sites[ctg].tolist() == want["known"]
        for key, ch in want["chunks"].items():
            cid, n = (int(x) for x in key.split("/"))
            c = known_sites_chunk(t.sites[ctg], cid, n)
            if ch["range"] is None:
                assert c is None
            else:
                assert [c[0], c[1]] == ch["range"] and c[2].tolist() == ch["sites"]
            ct = t.contig(ctg, chunk=(cid, n))
            got = ct.keep(PROBE)
            assert np.array_equal(got, _bits(ch["keep"])), key
            assert ct.known.tolist() == ch["sites"]
            kept_by_neighbour += int(sum(got[p - 1] for p in ch["sites"] if p <= 33))
    if name == "mixed":
        assert kept_by_neighbour > 0, "a site at pos <= 33 must be kept through a neighbour's interval"


def test_chunk_ids_are_checked():
    for fn, args in ((bed_chunk_region, (0, 100)), (known_sites_chunk, ([1, 2, 3],))):
        for cid in (0, 4):
            with pytest.raises(C3BError, match="chunk_id"):
                fn(*args, cid, 3)


def test_contents_and_paths_agree(tmp_path):
    case = G["bed"]["mixed"]
    a = targets.read_bed(case["text"]).contig("ctg1")
    b = targets.read_bed(_source(case, tmp_path, "m.bed")).contig("ctg1")
    assert np.array_equal(a.starts, b.starts) and np.array_equal(a.end_max, b.end_max)
    empty = targets.read_bed(case["text"]).contig("absent")
    assert empty.bed_region() is None and not empty.keep(PROBE).any()


@pytest.mark.parametrize("q", G["qual"], ids=lambda q: "%s-%s" % (q["case"], q["ref_pct"]))
def test_qual_cutoffs_genotyping(q):
    platform, pileup, _ = cc.case(q["case"])
    var_q, ref_q = cascade.qual_cutoffs([pileup], platform, var_pct_full=q["var_pct"], ref_pct_full=q["ref_pct"], genotyping=True)
    assert str(var_q) + " " + str(ref_q) == q["qual"]


def test_qual_cutoffs_genotyping_only_changes_zero_ref_pct():
    platform, pileup, _ = cc.case("ont")
    assert cascade.qual_cutoffs([pileup], platform, genotyping=True) == cascade.qual_cutoffs([pileup], platform)
    assert (cascade.qual_cutoffs([pileup], platform, ref_pct_full=0.0) ==
            cascade.qual_cutoffs([pileup], platform, ref_pct_full=cascade.PCT_FULL[platform][0]))


@pytest.mark.parametrize("case", G["addback"], ids=lambda c: c["name"])
def test_add_back_missing(case):
    assert cascade.add_back_missing(case["body"], targets.read_vcf(case["known"])) == case["out"]


def test_add_back_missing_in_a_region():
    case = G["addback"][0]
    known = targets.read_vcf(case["known"])
    whole = cascade.add_back_missing(case["body"], known)
    part = cascade.add_back_missing(case["body"], known.contig("ctg1"), region=("ctg1", 0, 400))
    assert part == "".join(r for r in whole.splitlines(keepends=True) if r.split("\t")[0] == "ctg1" and int(r.split("\t")[1]) <= 400)
    assert part.count("\n") == 4


def test_bed_with_known_sites_is_refused():
    bed, vcf = targets.read_bed(G["bed"]["mixed"]["text"]), targets.read_vcf(G["vcf"]["sparse"]["text"])
    with pytest.raises(ValueError, match="either bed or known_sites"):
        cascade.contig_targets("ctg1", bed=bed, known_sites=vcf)
    with pytest.raises(ValueError, match="needs"):
        cascade.contig_targets("ctg1", bed=vcf)
    assert cascade.contig_targets("ctg1") is None
    assert cascade.contig_targets("ctg1", known_sites=vcf).known.tolist() == [50, 60, 700]
