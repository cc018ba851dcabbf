"""The phasing statement (clair3_b200/phasing.py) against independent references at full width (tests/phase_refs.py): its
optimum equals a DP over unnormalised states on every layout, and exhaustive enumeration where a block has at most 20 reads,
and its haplotypes reach that optimum - on blocks with 15 active reads, on layouts shaped to the GPU kernel's edges (segment
edges, 14 reads leaving at once, the parity of the backtrace, one-read columns, ties, thousands of blocks) and on wide random
layouts.  Then the observations (``phasing.fragments``) pinned on crafted records at the CIGAR and record edges, and every
crafted contig read back from its BAM as written (tests/phase_records.py)."""
import numpy as np
import pytest

from clair3_b200 import bam_io, phasing
from phase_cases import random_fragments
from phase_records import CASES, FLAG_BITS, Case, Read
from phase_refs import SHAPED, assert_shape, brute_force, full_state_dp, hap_cost, shaped_case, shaped_fragments

BRUTE_MAX_READS = 20


def _check(frag, lay):
    """The statement's cost equals full_state_dp per block (and brute force on blocks of at most 20 reads); its haplotypes reach
    that cost.  Returns the number of blocks brute force checked."""
    hap, cost = phasing.solve(lay)
    want = np.array([full_state_dp(lay, b) for b in range(lay.n_blocks)], np.int64)
    assert np.array_equal(cost, want), np.flatnonzero(cost != want)[:10]
    assert np.array_equal(hap_cost(frag, lay, hap), cost)
    assert (hap[lay.blk_col_off[:-1]] == 0).all()
    n = 0
    for b in range(lay.n_blocks):
        if lay.blk_read_off[b + 1] - lay.blk_read_off[b] <= BRUTE_MAX_READS:
            assert brute_force(lay, b) == cost[b], b
            n += 1
    return n


def _kmax15_block(seed):
    """One block of 15 to 20 reads over 8 columns, 15 of them active at column 4, some reads missing inner entries."""
    rng = np.random.default_rng(seed)
    while True:
        n = int(rng.integers(15, BRUTE_MAX_READS + 1))
        spans = [(int(rng.integers(0, 4)), int(rng.integers(4, 8))) for _ in range(15)]
        spans += [(0, int(rng.integers(1, 3))) if rng.random() < 0.5 else (int(rng.integers(5, 7)), 7) for _ in range(n - 15)]
        reads = []
        for a, b in spans:
            vs = np.arange(a, b + 1)
            vs = vs[(rng.random(len(vs)) > 0.25) | (vs == a) | (vs == b)]
            reads.append((vs, rng.integers(0, 2, len(vs)), rng.integers(1, 41, len(vs))))
        try:
            frag, lay = shaped_fragments(reads)
        except AssertionError:            # a column over the cap: the selection left a read out
            continue
        if lay.n_blocks == 1:
            return frag, lay


@pytest.mark.parametrize("seed", range(12))
def test_kmax15_blocks_equal_enumeration(seed):
    frag, lay = _kmax15_block(seed)
    plan = phasing.column_plan(lay, 0)
    assert lay.blk_kmax[0] == 15 and max(p[0] for p in plan) == 15 and 15 <= len(lay.read_id) <= BRUTE_MAX_READS
    assert _check(frag, lay) == 1


@pytest.mark.parametrize("name", SHAPED)
def test_shaped_layouts(name):
    frag, lay, expect = shaped_case(name)
    assert_shape(lay, expect)
    n = _check(frag, lay)
    if name == "many":
        assert n >= 2000
        m, slot = np.diff(lay.blk_col_off), 1 << (lay.blk_kmax.astype(np.int64) - 1)
        assert len(np.unique(m * slot)) < lay.n_blocks - 1000          # blocks of equal size: ties in the largest-first order
        assert len(np.unique(lay.blk_kmax)) >= 5


@pytest.mark.parametrize("seed", range(20))
def test_wide_random_layouts(seed):
    rng = np.random.default_rng(1000 + seed)
    frag = random_fragments(1000 + seed, 400, 700, max_span=int(rng.integers(30, 60)))
    lay = phasing.layout(frag, 700)
    ks = [p[0] for b in range(lay.n_blocks) for p in phasing.column_plan(lay, b)]
    assert max(ks) == phasing.MAX_COVERAGE
    _check(frag, lay)


def test_tie_rules_pinned():
    # every weight 0: every state costs 0, so the lowest leaving pattern, the lowest final state and allele 0 to part 0 make
    # haplotype 0 all 0 - whatever parity flips the backtrace crosses
    frag, lay, expect = shaped_case("tie_w0")
    assert any(x.get("flip") for x in expect)
    hap, cost = phasing.solve(lay)
    assert cost.tolist() == [0] and not hap.any()
    # every read agreeing: cost 0, and haplotype 0 is allele 0 wherever every read shows 0 (part 0 holds every read)
    frag, lay, _ = shaped_case("tie_agree")
    hap, cost = phasing.solve(lay)
    col_allele = np.zeros(len(lay.col_var), np.uint8)
    col_allele[frag.var - frag.var.min()] = frag.allele
    assert cost.tolist() == [0] and np.array_equal(hap, col_allele ^ col_allele[0])


# ---------------------------------------------------------------------------------------------- the observations
def test_fragments_at_record_edges():
    """Hand-computed entries: each read shows allele (variant + hap) % 2 where not overridden."""
    var = [10, 19, 20, 27, 28, 30, 35, 37, 40, 43, 46, 52]
    N, R = 15, 5
    reads = [Read(10, "10M3I8=2D6X4N1M5D7M", qual=30),                  # D over 28 and 43, N over 37
             Read(10, "5H10M2P10=1P23X5H", mapq=255, qual=31, hap=1),   # H / P inside, = then X to the end
             Read(10, "43M", mapq=19),                                   # MAPQ 19: dropped
             Read(10, "43M", mapq=20, flag=0x1, qual=0, bases={0: N, 1: R}),   # kept; N and R: no entry
             Read(10, "43M", flag=0x800),                                # supplementary: dropped
             Read(25, "3I0M20M0D5X", qual=93, lq=20),                    # leading I, zero-length ops, sequence cut at 20
             Read(30, "8M", qual=0xFF)]
    c = Case(60, var, reads)
    f = phasing.fragments(c.rec, phasing.het_snvs(c.rows))
    want = ([(0, v, v % 2, 30) for v in (0, 1, 2, 3, 5, 6, 8, 10, 11)] + [(1, v, (v + 1) % 2, 31) for v in range(12)]
            + [(3, v, v % 2, 0) for v in range(2, 12)] + [(5, v, v % 2, 93) for v in range(3, 9)]
            + [(6, v, v % 2, 255) for v in (5, 6, 7)])
    got = list(zip(f.read.tolist(), f.var.tolist(), f.allele.tolist(), f.weight.tolist()))
    assert got == want


def test_fragments_flags_and_counts():
    c = CASES["flags"]()
    f = phasing.fragments(c.rec, phasing.het_snvs(c.rows))
    kept = set(np.unique(f.read).tolist())
    flag, mapq = c.rec["flag"], c.rec["mapq"]
    for r in range(len(flag)):
        drop = bool(flag[r] & phasing.FLAG_SKIP) or mapq[r] < 20
        assert (r in kept) != drop, (r, int(flag[r]), int(mapq[r]))
    assert sorted(int(flag[r]) for r in kept if flag[r]) == [b for b in FLAG_BITS if not b & phasing.FLAG_SKIP]
    assert sorted(int(mapq[r]) for r in kept if mapq[r] != 60) == [20, 255]
    c = CASES["few"]()
    f = phasing.fragments(c.rec, phasing.het_snvs(c.rows))
    # the 10M read covers one variant, the 10M5D8M read shows N at its second: both dropped; the 20M reads keep two entries
    assert f.read.tolist() == [1, 1, 2, 2, 3, 3, 5, 5] and f.var.tolist() == [0, 1, 0, 1, 2, 3, 2, 3]


@pytest.mark.parametrize("name", sorted(CASES))
def test_record_cases_read_back(tmp_path, name):
    """Each crafted contig through write_bam / read_bam gives the observations of its records in memory, and phases."""
    c = CASES[name]()
    bam = str(tmp_path / "c.bam")
    bam_io.write_bam(bam, c.rec, [(c.ctg, c.length)])
    back = bam_io.read_bam(bam, c.ctg, fa_fields=True)[0]
    v = phasing.het_snvs(c.rows)
    a, b = phasing.fragments(c.rec, v), phasing.fragments(back, v)
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and np.array_equal(x, y)
    assert len(a.read) and phasing.layout(a, len(v.pos)).n_blocks > 0
    if name == "ciglen":
        n_ops = np.diff(back["cigar_off"])
        assert n_ops.max() > 65535 and {31, 32, 33, 64, 65} <= set(n_ops.tolist())
