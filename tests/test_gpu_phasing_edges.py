"""The GPU phasing DP and observations (csrc/phase.cu via clair3_b200/phase_gpu.py) at their edges, exactly equal to the
statement (clair3_b200/phasing.py) and, for the DP, to the independent references of tests/phase_refs.py.

* The DP on the shaped layouts: block lengths around the 128-column backtrace segments with k changing across the edges,
  columns where 14 of 15 reads leave, the parity flip of the backtrace, one-read columns, tie-heavy weights and ~2,000 blocks,
  on one CTA, three and one per SM.  Layouts the kernel must refuse by itself name their block, and the next solve is right.
* The observations on crafted records (tests/phase_records.py): every CIGAR operation, zero-length operations, 31 to 65
  operations and one CIGAR past 65,535 through the CG tag, qualities 0 / 1 / 93 / 0xFF, N and IUPAC bases, a CIGAR past its
  sequence, MAPQ and each FLAG bit, one- and two-entry reads, and variants and reads at contig and span edges."""
import numpy as np
import pytest
import torch

from clair3_b200 import bam_io, phase_gpu, phasing
from clair3_b200._ffi import C3BError
from clair3_b200.bam_decode import BamDecoder
from phase_records import CASES
from phase_refs import SHAPED, assert_shape, full_state_dp, hap_cost, profile_spans, shaped_case, shaped_fragments

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _solve_all_ways(frag, lay):
    want = phasing.solve(lay)
    ref = np.array([full_state_dp(lay, b) for b in range(lay.n_blocks)], np.int64)
    assert np.array_equal(want[1], ref)
    for n_ctas in (1, 3, None):
        hap, cost = phase_gpu.solve(lay, DEV, n_ctas=n_ctas)
        assert np.array_equal(hap, want[0]), (n_ctas, np.flatnonzero(hap != want[0])[:10])
        assert np.array_equal(cost, want[1]), (n_ctas, np.flatnonzero(cost != want[1])[:10])
        assert np.array_equal(hap_cost(frag, lay, hap), cost)


@pytest.mark.parametrize("name", SHAPED)
def test_dp_shaped_layouts(name):
    frag, lay, expect = shaped_case(name)
    assert_shape(lay, expect)
    _solve_all_ways(frag, lay)


# ---------------------------------------------------------------------------------------------- layouts the kernel refuses
def _three_blocks():
    """Blocks of 10, 40 and 12 columns; the middle one has 15 active reads over its last three columns."""
    rng = np.random.default_rng(7)
    reads, col = [], 0
    for m, kw in ((10, dict(hi=6)), (40, dict(pin={37: 15, 38: 15, 39: 15})), (12, dict(hi=6))):
        spans, _ = profile_spans(m, rng, **kw)
        reads += [(np.arange(a, b + 1) + col, rng.integers(0, 2, b - a + 1), rng.integers(1, 41, b - a + 1)) for a, b in spans]
        col += m
    frag, lay = shaped_fragments(reads)
    assert lay.n_blocks == 3 and np.diff(lay.blk_col_off).tolist() == [10, 40, 12] and lay.blk_kmax[1] == 15
    return frag, lay


def _sixteenth_read(lay):
    """Block 1 gets a read entering with its last-entering read, where 15 are already active."""
    r1 = int(lay.blk_read_off[2])
    f = int(lay.read_first[r1 - 1])
    assert phasing.column_plan(lay, 1)[f][0] == 15
    ins = lambda a, x: np.insert(a, r1, x).astype(a.dtype)     # noqa: E731
    off = lay.blk_read_off.copy()
    off[2:] += 1
    return lay._replace(blk_read_off=off, read_id=ins(lay.read_id, lay.read_id.max() + 1), read_first=ins(lay.read_first, f),
                        read_last=ins(lay.read_last, int(np.diff(lay.blk_col_off)[1]) - 1)), 1


def _no_shared_read(lay):
    """Blocks 0 and 1 as one block: its column 10 shares no read with column 9."""
    m0, n0 = int(lay.blk_col_off[1]), int(lay.blk_read_off[1])
    first, last = lay.read_first.copy(), lay.read_last.copy()
    r1 = int(lay.blk_read_off[2])
    first[n0:r1] += m0
    last[n0:r1] += m0
    ent = lay.ent_read.copy()
    e0, e1 = lay.col_ent_off[m0], lay.col_ent_off[lay.blk_col_off[2]]
    ent[e0:e1] += n0
    return lay._replace(blk_col_off=np.delete(lay.blk_col_off, 1), blk_read_off=np.delete(lay.blk_read_off, 1),
                        blk_kmax=np.array([lay.blk_kmax[:2].max(), lay.blk_kmax[2]], lay.blk_kmax.dtype), read_first=first,
                        read_last=last, ent_read=ent), 0


def _inactive_entry(lay):
    """An entry of block 2 moved to a read of the block that is not active at its column."""
    c0, r0, r1 = int(lay.blk_col_off[2]), int(lay.blk_read_off[2]), int(lay.blk_read_off[3])
    first, last = lay.read_first[r0:r1], lay.read_last[r0:r1]
    for j in range(int(lay.blk_col_off[3]) - c0):
        off = np.flatnonzero((first > j) | (last < j))
        if len(off) and lay.col_ent_off[c0 + j + 1] > lay.col_ent_off[c0 + j]:
            ent = lay.ent_read.copy()
            ent[lay.col_ent_off[c0 + j]] = off[0]
            return lay._replace(ent_read=ent), 2
    raise AssertionError("no column of block 2 leaves a read inactive")


def _k_over_kmax(lay):
    """Block 1 claims at most 14 active reads; it has 15."""
    kmax = lay.blk_kmax.copy()
    kmax[1] -= 1
    return lay._replace(blk_kmax=kmax), 1


@pytest.mark.parametrize("breach", [_sixteenth_read, _no_shared_read, _inactive_entry, _k_over_kmax])
def test_dp_refuses_a_broken_layout(breach):
    frag, lay = _three_blocks()
    bad, b = breach(lay)
    for n_ctas in (1, None):
        with pytest.raises(C3BError, match=r"block %d breaks" % b):
            phase_gpu.solve(bad, DEV, n_ctas=n_ctas)
    want = phasing.solve(lay)
    hap, cost = phase_gpu.solve(lay, DEV)
    assert np.array_equal(hap, want[0]) and np.array_equal(cost, want[1])


# ---------------------------------------------------------------------------------------------- the observations
@pytest.fixture(scope="module")
def decoder():
    d = BamDecoder(0)
    yield d
    d.close()


def _same(a, b):
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and np.array_equal(x, y)


@pytest.mark.parametrize("name", sorted(CASES))
def test_observations_at_record_edges(decoder, tmp_path, name):
    c = CASES[name]()
    bam = str(tmp_path / "c.bam")
    bam_io.write_bam(bam, c.rec, [(c.ctg, c.length)])
    bam_io.write_bai(bam)
    rec = bam_io.read_bam(bam, c.ctg, fa_fields=True)[0]
    v = phasing.het_snvs(c.rows)
    want = phasing.phase_contig(c.rows, rec)
    assert len(want[2].read) and want[3].n_blocks > 0
    ends = rec["pos"] + np.array([sum(int(w >> 4) for w in rec["cigar"][a:b] if (w & 15) in (0, 2, 3, 7, 8))
                                  for a, b in zip(rec["cigar_off"][:-1], rec["cigar_off"][1:])])
    for span in c.spans:
        _same(phase_gpu.contig_fragments(decoder, bam, c.ctg, c.length, v, span), want[2])
        got = phase_gpu.phase_contig(decoder, bam, c.ctg, c.length, c.rows, span)
        assert got[0] == want[0]
        _same(got[3], want[3])
        assert np.array_equal(got[4], want[4]) and np.array_equal(got[5], want[5])
    if name == "span":
        assert (rec["pos"] // 500 + 2 <= (ends - 1) // 500).any()                 # a read over three spans of 500
        assert ((rec["pos"] % 500 == 0) & (rec["pos"] > 0)).sum() >= 3             # reads starting on a span edge
        assert v.pos[0] == 0 and v.pos[-1] == c.length - 1
    if name == "last_span":
        assert all((rec["pos"] >= range(0, c.length, span)[-1]).all() for span in c.spans)    # every read in the last span
    if name == "ciglen":
        assert np.diff(rec["cigar_off"]).max() > 65535
