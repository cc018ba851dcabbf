"""The phasing statement (clair3_b200/phasing.py) on the host: the DP's optimum against exhaustive enumeration of the read
bipartitions, the coverage cap of the read selection, the blocks, PS and the first variant's ``0|1``, the rows it leaves alone,
the header line, and the true phase of a synthetic diploid contig."""
import numpy as np
import pytest

from clair3_b200 import genome, phasing
from phase_cases import diploid_contig, random_fragments
from phase_refs import hap_cost


def _brute_force(frag, admitted):
    """The least all-heterozygous cost over every bipartition of the admitted reads."""
    keep = np.isin(frag.read, admitted)
    read, var, al, w = (a[keep] for a in frag)
    idx = np.searchsorted(admitted, read)
    vars_ = np.unique(var)
    best = None
    for mask in range(1 << max(len(admitted) - 1, 0)):
        part = (mask << 1 >> idx) & 1                       # the first read fixed in part 0
        total = 0
        for v in vars_:
            s = var == v
            o1 = int((w[s].astype(np.int64) * ((part[s] ^ al[s]) & 1)).sum())
            total += min(o1, int(w[s].astype(np.int64).sum()) - o1)
        best = total if best is None else min(best, total)
    return best


@pytest.mark.parametrize("seed", range(60))
def test_dp_optimum_equals_enumeration(seed):
    rng = np.random.default_rng(seed)
    frag = random_fragments(seed, int(rng.integers(2, 11)), int(rng.integers(2, 9)), max_span=int(rng.integers(2, 9)))
    n_var = int(frag.var.max()) + 1 if len(frag.var) else 0
    lay = phasing.layout(frag, n_var)
    hap, cost = phasing.solve(lay)
    admitted = np.sort(lay.read_id)
    assert int(cost.sum()) == _brute_force(frag, admitted)
    assert np.array_equal(hap_cost(frag, lay, hap), cost)
    for b in range(lay.n_blocks):
        assert hap[lay.blk_col_off[b]] == 0


@pytest.mark.parametrize("seed", range(8))
def test_selection_keeps_coverage_at_most_15(seed):
    frag = random_fragments(100 + seed, 300, 60, max_span=25)
    admitted, cov = phasing.select_reads(frag, 60)
    assert cov.max() <= phasing.MAX_COVERAGE
    again = np.zeros(60, np.int64)
    for r in admitted:
        v = frag.var[frag.read == r]
        again[v.min():v.max() + 1] += 1
    assert np.array_equal(again, cov)
    # greedy: every rejected read would push some variant of its range past the cap
    for r in np.setdiff1d(np.unique(frag.read), admitted):
        v = frag.var[frag.read == r]
        assert cov[v.min():v.max() + 1].max() == phasing.MAX_COVERAGE
    lay = phasing.layout(frag, 60)
    assert lay.blk_kmax.max() <= phasing.MAX_COVERAGE
    phasing.solve(lay)


def test_selection_order():
    # read 1 has more entries; reads 0 and 2 tie on entries, 2 weighs more; with a cap of 2 read 0 is left out
    frag = phasing.Fragments(np.array([0, 0, 1, 1, 1, 2, 2]), np.array([0, 1, 0, 1, 2, 0, 1], np.int32),
                             np.zeros(7, np.uint8), np.array([5, 5, 1, 1, 1, 9, 9], np.uint8))
    admitted, cov = phasing.select_reads(frag, 3, cap=2)
    assert admitted.tolist() == [1, 2] and cov.tolist() == [2, 2, 1]


def _components(frag, admitted, n_var):
    adj = {v: set() for v in range(n_var)}
    for r in admitted:
        v = frag.var[frag.read == r].tolist()
        for a, b in zip(v, v[1:]):
            adj[a].add(b)
            adj[b].add(a)
    seen, comps = set(), []
    for v in range(n_var):
        if v in seen or not adj[v]:
            continue
        stack, comp = [v], []
        seen.add(v)
        while stack:
            x = stack.pop()
            comp.append(x)
            for y in adj[x] - seen:
                seen.add(y)
                stack.append(y)
        comps.append(sorted(comp))
    return sorted(comps)


@pytest.mark.parametrize("seed", range(4))
def test_blocks_ps_and_first_variant(seed):
    rec, _, rows, truth = diploid_contig(seed, 30000, 12, 1500, het_rate=2e-3)
    out, v, frag, lay, hap, cost = phasing.phase_contig(rows, rec)
    assert lay.n_blocks > 0
    blocks = sorted(sorted(lay.col_var[a:b].tolist()) for a, b in zip(lay.blk_col_off[:-1], lay.blk_col_off[1:]))
    assert blocks == _components(frag, lay.read_id, len(v.pos))
    first = [int(lay.col_var[a]) for a in lay.blk_col_off[:-1]]
    assert first == sorted(first)
    phased = 0
    for b in range(lay.n_blocks):
        cols = lay.col_var[lay.blk_col_off[b]:lay.blk_col_off[b + 1]]
        ps = int(v.pos[cols.min()]) + 1
        for j, c in enumerate(cols):
            f = out[v.row[c]].rstrip("\n").split("\t")
            assert f[8].endswith(":PS") and f[9].split(":")[-1] == str(ps)
            gt = f[9].split(":")[0]
            assert gt in ("0|1", "1|0") and (j > 0 or gt == "0|1")
            phased += 1
    assert sum(r != o for r, o in zip(out, rows)) == phased


def test_rows_left_alone_are_byte_identical():
    rec, _, rows, _ = diploid_contig(7, 20000, 10, 1200, het_rate=2e-3)
    out, v, _, lay, _, _ = phasing.phase_contig(rows, rec)
    phased_rows = set(v.row[lay.col_var].tolist())
    assert len(out) == len(rows)
    others = [i for i in range(len(rows)) if i not in phased_rows]
    assert any("RefCall" in rows[i] for i in others) and any("1/1" in rows[i] for i in others)
    assert any(",".join([""]) in rows[i] and "1/2" in rows[i] for i in others)
    for i in others:
        assert out[i] == rows[i]
    for i in phased_rows:
        a, b = rows[i].split("\t"), out[i].split("\t")
        assert a[:8] == b[:8]
        assert b[8] == a[8] + ":PS"
        assert b[9].rstrip("\n").split(":")[1:-1] == a[9].rstrip("\n").split(":")[1:]


def test_variant_selection():
    rows = ["c\t10\t.\tA\tG\t3\tLowQual\tP\tGT:GQ\t0/1:3\n", "c\t11\t.\tA\tG\t3\tPASS\tP\tGT:GQ\t1/1:3\n",
            "c\t12\t.\tAC\tA\t3\tPASS\tP\tGT:GQ\t0/1:3\n", "c\t13\t.\tA\tG,T\t3\tPASS\tP\tGT:GQ\t1/2:3\n",
            "c\t14\t.\tN\tG\t3\tPASS\tP\tGT:GQ\t0/1:3\n", "c\t15\t.\tC\tT\t3\tPASS\tF\tGT:GQ\t0/1:3\n",
            "c\t16\t.\tC\t.\t3\tRefCall\tP\tGT:GQ\t0/0:3\n"]
    v = phasing.het_snvs(rows)
    assert v.row.tolist() == [0, 5] and v.pos.tolist() == [9, 14] and v.ref.tolist() == [1, 2] and v.alt.tolist() == [4, 8]


def test_header_line():
    head = genome._HEADER.format("x") + "\n##contig=<ID=chr1,length=10>\n#CHROM\tPOS"
    out = phasing.phase_header(head).split("\n")
    at = out.index(phasing.PS_HEADER)
    assert out[at - 1].startswith("##FORMAT=<ID=AF") and out[at + 1].startswith("##contig")
    assert [x for x in out if x != phasing.PS_HEADER] == head.split("\n")
    assert sum(x.startswith("##FORMAT") for x in out) == 7


def test_fragments_rules():
    # one read over three SNPs: REF, ALT, a third base (no entry); MAPQ 19, a duplicate and a one-entry read are dropped
    from clair3_b200.synth_reads import records_from_lists
    ref = "ACGTACGTAC"
    rows = ["c\t3\t.\tG\tT\t9\tPASS\tP\tGT\t0/1\n", "c\t5\t.\tA\tC\t9\tPASS\tP\tGT\t0/1\n", "c\t8\t.\tT\tG\t9\tPASS\tP\tGT\t0/1\n"]
    v = phasing.het_snvs(rows)
    items = [(0, 0, 60, [("S", 2), ("M", 3), ("I", 1), ("M", 3), ("D", 1), ("M", 3)], "TT" + "ACG" + "G" + "TCC" + "CAC"),
             (0, 0, 19, [("M", 10)], ref), (0, 1024, 60, [("M", 10)], ref), (4, 0, 60, [("M", 6)], "AAGCAC"),
             (2, 0, 60, [("M", 7)], "TTACGGA")]
    rec = records_from_lists(items)
    rec["qual"] = np.arange(int(rec["l_qseq"].sum()), dtype=np.uint8) % 50
    rec["qual_off"] = np.concatenate([[0], np.cumsum(rec["l_qseq"])]).astype(np.int64)
    f = phasing.fragments(rec, v)
    # sorted by pos: record 0 shows G at 2 (REF, query 4), C at 4 (ALT, query 7 past the insertion), C at 7 (neither T nor G);
    # record 3 (pos 2) shows T (ALT), A (REF) and G (ALT); record 4 (pos 4) shows A at 4 (REF) and C at 7 (neither): one entry, dropped
    assert f.read.tolist() == [0, 0, 3, 3, 3]
    assert f.var.tolist() == [0, 1, 0, 1, 2] and f.allele.tolist() == [0, 1, 1, 0, 1]
    q, o = rec["qual"], int(rec["qual_off"][3])
    assert f.weight.tolist() == [q[4], q[7], q[o], q[o + 2], q[o + 5]]


@pytest.mark.parametrize("seed", range(3))
def test_known_phase_of_a_diploid_contig(seed):
    rec, _, rows, truth = diploid_contig(20 + seed, 60000, 30, 3000)
    out, v, frag, lay, hap, cost = phasing.phase_contig(rows, rec)
    _check_truth(v, frag, lay, hap, truth)


def _check_truth(v, frag, lay, hap, truth):
    linked = np.unique(frag.var[np.isin(frag.read, lay.read_id)])
    assert np.array_equal(np.sort(lay.col_var), linked)
    for b in range(lay.n_blocks):
        cols = lay.col_var[lay.blk_col_off[b]:lay.blk_col_off[b + 1]]
        h = hap[lay.blk_col_off[b]:lay.blk_col_off[b + 1]]
        t = truth[cols]
        assert np.array_equal(h, t) or np.array_equal(h, 1 - t), "switch error in block %d" % b
