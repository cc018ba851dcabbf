"""Independent references for the phasing DP (clair3_b200/phasing.py's ``solve_block``) and deterministic layouts shaped to the
GPU kernel's edges.

* ``brute_force``: every bipartition of a block's reads, column by column, vectorised over the masks.
* ``full_state_dp``: a DP over unnormalised states - every bipartition of the active reads, both halves kept - whose
  projection matches the previous column's states to the current ones by the shared reads' identities.
* ``hap_cost``: the cost each block's haplotype pair achieves, each read taking its cheaper haplotype.

None of them shares code with ``solve_block``: no deposit, no normalised state, no prefix order of the shared reads.

``shaped_fragments`` places reads on explicit variant ranges; ``profile_spans`` finds read ranges whose active counts follow a
given profile; ``shaped_case`` builds the named layouts the DP tests run, each with the column shapes it claims
(``assert_shape`` reads them back from ``phasing.column_plan``).
"""
from __future__ import annotations

import numpy as np

from clair3_b200 import phasing

SEGMENT = 128      # include/clair3_b200_phase.h C3B_PHASE_SEGMENT: the DP's backtrace segment
_BIT = [((np.arange(1 << phasing.MAX_COVERAGE) >> i) & 1).astype(np.int64) for i in range(phasing.MAX_COVERAGE)]   # bit i of each state


def _block_entries(lay, b):
    """Per column of block b: (block-local reads, alleles, weights as int64)."""
    c0, c1 = lay.blk_col_off[b], lay.blk_col_off[b + 1]
    out = []
    for c in range(c0, c1):
        e = slice(lay.col_ent_off[c], lay.col_ent_off[c + 1])
        out.append((lay.ent_read[e].astype(np.int64), lay.ent_allele[e].astype(np.int32), lay.ent_weight[e].astype(np.int64)))
    return out


# ------------------------------------------------------------------------------------------------ the references
def brute_force(lay, b):
    """The least all-heterozygous cost of block b over every bipartition of its reads (read 0 fixed in part 0)."""
    n = int(lay.blk_read_off[b + 1] - lay.blk_read_off[b])
    assert n <= 21, "brute force over %d reads" % n
    masks = np.arange(1 << max(n - 1, 0), dtype=np.int64) << 1
    total = np.zeros(len(masks), np.int64)
    for reads, allele, weight in _block_entries(lay, b):
        o1 = np.zeros(len(masks), np.int64)
        for r, a, w in zip(reads.tolist(), allele.tolist(), weight.tolist()):
            if w:
                o1 += w * (((masks >> r) & 1) ^ a)
        total += np.minimum(o1, int(weight.sum()) - o1)
    return int(total.min())


def full_state_dp(lay, b):
    """The optimal cost of block b by a DP over all 2^k bipartitions of each column's active reads (both halves kept): a state
    is matched to the previous column's states that put every shared read in the same part, found by read identity."""
    r0, r1 = lay.blk_read_off[b], lay.blk_read_off[b + 1]
    first, last = lay.read_first[r0:r1], lay.read_last[r0:r1]
    D, prev = None, None
    for j, (reads, allele, weight) in enumerate(_block_entries(lay, b)):
        act = np.flatnonzero((first <= j) & (last >= j))
        k = len(act)
        assert 1 <= k <= phasing.MAX_COVERAGE
        at = np.full(r1 - r0, -1, np.int64)            # the bit of each active read in this column's states
        at[act] = np.arange(k)
        n = 1 << k
        assert (at[reads] >= 0).all()
        o1 = np.zeros(n, np.int64)
        for r, a, w in zip(reads.tolist(), allele.tolist(), weight.tolist()):
            o1 += w * (_BIT[at[r]][:n] ^ a)
        cost = np.minimum(o1, int(weight.sum()) - o1)
        if D is None:
            D, prev = cost, at
            continue
        shared = act[prev[act] >= 0]
        assert len(shared) > 0, "column %d shares no read with the one before" % j
        key_prev, key = np.zeros(len(D), np.int64), np.zeros(n, np.int64)
        for i, r in enumerate(shared.tolist()):
            key_prev |= _BIT[prev[r]][:len(D)] << i
            key |= _BIT[at[r]][:n] << i
        best = np.full(1 << len(shared), np.iinfo(np.int64).max, np.int64)
        np.minimum.at(best, key_prev, D)
        D, prev = cost + best[key], at
    return int(D.min())


def hap_cost(frag, lay, hap):
    """Per block, the cost the haplotype pair ``hap`` (haplotype 0's allele per column) achieves over the fragments of the
    block's reads: each read takes its cheaper haplotype."""
    if not lay.n_blocks:
        return np.zeros(0, np.int64)
    n_var = int(max(lay.col_var.max(), frag.var.max())) + 1
    allele = np.full(n_var, 255, np.int64)
    allele[lay.col_var] = hap
    blk = np.repeat(np.arange(lay.n_blocks), np.diff(lay.blk_read_off))
    keep = np.isin(frag.read, lay.read_id)
    read, var, al, w = frag.read[keep], frag.var[keep], frag.allele[keep].astype(np.int64), frag.weight[keep].astype(np.int64)
    assert (allele[var] < 2).all(), "an admitted read's entry at an unphased variant"
    r = np.searchsorted(np.sort(lay.read_id), read)
    mism, tot = np.zeros(len(lay.read_id), np.int64), np.zeros(len(lay.read_id), np.int64)
    np.add.at(mism, r, w * (al != allele[var]))
    np.add.at(tot, r, w)
    per_read = np.minimum(mism, tot - mism)
    out = np.zeros(lay.n_blocks, np.int64)
    np.add.at(out, blk[np.argsort(lay.read_id)], per_read)
    return out


# ------------------------------------------------------------------------------------------------ shaped layouts
def shaped_fragments(reads, n_var=None):
    """(fragments, layout) of reads given as (variant indices ascending, alleles, weights): read i's id is i.  Every read must
    be admitted, so each variant's range coverage stays at or under the cap."""
    out = [[], [], [], []]
    for i, (vs, al, w) in enumerate(reads):
        vs = np.asarray(vs, np.int64)
        out[0].append(np.full(len(vs), i, np.int64))
        out[1].append(vs.astype(np.int32))
        out[2].append(np.broadcast_to(np.asarray(al, np.uint8), vs.shape).copy())
        out[3].append(np.broadcast_to(np.asarray(w, np.uint8), vs.shape).copy())
    frag = phasing.Fragments(*(np.concatenate(a) for a in out))
    n_var = int(frag.var.max()) + 1 if n_var is None else n_var
    lay = phasing.layout(frag, n_var)
    assert len(lay.read_id) == len(reads), "the read selection left %d reads out" % (len(reads) - len(lay.read_id))
    return frag, lay


def profile_spans(m, rng, lo=2, hi=phasing.MAX_COVERAGE, pin=None, churn=None, oldest=(), newest=()):
    """(read [first, last] column ranges in the block's read order, active reads per column) of m columns.  Column j has
    ``pin[j]`` active reads if pinned, else a random count in [lo, hi] that the reads before it allow; the reads beyond it
    leave, plus ``churn.get(j, 1)`` more that new reads replace where a shared read stays.  Only reads active for two columns
    or more may leave, so the column before a pinned one holds its reads (no read leaves or enters there).  The leaving reads
    are the oldest at the columns in ``oldest`` (read 0 of the previous column among them), the newest at those in
    ``newest``, random elsewhere.  No read enters at the last column: every read has two entries or more."""
    pin, churn = pin or {}, churn or {}
    spans, active, ks = [], [], []
    for j in range(m):
        last = j == m - 1
        hold = j + 1 in pin and j not in pin
        go = []
        if j:
            can = [i for i in active if spans[i][0] <= j - 2]
            most = min(len(can), len(active) - 1)
            if j in pin:
                k = pin[j]
            elif hold:
                k = len(active)
            else:
                kmin = max(min(lo, len(active)), len(active) - most)
                k = int(rng.integers(kmin, (len(active) if last else max(hi, kmin)) + 1))
            need = max(0, len(active) - k)
            n_leave = min(need + churn.get(j, 0 if hold or last else 1), most)
            assert n_leave >= need, "column %d: %d reads must leave, %d can" % (j, need, most)
            if j in oldest:
                go = can[:n_leave]
            elif j in newest:
                go = can[len(can) - n_leave:]
            else:
                go = [active[i] for i in sorted(rng.choice([active.index(x) for x in can], n_leave, replace=False).tolist())]
            for i in go:
                spans[i][1] = j - 1
            active = [i for i in active if i not in go]
        else:
            k = pin.get(0, int(rng.integers(lo, hi + 1)))
        assert not last or len(active) >= k, "a read entering at the last column would have one entry"
        while len(active) < k:
            active.append(len(spans))
            spans.append([j, None])
        ks.append(len(active))
    for i in active:
        spans[i][1] = m - 1
    return [tuple(s) for s in spans], ks


def _entries(spans, col0, rng, alleles="random", weights="random"):
    """Shaped reads (every column of each span) at variant offset col0, with allele and weight schemes."""
    out = []
    for first, last in spans:
        vs = np.arange(first, last + 1) + col0
        n = len(vs)
        if alleles == "random":
            al = rng.integers(0, 2, n)
        elif alleles == "agree":
            al = (vs * 2654435761 >> 7) & 1                 # one allele per column for every read
        else:
            raise ValueError(alleles)
        if isinstance(weights, int):
            w = np.full(n, weights)
        elif weights == "random":
            w = rng.integers(1, 41, n)
        elif weights == "halfzero":                          # half the entries, and every third column whole, at weight 0
            w = np.where((rng.random(n) < 0.5) | (vs % 3 == 0), 0, rng.integers(1, 41, n))
        else:
            raise ValueError(weights)
        out.append((vs, al, w))
    return out


EDGE_PINS = {"15-15": {-1: 15, 0: 15}, "15-3": {-2: 14, -1: 15, 0: 3}, "3-15": {-1: 3, 0: 15}}


def _len_case(m, rng):
    """m columns; at the segment edges k goes 15 -> 15, 15 -> 3 or 3 -> 15 (the last losing the previous column's read 0)."""
    kinds = {129: ["15-15"], 255: ["15-3"], 256: ["3-15"], 257: ["15-15", "15-3"], 1000: ["15-15", "15-3", "3-15"] * 3}
    pin, oldest = {}, set()
    for i, x in enumerate(kinds.get(m, [])):
        e = SEGMENT * (i + 1)
        if e < m:
            pin.update({e + d: k for d, k in EDGE_PINS[x].items()})
            if x == "3-15":
                oldest.add(e)
    if m == 2:
        pin = {0: 15, 1: 15}
    if m == 128:
        pin = {126: 15, 127: 15}                             # the last column is the checkpoint column, and none is written
    spans, ks = profile_spans(m, rng, pin=pin, oldest=oldest)
    return spans, [dict(j=j, k=k) for j, k in sorted(pin.items())] + [dict(j=e, flip=True) for e in sorted(oldest)]


def _leave14_case(rng):
    """Columns where 14 of 15 reads leave and 14 enter around the one that stays: inside a segment and at segment edges, with
    the staying read the previous column's read 0 (newest leave) or its last (oldest leave)."""
    at = {60: "newest", 128: "oldest", 200: "oldest", 256: "newest"}
    pin = {}
    for j in at:
        pin.update({j - 2: 15, j - 1: 15, j: 15})
    spans, _ = profile_spans(300, rng, lo=8, pin=pin, churn={j: 14 for j in at} | {j - 1: 0 for j in at},
                             oldest={j for j, p in at.items() if p == "oldest"}, newest={j for j, p in at.items() if p == "newest"})
    return spans, [dict(j=j, k=15, ns=1, leave=14, flip=(p == "oldest")) for j, p in at.items()]


def _flip_case(rng):
    """Columns where read 0 of the previous column leaves, at segment edges and inside segments."""
    flips = [5, 6, 7, 127, 128, 129, 255, 256, 300]
    spans, _ = profile_spans(400, rng, lo=4, hi=14, churn={j: 2 for j in flips}, oldest=set(flips))
    return spans, [dict(j=j, flip=True) for j in flips]


def _k1_case(rng):
    """Columns with one active read inside a block: the read that links its two parts."""
    ones = [0, 1, 40, 41, 127, 128, 200]
    spans, _ = profile_spans(300, rng, lo=3, hi=12, pin={j: 1 for j in ones})
    return spans, [dict(j=j, k=1) for j in ones]


TIE_SCHEMES = {"w0": ("random", 0), "w1": ("random", 1), "w30": ("random", 30), "w255": ("random", 255),
               "agree": ("agree", "random"), "halfzero": ("random", "halfzero")}


def _many_case(rng):
    """About 2,000 blocks of two to five columns, then three long blocks with kmax 15, 9 and 4."""
    reads, col = [], 0
    for _ in range(2000):
        m = int(rng.integers(2, 6))
        reads.append((np.arange(col, col + m), rng.integers(0, 2, m), rng.integers(1, 41, m)))     # links the whole block
        for _ in range(int(rng.integers(0, 6))):
            a = int(rng.integers(0, m - 1))
            b = int(rng.integers(a + 1, m))
            vs = np.arange(col + a, col + b + 1)
            reads.append((vs, rng.integers(0, 2, len(vs)), rng.integers(1, 41, len(vs))))
        col += m
    long_blocks = []
    for m, kmax in ((300, 15), (400, 9), (260, 4)):
        spans, _ = profile_spans(m, rng, lo=max(kmax - 6, 2), hi=kmax, pin={m // 2: kmax})
        long_blocks.append((col, kmax))
        reads += _entries(spans, col, rng)
        col += m
    return reads, long_blocks


SHAPED = (["len%d" % m for m in (2, 127, 128, 129, 255, 256, 257, 1000)] + ["leave14", "flip", "k1"]
          + ["tie_" + t for t in TIE_SCHEMES] + ["many"])


def shaped_case(name):
    """(fragments, layout, expected shapes) of a named case: the shapes are dicts of block ``b`` (default 0), column ``j``
    and any of ``k``, ``ns``, ``leave`` (popcount of the leaving mask) and ``flip`` (read 0 of the previous column leaves)."""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name.startswith("len"):
        spans, expect = _len_case(int(name[3:]), rng)
        frag, lay = shaped_fragments(_entries(spans, 0, rng))
    elif name == "leave14":
        spans, expect = _leave14_case(rng)
        frag, lay = shaped_fragments(_entries(spans, 0, rng))
    elif name == "flip":
        spans, expect = _flip_case(rng)
        frag, lay = shaped_fragments(_entries(spans, 0, rng))
    elif name == "k1":
        spans, expect = _k1_case(rng)
        frag, lay = shaped_fragments(_entries(spans, 0, rng))
    elif name.startswith("tie_"):
        alleles, weights = TIE_SCHEMES[name[4:]]
        pin, flips = {127: 15, 128: 15, 255: 15, 256: 15}, set(range(3, 300, 11))
        spans, _ = profile_spans(300, rng, lo=12, pin=pin, churn={j: 3 for j in flips}, oldest=flips)
        frag, lay = shaped_fragments(_entries(spans, 0, rng, alleles, weights))
        expect = [dict(j=j, k=k) for j, k in pin.items()] + [dict(j=j, flip=True) for j in sorted(flips)]
    elif name == "many":
        reads, long_blocks = _many_case(rng)
        frag, lay = shaped_fragments(reads)
        assert lay.n_blocks == 2003
        starts = lay.col_var[lay.blk_col_off[:-1]]
        expect = []
        for col, kmax in long_blocks:
            b = int(np.flatnonzero(starts == col)[0])
            assert lay.blk_kmax[b] == kmax
            expect.append(dict(b=b, j=0))
    else:
        raise KeyError(name)
    return frag, lay, expect


def assert_shape(lay, expect):
    """Each expected column shape, read back from ``phasing.column_plan``."""
    plans = {}
    for x in expect:
        b = x.get("b", 0)
        if b not in plans:
            plans[b] = phasing.column_plan(lay, b)
        k, ns, sh, lv, _ = plans[b][x["j"]]
        got = dict(k=k, ns=ns, leave=bin(lv).count("1"), flip=bool(lv & 1))
        for key in ("k", "ns", "leave", "flip"):
            if key in x:
                assert got[key] == x[key], "block %d column %d: %s = %s, not %s" % (b, x["j"], key, got[key], x[key])
