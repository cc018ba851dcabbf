"""Read-based phasing of the merged calls: the statement the GPU route (``clair3_b200/phase_gpu.py``, ``csrc/phase.cu``) is held
to, in plain Python and numpy (DESIGN.md 5g.3).

Clair3's ``--enable_phasing`` runs ``whatshap phase --ignore-read-groups`` on each contig's ``merge_output`` rows.  This module
states WhatsHap's model - the all-heterozygous weighted minimum-error-correction (wMEC) problem over reads with a coverage cap
of 15 - exactly, so that the phase sets come from the same model; the file is not WhatsHap's byte for byte (its allele
detection realigns each read around each variant, and its read selection and output carry more than is stated here).

Per contig:

* **Variants** (``het_snvs``): the rows whose GT is ``0/1`` with a REF and an ALT of one base each, A, C, G or T.  FILTER is
  not read, so LowQual rows are phased too.  Every other row passes through unchanged.
* **Fragments** (``fragments``): records that are not unmapped, secondary, QC-fail, duplicate or supplementary and have
  MAPQ >= 20.  At each variant a read covers with an aligned base (CIGAR M / = / X) the read base equal to REF is allele 0,
  equal to ALT allele 1, anything else no entry; the entry's weight is the base quality.  A read of fewer than two entries
  is dropped.  A read's id is its index among the contig's records in file order.
* **Read selection** (``select_reads``): reads sorted by (entries desc, summed weight desc, id asc) and admitted greedily: a
  read is admitted only if every variant from its first entry to its last still has a coverage of at most 15 with it.
* **Blocks** (``layout``): connected components of variants linked by admitted reads (a read links the variants of its
  entries), ordered by first variant.  A block's columns are its variants, ascending; its reads are ordered by (first column,
  id).  A variant that no admitted read links stays unphased.
* **DP** (``solve_block``): a read is active from its first column to its last.  A state is a bipartition (S0, S1) of the
  reads active at column j, as a bit mask over them in block order, with the lowest active read in S0 (bit 0 clear).  The
  column cost is ``min(W1(S0) + W0(S1), W0(S0) + W1(S1))`` with ``Wa(S)`` the summed weight of the reads of S that show
  allele a, and ``D(j, B) = cost(j, B) + min D(j - 1, B')`` over the B' that agree with B on the reads active at both
  columns - up to swapping the parts, since D does not change when they swap.  The reads active at j that were active at
  j - 1 come first in B, those entering at j after them, so B' is B's shared bits deposited at their places among the reads
  of column j - 1 plus a pattern l of the leaving reads' bits (the predecessor choice).  Ties: the lowest l, then at the last
  column the lowest state; a column gives allele 0 to S0 of its own state (bit 0 clear) when both assignments cost the same.
  Costs are integer sums, so any implementation that follows these rules gets the same optimum and the same haplotypes.
* **Output** (``phase_rows``): haplotype 0 carries allele 0 at a block's first variant, so that row's GT is ``0|1``; ``PS``
  is the 1-based position of the block's first variant.  A phased row gets GT ``h0|h1`` and ``:PS`` appended to FORMAT and
  the sample column; every other row is byte-identical.  ``phase_header`` inserts the PS FORMAT line after the last
  ``##FORMAT`` line.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

MIN_MAPQ = 20                      # whatshap phase --mapping-quality default
MAX_COVERAGE = 15                  # whatshap phase --max-coverage default
FLAG_SKIP = 0x4 | 0x100 | 0x200 | 0x400 | 0x800      # unmapped, secondary, QC-fail, duplicate, supplementary
PS_HEADER = '##FORMAT=<ID=PS,Number=1,Type=Integer,Description="Phase set">'
MAX_BLOCK_WEIGHT = (1 << 32) - 1   # D is held in 32 bits: a block's summed entry weights bound it
_NT16 = {"A": 1, "C": 2, "G": 4, "T": 8}
_ALIGNED = (0, 7, 8)               # M, =, X
_REF_OPS = (0, 2, 3, 7, 8)
_QUERY_OPS = (0, 1, 4, 7, 8)


class Variants(NamedTuple):
    """The phasable rows of a contig: ``row`` index into its rows, 0-based ``pos`` ascending, ``ref`` / ``alt`` nt16 codes."""
    row: np.ndarray
    pos: np.ndarray
    ref: np.ndarray
    alt: np.ndarray


class Fragments(NamedTuple):
    """Allele observations sorted by (read, variant): read id, variant index, allele (0 REF / 1 ALT), weight (base quality)."""
    read: np.ndarray
    var: np.ndarray
    allele: np.ndarray
    weight: np.ndarray


def empty_fragments():
    return Fragments(np.zeros(0, np.int64), np.zeros(0, np.int32), np.zeros(0, np.uint8), np.zeros(0, np.uint8))


# ------------------------------------------------------------------------------------------------ variants and reads
def het_snvs(rows):
    """The ``Variants`` of a contig's VCF rows (row texts, sorted by position)."""
    keep, pos, ref, alt = [], [], [], []
    for i, row in enumerate(rows):
        c = row.rstrip("\n").split("\t")
        if len(c) < 10 or c[9].split(":", 1)[0] != "0/1" or c[3] not in _NT16 or c[4] not in _NT16:
            continue
        keep.append(i)
        pos.append(int(c[1]) - 1)
        ref.append(_NT16[c[3]])
        alt.append(_NT16[c[4]])
    return Variants(np.array(keep, np.int64), np.array(pos, np.int64), np.array(ref, np.uint8), np.array(alt, np.uint8))


def fragments(rec, variants):
    """The ``Fragments`` of a contig's records (``bam_io.read_bam(..., fa_fields=True)``'s dict, every record of the contig)
    at ``variants``."""
    vpos = np.asarray(variants.pos, np.int64)
    out = [[], [], [], []]
    if not len(vpos):
        return empty_fragments()
    flag, mapq, pos = np.asarray(rec["flag"]), np.asarray(rec["mapq"]), np.asarray(rec["pos"], np.int64)
    cig_all, coff = np.asarray(rec["cigar"], np.uint32), np.asarray(rec["cigar_off"], np.int64)
    seq, soff = np.asarray(rec["seq"], np.uint8), np.asarray(rec["seq_off"], np.int64)
    qual, qoff = np.asarray(rec["qual"], np.uint8), np.asarray(rec["qual_off"], np.int64)
    for r in np.flatnonzero(((flag & FLAG_SKIP) == 0) & (mapq >= MIN_MAPQ)):
        cig = cig_all[coff[r]:coff[r + 1]]
        if not len(cig):
            continue
        op, ln = (cig & 15).astype(np.int64), (cig >> 4).astype(np.int64)
        rl = np.where(np.isin(op, _REF_OPS), ln, 0)
        ql = np.where(np.isin(op, _QUERY_OPS), ln, 0)
        r0 = pos[r] + np.cumsum(rl) - rl
        q0 = np.cumsum(ql) - ql
        al = np.isin(op, _ALIGNED) & (ln > 0)
        r0, q0, ln = r0[al], q0[al], ln[al]
        if not len(r0):
            continue
        v0, v1 = np.searchsorted(vpos, r0[0]), np.searchsorted(vpos, r0[-1] + ln[-1])
        v = np.arange(v0, v1)
        k = np.searchsorted(r0, vpos[v], side="right") - 1
        inside = vpos[v] < r0[k] + ln[k]
        v, k = v[inside], k[inside]
        q = q0[k] + vpos[v] - r0[k]
        lq = int(rec["l_qseq"][r])
        b = seq[soff[r] + (np.minimum(q, max(lq - 1, 0)) >> 1)] if lq else np.zeros(len(q), np.uint8)
        base = np.where(q < lq, np.where(q & 1, b & 15, b >> 4), 0)        # a base past the read: none, as the GPU reads it
        allele = np.where(base == variants.ref[v], 0, np.where(base == variants.alt[v], 1, 2))
        hit = allele < 2
        if hit.sum() < 2:
            continue
        out[0].append(np.full(int(hit.sum()), r, np.int64))
        out[1].append(v[hit].astype(np.int32))
        out[2].append(allele[hit].astype(np.uint8))
        out[3].append(qual[qoff[r] + q[hit]])
    if not out[0]:
        return empty_fragments()
    return Fragments(*(np.concatenate(a) for a in out))


# ------------------------------------------------------------------------------------------------ selection and blocks
def _per_read(frag):
    """(read ids, first entry index, entry counts) of the reads of sorted fragments."""
    ids, start, count = np.unique(frag.read, return_index=True, return_counts=True)
    return ids, start, count


def select_reads(frag, n_var, cap=MAX_COVERAGE):
    """The admitted read ids, ascending, and the coverage over the variants they leave (each read counted from its first entry's
    variant to its last's)."""
    cov = np.zeros(n_var, np.int64)
    if not len(frag.read):
        return np.zeros(0, np.int64), cov
    ids, start, count = _per_read(frag)
    wsum = np.add.reduceat(frag.weight.astype(np.int64), start)
    first, last = frag.var[start].astype(np.int64), frag.var[start + count - 1].astype(np.int64)
    admitted = []
    for i in np.lexsort((ids, -wsum, -count)):
        a, b = first[i], last[i] + 1
        if cov[a:b].max() < cap:
            cov[a:b] += 1
            admitted.append(ids[i])
    return np.sort(np.array(admitted, np.int64)), cov


class Layout(NamedTuple):
    """The blocks of a contig as both DP implementations read them.  Block b's columns are ``[blk_col_off[b],
    blk_col_off[b + 1])`` of the global column numbering and its reads ``[blk_read_off[b], blk_read_off[b + 1])``; per column
    the variant index (``col_var``) and its entries ``[col_ent_off[c], col_ent_off[c + 1])`` (block-local read index, allele,
    weight; ascending by read); per read its id and first / last column within the block; per block the most reads active
    at one column (``blk_kmax``)."""
    blk_col_off: np.ndarray
    blk_read_off: np.ndarray
    blk_kmax: np.ndarray
    col_var: np.ndarray
    col_ent_off: np.ndarray
    read_id: np.ndarray
    read_first: np.ndarray
    read_last: np.ndarray
    ent_read: np.ndarray
    ent_allele: np.ndarray
    ent_weight: np.ndarray

    @property
    def n_blocks(self):
        return len(self.blk_col_off) - 1


def _components(frag, n_var):
    """Component label per variant (-1: linked by no read) of the variants linked by consecutive entries of each read."""
    parent = np.arange(n_var)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    same = frag.read[1:] == frag.read[:-1]
    for a, b in zip(frag.var[:-1][same].tolist(), frag.var[1:][same].tolist()):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    label = np.array([find(x) for x in range(n_var)], np.int64)
    label[np.setdiff1d(np.arange(n_var), frag.var)] = -1
    return label


def layout(frag, n_var, cap=MAX_COVERAGE):
    """Read selection and blocks of a contig's fragments over ``n_var`` variants: its ``Layout``."""
    admitted, _ = select_reads(frag, n_var, cap)
    keep = np.isin(frag.read, admitted)
    f = Fragments(*(a[keep] for a in frag))
    label = _components(f, n_var)
    roots = np.unique(label[label >= 0])                     # each root is its component's lowest variant: ordered by it
    block_of_var = np.full(n_var, -1, np.int64)
    block_of_var[label >= 0] = np.searchsorted(roots, label[label >= 0])
    cols = np.flatnonzero(label >= 0)
    cols = cols[np.lexsort((cols, block_of_var[cols]))]      # by block, then variant
    nb = len(roots)
    blk_col_off = np.zeros(nb + 1, np.int64)
    blk_col_off[1:] = np.cumsum(np.bincount(block_of_var[cols], minlength=nb))
    col_of_var = np.full(n_var, -1, np.int64)
    col_of_var[cols] = np.arange(len(cols))
    ids, start, count = _per_read(f)
    rblk = block_of_var[f.var[start]]
    rfirst = col_of_var[f.var[start]] - blk_col_off[rblk]
    rlast = col_of_var[f.var[start + count - 1]] - blk_col_off[rblk]
    order = np.lexsort((ids, rfirst, rblk))
    blk_read_off = np.zeros(nb + 1, np.int64)
    blk_read_off[1:] = np.cumsum(np.bincount(rblk, minlength=nb))
    local = np.empty(len(ids), np.int64)
    local[order] = np.arange(len(ids)) - blk_read_off[rblk[order]]
    e_col = col_of_var[f.var]
    e_read = np.repeat(local, count)
    eo = np.lexsort((e_read, e_col))
    col_ent_off = np.zeros(len(cols) + 1, np.int64)
    col_ent_off[1:] = np.cumsum(np.bincount(e_col, minlength=len(cols)))
    # the most reads active at one column of each block
    act = np.zeros(len(cols) + 1, np.int64)
    c0 = blk_col_off[rblk]
    np.add.at(act, c0 + rfirst, 1)
    np.add.at(act, c0 + rlast + 1, -1)
    act = np.cumsum(act)[:-1]
    kmax = np.array([act[a:b].max() for a, b in zip(blk_col_off[:-1], blk_col_off[1:])], np.int32)
    lay = Layout(blk_col_off, blk_read_off, kmax, cols.astype(np.int64), col_ent_off, ids[order], rfirst[order].astype(np.int32),
                 rlast[order].astype(np.int32), e_read[eo].astype(np.int32), f.allele[eo], f.weight[eo])
    for b in range(nb):
        w = int(lay.ent_weight[col_ent_off[blk_col_off[b]]:col_ent_off[blk_col_off[b + 1]]].astype(np.int64).sum())
        if w > MAX_BLOCK_WEIGHT:
            raise ValueError("phasing: a block's summed weights (%d) exceed 2^32 - 1" % w)
    return lay


# ------------------------------------------------------------------------------------------------ the DP
def _deposit(x, mask):
    """pdep: the low bits of x (an array) placed at the set bits of ``mask``, lowest first."""
    out = np.zeros_like(x)
    i = 0
    for b in range(16):
        if mask >> b & 1:
            out |= ((x >> i) & 1) << b
            i += 1
    return out


def _subsets(mask):
    """The subsets of ``mask`` in increasing order: subset l is the l-th leaving-read pattern."""
    sub = 0
    while True:
        yield sub
        sub = (sub - mask) & mask
        if sub == 0:
            return


def column_plan(lay, b):
    """Per column of block b: (k, ns, shared mask, leaving mask, entry bit positions) - the active reads' count, the count of
    those active at the previous column too, and which bits of the previous column's state are shared / leaving."""
    c0, c1 = lay.blk_col_off[b], lay.blk_col_off[b + 1]
    r0, r1 = lay.blk_read_off[b], lay.blk_read_off[b + 1]
    first, last = lay.read_first[r0:r1], lay.read_last[r0:r1]
    act, nxt, plan = [], 0, []
    for j in range(c1 - c0):
        sh = lv = 0
        new = []
        for i, r in enumerate(act):
            if last[r] >= j:
                sh |= 1 << i
                new.append(r)
            else:
                lv |= 1 << i
        ns = len(new)
        while nxt < len(first) and first[nxt] == j:
            new.append(nxt)
            nxt += 1
        act = new
        if len(act) > MAX_COVERAGE or (j > 0 and ns == 0):
            raise ValueError("phasing: block %d column %d: %d active reads, %d shared" % (b, j, len(act), ns))
        e = slice(lay.col_ent_off[c0 + j], lay.col_ent_off[c0 + j + 1])
        bits = np.array([act.index(r) for r in lay.ent_read[e]], np.int64)
        plan.append((len(act), ns, sh, lv, bits))
    return plan


def _column_costs(states, bits, allele, weight):
    """(cost, a0) per normalized state: a0 = the allele of part 0 (0 on a tie)."""
    B = states << 1
    opt1 = np.zeros(len(states), np.int64)
    for bt, a, w in zip(bits.tolist(), allele.tolist(), weight.tolist()):
        opt1 += w * (((B >> bt) ^ a) & 1)
    opt2 = int(weight.astype(np.int64).sum()) - opt1
    return np.minimum(opt1, opt2), (opt1 > opt2).astype(np.uint8)


def solve_block(lay, b):
    """The DP of block b: (haplotype 0's allele per column of the block, uint8; the optimal cost)."""
    c0 = lay.blk_col_off[b]
    plan = column_plan(lay, b)
    m = len(plan)
    ent = lambda j: slice(lay.col_ent_off[c0 + j], lay.col_ent_off[c0 + j + 1])    # noqa: E731
    args, D = [None] * m, None
    for j, (k, ns, sh, lv, bits) in enumerate(plan):
        states = np.arange(1 << (k - 1), dtype=np.int64)
        cost, _ = _column_costs(states, bits, lay.ent_allele[ent(j)], lay.ent_weight[ent(j)])
        if j == 0:
            D = cost
            continue
        kp = plan[j - 1][0]
        full_p = (1 << kp) - 1
        base = _deposit(np.arange(1 << (ns - 1), dtype=np.int64) << 1, sh)
        best = np.full(len(base), np.iinfo(np.int64).max, np.int64)
        arg = np.zeros(len(base), np.int64)
        for l, sub in enumerate(_subsets(lv)):
            full = base | sub
            v = D[np.where(full & 1, ~full & full_p, full) >> 1]
            better = v < best
            best = np.where(better, v, best)
            arg = np.where(better, l, arg)
        args[j] = arg
        D = cost + best[states & ((1 << (ns - 1)) - 1)]
    s = int(np.argmin(D))
    total = int(D[s])
    hap = np.zeros(m, np.uint8)
    f = 0
    for j in range(m - 1, -1, -1):
        k, ns, sh, lv, bits = plan[j]
        _, a0 = _column_costs(np.array([s], np.int64), bits, lay.ent_allele[ent(j)], lay.ent_weight[ent(j)])
        hap[j] = a0[0] ^ f
        if j:
            t = s & ((1 << (ns - 1)) - 1)
            l = int(args[j][t])
            full = int(_deposit(np.array([t << 1], np.int64), sh)[0] | _deposit(np.array([l], np.int64), lv)[0])
            if full & 1:
                full = ~full & ((1 << plan[j - 1][0]) - 1)
                f ^= 1
            s = full >> 1
    return hap ^ hap[0], total


def solve(lay):
    """Every block's DP: (haplotype 0's allele per column, uint8 [columns]; optimal cost per block, int64 [blocks])."""
    hap = np.zeros(len(lay.col_var), np.uint8)
    cost = np.zeros(lay.n_blocks, np.int64)
    for b in range(lay.n_blocks):
        hap[lay.blk_col_off[b]:lay.blk_col_off[b + 1]], cost[b] = solve_block(lay, b)
    return hap, cost


# ------------------------------------------------------------------------------------------------ output
def phase_header(head):
    """A VCF header with ``PS_HEADER`` after its last ``##FORMAT`` line (after the last meta line when it has none)."""
    lines = head.split("\n")
    at = max((i for i, x in enumerate(lines) if x.startswith("##FORMAT")), default=None)
    if at is None:
        at = max((i for i, x in enumerate(lines) if x.startswith("##")), default=-1)
    lines.insert(at + 1, PS_HEADER)
    return "\n".join(lines)


def phase_rows(rows, variants, lay, hap):
    """The contig's rows with the phased ones rewritten: GT ``h0|h1`` and ``:PS`` on FORMAT and the sample column."""
    out = list(rows)
    for b in range(lay.n_blocks):
        c0, c1 = lay.blk_col_off[b], lay.blk_col_off[b + 1]
        ps = int(variants.pos[lay.col_var[c0]]) + 1
        for c in range(c0, c1):
            i = int(variants.row[lay.col_var[c]])
            row = out[i]
            end = "\n" if row.endswith("\n") else ""
            f = row[:len(row) - len(end)].split("\t")
            h = int(hap[c])
            sample = f[9].split(":")
            sample[0] = "%d|%d" % (h, 1 - h)
            f[8] += ":PS"
            f[9] = ":".join(sample) + ":%d" % ps
            out[i] = "\t".join(f) + end
    return out


def phase_contig(rows, rec):
    """The host statement end to end for one contig: ``rows`` its VCF rows, ``rec`` every record of the contig
    (``bam_io.read_bam(bam, ctg, fa_fields=True)[0]``).  Returns (phased rows, variants, fragments, layout, haplotypes, costs)."""
    v = het_snvs(rows)
    frag = fragments(rec, v)
    lay = layout(frag, len(v.pos))
    hap, cost = solve(lay)
    return phase_rows(rows, v, lay, hap), v, frag, lay, hap, cost


def split_contigs(body):
    """{contig: [row texts]} of a sorted VCF body, in order."""
    out = {}
    for row in body.splitlines(keepends=True):
        out.setdefault(row.split("\t", 1)[0], []).append(row)
    return out
