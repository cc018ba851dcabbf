"""Crafted pileup and full-alignment call results for the cascade's host layer (clair3_b200/cascade.py), rebuilt from this
module's code by tests/golden/make_cascade_golden.py (which runs the reference's SelectQual, SelectCandidates and MergeVcf on
their VCF text) and by tests/test_cascade_cpu.py (which holds ``qual_cutoffs``, ``select`` and ``merge`` to those outputs).

A call result here has the fields of ``decode.batch_calls``' dict (``calls`` as ``model.CALL_DTYPE`` records, the ``text`` /
``ad`` pools, ``start``) plus ``cand_ok`` for pileup calls, so ``decode.calls_text`` formats it as the decoder would."""
import numpy as np

from clair3_b200 import cascade, decode
from clair3_b200.model import CALL_DTYPE

CTG = "chr20"
HEADER = "##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE\n"
CFG_P = decode.replay_config(pileup=True, add_indel_length=False)._replace(is_show_reference=True)
CFG_F = decode.replay_config(pileup=False, add_indel_length=True)._replace(is_show_reference=True)


def prob_of_qual(q):
    """A float32 probability whose QUAL is exactly ``q`` (the smallest such bit pattern)."""
    t = cascade.prob_threshold(q)
    p = np.array(t, np.uint32).view(np.float32)[()]
    assert decode.quality_score_from(p) == q
    return p


def result(rows, cand_ok=None):
    """rows: (1-based position, genotype code, float32 prob, REF, ALT) with ALT "." for a reference row; is_ref (FILTER
    RefCall) follows the genotype, so a row can disagree with its ALT text."""
    n = len(rows)
    calls = np.zeros(n, CALL_DTYPE)
    text, ad, start = [], [], np.zeros(n, np.int64)
    o = 0
    for s, (pos, gt, prob, ref, alt) in enumerate(rows):
        counts = [] if alt == "." else [7] * (alt.count(",") + 1)
        c = calls[s]
        c["dp"], c["ref_count"], c["support"] = 30, 12, sum(counts) if counts else 12
        c["prob"], c["genotype"], c["printed"] = prob, gt, 1
        c["flags"] = 1 if gt == 0 else 2
        c["ref_len"], c["alt_len"], c["n_ad"] = len(ref), len(alt), len(counts)
        b = (ref + alt).encode()
        start[s] = o
        text.append(b)
        ad.extend(counts + [0] * (len(b) - len(counts)))
        o += len(b)
    res = {"chromosome": [CTG] * n, "position": np.array([r[0] for r in rows], np.int64), "calls": calls,
           "text": np.frombuffer(b"".join(text) or b"\0", np.uint8).copy(), "ad": np.array(ad or [0], np.int64), "start": start}
    if cand_ok is not None:
        res["cand_ok"] = np.asarray(cand_ok, np.uint8)
    return res


def _random_rows(rng, positions, ref_frac, q2=(), tie_prob=None, tie_every=0):
    rows = []
    p2 = prob_of_qual(2.0)
    for i, pos in enumerate(positions):
        base = "ACGT"[rng.integers(0, 4)]
        prob = np.float32(rng.uniform(0.45, 1.0))
        if tie_prob is not None and tie_every and i % tie_every == 0:
            prob = tie_prob
        if i in q2:
            prob = p2
        if rng.random() < ref_frac:
            rows.append((int(pos), 0, prob, base, "."))
        else:
            alt = "ACGT"[("ACGT".index(base) + 1 + rng.integers(0, 3)) % 4]
            kind = rng.integers(0, 4)
            if kind == 0:
                rows.append((int(pos), 2, prob, base, alt))
            elif kind == 1:
                rows.append((int(pos), 1, prob, base, alt))
            elif kind == 2:
                rows.append((int(pos), 1, prob, base, base + "GT"))
            else:
                rows.append((int(pos), 3, prob, base + "CA", base + "," + base + "C"))
    return rows


def _fa_rows(rng, pileup_rows, positions):
    """Full-alignment calls at some candidates: a RefCall over a pileup variant, variants, QUAL exactly 2.00."""
    by_pos = {r[0]: r for r in pileup_rows}
    out = []
    p2 = prob_of_qual(2.0)
    for j, pos in enumerate(positions):
        r = by_pos[int(pos) + 1]
        prob = p2 if j % 7 == 3 else np.float32(rng.uniform(0.1, 1.0) ** 2)
        if j % 5 == 0 or r[4] == ".":
            out.append((r[0], 0, prob, r[3][0], "."))
        else:
            out.append((r[0], int(rng.integers(1, 3)), prob, r[3][0], "ACGT"[("ACGT".index(r[3][0]) + 1) % 4]))
    return out


def phased_vcf(positions):
    """A phased VCF body: 0|1 / 1|0 SNPs (and one unphased) at ``positions`` (1-based)."""
    rows = []
    for i, p in enumerate(positions):
        gt = "0/1" if i == 2 else ("0|1" if i % 2 else "1|0")
        rows.append("%s\t%d\t.\tA\tC\t30\tPASS\t.\tGT:GQ:DP:AD:AF:PS\t%s:30:30:10,10:0.5:%d\n" % (CTG, p, gt, 1000))
    return HEADER + "".join(rows)


def case(name):
    """(platform, pileup call result, phased VCF text or None) of case ``name``."""
    rng = np.random.default_rng({"ont": 1, "hifi": 2, "zero_ref": 3, "two_chunks": 4}[name])
    if name in ("ont", "hifi"):
        positions = np.unique(np.concatenate([[1, 2, 5, 16, 17, 18, 19, 40], rng.integers(50, 400000, 600)]))
        tie = np.float32(0.47)              # about the tenth-lowest reference QUAL: ties at the ont cut-off
        rows = _random_rows(rng, positions, 0.55, q2=(3, 11, 29), tie_prob=tie, tie_every=9)
        # rows whose GT and ALT text disagree: 0/0 with an ALT, 0/1 with ALT "." and with ALT == REF
        rows[20] = (rows[20][0], 0, rows[20][2], "A", "C")
        rows[21] = (rows[21][0], 1, rows[21][2], "A", ".")
        rows[22] = (rows[22][0], 1, rows[22][2], "G", "G")
        ok = (rng.random(len(rows)) > 0.03).astype(np.uint8)
        phased = phased_vcf([10, 30, int(positions[100]), int(positions[300]), 500000, 900000])
        return name, result(rows, ok), phased
    if name == "zero_ref":
        positions = np.arange(100, 100 + 80 * 37, 37)
        rows = _random_rows(rng, positions, 0.0)
        for i in (4, 30, 60):
            rows[i] = (rows[i][0], 0, rows[i][2], "T", ".")
        return "ont", result(rows, np.ones(len(rows), np.uint8)), None
    if name == "two_chunks":
        positions = np.unique(rng.integers(1, 3_000_000, 17000))
        rows = _random_rows(rng, positions, 0.05)
        return "ont", result(rows, np.ones(len(rows), np.uint8)), None
    raise KeyError(name)


NAMES = ("ont", "hifi", "zero_ref", "two_chunks")


def fa_results(pileup, positions, chunks, seed):
    """One full-alignment call result per chunk, at a subset of the chunk's candidates."""
    rng = np.random.default_rng(seed)
    rows = [(int(p), int(g), pr, r, a) for p, g, pr, r, a in _rows_of(pileup)]
    out = []
    for lo, hi in chunks:
        pick = positions[lo:hi][rng.random(hi - lo) < 0.6]
        out.append(result(_fa_rows(rng, rows, pick)))
    return out


def _rows_of(res):
    calls, text, start = res["calls"], res["text"], res["start"]
    for s in range(len(calls)):
        o, rl, al = int(start[s]), int(calls["ref_len"][s]), int(calls["alt_len"][s])
        yield (res["position"][s], calls["genotype"][s], calls["prob"][s], text[o:o + rl].tobytes().decode(),
               text[o + rl:o + rl + al].tobytes().decode())


def vcf_text(res, cfg):
    """The VCF a call result prints: header and its rows (printed, cand_ok)."""
    return HEADER + "".join(cascade.row_texts(res, cfg)[1])
