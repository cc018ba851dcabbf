"""Mint the targeted vectors of the decoder's calls from the REAL reference (a Clair3 checkout, named by CLAIR3_REFERENCE).

    CLAIR3_REFERENCE=/path/to/Clair3 PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_decode_calls_golden.py

Every alt_info case below targets one rule of ``output_from`` / ``output_with`` (``clair3/CallVariants.py:676-1394``).  Each case
is decoded under a set of crafted probability rows, each of which points the walk at one outcome category and indel length
(plus flat rows, whose walks pass many entries before homo_Ref), for both output widths.  For every (case, row) the reference's
own ``output_from`` result and its ``batch_output`` text under six output configs are recorded, one site per call, with the name
of the exception where the reference raises.  Only the data goes into the ``.npz``.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CENTER = 16
CONFIGS = {
    "default": {},
    "show_ref": {"is_show_reference": True},
    "haploid_precise": {"is_haploid_precise_mode_enabled": True},
    "haploid_sensitive": {"is_haploid_sensitive_mode_enabled": True},
    "long_indel": {"enable_long_indel": True, "is_show_reference": True},
    "qual_iupac": {"quality_score_for_pass": 12.0, "keep_iupac_bases": True},
}


def _bases(r, n, alphabet="ACGT"):
    return "".join(r.choice(list(alphabet), size=n))


def cases():
    """(centre base, alt_info) pairs; each targets one rule."""
    r = np.random.Generator(np.random.PCG64(77))
    b = lambda n: _bases(r, n)                                          # noqa: E731
    out = [
        ("A", "40-XC 10 XG 10 XT 3 R 20"),              # SNP count tie: the first maximum in alt_info order
        ("A", "40-XG 10 XC 10 R 20"),
        ("A", "40-XC 12 XG 20 R 5"),                    # 8 reads behind the best: the proposed base stays
        ("A", "40-XC 11 XG 20 R 5"),                    # 9 reads behind: replaced
        ("A", "40-XC 10 R 20"),                         # both SNP bases non-reference, fewer than two SNP alleles
        ("C", "40-XA 4 R 20"),
        ("A", "40-IAC 5 IAG 5 IACG 5 IACT 5 R 3"),      # insertion ties (proposed, unproposed, return_multi)
        ("A", "40-IACGT 7 IAC 7 IATT 7 R 3"),
        ("A", "40-DC 5 DG 5 DCG 5 DTT 5 R 3"),          # deletion ties
        ("A", "40-DCCC 6 DGG 6 DT 6 R 1"),
        ("A", "40-DCC 6 DGG 6 DT 2 R 4"),               # two deletions of equal length (DelDel)
        ("A", "40-DCC 6 DGG 6 R 4"),
        ("G", "40-IG%s 5 IG%s 6 IG%s 7 D%s 4 D%s 5 D%s 6 R 2" % (b(15), b(16), b(17), b(15), b(16), b(17))),   # 15 / 16 / 17
        ("T", "40-IT%s 5 IT%s 6 IT%s 3 IT%s 4 D%s 5 D%s 6 R 1" % (b(50), b(51), b(49), b(55), b(50), b(51))),  # 50 / 51
        ("T", "40-IT%s 9 IT%s 6 IT%s 3 R 1" % (b(51), b(50), b(56))),
        ("C", "40-IC%s 8 IC%s 8 IC%s 2 D%s 3 R 1" % (b(60), b(61), b(54), b(52))),
        ("R", "40-XA 8 XG 9 DRyN 5 DAC 4 IAT 3 R 2"),   # IUPAC reference bases and deletion text
        ("N", "40-Dacgt 6 DNNa 6 XC 4 R 2"),
        ("Y", "40-XT 7 ICG 5 Dwsk 4 R 2"),
        ("K", "40-XG 3 DGT 5 IGA 5 R 2"),
        ("A", "0-XC 5 IAC 3 DC 2 R 3"),                 # depth 0 (single count)
        ("A", "5-XC 30 IAG 20 DT 9 R 2"),               # support above depth
        ("A", "40-XC 5 IAG 4 DT 3"),                    # no R
        ("A", "40-XC 5 R -3"),                          # negative R: the '-' splits the string
        ("A", "40"),                                    # no '-'
        ("A", "40-"),                                   # empty body
        ("A", "40-XC 5 XG 3 XC 9 R 1 R 4"),             # repeated keys: first position, last count
        ("A", "40-XC 5-XG 9"),                          # a second '-'
        ("A", "40-XC 5 IAG 3 R 2   "),                  # trailing space
        ("A", "40-XC 5 XG"),                            # a key without a count
        ("A", "x-XC 5"),                                # depth does not parse
        ("A", "40-XC five"),                            # count does not parse
        ("A", "40-X 5 XC 3"),                           # a bare X key
        ("A", "40- 5"),                                 # an empty key
        ("A", "40-" + " ".join("IA%s %d" % (b(1 + i % 20), 1 + (i * 7) % 13) for i in range(60)) + " R 3"),  # 60 insertions
        ("A", "40-IA%s 12 IA%s 3 XC 2 R 4" % (b(500), b(480))),                # a 500-base insertion
        ("A", "40-R 30"),                               # nothing but reference reads: long walks
        ("A", "40-XA 3 IAA 2 R 30"),
    ]
    return out


def rows(out_dim, r):
    """Crafted rows: each points the walk at one category / length pair; flat and quarter rows walk far."""
    def row(gt=None, geno=None, l1=0, l2=0):
        y = np.full(out_dim, 0.01, np.float32)
        if gt is not None:
            y[gt] = 0.9
        y[21 + (geno if geno is not None else 0)] = 0.9
        if out_dim == 90:
            y[24 + 16 + l1] = 0.9
            y[57 + 16 + l2] = 0.9
        return y
    out = [row(4, 1), row(7, 1), row(1, 2), row(5, 2), row(2, 2)]                            # SNPs
    lens = (1, 2, 3, 15, 16) if out_dim == 90 else (0,)
    for L in lens:
        out += [row(15, 1, L, L), row(16 + 1, 2, 0, L), row(10, 1, -L, -L), row(11 + 2, 2, -L, 0)]
    if out_dim == 90:
        out += [row(15, 2, 1, 2), row(15, 2, 16, 16), row(10, 2, -2, -1), row(10, 2, -16, -16), row(10, 2, -3, -3),
                row(20, 2, -1, 1), row(20, 2, -16, 16)]
    else:
        out += [row(15, 2), row(10, 2), row(20, 2)]
    out += [np.full(out_dim, 0.3, np.float32), (r.integers(0, 5, size=out_dim) / 4.0).astype(np.float32),
            r.uniform(0.05, 1.0, size=out_dim).astype(np.float32)]
    out[-1][21] = np.float32(1e-6)
    return np.stack(out)


def config(CV, out_dim, **kw):
    base = dict(is_show_reference=False, is_debug=False, is_haploid_precise_mode_enabled=False,
                is_haploid_sensitive_mode_enabled=False, is_output_for_ensemble=False, quality_score_for_pass=None, tensor_fn="PIPE",
                input_probabilities=True, add_indel_length=(out_dim == 90), gvcf=False, pileup=(out_dim == 24),
                enable_long_indel=False, maximum_variant_length_that_need_infer=50, keep_iupac_bases=False)
    base.update(kw)
    if base["enable_long_indel"]:
        base["maximum_variant_length_that_need_infer"] = 100000
    return CV.OutputConfig(**base)


def split(row, out_dim):
    if out_dim == 90:
        return row[:21], row[21:24], row[24:57], row[57:90]
    return row[:21], row[21:24], 0, 0


def mint(reference):
    """The fixture's arrays, from the reference checkout at ``reference``."""
    if reference not in sys.path:
        sys.path.insert(0, reference)
    import clair3.CallVariants as CV

    r = np.random.Generator(np.random.PCG64(4041))
    out = {}
    for out_dim in (24, 90):
        crafted = rows(out_dim, r)
        ys, pos, alts = [], [], []
        for ci, (center, alt) in enumerate(cases()):
            for y in crafted:
                seq = _bases(r, CENTER, "acgtACGT") + center + _bases(r, CENTER, "acgtACGT")
                ys.append(y)
                pos.append("chr%d:%d:%s" % (1 + ci % 3, 1000 + len(pos), seq))
                alts.append(alt)
        y = np.stack(ys)
        res = {"y": y, "pos": np.array(pos), "alt": np.array(alts)}
        for tag, cfg in (("", config(CV, out_dim)), ("_long", config(CV, out_dim, enable_long_indel=True))):
            flags, refs, alts_o, probs, excs = [], [], [], [], []
            for i in range(len(y)):
                fl, rb, ab, p, exc = (0,) * 10, "", "", np.float32(0), ""
                try:
                    parts = alts[i].rstrip().split("-")
                    seqs = (parts[1] if len(parts) > 1 else "").split(" ")
                    d = dict(zip(seqs[::2], [int(v) for v in seqs[1::2]]))
                    int(parts[0])
                    fl, (rb, ab), p = CV.output_from(pos[i].split(":")[-1], "chr", 1, CENTER, *split(y[i], out_dim), cfg, None, d)
                except Exception as e:                                   # noqa: BLE001
                    exc = type(e).__name__
                flags.append(np.array(fl, np.uint8))
                refs.append(str(rb))
                alts_o.append(str(ab))
                probs.append(np.float32(p))
                excs.append(exc)
            res["of_flags" + tag] = np.array(flags)
            res["of_ref" + tag] = np.array(refs)
            res["of_alt" + tag] = np.array(alts_o)
            res["of_prob" + tag] = np.array(probs, np.float32)
            res["of_exc" + tag] = np.array(excs)
        for name, kw in CONFIGS.items():
            texts, excs = [], []
            cfg = config(CV, out_dim, **kw)
            for i in range(len(y)):
                try:
                    texts.append(CV.batch_output([pos[i]], [alts[i]], y[i:i + 1], cfg, None))
                    excs.append("")
                except Exception as e:                                   # noqa: BLE001
                    texts.append("")
                    excs.append(type(e).__name__)
            res["text_" + name] = np.array(texts)
            res["exc_" + name] = np.array(excs)
        for k, v in res.items():
            out["c%d_%s" % (out_dim, k)] = v
    return out


def main():
    sys.dont_write_bytecode = True
    out = mint(os.environ["CLAIR3_REFERENCE"])
    for out_dim in (24, 90):
        print(out_dim, "rows", len(out["c%d_y" % out_dim]),
              {n: int((out["c%d_text_%s" % (out_dim, n)] != "").sum()) for n in CONFIGS},
              "raises", sorted(set(out["c%d_exc_default" % out_dim]) - {""}))
    np.savez_compressed(os.path.join(HERE, "decode_calls.npz"), **out)


if __name__ == "__main__":
    main()
