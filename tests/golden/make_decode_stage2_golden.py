"""Mint the golden vectors of the decoder's second stage from the REAL reference (a Clair3 checkout, named by CLAIR3_REFERENCE).

    CLAIR3_REFERENCE=/path/to/Clair3 PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_decode_stage2_golden.py

Two kinds of data, for both output widths (24: no indel-length heads, 90: with them):

* **Attempt sequences.**  The reference's own ``output_from`` (``clair3/CallVariants.py:676-1012``) runs with its three
  alt-info helpers (``find_alt_base``, ``insertion_bases_using_alt_info_from``, ``deletion_bases_using_alt_info_from``) replaced
  by stubs that always fail and record the caller's ``maximum_probability``, ``idx`` and ``is_*`` locals.  Every attempt then
  fails, so the reference walks its whole order down to the homozygous-reference call and reveals it.  Rows include Dirichlet
  draws, rows quantised to quarters (exact ties across and inside categories, zeros, values of exactly 0.5) and rows whose
  homo_Ref probability is tiny, so that homo_Ref ranks last among hundreds of entries.
* **Real outputs.**  The reference's real ``output_from`` and ``batch_output`` on seeded ``depth-X.. n I.. n D.. n R.. n``
  alt_info strings that make attempts fail in every category, under several output configs (showRef, both haploid modes,
  ``enable_long_indel``, a ``quality_score_for_pass`` threshold, ``keep_iupac_bases``); reference windows carry lowercase
  flanks and IUPAC centre bases.

Only the data goes into the ``.npz``.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ["CLAIR3_REFERENCE"])
sys.dont_write_bytecode = True

import clair3.CallVariants as CV  # noqa: E402
from clair3.task.gt21 import gt21_enum_from_label  # noqa: E402
from shared.utils import IUPAC_base_to_ACGT_base_dict as BASE2ACGT  # noqa: E402

FLAG_NAMES = ("is_homo_SNP", "is_hetero_SNP", "is_homo_insertion", "is_hetero_ACGT_Ins", "is_hetero_InsIns", "is_homo_deletion",
              "is_hetero_ACGT_Del", "is_hetero_DelDel", "is_insertion_and_deletion")
CENTER = 16


def dirichlet_rows(r, n, out_dim):
    y = np.zeros((n, out_dim), dtype=np.float32)
    bounds = [0, 21, 24, 57, 90][: (5 if out_dim == 90 else 3)]
    for lo, hi in zip(bounds, bounds[1:]):
        conc = r.choice([0.05, 0.3, 2.0], size=n)
        for i in range(n):
            y[i, lo:hi] = r.dirichlet(np.full(hi - lo, conc[i])).astype(np.float32)
    return y


def quarter_rows(r, n, out_dim):
    """Values in {0, .25, .5, .75, 1}: products tie exactly across and inside the lists."""
    return (r.integers(0, 5, size=(n, out_dim)) / 4.0).astype(np.float32)


def late_ref_rows(r, n, out_dim):
    y = r.uniform(0.05, 1.0, size=(n, out_dim)).astype(np.float32)
    y[:, 21] = np.float32(1e-7)
    return y


def test_rows(r, out_dim):
    n_dirichlet, n_quarter, n_late = (160, 160, 20) if out_dim == 24 else (60, 30, 3)
    y = np.concatenate([dirichlet_rows(r, n_dirichlet, out_dim), quarter_rows(r, n_quarter, out_dim),
                        late_ref_rows(r, n_late, out_dim)])
    bases = r.choice(list("ACGT"), size=len(y))
    # drop the early-out rows: output_from returns before ranking anything for them
    keep = []
    for i in range(len(y)):
        res = CV.possible_outcome_probabilites_from(*split(y[i], out_dim), reference_base=str(bases[i]), alt_info_dict={},
                                                    add_indel_length=(out_dim == 90))
        if len(res) > 1:
            keep.append(i)
    return y[keep], bases[keep]


def split(row, out_dim):
    if out_dim == 90:
        return row[:21], row[21:24], row[24:57], row[57:90]
    return row[:21], row[21:24], 0, 0


def config(out_dim, **kw):
    base = dict(is_show_reference=False, is_debug=False, is_haploid_precise_mode_enabled=False,
                is_haploid_sensitive_mode_enabled=False, is_output_for_ensemble=False, quality_score_for_pass=None, tensor_fn="PIPE",
                input_probabilities=True, add_indel_length=(out_dim == 90), gvcf=False, pileup=(out_dim == 24),
                enable_long_indel=False, maximum_variant_length_that_need_infer=50, keep_iupac_bases=False)
    base.update(kw)
    if base["enable_long_indel"]:
        base["maximum_variant_length_that_need_infer"] = 100000
    return CV.OutputConfig(**base)


CONFIGS = {
    "default": {},
    "show_ref": {"is_show_reference": True},
    "haploid_precise": {"is_haploid_precise_mode_enabled": True},
    "haploid_sensitive": {"is_haploid_sensitive_mode_enabled": True},
    "long_indel": {"enable_long_indel": True, "is_show_reference": True},
    "qual_iupac": {"quality_score_for_pass": 12.0, "keep_iupac_bases": True},
}


def record_sequences(y, bases, out_dim):
    """Attempt order of the reference's own output_from with always-failing, recording alt-info helpers."""
    log = []

    def stub(*args, _find=False, **kwargs):
        f = sys._getframe(2 if _find else 1).f_locals
        flags = tuple(bool(f[n]) for n in FLAG_NAMES)
        cat = 1 + flags.index(True)
        entry = (cat, int(f["idx"]), np.float32(f["maximum_probability"]), flags)
        if not log or not (log[-1][0] == entry[0] and log[-1][1] == entry[1] and log[-1][2] == entry[2] and log[-1][3] == flags):
            log.append(entry)          # one attempt may call the helpers twice (InsIns, DelDel, InsDel)
        return ([], None) if _find else ""

    saved = CV.find_alt_base, CV.insertion_bases_using_alt_info_from, CV.deletion_bases_using_alt_info_from
    CV.find_alt_base = lambda *a, **k: stub(*a, _find=True, **k)
    CV.insertion_bases_using_alt_info_from = stub
    CV.deletion_bases_using_alt_info_from = stub
    cfg = config(out_dim)
    rows, cats, idxs, probs, masks = [], [], [], [], []
    try:
        for i in range(len(y)):
            del log[:]
            seq = "a" * CENTER + str(bases[i]) + "c" * CENTER
            flags, _, p = CV.output_from(seq, "chr1", 100 + i, CENTER, *split(y[i], out_dim), cfg, None, {})
            assert flags[0], "every attempt fails, so the walk ends at homo_Ref"
            for cat, idx, prob, fl in log + [(0, 0, np.float32(p), (False,) * 9)]:
                rows.append(i)
                cats.append(cat)
                idxs.append(idx)
                probs.append(prob)
                masks.append((1 if cat == 0 else 0) | sum(1 << (b + 1) for b, v in enumerate(fl) if v))
    finally:
        CV.find_alt_base, CV.insertion_bases_using_alt_info_from, CV.deletion_bases_using_alt_info_from = saved
    return (np.array(rows, np.int32), np.array(cats, np.uint8), np.array(idxs, np.uint16), np.array(probs, np.float32),
            np.array(masks, np.uint16))


def rand_bases(r, n, alphabet="ACGT"):
    return "".join(r.choice(list(alphabet), size=n))


def alt_info_strings(r, n, centers):
    out = []
    for i in range(n):
        items = []
        c = centers[i]
        for b in r.choice(list("ACGT"), size=int(r.integers(0, 4)), replace=False):
            items.append(("X" + b, int(r.integers(1, 40))))
        for _ in range(int(r.integers(0, 4))):
            length = int(r.choice([1, 2, 3, 5, 8, 15, 16, 17, 30, 49, 60, 70, 120]))
            items.append(("I" + c + rand_bases(r, length), int(r.integers(1, 30))))
        for _ in range(int(r.integers(0, 4))):
            length = int(r.choice([1, 2, 3, 4, 6, 15, 16, 20, 45, 55, 64]))
            alphabet = "ACGT" if r.random() < 0.7 else "acgtRYN"
            items.append(("D" + rand_bases(r, length, alphabet), int(r.integers(1, 30))))
        if r.random() < 0.8:
            items.append(("R", int(r.integers(0, 50))))
        r.shuffle(items)
        depth = int(r.integers(1, 8)) if r.random() < 0.05 else int(r.integers(20, 120))
        dedup = {}
        for k, v in items:
            dedup.setdefault(k, v)
        body = " ".join("%s %d" % kv for kv in dedup.items())
        out.append("%d-%s" % (depth, body) if body else "%d" % depth)
    return out


def real_outputs(r, out_dim, n):
    y = np.concatenate([dirichlet_rows(r, n - n // 4, out_dim), quarter_rows(r, n // 4, out_dim)])
    # a share of confident reference rows so that showRef has early-out rows to print
    for i in r.choice(len(y), size=len(y) // 5, replace=False):
        y[i, 21] = np.float32(0.9)
        y[i, :21] = np.float32(0.02)
        y[i, [0, 4, 7, 9]] = np.float32(0.8)
        if out_dim == 90:
            y[i, 24 + 16] = y[i, 57 + 16] = np.float32(0.9)
    centers = [str(b) for b in r.choice(list("ACGTACGTACGTRYKMN"), size=len(y))]
    seqs = [rand_bases(r, CENTER, "acgtACGT") + c + rand_bases(r, CENTER, "acgtACGT") for c in centers]
    pos = ["chr%d:%d:%s" % (1 + i % 3, 1000 + 7 * i, s) for i, s in enumerate(seqs)]
    pos[1] = "HLA-A*01:01:01:01:%d:%s" % (77, seqs[1])                           # contig name with ':' in it
    alts = alt_info_strings(r, len(y), [BASE2ACGT[c] for c in centers])
    res = {"y": y, "pos": np.array(pos), "alt": np.array(alts)}
    cfg = config(out_dim, enable_long_indel=False)
    cfg_long = config(out_dim, enable_long_indel=True)
    for tag, c in (("", cfg), ("_long", cfg_long)):
        flags, refs, alts_o, probs = [], [], [], []
        for i in range(len(y)):
            _, depth_alt = alts[i].split("-", 1) if "-" in alts[i] else (alts[i], "")
            seqs_ = depth_alt.split(" ")
            d = dict(zip(seqs_[::2], [int(v) for v in seqs_[1::2]])) if depth_alt else {}
            fl, (rb, ab), p = CV.output_from(seqs[i], "chr", 1, CENTER, *split(y[i], out_dim), c, None, d)
            flags.append(np.array(fl, dtype=np.uint8))
            refs.append(rb)
            alts_o.append(ab)
            probs.append(np.float32(p))
        res["of_flags" + tag] = np.array(flags)
        res["of_ref" + tag] = np.array(refs)
        res["of_alt" + tag] = np.array(alts_o)
        res["of_prob" + tag] = np.array(probs, dtype=np.float32)
    for name, kw in CONFIGS.items():
        res["text_" + name] = np.array(CV.batch_output(pos, alts, y, config(out_dim, **kw), None))
    return res


def main():
    r = np.random.Generator(np.random.PCG64(3031))
    out = {}
    for out_dim in (24, 90):
        y, bases = test_rows(r, out_dim)
        gt = np.array([gt21_enum_from_label(b + b) for b in bases], dtype=np.uint8)
        rows, cats, idxs, probs, masks = record_sequences(y, bases, out_dim)
        out.update({"seq_y%d" % out_dim: y, "seq_gt%d" % out_dim: gt, "seq_row%d" % out_dim: rows, "seq_cat%d" % out_dim: cats,
                    "seq_idx%d" % out_dim: idxs, "seq_prob%d" % out_dim: probs, "seq_mask%d" % out_dim: masks})
        print(out_dim, "rows", len(y), "attempts", len(rows), "max walk", np.bincount(rows).max())
        for k, v in real_outputs(r, out_dim, 400).items():
            out["real%d_%s" % (out_dim, k)] = v
        print(out_dim, {name: out["real%d_text_%s" % (out_dim, name)].item().count("\n") for name in CONFIGS})
    np.savez_compressed(os.path.join(HERE, "decode_stage2.npz"), **out)


if __name__ == "__main__":
    main()
