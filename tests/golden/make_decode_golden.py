"""Mint the golden vectors of the decoder's first stage from the REAL reference (a Clair3 checkout, named by CLAIR3_REFERENCE).

    CLAIR3_REFERENCE=/path/to/Clair3 PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_decode_golden.py

Calls the reference's own ``possible_outcome_probabilites_from`` and ``quality_score_from``
(``clair3/CallVariants.py:510-576,375-381``) and ``gt21_enum_from_label`` site by site on seeded
probability rows (a mix of confident homozygous-reference rows, confident variants and rows sitting exactly on the 0.5
thresholds) and stores inputs + the early-out flag, the returned probability and the un-rounded QUAL as a small ``.npz``.
"""
import os
import sys
from math import log

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ["CLAIR3_REFERENCE"])
sys.dont_write_bytecode = True

from clair3.CallVariants import Phred_Trans, possible_outcome_probabilites_from, quality_score_from  # noqa: E402
from clair3.task.gt21 import gt21_enum_from_label  # noqa: E402


def rows(r, n, out_dim):
    y = np.zeros((n, out_dim), dtype=np.float32)
    bounds = [0, 21, 24, 57, 90][: (5 if out_dim == 90 else 3)]
    for lo, hi in zip(bounds, bounds[1:]):
        conc = r.choice([0.05, 0.3, 2.0], size=n)
        for i in range(n):
            y[i, lo:hi] = r.dirichlet(np.full(hi - lo, conc[i])).astype(np.float32)
    return y


def main():
    r = np.random.Generator(np.random.PCG64(2024))
    out = {}
    for out_dim in (24, 90):
        n = 600
        y = rows(r, n, out_dim)
        bases = r.choice(list("ACGT"), size=n)
        # rows exactly on / next to the thresholds
        for i in range(0, 40):
            g = int(gt21_enum_from_label(bases[i] * 2))
            y[i, 21] = np.float32(0.5) if i % 2 == 0 else np.nextafter(np.float32(0.5), np.float32(0))
            y[i, g] = np.float32(0.5) if i % 3 else np.nextafter(np.float32(0.5), np.float32(0))
            if out_dim == 90:
                y[i, 24 + 16] = np.float32(0.5) if i % 5 else np.float32(0.4999)
                y[i, 57 + 16] = np.float32(0.75)
        for i in range(40, 300):       # confident reference calls
            g = int(gt21_enum_from_label(bases[i] * 2))
            y[i, 21] = np.float32(r.uniform(0.5, 1.0))
            y[i, g] = np.float32(r.uniform(0.5, 1.0))
            if out_dim == 90:
                y[i, 24 + 16] = np.float32(r.uniform(0.45, 1.0))
                y[i, 57 + 16] = np.float32(r.uniform(0.45, 1.0))
        early = np.zeros(n, dtype=np.uint8)
        prob = np.zeros(n, dtype=np.float32)
        qual = np.zeros(n, dtype=np.float64)
        qual_rounded = np.zeros(n, dtype=np.float64)
        ref_gt21 = np.zeros(n, dtype=np.uint8)
        for i in range(n):
            ref_gt21[i] = int(gt21_enum_from_label(bases[i] * 2))
            vl1 = y[i, 24:57] if out_dim == 90 else 0
            vl2 = y[i, 57:90] if out_dim == 90 else 0
            res = possible_outcome_probabilites_from(y[i, :21], y[i, 21:24], vl1, vl2, reference_base=str(bases[i]),
                                                     alt_info_dict={}, add_indel_length=(out_dim == 90))
            early[i] = 1 if len(res) == 1 else 0
            p = res[0]                                     # homo_Ref_probability is element 0 in both shapes of the result
            prob[i] = p
            qual_rounded[i] = quality_score_from(p)
            qual[i] = max(Phred_Trans * log(((1.0 - p) + 1e-10) / (p + 1e-10)) + 10, 0)    # quality_score_from without round()
        out["y%d" % out_dim] = y
        out["bases%d" % out_dim] = np.array("".join(bases))
        out["ref_gt21_%d" % out_dim] = ref_gt21
        out["early%d" % out_dim] = early
        out["prob%d" % out_dim] = prob
        out["qual%d" % out_dim] = qual
        out["qual_rounded%d" % out_dim] = qual_rounded
    np.savez_compressed(os.path.join(HERE, "decode_stage1.npz"), **out)
    print("early-out fraction:", out["early24"].mean(), out["early90"].mean())


if __name__ == "__main__":
    main()
