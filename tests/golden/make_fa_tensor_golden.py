"""Mint tests/golden/fa_tensor.npz from the reference's own calculate_clair3_full_alignment, compiled by oracle/fa_ref.py
(CLAIR3_REFERENCE must point at the reference checkout when oracle/_ref is not built yet):

    CLAIR3_REFERENCE=/path/to/Clair3 python tests/golden/make_fa_tensor_golden.py

Records, candidates, phased variants and parameters in; matrix, all_alt_info strings and the number of rand() draws out.  The
case has more reads than rows at some candidates (so the shuffle is exercised), haplotagging and dwell time on."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from clair3_b200 import synth_reads as sr          # noqa: E402
from oracle import fa_ref                          # noqa: E402

PARAMS = dict(need_haplotagging=True, min_mq=5, matrix_depth=55, max_indel_length=50, enable_dwell_time=True, rand_seed=1,
              rand_skip=0)
FIELDS = ("pos", "flag", "mapq", "cigar_off", "cigar", "seq_off", "seq", "l_qseq", "qual", "qual_off", "qname", "qname_off", "mv",
          "mv_off")


def main():
    rec, ref, cand, var = sr.random_fa_case(21, region_len=1500, depth=70, read_len=900, n_cand=24, n_var=10, dwell=True)
    m, alt, draws = fa_ref.full_alignment(rec, cand, ref, variants=var, **PARAMS)
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fa_tensor.npz")
    np.savez_compressed(out, **{k: rec[k] for k in FIELDS}, ref=np.frombuffer(ref.encode(), np.uint8), candidates=cand,
                        var_pos=np.array([v[0] for v in var], np.int32), var_ref=np.array([v[1] for v in var]),
                        var_alt=np.array([v[2] for v in var]), var_gt=np.array([v[3] for v in var], np.int32),
                        var_ps=np.array([v[4] for v in var], np.int32), matrix=m, alt_info=np.array(alt), draws=np.int64(draws),
                        params=np.array(repr(PARAMS)))
    print("%s: %d candidates, %d reads, %d draws, %d bytes" % (out, len(cand), len(rec["pos"]), draws, os.path.getsize(out)))


if __name__ == "__main__":
    main()
