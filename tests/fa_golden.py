"""Shared by the full-alignment tests: the golden fixture's inputs and outputs as the builder and the oracle take them."""
import ast
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fa_tensor.npz")
RECORD_FIELDS = ("pos", "flag", "mapq", "cigar_off", "cigar", "seq_off", "seq", "l_qseq", "qual", "qual_off", "qname", "qname_off",
                 "mv", "mv_off")


def load_fa_golden():
    """(records, ref_seq, candidates, variants, params, matrix, alt_info strings, draws)."""
    z = np.load(GOLDEN)
    rec = {k: z[k] for k in RECORD_FIELDS}
    ref = z["ref"].tobytes().decode()
    var = [(int(p), str(r), str(a), int(g), int(s)) for p, r, a, g, s in
           zip(z["var_pos"], z["var_ref"], z["var_alt"], z["var_gt"], z["var_ps"])]
    return rec, ref, z["candidates"], var, ast.literal_eval(str(z["params"])), z["matrix"], [str(s) for s in z["alt_info"]], int(z["draws"])


def builder_kwargs(params):
    """oracle.fa_ref.full_alignment keyword arguments -> FullAlignmentBuilder.build keyword arguments."""
    p = dict(params)
    p["dwell"] = p.pop("enable_dwell_time")
    return p
