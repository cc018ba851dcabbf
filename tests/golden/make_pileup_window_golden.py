"""Mints tests/golden/pileup_window_cases.npz from the reference's own CreateTensorPileup (preprocess/CreateTensorPileupFromCffi.py,
run live by oracle/pileup_tensor_ref.py; needs the reference checkout: CLAIR3_REFERENCE or a sibling directory).

Per case of tests/plp_window_cases.py (the inputs are rebuilt from that module's code): ``<name>/positions`` the 1-based
positions of the windows the reference keeps, in its order; ``<name>/tensors`` int32 [k, 33, 18] those windows;
``<name>/pos_info`` / ``<name>/alt_info`` its ``"ctg:pos:ref_base"`` and ``"depth-alt"`` strings.  These pin the C oracle and
the GPU counter's window verdicts and gather where the reference checkout is absent (the GPU machines).
    python tests/golden/make_pileup_window_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import pileup_tensor_ref as ptr  # noqa: E402
import plp_window_cases as cases  # noqa: E402

if not ptr.available():
    sys.exit("the reference checkout is needed: set CLAIR3_REFERENCE")

out = {"names": np.array(cases.IDS)}
for name, build in cases.ALL:
    c = build()
    tensors, pos_info, alt_info = ptr.create_tensor_pileup(c["records"], c["ref"], c["ref_start"], c["ctg_start"], c["ctg_end"],
                                                           **c["kw"])
    out["%s/positions" % name] = ptr.kept_positions(pos_info)
    out["%s/tensors" % name] = tensors.astype(np.int32)
    out["%s/pos_info" % name] = np.array(pos_info, dtype=str)
    out["%s/alt_info" % name] = np.array(alt_info, dtype=str)
np.savez_compressed(os.path.join(ROOT, "tests", "golden", "pileup_window_cases.npz"), **out)
print("%d cases, %d windows" % (len(cases.IDS), sum(len(out["%s/positions" % n]) for n in cases.IDS)))
