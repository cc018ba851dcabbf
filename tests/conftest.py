import ast
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with `pytest -m gpu` on a GPU machine)")


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests need an H100 (compute capability 9.0): skip them cleanly anywhere else, so a plain `pytest` on a CPU
    host passes instead of dying in the CUDA driver."""
    try:
        import torch
        ok = torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0)
    except Exception:
        ok = False
    if ok:
        return
    skip = pytest.mark.skip(reason="needs an H100 (sm_90) GPU")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    meta = ast.literal_eval(str(z["meta"]))
    return z, meta


def golden_case(name):
    """Rebuild (state_dict, inputs) from the seeds recorded in a golden fixture."""
    from clair3_b200 import synth
    z, meta = load_golden(name)
    if meta["kind"] == "pileup":
        sd = synth.pileup_state_dict(meta["add_indel_length"], seed=meta["seed"])
        x = synth.pileup_inputs(meta["batch"], seed=meta["seed"], realistic=meta["realistic"],
                                dtype=np.dtype(meta["dtype"]))
    else:
        sd = synth.fa_state_dict(meta["add_indel_length"], channels=meta["channels"], seed=meta["seed"])
        x = synth.fa_inputs(meta["batch"], depth=meta["depth"], channels=meta["channels"],
                            seed=meta["seed"], realistic=meta["realistic"])
    return z, meta, sd, x


GOLDEN_PILEUP = ["p24", "p90", "p24_int8"]
GOLDEN_FA = ["f8", "f9_dwell", "f55", "f8_24"]
