"""Mint golden vectors from the REAL reference (a Clair3 checkout, named by CLAIR3_REFERENCE).

    CLAIR3_REFERENCE=/path/to/Clair3 PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden.py

Imports the reference's ``clair3/model.py`` unmodified, loads the seeded synthetic checkpoints of
``clair3_b200.synth`` through the reference's own ``load_state_dict`` (strict), runs the fp32 CPU
forward under ``torch.inference_mode`` exactly like ``_torch_predict``
(``clair3/CallVariantsFromCffi.py:48-52``) and stores outputs plus intermediate taps as small
``.npz`` fixtures.  Inputs/weights are NOT stored: tests rebuild them from the recorded seeds.
The tests read only the committed fixtures.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ["CLAIR3_REFERENCE"])
sys.dont_write_bytecode = True

from clair3.model import Clair3_P, Clair3_F  # noqa: E402  (the reference)
from clair3_b200 import synth  # noqa: E402

CASES = [
    # name, kind, kwargs
    ("p24", "pileup", dict(add_indel_length=False, batch=48, seed=1, realistic=True, dtype="int32")),
    ("p90", "pileup", dict(add_indel_length=True, batch=16, seed=2, realistic=False, dtype="int32")),
    ("p24_int8", "pileup", dict(add_indel_length=False, batch=8, seed=6, realistic=True, dtype="int8")),
    ("f8", "fa", dict(add_indel_length=True, batch=12, seed=3, depth=89, channels=8, realistic=True, conv_taps=True)),
    ("f9_dwell", "fa", dict(add_indel_length=True, batch=6, seed=4, depth=89, channels=9, realistic=True)),
    ("f55", "fa", dict(add_indel_length=True, batch=6, seed=5, depth=55, channels=8, realistic=True)),
    ("f8_24", "fa", dict(add_indel_length=False, batch=4, seed=7, depth=89, channels=8, realistic=False)),
]


def to_torch_sd(sd):
    return {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}


def run_case(name, kind, kw):
    torch.manual_seed(0)
    taps = {}
    if kind == "pileup":
        sd = synth.pileup_state_dict(kw["add_indel_length"], seed=kw["seed"])
        x = synth.pileup_inputs(kw["batch"], seed=kw["seed"], realistic=kw["realistic"], dtype=np.dtype(kw["dtype"]))
        m = Clair3_P(add_indel_length=kw["add_indel_length"], predict=True, input_channels=18)
        m.LSTM1.register_forward_hook(lambda mod, i, o: taps.__setitem__("lstm1", o[0].numpy().copy()))
        m.LSTM2.register_forward_hook(lambda mod, i, o: taps.__setitem__("lstm2", o[0].numpy().copy()))
        m.L4.register_forward_hook(lambda mod, i, o: taps.__setitem__("l4_pre", o.numpy().copy()))
    else:
        sd = synth.fa_state_dict(kw["add_indel_length"], channels=kw["channels"], seed=kw["seed"])
        x = synth.fa_inputs(kw["batch"], depth=kw["depth"], channels=kw["channels"], seed=kw["seed"],
                            realistic=kw["realistic"])
        m = Clair3_F(add_indel_length=kw["add_indel_length"], predict=True, input_channels=kw["channels"])
        for tap in ("conv1", "res_block1", "conv3", "res_block2", "conv5", "res_block3"):
            getattr(m, tap).register_forward_hook(
                lambda mod, i, o, tap=tap: taps.__setitem__(tap, o.numpy().copy()))
        m.pyramidpolling.register_forward_hook(lambda mod, i, o: taps.__setitem__("spp", o.numpy().copy()))
        m.L4.register_forward_hook(lambda mod, i, o: taps.__setitem__("l4_pre", o.numpy().copy()))
    m.eval()
    missing = m.load_state_dict(to_torch_sd(sd), strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    with torch.inference_mode():
        y = m(torch.from_numpy(x)).detach().cpu().numpy()
    out = {"y": y.astype(np.float32)}
    keep_sites = 2
    for k, v in taps.items():
        if k in ("conv1", "res_block1", "conv3", "res_block2", "conv5", "res_block3"):
            if not kw.get("conv_taps"):
                continue
            out["tap_" + k] = v[:1].astype(np.float32)
        elif k in ("lstm1", "lstm2"):
            out["tap_" + k] = v[:keep_sites].astype(np.float32)
        else:
            out["tap_" + k] = v.astype(np.float32)
    meta = dict(kw)
    meta["kind"] = kind
    meta["torch"] = torch.__version__
    out["meta"] = np.array(repr(meta))
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **out)
    print(name, y.shape, "row sums", y.sum(1)[:3], os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    for c in CASES:
        run_case(*c)
