"""ORACLE (timing port) — test/bench infrastructure only, never imported by the product path.

The reference's CPU implementation of the hot path is ``torch.nn`` modules executed by ATen/oneDNN
(``clair3/model.py:96-125,130-161`` pileup; ``:183-279,317-416`` full-alignment), run under
``torch.inference_mode`` by ``_torch_predict`` (``clair3/CallVariantsFromCffi.py:48-52``).
The reference's source is not part of this repository, so this file restates the two forwards with the
same torch CPU operators (``torch.lstm``, ``conv2d``, ``batch_norm``, ``max_pool2d``, ``linear``,
``selu``, ``softmax``) so ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs time the very
kernels the reference would execute (kind = "port").  Pinned against the golden fixtures minted
from the real reference in ``tests/test_oracle.py``.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F


def _t(sd):
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in sd.items()}


class PileupPort:
    """Clair3_P.forward restated with torch CPU ops (clair3/model.py:130-161)."""

    def __init__(self, sd, add_indel_length=False):
        self.sd = _t(sd)
        self.add_indel_length = add_indel_length
        self.flat = {}
        for name in ("LSTM1", "LSTM2"):
            self.flat[name] = [self.sd[f"{name}.{p}_l0{s}"] for s in ("", "_reverse")
                               for p in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]

    def _lstm(self, x, name, hidden):
        b = x.shape[0]
        h0 = x.new_zeros(2, b, hidden)
        out, _, _ = torch.lstm(x, (h0, h0.clone()), self.flat[name], True, 1, 0.0, False, True, True)
        return out

    def __call__(self, x):
        sd = self.sd
        with torch.inference_mode():
            x = torch.as_tensor(x).float()
            x = self._lstm(x, "LSTM1", 128)
            x = self._lstm(x, "LSTM2", 160)
            x = torch.flatten(x, 1)
            x = F.selu(F.linear(x, sd["L4.weight"], sd["L4.bias"]))
            return _heads(x, sd, self.add_indel_length)


def _heads(x, sd, add_indel_length):
    names = [("L5_1", "Y_gt21_logits"), ("L5_2", "Y_genotype_logits")]
    if add_indel_length:
        names += [("L5_3", "Y_indel_length_logits_1"), ("L5_4", "Y_indel_length_logits_2")]
    outs = []
    for l5, y in names:
        z = F.selu(F.linear(x, sd[f"{l5}.weight"], sd[f"{l5}.bias"]))
        z = F.selu(F.linear(z, sd[f"{y}.weight"], sd[f"{y}.bias"]))
        outs.append(torch.softmax(z, dim=-1))
    return torch.cat(outs, dim=1)


class FullAlignmentPort:
    """Clair3_F.forward restated with torch CPU ops (clair3/model.py:377-416)."""

    def __init__(self, sd, add_indel_length=True):
        self.sd = _t(sd)
        self.add_indel_length = add_indel_length
        self.cin = self.sd["conv1.conv.weight"].shape[1]

    def _cbr(self, x, conv, bn, stride, relu=True):
        sd = self.sd
        x = F.conv2d(x, sd[f"{conv}.weight"], sd[f"{conv}.bias"], stride=stride, padding=1)
        x = F.batch_norm(x, sd[f"{bn}.running_mean"], sd[f"{bn}.running_var"], sd[f"{bn}.weight"],
                         sd[f"{bn}.bias"], False, 0.0, 1e-3)
        return F.relu(x) if relu else x

    def _block(self, x, p):
        y = self._cbr(x, f"{p}.conv1", f"{p}.bn1", 1)
        y = self._cbr(y, f"{p}.conv2", f"{p}.bn2", 1, relu=False)
        return F.relu(x + y)

    @staticmethod
    def _spp(x):
        pooled = []
        h, w = x.shape[-2:]
        for p in (3, 2, 1):
            wh, ww = math.ceil(h / p), math.ceil(w / p)
            oh, ow = math.ceil(h / wh), math.ceil(w / ww)
            ph = max((oh - 1) * wh + wh - h, 0)
            pw = max((ow - 1) * ww + ww - w, 0)
            xp = F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2)) if (ph or pw) else x
            mp = F.max_pool2d(xp, (wh, ww), (wh, ww)).permute(0, 2, 3, 1)
            pooled.append(torch.flatten(mp, 1))
        return torch.cat(pooled, 1)

    def __call__(self, x):
        sd = self.sd
        with torch.inference_mode():
            x = torch.as_tensor(x).float() / 100.0
            if x.ndim == 4 and x.shape[-1] == self.cin:
                x = x.permute(0, 3, 1, 2)
            x = self._cbr(x, "conv1.conv", "conv1.bn", 2)
            x = self._block(x, "res_block1.0")
            x = self._cbr(x, "conv3.conv", "conv3.bn", 2)
            x = self._block(x, "res_block2.0")
            x = self._cbr(x, "conv5.conv", "conv5.bn", 2)
            x = self._block(x, "res_block3.0")
            x = self._spp(x)
            x = F.selu(F.linear(x, sd["L4.weight"], sd["L4.bias"]))
            return _heads(x, sd, self.add_indel_length)


if __name__ == "__main__":
    # Worker of bench.py's cpu_baseline "deployment shape" leg: one single-threaded process of the reference's CPU forward
    # (what `--threads 1` gives each worker, clair3/CallVariantsFromCffi.py:56-63), run N at a time and summed by the caller.
    #   python -m oracle.torch_port <pileup|fa> <seconds> <sites per call>
    import json
    import sys
    import time

    from clair3_b200 import synth

    workload, seconds, sites = sys.argv[1], float(sys.argv[2]), int(sys.argv[3])
    steps = int(sys.argv[4]) if len(sys.argv) > 4 else 0      # > 0: exactly that many calls, sized to take ~`seconds` in total
    torch.set_num_threads(1)
    full = 1024 if workload == "pileup" else 256
    if workload == "pileup":
        port = PileupPort(synth.pileup_state_dict(False, seed=0), False)
        make = synth.pileup_inputs
    else:
        port = FullAlignmentPort(synth.fa_state_dict(True, channels=8, seed=0), True)
        make = synth.fa_inputs
    x = make(sites, seed=900)
    port(x)
    if steps > 0:
        t0 = time.perf_counter()
        port(x)
        rate = sites / (time.perf_counter() - t0)
        sites = max(8, min(full, int(rate * seconds / steps) // 8 * 8))
        x = make(sites, seed=900)
        port(x)
    t0 = time.perf_counter()
    n = 0
    while (n < steps) if steps > 0 else (time.perf_counter() - t0 < seconds):
        port(x)
        n += 1
    print(json.dumps({"sites": n * sites, "seconds": time.perf_counter() - t0, "sites_per_call": sites, "calls": n}), flush=True)
