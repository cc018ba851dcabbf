"""Cost of the decoder with GPU ranking (``c3b_decode_stage1`` + ``c3b_decode_stage2`` + ``clair3_b200.decode``).

    python tools/bench_decode.py [--iters 200] [--sites 4096]
    CLAIR3_REFERENCE=/path/to/Clair3 python tools/bench_decode.py --reference      # CPU only: the reference's decoder

With a GPU it prints one JSON line per measurement:

* ``device``: device time of stage 1 + stage 2 (k = 16, chained on ``nonref_idx`` / ``n_nonref``) per 256-site Clair3_F batch
  (90 outputs) and per 1024-site Clair3_P batch (24 outputs), from CUDA events around ``--iters`` back-to-back batches;
* ``host``: wall time of ``decode.batch_output`` per non-reference site on seeded rows and alt_info strings, split into the
  time spent in the two stage calls (host pointers: copies and synchronisation included) and the host walk + formatting.

``--reference`` (no GPU needed; reads the reference named by ``CLAIR3_REFERENCE``) times the reference's own ``batch_output``
on the same rows, and the host walk of ``decode.batch_output`` with the numpy oracle standing in for the GPU stages, both per
non-reference site on this CPU.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from clair3_b200 import decode  # noqa: E402


def rows(n, out_dim, seed):
    """Softmax heads at mixed temperatures with a third of the sites confidently homozygous-reference, seeded alt_info."""
    r = np.random.default_rng(seed)
    bounds = [0, 21, 24, 57, 90][: (5 if out_dim == 90 else 3)]
    y = np.empty((n, out_dim), dtype=np.float32)
    scale = r.choice([0.3, 2.0, 6.0], size=(n, 1))
    for lo, hi in zip(bounds, bounds[1:]):
        z = np.exp(r.standard_normal((n, hi - lo)) * scale)
        y[:, lo:hi] = z / z.sum(1, keepdims=True)
    bases = r.choice(list("ACGT"), size=n)
    ref = r.random(n) < 1 / 3
    col = np.array([decode.GT21_OF_BASE[b] for b in bases])
    y[ref, :21] = np.float32(0.01)
    y[ref, col[ref]] = np.float32(0.8)
    y[ref, 21] = np.float32(0.9)
    if out_dim == 90:
        y[ref, 40] = y[ref, 73] = np.float32(0.9)
    pos, alts = [], []
    for i in range(n):
        seq = "".join(r.choice(list("ACGT"), size=16)) + bases[i] + "".join(r.choice(list("ACGT"), size=16))
        pos.append("chr20:%d:%s" % (100 + i, seq))
        items = ["X%s %d" % (b, r.integers(1, 30)) for b in r.choice(list("ACGT"), size=int(r.integers(0, 3)), replace=False)]
        items += ["I%s%s %d" % (bases[i], "".join(r.choice(list("ACGT"), size=int(r.integers(1, 12)))), r.integers(1, 20))
                  for _ in range(int(r.integers(0, 3)))]
        items += ["D%s %d" % ("".join(r.choice(list("ACGT"), size=int(r.integers(1, 12)))), r.integers(1, 20))
                  for _ in range(int(r.integers(0, 3)))]
        items.append("R %d" % r.integers(0, 40))
        alts.append("%d-%s" % (r.integers(20, 90), " ".join(items)))
    return y, pos, alts


class Timed:
    """Wraps a model's decode stages and accumulates their wall time."""

    def __init__(self, m):
        self.m, self.t = m, 0.0

    def decode_stage1(self, *a, **k):
        t0 = time.perf_counter()
        out = self.m.decode_stage1(*a, **k)
        self.t += time.perf_counter() - t0
        return out

    def decode_stage2(self, *a, **k):
        t0 = time.perf_counter()
        out = self.m.decode_stage2(*a, **k)
        self.t += time.perf_counter() - t0
        return out


def host_cost(m, out_dim, sites, batch, seed=5):
    y, pos, alts = rows(sites, out_dim, seed)
    cfg = decode.replay_config(pileup=out_dim == 24, add_indel_length=out_dim == 90)
    tm = Timed(m)
    decode.batch_output(tm, pos[:batch], alts[:batch], y[:batch], cfg)        # warm-up
    tm.t = 0.0
    nonref = 0
    for s in range(0, sites, batch):
        d = tm.decode_stage1(y[s:s + batch], np.array([decode.GT21_OF_BASE[p[-17]] for p in pos[s:s + batch]], np.uint8))
        nonref += int(np.asarray(d["n_nonref"].cpu() if hasattr(d["n_nonref"], "cpu") else d["n_nonref"])[0])
    tm.t = 0.0
    t0 = time.perf_counter()
    for s in range(0, sites, batch):
        decode.batch_output(tm, pos[s:s + batch], alts[s:s + batch], y[s:s + batch], cfg)
    total = time.perf_counter() - t0
    return {"sites": sites, "nonref_sites": nonref, "us_per_nonref_site": 1e6 * total / nonref,
            "stage_calls_us_per_nonref_site": 1e6 * tm.t / nonref, "walk_us_per_nonref_site": 1e6 * (total - tm.t) / nonref}


def gpu(args):
    import torch

    from clair3_b200 import synth
    from clair3_b200.model import Clair3_F, Clair3_P
    f = Clair3_F(add_indel_length=True, predict=True, input_channels=8)
    f.to(torch.device("cuda"))
    f.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=8, seed=1).items()})
    p = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    p.to(torch.device("cuda"))
    p.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()})
    for name, m, out_dim, batch in (("Clair3_F", f, 90, 256), ("Clair3_P", p, 24, 1024)):
        y, pos, _ = rows(batch, out_dim, seed=out_dim)
        yd = torch.from_numpy(y).cuda()
        gd = torch.from_numpy(np.array([decode.GT21_OF_BASE[s[-17]] for s in pos], np.uint8)).cuda()

        def once():
            s1 = m.decode_stage1(yd, gd)
            return m.decode_stage2(yd, gd, sites=s1["nonref_idx"], n_sites=s1["n_nonref"], k=16)

        for _ in range(20):
            once()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            once()
        e1.record()
        e1.synchronize()
        us = 1e3 * e0.elapsed_time(e1) / args.iters
        # the events above include the gaps while Python issues each call; the profiler reports the kernels' own time
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                once()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "decode_stage" in ev.key:
                kern["stage1" if "stage1" in ev.key else "stage2"] = ev.device_time_total / args.iters
        print(json.dumps({"measure": "device", "model": name, "out_dim": out_dim, "batch_sites": batch, "k": 16,
                          "us_per_batch_stage1_plus_stage2": round(us, 2),
                          "kernel_us_per_batch": {k: round(v, 2) for k, v in sorted(kern.items())}, "iters": args.iters,
                          "device": torch.cuda.get_device_name()}), flush=True)
        res = host_cost(m, out_dim, args.sites, batch)
        print(json.dumps({"measure": "host", "model": name, "out_dim": out_dim, "batch_sites": batch,
                          **{k: (round(v, 2) if isinstance(v, float) else v) for k, v in res.items()}}), flush=True)


def reference(args):
    sys.path.insert(0, os.environ["CLAIR3_REFERENCE"])
    import clair3.CallVariants as CV

    from oracle import decode_oracle as dec1
    from oracle import decode_stage2_oracle as dec2

    class OracleStages:
        def decode_stage1(self, y, g):
            return dec1.decode_stage1(y, g)

        def decode_stage2(self, y, g, sites=None, n_sites=None, k=16):
            return dec2.decode_stage2(y, g, sites, n_sites, k)

    for out_dim, batch in ((90, 256), (24, 1024)):
        y, pos, alts = rows(args.sites, out_dim, seed=5)
        cfg = CV.OutputConfig(**decode.replay_config(pileup=out_dim == 24, add_indel_length=out_dim == 90)._asdict())
        nonref = sum(int(dec1.decode_stage1(y[s:s + batch], np.array([decode.GT21_OF_BASE[p[-17]] for p in pos[s:s + batch]],
                                                                          np.uint8))["n_nonref"][0]) for s in range(0, args.sites, batch))
        t0 = time.perf_counter()
        ref_text = "".join(CV.batch_output(pos[s:s + batch], alts[s:s + batch], y[s:s + batch], cfg, None)
                           for s in range(0, args.sites, batch))
        t_ref = time.perf_counter() - t0
        res = host_cost(OracleStages(), out_dim, args.sites, batch)
        ours = "".join(decode.batch_output(OracleStages(), pos[s:s + batch], alts[s:s + batch], y[s:s + batch],
                                           decode.replay_config(out_dim == 24, out_dim == 90)) for s in range(0, args.sites, batch))
        print(json.dumps({"measure": "reference_cpu", "out_dim": out_dim, "sites": args.sites, "nonref_sites": nonref,
                          "reference_us_per_nonref_site": round(1e6 * t_ref / nonref, 2),
                          "host_walk_us_per_nonref_site": round(res["walk_us_per_nonref_site"], 2),
                          "same_text": ours == ref_text}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--sites", type=int, default=4096)
    ap.add_argument("--reference", action="store_true", help="CPU only: time the reference's batch_output (CLAIR3_REFERENCE)")
    args = ap.parse_args()
    if args.reference:
        reference(args)
    else:
        gpu(args)


if __name__ == "__main__":
    main()
