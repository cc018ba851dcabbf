"""Cost of the decoder with GPU ranking (``c3b_decode_stage1`` + ``c3b_decode_stage2`` + ``clair3_b200.decode``).

    python tools/bench_decode.py [--iters 200] [--sites 4096]
    CLAIR3_REFERENCE=/path/to/Clair3 python tools/bench_decode.py --reference      # CPU only: the reference's decoder

With a GPU it prints one JSON line per measurement:

* ``device``: device time of stage 1 + stage 2 (k = 16, chained on ``nonref_idx`` / ``n_nonref``) per 256-site Clair3_F batch
  (90 outputs) and per 1024-site Clair3_P batch (24 outputs), from CUDA events around ``--iters`` back-to-back batches;
* ``device_calls``: device time per batch of each kernel ``c3b_decode_calls`` launches (device pointers, k = 16);
* ``host``, ``route: host_walk``: wall time of ``decode.batch_output`` with only the two stages (the host walk) per
  non-reference site on seeded rows and alt_info strings, split into the time spent in the two stage calls (host pointers:
  copies and synchronisation included) and the host walk + formatting;
* ``host``, ``route: device_calls``: the same rows through ``decode.batch_output``'s records route (``c3b_decode_calls`` on host
  pointers, then ``calls_text``), and the part of it spent formatting the rows.

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


def calls_cost(m, out_dim, sites, batch, nonref, seed=5):
    """decode.batch_output through the records route (decode.batch_calls + calls_text) on the same rows, per non-reference
    site: the whole call, and the part spent formatting the printed rows."""
    y, pos, alts = rows(sites, out_dim, seed)
    cfg = decode.replay_config(pileup=out_dim == 24, add_indel_length=out_dim == 90)
    decode.batch_output(m, pos[:batch], alts[:batch], y[:batch], cfg)        # warm-up
    t_fmt = 0.0
    t0 = time.perf_counter()
    for s in range(0, sites, batch):
        res = decode.batch_calls(m, pos[s:s + batch], alts[s:s + batch], y[s:s + batch], cfg)
        t1 = time.perf_counter()
        decode.calls_text(res, cfg)
        t_fmt += time.perf_counter() - t1
    total = time.perf_counter() - t0
    return {"sites": sites, "nonref_sites": nonref, "us_per_nonref_site": 1e6 * total / nonref,
            "row_format_us_per_nonref_site": 1e6 * t_fmt / nonref}


def card():
    """The GPU's name and power limit, as nvidia-smi reports them when the bench runs (part of every number)."""
    import subprocess
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    return {"device": out[0], "power_limit_w": float(out[1])} if len(out) == 2 else {"device": "unknown", "power_limit_w": None}


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
    gpu_card = card()
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
                          "kernel_us_per_batch": {k: round(v, 2) for k, v in sorted(kern.items())}, "iters": args.iters, **gpu_card}), flush=True)
        # stage 3 (c3b_decode_calls: stages 1 and 2, the walk, the full re-rank and the row counts), device pointers
        ab = [a.encode() for a in rows(batch, out_dim, seed=out_dim)[2]]
        off = np.zeros(batch + 1, np.int64)
        np.cumsum([len(a) for a in ab], out=off[1:])
        abd, offd = torch.from_numpy(np.frombuffer(b"".join(ab), np.uint8).copy()).cuda(), torch.from_numpy(off).cuda()
        rbd = torch.from_numpy(np.array([ord(s[-17]) for s in pos], np.uint8)).cuda()
        cfg = decode.replay_config(pileup=out_dim == 24, add_indel_length=out_dim == 90)
        for _ in range(5):
            m.decode_calls(yd, rbd, abd, offd, cfg)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                m.decode_calls(yd, rbd, abd, offd, cfg)
            torch.cuda.synchronize()
        calls_kern = {}
        for ev in prof.key_averages():
            if "decode" in ev.key or "calls_" in ev.key:
                key = next(n for n in ("decode_calls_kernel", "calls_compact", "calls_gt21", "stage1", "stage2") if n in ev.key)
                calls_kern[key] = calls_kern.get(key, 0.0) + ev.device_time_total / args.iters
        print(json.dumps({"measure": "device_calls", "model": name, "out_dim": out_dim, "batch_sites": batch, "k": 16,
                          "kernel_us_per_batch": {k: round(v, 2) for k, v in sorted(calls_kern.items())}, "iters": args.iters, **gpu_card}), flush=True)
        res = host_cost(m, out_dim, args.sites, batch)
        print(json.dumps({"measure": "host", "route": "host_walk", "model": name, "out_dim": out_dim, "batch_sites": batch,
                          **{k: (round(v, 2) if isinstance(v, float) else v) for k, v in res.items()}, **gpu_card}), flush=True)
        res = calls_cost(m, out_dim, args.sites, batch, res["nonref_sites"])
        print(json.dumps({"measure": "host", "route": "device_calls", "model": name, "out_dim": out_dim, "batch_sites": batch,
                          **{k: (round(v, 2) if isinstance(v, float) else v) for k, v in res.items()}, **gpu_card}), flush=True)


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
