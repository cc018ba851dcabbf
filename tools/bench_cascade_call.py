"""What a region costs through Clair3's pileup -> full-alignment cascade on the GPU, against the same calls assembled through
the host route.

    python tools/bench_cascade_call.py [--region 131072] [--iters 5] [--warmup 1] [--out FILE]

Writes the region of ``tools/bench_bam_decode.py`` (depth 40, ``--region`` columns, 8 kb reads and 150 bp reads, seeded) to a
temporary directory as an indexed BAM, with seeded ``Clair3_P(False)`` / ``Clair3_F(True, 8 channels)`` weights, and measures
in one process after warm-up:

* ``cascade.call_region`` (one ``BamDecoder.decode``, the counter, Clair3_P, the device selection, one full-alignment build
  per 10,000 candidates, Clair3_F, the merge): wall time, and wall and device time per stage (CUDA events at the stage
  boundaries), the full-alignment candidate count, and the host waits (``cudaStreamSynchronize`` / synchronous copies seen by
  ``torch.profiler`` in one profiled run of its own, when the profiler sees the library's runtime calls);
* ``cascade.call_region_host``: ``bam_io.read_bam`` -> count -> call -> host ``select`` -> host-candidate builds -> call ->
  ``merge``, with the merged body and the call records asserted identical.

The cut-offs are the region's own (``qual_cutoffs``, ont defaults).  Prints one JSON line with the card's name and power limit
read in the same run.  Needs an H100; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from clair3_b200 import bam_io, cascade, decode, synth, synth_reads as sr  # noqa: E402
from clair3_b200.model import Clair3_F, Clair3_P  # noqa: E402

CFG = dict(depth=40, indel_rate=0.04, origin=10000, seed=5)        # tools/bench_bam_decode.py
CFG_P = decode.replay_config(pileup=True, add_indel_length=False)._replace(is_show_reference=True)
CFG_F = decode.replay_config(pileup=False, add_indel_length=True)._replace(is_show_reference=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ")
    return name or torch.cuda.get_device_name(0), limit or "unknown"


def med(v):
    return float(np.median(v))


def host_waits(fn):
    """Synchronising runtime calls in one profiled run of fn (None when the profiler shows none at all)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
    names = [e.name for e in prof.events()]
    n = sum(1 for x in names if x in ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cudaEventSynchronize", "cudaMemcpy"))
    return n or None


def workload(tmp, read_len, region, models, ws, iters, warmup):
    rec, ref, rs = sr.random_alignment(region, depth=CFG["depth"], read_len=read_len, seed=CFG["seed"], indel_rate=CFG["indel_rate"],
                                       origin=CFG["origin"])
    path = os.path.join(tmp, "w%d.bam" % read_len)
    bam_io.write_bam(path, rec, [("ctg", rs + len(ref))])
    bam_io.write_bai(path)
    idx = bam_io.read_bai(path + ".bai")
    start, end = CFG["origin"], CFG["origin"] + region
    args = (path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F)

    def dev():
        r = cascade.call_region(*args, index=idx, workspaces=ws)
        torch.cuda.synchronize()
        return r

    def host():
        r = cascade.call_region_host(*args, workspaces=ws)
        torch.cuda.synchronize()
        return r

    for _ in range(warmup):
        a, b = dev(), host()
    same = bool(a["vcf"] == b["vcf"] and np.array_equal(a["candidates"], b["candidates"])
                and np.array_equal(a["pileup"]["calls"], b["pileup"]["calls"])
                and all(np.array_equal(x["calls"], y["calls"]) for x, y in zip(a["full_alignment"], b["full_alignment"])))
    t_dev, t_host, stages = [], [], []
    for _ in range(iters):
        t0 = time.perf_counter()
        r = dev()
        t1 = time.perf_counter()
        host()
        t2 = time.perf_counter()
        t_dev.append(1e3 * (t1 - t0))
        t_host.append(1e3 * (t2 - t1))
        stages.append(r["stages"])
    per_stage = [{"stage": s["stage"], "wall_ms": med([run[i]["wall_ms"] for run in stages]),
                  "device_ms": med([run[i]["device_ms"] for run in stages])} for i, s in enumerate(stages[0])]
    return {"read_len": read_len, "records": int(len(rec["pos"])), "pileup_calls": int(len(a["pileup"]["calls"])),
            "vcf_rows": a["vcf"].count("\n"), "qual_cutoffs": list(a["qual_cutoffs"]), "fa_candidates": int(len(a["candidates"])),
            "fa_builds": len(a["chunks"]), "call_region_ms": med(t_dev), "call_region_ms_min_max": [min(t_dev), max(t_dev)],
            "host_route_ms": med(t_host), "host_route_ms_min_max": [min(t_host), max(t_host)], "stages": per_stage,
            "host_waits_profiled": host_waits(dev), "identical": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--region", type=int, default=1 << 17)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cascade_call: needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda:0")
    p = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    p.to(dev)
    p.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()})
    f = Clair3_F(add_indel_length=True, predict=True, input_channels=8)
    f.to(dev)
    f.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=8, seed=1).items()})
    ws = cascade.Workspaces(0)
    line = {"bench": "cascade_call", "region_columns": args.region, "depth": CFG["depth"], "iters": args.iters, "warmup": args.warmup}
    with tempfile.TemporaryDirectory() as tmp:
        line["workloads"] = [workload(tmp, n, args.region, (p, f), ws, args.iters, args.warmup) for n in (8000, 150)]
    ws.close()
    name, limit = card()
    line.update(gpu=name, power_limit=limit)
    out = json.dumps(line)
    print(out)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(out + "\n")
    if not all(w["identical"] for w in line["workloads"]):
        raise SystemExit("bench_cascade_call: the device route and the host route disagree")


if __name__ == "__main__":
    main()
