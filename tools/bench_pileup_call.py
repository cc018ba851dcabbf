"""What one region costs from counted records to call records, with and without the trip through host strings.

    python tools/bench_pileup_call.py [--region 131072] [--iters 40] [--warmup 2] [--out FILE]

On the seeded alignment of ``bench.py``'s ``pileup_counts`` sub-record (depth 40, 8 kb reads, 4 % indels; ``--region`` columns of
it) and seeded Clair3_P weights it alternates, in one process after warm-up,

* the route through the host: ``count`` -> ``fetch`` -> ``alt_info_strings`` (``format_alt_info`` per candidate) ->
  ``forward`` -> ``decode.batch_calls`` (parses ``ctg:pos:ref``, encodes the strings, sends them back), and
* ``PileupCounter.call``: the text stage, Clair3_P and the decoder on device views,

each region timed on the host clock from before ``count`` to a device synchronise after the results are on the host, and prints
one JSON line: wall time per candidate of both (median over ``--iters`` regions each, with the quartiles and extremes), the
count's and the text stage's device time (medians over the ``call`` regions) and launches, the bytes of text, and the card's
name and power limit read in the same run.  Needs an H100; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from clair3_b200 import decode, pileup_counts as pc, synth, synth_reads as sr  # noqa: E402
from clair3_b200.model import Clair3_P  # noqa: E402

CFG = dict(depth=40, read_len=8000, indel_rate=0.04, origin=10000, seed=5)       # bench.py: PLP_CFG


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ")
    return name or torch.cuda.get_device_name(0), limit or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--region", type=int, default=1 << 17)
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pileup_call: needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda:0")
    rec, ref, rs = sr.random_alignment(args.region, depth=CFG["depth"], read_len=CFG["read_len"], seed=CFG["seed"],
                                       indel_rate=CFG["indel_rate"], origin=CFG["origin"])
    start, end = CFG["origin"], CFG["origin"] + args.region
    host = pc.BamRecords.from_dict(rec)
    model = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    model.to(dev)
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()})
    cfg = decode.replay_config(pileup=True, add_indel_length=False)
    ctr = pc.PileupCounter(0)

    def host_route():
        r = ctr.count(host, start, end, ref, rs, alt_info=True).fetch()
        strings = ctr.alt_info_strings(r)
        Y, ok = ctr.forward(model)
        t = pc.alt_info_list(strings, "ctg")
        res = decode.batch_calls(model, [x[1] for x in t], [x[2] for x in t], Y, cfg)
        torch.cuda.synchronize()
        return res

    def device_route():
        res = ctr.count(host, start, end, ref, rs, alt_info=True).call(model, cfg, "ctg")
        torch.cuda.synchronize()
        return res

    for _ in range(max(1, args.warmup)):                         # at least one: it is also the parity check
        a, b = host_route(), device_route()
    same = bool(np.array_equal(a["calls"], b["calls"]) and decode.calls_text(a, cfg) == decode.calls_text(b, cfg))
    t_host, t_dev, ms_count, ms_text = [], [], [], []
    for _ in range(args.iters):                                  # alternated: both see the same neighbours on the card
        t0 = time.perf_counter()
        host_route()
        t1 = time.perf_counter()
        device_route()
        t2 = time.perf_counter()
        t_host.append(t1 - t0)
        t_dev.append(t2 - t1)
        ms_count.append(ctr.last_ms()[0])                        # outside the timed windows
        ms_text.append(ctr.alt_text_last_ms()[0])
    n_cand = len(b["calls"])
    count_launches, text_launches = ctr.last_ms()[1], ctr.alt_text_last_ms()[1]
    n_text, n_dec = ctr.alt_text_sizes()
    name, limit = card()
    med = lambda v: float(np.median(v))                          # noqa: E731
    spread = lambda v: [round(1e3 * float(x), 3) for x in np.percentile(v, [0, 25, 75, 100])]      # noqa: E731
    line = {"bench": "pileup_call", "gpu": name, "power_limit": limit, "region_columns": args.region, "reads": host.n_reads,
            "candidates": n_cand, "kept_candidates": int(b["cand_ok"].sum()), "iters": args.iters, "warmup": args.warmup,
            "records_identical": same,
            "host_route_us_per_candidate": 1e6 * med(t_host) / max(n_cand, 1), "call_us_per_candidate": 1e6 * med(t_dev) / max(n_cand, 1),
            "host_route_ms_min_q1_q3_max": spread(t_host), "call_ms_min_q1_q3_max": spread(t_dev),
            "timed_s": round(sum(t_host) + sum(t_dev), 3),
            "count_device_ms": med(ms_count), "count_launches": count_launches, "text_device_ms": med(ms_text),
            "text_launches": text_launches,
            "text_bytes": n_text, "decoder_bytes": n_dec}
    out = json.dumps(line)
    print(out)
    if args.out:
        with open(args.out, "w") as f:
            f.write(out + "\n")
    ctr.close()
    if not same:
        raise SystemExit("bench_pileup_call: call() and the host route disagree")


if __name__ == "__main__":
    main()
