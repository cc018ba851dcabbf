"""What a region's full-alignment candidates cost from records to call records, with and without the trip through host strings.

    python tools/bench_fa_call.py [--region 200000] [--depth 50] [--iters 20] [--warmup 2] [--out FILE]

On the seeded region of ``tools/bench_fa_tensor.py`` (``random_fa_case``: 10 kb reads at depth ~``--depth``, one candidate per
~100 bp, one phased heterozygous SNP per ~1 kb) and seeded ``Clair3_F(True, True, 8)`` weights it alternates, in one process
after warm-up,

* the route through the host: ``build`` -> ``fetch`` -> ``alt_info_strings`` (``format_alt_info`` per candidate) -> the
  ``ctg:pos:ref`` / ``depth-alt`` split of ``create_tensor_full_alignment`` -> ``forward`` -> ``decode.batch_calls`` (parses
  the strings, encodes them, sends them back), and
* ``build`` -> ``FullAlignmentBuilder.call``: the text stage, Clair3_F and the decoder on device views,

both on host records, each region timed on the host clock from before ``build`` to a device synchronise after the results are
on the host, and prints one JSON line: whether both routes gave the same call records and VCF rows, wall time per candidate of
both (median over ``--iters`` regions each, with the quartiles and extremes), the build's and the text stage's device time
(medians over the ``call`` regions) and launches, the bytes of text, and the card's name and power limit read in the same run.
Exits non-zero when the routes disagree.  Needs an H100; there is no CPU fallback.
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

from clair3_b200 import decode, synth, synth_reads as sr  # noqa: E402
from clair3_b200.fa_tensor import FullAlignmentBuilder  # noqa: E402
from clair3_b200.model import Clair3_F  # noqa: E402
from clair3_b200.pileup_counts import BamRecords  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ")
    return name or torch.cuda.get_device_name(0), limit or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--region", type=int, default=200000)
    ap.add_argument("--depth", type=int, default=50)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fa_call: needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda:0")
    # tools/bench_fa_tensor.py: make_case
    rec, ref, cand, var = sr.random_fa_case(args.depth, region_len=args.region, depth=args.depth, read_len=10000,
                                            n_cand=args.region // 100, n_var=args.region // 1000, dup_frac=0.0)
    host = BamRecords.from_dict(rec)
    model = Clair3_F(add_indel_length=True, predict=True, input_channels=8)
    model.to(dev)
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=8, seed=1).items()})
    cfg = decode.replay_config(pileup=False, add_indel_length=True)
    b = FullAlignmentBuilder(0)

    def host_route():
        b.build(host, cand, ref, 0, variants=var)
        b.fetch()
        pos_info, alt_info = [], []
        for s in b.alt_info_strings():
            pos, depth, center_ref_base, alt = s.rstrip().split("-")[:4]
            pos_info.append("ctg:" + pos + ":" + center_ref_base)
            alt_info.append(depth + "-" + alt)
        Y = b.forward(model)
        res = decode.batch_calls(model, pos_info, alt_info, Y, cfg)
        torch.cuda.synchronize()
        return res

    def device_route():
        res = b.build(host, cand, ref, 0, variants=var).call(model, cfg, "ctg")
        torch.cuda.synchronize()
        return res

    for _ in range(max(1, args.warmup)):                         # at least one: it is also the parity check
        a, c = host_route(), device_route()
    same = bool(np.array_equal(a["position"], c["position"]) and np.array_equal(a["calls"], c["calls"])
                and decode.calls_text(a, cfg) == decode.calls_text(c, cfg))
    t_host, t_dev, ms_build, ms_text = [], [], [], []
    for _ in range(args.iters):                                  # alternated: both see the same neighbours on the card
        t0 = time.perf_counter()
        host_route()
        t1 = time.perf_counter()
        device_route()
        t2 = time.perf_counter()
        t_host.append(t1 - t0)
        t_dev.append(t2 - t1)
        ms_build.append(b.last_ms()[0])                          # outside the timed windows
        ms_text.append(b.alt_text_last_ms()[0])
    n_cand = len(c["calls"])
    build_launches, text_launches = b.last_ms()[1], b.alt_text_last_ms()[1]
    n_text, n_dec = b.alt_text_sizes()
    n_kept = b.sizes()[1]
    name, limit = card()
    med = lambda v: float(np.median(v))                          # noqa: E731
    spread = lambda v: [round(1e3 * float(x), 3) for x in np.percentile(v, [0, 25, 75, 100])]      # noqa: E731
    line = {"bench": "fa_call", "gpu": name, "power_limit": limit, "region_bp": args.region, "depth": args.depth,
            "reads": host.n_reads, "kept_reads": n_kept, "candidates": n_cand, "printed_rows": int(c["calls"]["printed"].sum()),
            "iters": args.iters, "warmup": args.warmup, "records_identical": same,
            "host_route_us_per_candidate": 1e6 * med(t_host) / max(n_cand, 1), "call_us_per_candidate": 1e6 * med(t_dev) / max(n_cand, 1),
            "host_route_ms_min_q1_q3_max": spread(t_host), "call_ms_min_q1_q3_max": spread(t_dev),
            "timed_s": round(sum(t_host) + sum(t_dev), 3),
            "build_device_ms": med(ms_build), "build_launches": build_launches, "text_device_ms": med(ms_text),
            "text_launches": text_launches, "text_bytes": n_text, "decoder_bytes": n_dec}
    out = json.dumps(line)
    print(out)
    if args.out:
        with open(args.out, "w") as f:
            f.write(out + "\n")
    b.close()
    if not same:
        raise SystemExit("bench_fa_call: call() and the host route disagree")


if __name__ == "__main__":
    main()
