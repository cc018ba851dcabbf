"""Device time per launch of the networks' feed-forward GEMM kernels and the heads kernel, each timed on its own.

    python tools/bench_pileup_gemms.py [--iters 50] [--out FILE]

Runs the pileup network at 1024 sites per forward and the full-alignment network at 256 sites per forward (the shapes
``bench.py`` times), one stream, device-resident seeded inputs rotated over distinct batches, under ``torch.profiler`` with CUDA
activities.  It prints one JSON line: for each of ``proj2_kernel``, ``l4_kernel<128>`` (pileup), ``heads_kernel`` (pileup),
``l4_kernel<256>`` and ``heads_kernel`` (full alignment) the median and mean device time per launch, the FLOPs and the
compulsory HBM bytes of one launch from its shapes, and the two floors those give: FLOPs over the dense FP16 tensor rate at
the SM clock read in the same run (4096 FLOP per clock and SM), and bytes over the 3.35 TB/s of the H100 SXM data sheet.
The card's name and power limit come from ``nvidia-smi`` in the same run, and the SM clocks from ``nvidia-smi`` samples taken every
100 ms while the profiled forwards run (``clocks``; the floors use their median).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from clair3_b200 import synth  # noqa: E402
from clair3_b200.model import Clair3_F, Clair3_P  # noqa: E402
from bench import ClockSampler  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
FLOP_PER_CLK_SM = 4096             # dense FP16 tensor rate per SM (989 TFLOP/s = 132 SMs x 1830 MHz x 4096)
T, L4_IN_P, L4_IN_F = 33, 10560, 3584


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_mhz": float(sm), "sm_max_mhz": float(smax)}
    except Exception as e:  # noqa: BLE001
        return {"error": "%s: %s" % (type(e).__name__, e)}


def make(kind, channels, add_indel, dev):
    if kind == "pileup":
        sd = synth.pileup_state_dict(add_indel, seed=0)
        m = Clair3_P(add_indel_length=add_indel, predict=True, input_channels=channels)
    else:
        sd = synth.fa_state_dict(add_indel, channels=channels, seed=0)
        m = Clair3_F(add_indel_length=add_indel, predict=True, input_channels=channels)
    m.to(dev)
    m.eval()
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    return m


def profile(m, xs, ys, iters):
    """{kernel name: [device us per launch]} of `iters` forwards on the current stream."""
    for i in range(4):
        m.forward_into(xs[i % len(xs)], ys)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for i in range(iters):
            m.forward_into(xs[i % len(xs)], ys)
        torch.cuda.synchronize()
    times = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            times.setdefault(ev.name, []).append(ev.time_range.elapsed_us())
    return times


def pick(times, needle):
    hits = [v for k, v in times.items() if needle in k]
    if len(hits) != 1:
        raise SystemExit("expected one kernel matching %r, found %d: %s" % (needle, len(hits), sorted(times)))
    return hits[0]


def row(us, flop, nbytes, sm_mhz, n_sm):
    med = float(np.median(us))
    t_mma = flop / (n_sm * FLOP_PER_CLK_SM * sm_mhz * 1e6) * 1e6
    t_hbm = nbytes / HBM_BYTES_PER_S * 1e6
    return {"us_median": med, "us_mean": float(np.mean(us)), "launches": len(us), "gflop": flop / 1e9, "hbm_mb": nbytes / 1e6,
            "floor_mma_us": t_mma, "floor_hbm_us": t_hbm, "floor_over_median": max(t_mma, t_hbm) / med}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pileup_gemms: no CUDA device")
    dev = torch.device("cuda:0")
    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
    info = card()
    sampler = ClockSampler(0).start()
    t0 = sampler.mark()

    bp = 1024
    mp = make("pileup", 18, False, dev)
    xp = [torch.from_numpy(synth.pileup_inputs(bp, seed=100 + i)).to(dev) for i in range(8)]
    yp = torch.empty((bp, mp.out_dim), dtype=torch.float32, device=dev)
    tp = profile(mp, xp, yp, args.iters)

    bf = 256
    mf = make("fa", 8, True, dev)
    xf = [torch.from_numpy(synth.fa_inputs(bf, depth=89, channels=8, seed=200 + i)).to(dev) for i in range(4)]
    yf = torch.empty((bf, mf.out_dim), dtype=torch.float32, device=dev)
    tf = profile(mf, xf, yf, args.iters)
    clocks = sampler.window(t0, sampler.mark())
    sampler.stop()
    if not clocks.get("sm_mhz"):
        raise SystemExit("bench_pileup_gemms: no SM clock samples from nvidia-smi")
    clk = clocks["sm_mhz"]
    m_p = T * bp
    kernels = {
        # h1 read once, pre-gates written once, the weight slabs once per CTA (served from L2 after the first)
        "proj2": row(pick(tp, "proj2_kernel"), 2.0 * m_p * 1280 * 256, m_p * 256 * 2 + m_p * 1280 * 2 + 1280 * 256 * 2, clk, n_sm),
        # activations and weights read once; the fp32 partials the heads kernel reads are not counted
        "l4_pileup": row(pick(tp, "l4_kernel<128>"), 2.0 * bp * L4_IN_P * 128, bp * L4_IN_P * 2 + L4_IN_P * 128 * 2, clk, n_sm),
        "heads_pileup": row(pick(tp, "heads_kernel"), 2.0 * bp * (128 * 128 * 2 + 128 * 24), bp * 128 * 4, clk, n_sm),
        "l4_fa": row(pick(tf, "l4_kernel<256>"), 2.0 * bf * L4_IN_F * 256, bf * L4_IN_F * 2 + L4_IN_F * 256 * 2, clk, n_sm),
        "heads_fa": row(pick(tf, "heads_kernel"), 2.0 * bf * (256 * 128 * 4 + 128 * 90), bf * 256 * 4, clk, n_sm),
    }
    line = {"tool": "bench_pileup_gemms", "card": info, "clocks": clocks, "sm_count": n_sm,
            "floor_clock_mhz": clk, "iters": args.iters, "pileup_sites": bp, "fa_sites": bf, "kernels": kernels}
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
