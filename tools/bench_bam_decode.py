"""What reading a region of a BAM file costs on the GPU reader against the host's zlib and ``bam_io.read_bam``.

    python tools/bench_bam_decode.py [--region 131072] [--iters 20] [--warmup 2] [--out FILE]

Writes two seeded workloads to a temporary directory with ``bam_io.write_bam`` (zlib level 6) and an index (``write_bai``): the
region of ``tools/bench_pileup_call.py`` (depth 40, ``--region`` columns) with 8 kb reads and with 150 bp reads.  For each it
measures, in one process after warm-up,

* ``BamDecoder.decode``'s device time (CUDA events around its kernels, ``last_ms``; median over ``--iters`` decodes) with
  compressed and uncompressed MB/s, and its wall time from the file to the sized records;
* the same blocks inflated one by one with ``zlib.decompress`` on one host thread (inflate only, nothing parsed), and
  ``bam_io.read_bam`` on the same file and region;

and for the 8 kb workload the route from the file to call records both ways, ``read_bam`` -> ``count`` -> ``call`` and
``BamDecoder.decode`` -> ``count`` -> ``call``, with the call records asserted identical.  Prints one JSON line with the card's
name and power limit read in the same run.  Needs an H100; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from clair3_b200 import bam_io, decode, pileup_counts as pc, synth, synth_reads as sr  # noqa: E402
from clair3_b200.bam_decode import BamDecoder  # noqa: E402
from clair3_b200.model import Clair3_P  # noqa: E402

CFG = dict(depth=40, indel_rate=0.04, origin=10000, seed=5)        # tools/bench_pileup_call.py


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ")
    return name or torch.cuda.get_device_name(0), limit or "unknown"


def med(v):
    return float(np.median(v))


def zlib_inflate_ms(path, c0, c1):
    """Per-block zlib.decompress of the range's blocks on one thread (what htslib's bgzf loop does), in ms."""
    raw = open(path, "rb").read()[c0:c1]
    blocks = [(o + 18, o + n - 8) for o, n, _ in bam_io.bgzf_blocks(raw)]
    t0 = time.perf_counter()
    for a, b in blocks:
        zlib.decompress(raw[a:b], -15)
    return 1e3 * (time.perf_counter() - t0)


def workload(tmp, read_len, region, dec, iters, warmup):
    rec, ref, rs = sr.random_alignment(region, depth=CFG["depth"], read_len=read_len, seed=CFG["seed"], indel_rate=CFG["indel_rate"],
                                       origin=CFG["origin"])
    path = os.path.join(tmp, "w%d.bam" % read_len)
    bam_io.write_bam(path, rec, [("ctg", CFG["origin"] + region + 4 * read_len + 100000)])
    bam_io.write_bai(path)
    start, end = CFG["origin"], CFG["origin"] + region
    idx = bam_io.read_bai(path + ".bai")
    c0, c1, u0, u1 = bam_io.bai_range(idx, 0, start, end, path)
    n_blocks = len(bam_io.bgzf_blocks(open(path, "rb").read()[c0:c1]))
    for _ in range(warmup):
        got = dec.decode(path, "ctg", start, end, index=idx)
    want, _ = bam_io.read_bam(path, "ctg", start, end)
    h = got.host()
    same = all(np.array_equal(h[k], want[k]) for k in h)
    dev_ms, wall_ms, zl_ms, rb_ms = [], [], [], []
    for _ in range(iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dec.decode(path, "ctg", start, end, index=idx)
        torch.cuda.synchronize()
        wall_ms.append(1e3 * (time.perf_counter() - t0))
        dev_ms.append(dec.last_ms()[0])
    for _ in range(max(3, iters // 4)):
        zl_ms.append(zlib_inflate_ms(path, c0, c1))
    for _ in range(3):
        t0 = time.perf_counter()
        bam_io.read_bam(path, "ctg", start, end)
        rb_ms.append(1e3 * (time.perf_counter() - t0))
    d = med(dev_ms)
    return path, (start, end, ref, rs), {
        "read_len": read_len, "records": int(len(want["pos"])), "blocks": n_blocks, "compressed_bytes": c1 - c0,
        "uncompressed_bytes": u1, "records_identical": bool(same), "decode_device_ms": d, "decode_launches": dec.last_ms()[1],
        "decode_device_ms_min_max": [round(min(dev_ms), 4), round(max(dev_ms), 4)],
        "compressed_MB_per_s": (c1 - c0) / d / 1e3, "uncompressed_MB_per_s": u1 / d / 1e3, "decode_wall_ms": med(wall_ms),
        "zlib_per_block_ms": med(zl_ms), "read_bam_ms": med(rb_ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--region", type=int, default=1 << 17)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bam_decode: needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda:0")
    dec = BamDecoder(0)
    line = {"bench": "bam_decode", "region_columns": args.region, "depth": CFG["depth"], "iters": args.iters, "warmup": args.warmup}
    with tempfile.TemporaryDirectory() as tmp:
        path8, (start, end, ref, rs), w8 = workload(tmp, 8000, args.region, dec, args.iters, args.warmup)
        _, _, w150 = workload(tmp, 150, args.region, dec, args.iters, args.warmup)
        line["workloads"] = [w8, w150]
        # file -> call records, both ways, on the 8 kb workload
        model = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
        model.to(dev)
        model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()})
        cfg = decode.replay_config(pileup=True, add_indel_length=False)
        ctr = pc.PileupCounter(0)
        idx = bam_io.read_bai(path8 + ".bai")

        def host_route():
            rec, _ = bam_io.read_bam(path8, "ctg", start, end)
            res = ctr.count(rec, start, end, ref, rs, alt_info=True).call(model, cfg, "ctg")
            torch.cuda.synchronize()
            return res

        def device_route():
            rec = dec.decode(path8, "ctg", start, end, ref_seq=ref, index=idx)
            res = ctr.count(rec, start, end, None, rs, alt_info=True).call(model, cfg, "ctg")
            torch.cuda.synchronize()
            return res

        for _ in range(max(1, args.warmup)):
            a, b = host_route(), device_route()
        same = bool(np.array_equal(a["calls"], b["calls"]) and decode.calls_text(a, cfg) == decode.calls_text(b, cfg))
        t_host, t_dev = [], []
        for _ in range(max(3, args.iters // 4)):
            t0 = time.perf_counter()
            host_route()
            t1 = time.perf_counter()
            device_route()
            t2 = time.perf_counter()
            t_host.append(1e3 * (t1 - t0))
            t_dev.append(1e3 * (t2 - t1))
        ctr.close()
    dec.close()
    name, limit = card()
    line.update(gpu=name, power_limit=limit, route_candidates=len(b["calls"]), route_call_records_identical=same,
                route_read_bam_ms=med(t_host), route_gpu_decode_ms=med(t_dev))
    out = json.dumps(line)
    print(out)
    if args.out:
        with open(args.out, "w") as f:
            f.write(out + "\n")
    if not same or not all(w["records_identical"] for w in line["workloads"]):
        raise SystemExit("bench_bam_decode: the two readers disagree")


if __name__ == "__main__":
    main()
