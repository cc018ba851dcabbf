"""What reading a bgzip-compressed reference FASTA costs: ``BamDecoder.fetch_fasta`` (the blocks inflated and the bases gathered
on the GPU) against ``bam_io.fetch_fasta`` (zlib on the host), and the genome route with a plain and a bgzipped FASTA.

    python tools/bench_fasta_fetch.py [--windows 24] [--warmup 4] [--contig-mb 40] [--out FILE]

A seeded ``--contig-mb`` Mb contig (60 bases per line, bgzipped as ``bgzip`` cuts it: 65,280-byte blocks) and windows of
5,002,001 bases (a 5 Mb chunk plus ``FETCH_EXPAND`` either side, what the genome route fetches per chunk) at seeded starts.
It reports, per window:

* ``device_ms``: the fetch's kernels (inflate and gather) between CUDA events on its stream, after ``--warmup`` windows;
* ``stream_ms``: the stream's time over all the windows fetched back to back from compressed bytes already in host memory
  (the staging copy and upload included), over the number of windows;
* ``call_ms``: host wall time of ``fetch_fasta`` from the file, with its wait;
* ``host_zlib_ms``: ``bam_io.fetch_fasta`` over the same windows (host wall time).

Then ``genome.call_genome`` on ``tools/bench_genome_call.py``'s first case (two 2 Mb contigs, 1 Mb chunks) with the plain
and the bgzipped FASTA, each after a warm-up run: the wall time, the stages (``cascade.Stages``) and whether the files are
equal apart from ``##reference=``.  Prints one JSON line with the card's name and power limit read in the same run.  Needs an
H100.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_cascade_call import card  # noqa: E402
from bench_genome_call import make  # noqa: E402
from clair3_b200 import bam_io, cascade, genome  # noqa: E402
from clair3_b200.bam_decode import BamDecoder  # noqa: E402
from clair3_b200.pileup_counts import FETCH_EXPAND  # noqa: E402
import bgzf_fasta as bf  # noqa: E402
import test_gpu_genome as tg  # noqa: E402

WINDOW = genome.CHUNK_SIZE + 2 * FETCH_EXPAND + 1


def fetch_windows(d, n_windows, warmup, contig_mb):
    rng = np.random.default_rng(11)
    length = int(contig_mb * 1e6)
    plain = bf.write_fasta(os.path.join(d, "w.fa"), [("chrW", bf.random_sequence(length, rng))], width=60)
    gz = plain + ".gz"
    blocks = len(bf.bgzip(plain, gz))
    starts = [int(s) for s in rng.integers(0, length - WINDOW, warmup + n_windows)]
    dec = BamDecoder(0)
    try:
        row = {r[0]: r for r in bam_io.read_fai(gz + ".fai")}["chrW"]
        gzi = bam_io.read_gzi(gz + ".gzi")
        raw = open(gz, "rb").read()
        pre = []
        for s in starts:
            _, _, c0, c1, u0 = bam_io.fasta_span(row, s, s + WINDOW, gzi)
            pre.append((raw[c0:c1], u0, s))
        device_ms, call_ms = [], []
        for i, s in enumerate(starts):
            t0 = time.perf_counter()
            out = dec.fetch_fasta(gz, "chrW", s, s + WINDOW)
            t1 = time.perf_counter()
            if i >= warmup:
                device_ms.append(dec.last_ms()[0])
                call_ms.append(1e3 * (t1 - t0))
        want = bam_io.fetch_fasta(gz, "chrW", starts[-1], starts[-1] + WINDOW)
        equal = out.cpu().numpy().tobytes().decode() == want
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for data, u0, s in pre[warmup:]:
            dec.fetch_fasta_bytes(data, u0, s, row[3], row[4], WINDOW, wait=False)
        ev[1].record()
        dec.fasta_status()
        torch.cuda.synchronize()
        stream_ms = ev[0].elapsed_time(ev[1]) / n_windows
        host_ms = []
        for s in starts[warmup:]:
            t0 = time.perf_counter()
            bam_io.fetch_fasta(gz, "chrW", s, s + WINDOW)
            host_ms.append(1e3 * (time.perf_counter() - t0))
    finally:
        dec.close()
    per_window_mib = (pre[-1][0].__len__()) / 2 ** 20
    med = lambda v: float(np.median(v))            # noqa: E731
    return {"window_bases": WINDOW, "windows": n_windows, "warmup": warmup, "contig_bases": length, "bgzf_blocks": blocks,
            "compressed_mib_per_window": round(per_window_mib, 3),
            "device_ms": {"median": med(device_ms), "min": min(device_ms), "max": max(device_ms)},
            "stream_ms": stream_ms,
            "call_ms": {"median": med(call_ms), "min": min(call_ms), "max": max(call_ms)},
            "host_zlib_ms": {"median": med(host_ms), "min": min(host_ms), "max": max(host_ms)},
            "bytes_equal_host": equal}


def genome_stages(d):
    bam, fa = make(d, [("chr1", 2.0), ("chr2", 2.0)], 101)
    gz = fa + ".gz"
    bf.bgzip(fa, gz)
    models = tg._models()
    ws = cascade.Workspaces(0)
    out = {}
    try:
        for label, ref in (("plain", fa), ("bgzf", gz)):
            genome.call_genome(bam, ref, models[0], models[1], os.path.join(d, label + "_warm"), chunk_size=1_000_000,
                               workspaces=ws, ctg_name="chr1")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = genome.call_genome(bam, ref, models[0], models[1], os.path.join(d, label), chunk_size=1_000_000, workspaces=ws)
            torch.cuda.synchronize()
            out[label] = {"wall_s": time.perf_counter() - t0, "rows": res["rows"],
                          "stages_ms": {k: {a: round(b, 3) for a, b in v.items()} for k, v in res["stages"].items()},
                          "texts": res["texts"]}
    finally:
        ws.close()
    strip = lambda t: [x for x in t.split("\n") if not x.startswith("##reference=")]     # noqa: E731
    equal = (sorted(out["plain"]["texts"]) == sorted(out["bgzf"]["texts"])
             and all(strip(out["plain"]["texts"][n]) == strip(out["bgzf"]["texts"][n]) for n in out["plain"]["texts"]))
    for v in out.values():
        del v["texts"]
    return {"case": "multi_contig_1mb_chunks (2 x 2 Mb)", "files_equal_apart_from_reference_line": equal, **out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--contig-mb", type=float, default=40.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    with tempfile.TemporaryDirectory() as d:
        fetch = fetch_windows(d, a.windows, a.warmup, a.contig_mb)
    with tempfile.TemporaryDirectory() as d:
        route = genome_stages(d)
    text = json.dumps({"bench": "fasta_fetch", "gpu": name, "power_limit": limit, "fetch": fetch, "genome": route})
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
