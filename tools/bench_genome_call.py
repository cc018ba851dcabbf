"""What a whole-genome run costs (``genome.call_genome``, DESIGN.md 5g), stage by stage.

    python tools/bench_genome_call.py [--contig-mb 2] [--contigs 2] [--out FILE]

A seeded synthetic genome: ``--contigs`` major contigs of ``--contig-mb`` Mb at depth 30 with 8 kb reads, called with a
1 Mb chunk size, and one contig of exactly 5,000,000 bases called at the reference's 5 Mb chunk size (one 5 Mb chunk), each
written as an indexed BAM and an indexed FASTA; seeded weights.  For each case it reports the wall time, the summed wall and
device ms of every stage (CUDA events at the stage boundaries), the rows per file and, from one more run of the same call
in a fresh child process (so nothing an earlier run freed is reused), sampled every 10 ms by a thread during the call:

* ``peak_device_mib``: this process's device memory as NVML reports it (``nvmlDeviceGetComputeRunningProcesses``, read only):
  the CUDA context, the torch caching allocator and the library's own ``cudaMalloc`` workspaces together;
  ``torch_allocated_peak_mib`` is the torch allocator's part alone (``max_memory_allocated``); ``card_used_peak_mib`` is the
  whole card's used memory (``cudaMemGetInfo``) and ``card_used_before_workspaces_mib`` the same before the workspaces were
  created (models loaded), so their difference bounds what the route's workspaces and buffers take;
* ``host_peak_rss_delta_mib``: the child's peak resident set size during the call less the one just before it, with the
  models loaded and the workspaces created (``/proc/self/statm``).

It also reports whether the three files equal the host route of tests/test_gpu_genome.py, with that route's time.  Several
GPUs are not measured here (one process); prints one JSON line with the card's name and power limit read in the same run.
Needs an H100.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_cascade_call import card  # noqa: E402
from clair3_b200 import bam_io, cascade, genome, synth_reads as sr  # noqa: E402
import test_gpu_genome as tg  # noqa: E402


def make(d, sizes, seed):
    seqs, parts = [], []
    for tid, (name, mb) in enumerate(sizes):
        rec, ref, rs = sr.random_alignment(int(mb * 1e6), depth=30, read_len=8000, seed=seed + tid, origin=0)
        seqs.append((name, ref))
        parts.append((rec, tid))
    bam, fa = os.path.join(d, "g.bam"), os.path.join(d, "g.fa")
    bam_io.write_bam(bam, tg._concat_records(parts), [(n, len(s)) for n, s in seqs])
    bam_io.write_bai(bam)
    bam_io.write_fasta(fa, seqs)
    bam_io.write_fai(fa)
    return bam, fa


def card_used():
    free, total = torch.cuda.mem_get_info()
    return total - free


class _Sampler(threading.Thread):
    """Peak device memory of this process (NVML) and peak resident set size, sampled until ``stop``."""

    def __init__(self):
        super().__init__(daemon=True)
        self.dev_peak, self.rss_peak, self.card_peak, self.halt = None, 0, 0, threading.Event()
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nvml, self.handle = pynvml, pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        except Exception:                                # no NVML: device memory is "not measured"
            self.nvml = None
        self.rss0 = self.rss()

    @staticmethod
    def rss():
        with open("/proc/self/statm") as f:
            return int(f.read().split()[1]) * os.sysconf("SC_PAGE_SIZE")

    def device(self):
        if self.nvml is None:
            return None
        for p in self.nvml.nvmlDeviceGetComputeRunningProcesses(self.handle):
            if p.pid == os.getpid() and p.usedGpuMemory is not None:
                return p.usedGpuMemory
        return None

    def run(self):
        while not self.halt.is_set():
            d = self.device()
            if d is not None:
                self.dev_peak = max(self.dev_peak or 0, d)
            self.rss_peak = max(self.rss_peak, self.rss())
            self.card_peak = max(self.card_peak, card_used())
            time.sleep(0.01)

    def stop(self):
        self.halt.set()
        self.join()
        mib = 2 ** 20
        return {"peak_device_mib": "not measured (NVML shows no entry for this process)" if self.dev_peak is None else self.dev_peak / mib,
                "card_used_peak_mib": self.card_peak / mib,
                "host_peak_rss_delta_mib": (self.rss_peak - self.rss0) / mib}


def _memory_child(bam, fa, out, chunk_size, q):
    """``call_genome`` once in a fresh process, under the sampler."""
    models = tg._models()
    torch.cuda.synchronize()
    before = card_used()
    ws = cascade.Workspaces(0)
    try:
        sampler = _Sampler()
        sampler.start()
        genome.call_genome(bam, fa, models[0], models[1], out, chunk_size=chunk_size, workspaces=ws)
        torch.cuda.synchronize()
        mem = sampler.stop()
    finally:
        ws.close()
    mem["card_used_before_workspaces_mib"] = before / 2 ** 20
    q.put(mem)


def case(ws, models, sizes, chunk_size, seed, host):
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        bam, fa = make(d, sizes, seed)
        made = time.perf_counter() - t0
        out = os.path.join(d, "out")
        genome.call_genome(bam, fa, models[0], models[1], out + "_warm", chunk_size=chunk_size, workspaces=ws, ctg_name=sizes[0][0])
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        res = genome.call_genome(bam, fa, models[0], models[1], out, chunk_size=chunk_size, workspaces=ws)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        torch_peak = torch.cuda.max_memory_allocated() / 2 ** 20
        import multiprocessing as mp
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        child = ctx.Process(target=_memory_child, args=(bam, fa, out + "_child", chunk_size, q))
        child.start()
        memory = q.get(timeout=900)
        child.join(timeout=120)
        row = {"contigs": [[n, len_] for n, len_ in res["contigs"]], "chunk_size": chunk_size, "chunks": len(res["chunks"]),
               "beds": res["beds"], "rows": res["rows"], "wall_s": wall, "make_input_s": made,
               "stages_ms": {k: {a: round(b, 3) for a, b in v.items()} for k, v in res["stages"].items()},
               "chunk_lengths": sorted({int(genome.chunk_region(dict(res["contigs"])[c], i, n)[1]
                                            - genome.chunk_region(dict(res["contigs"])[c], i, n)[0]) for c, i, n in res["chunks"]}),
               "torch_allocated_peak_mib": torch_peak, **memory}
        if host:
            t0 = time.perf_counter()
            want = tg.host_route(ws, models[0], models[1], bam, fa, include_all=False, chunk_size=chunk_size,
                                 split_bed_size=cascade.SPLIT_BED_SIZE, min_contig_size=0)
            row["host_route_s"] = time.perf_counter() - t0
            row["equal_host_route"] = want == res["texts"]
        return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contig-mb", type=float, default=2.0)
    ap.add_argument("--contigs", type=int, default=2)
    ap.add_argument("--no-host", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    models = tg._models()
    ws = cascade.Workspaces(0)
    try:
        rows = {"multi_contig_1mb_chunks": case(ws, models, [("chr%d" % (i + 1), a.contig_mb) for i in range(a.contigs)], 1_000_000,
                                                 101, not a.no_host),
                # 4,959,800 bases of reads give a 5,000,000-base contig (random_alignment adds 5 read lengths and 200):
                # chunk_num 1, one 5 Mb chunk
                "one_5mb_chunk": case(ws, models, [("chr1", (genome.CHUNK_SIZE - 5 * 8000 - 200) / 1e6)], genome.CHUNK_SIZE,
                                      201, False)}
    finally:
        ws.close()
    line = {"bench": "genome_call", "gpu": name, "power_limit": limit, "world": 1, "multi_gpu": "not measured",
            "cases": rows}
    text = json.dumps(line)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
