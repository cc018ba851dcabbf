"""What ``--enable_phasing`` costs (DESIGN.md 5g.3): the phase stage on the GPU next to the CPU statement on the same input.

    python tools/bench_phase.py [--out FILE]

Two cases:

* ``genome_call_case``: tools/bench_genome_call.py's first case (two 2 Mb contigs at depth 30 with 8 kb reads, 1 Mb chunks,
  seed 101) through ``genome.call_genome(enable_phasing=True)``: the ``phase`` stage's wall and device ms from the route's
  stage marks, and ``clair3_b200.phasing.phase_contig`` over the same merged rows and records on the host.
* ``diploid_5mb``: one 5 Mb contig of a seeded diploid genome (het SNPs every 1 kb on average, two haplotypes, reads drawn
  from each with 3 % errors, depth 30, 8 kb reads), phased with ``phase_gpu.phase_contig`` in one 5 Mb span: wall time and
  device time (CUDA events) of the whole contig and of its parts (observations, host layout, DP), and the host statement's
  time on the same rows and records.  Both must give the same rows.

WhatsHap's own time is not measured: it is not part of this project.  Prints one JSON line with the card's name and power
limit read in the same run.  Needs an H100.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_cascade_call import card  # noqa: E402
from bench_genome_call import make  # noqa: E402
from clair3_b200 import bam_io, cascade, genome, phase_gpu, phasing  # noqa: E402
from clair3_b200.bam_decode import BamDecoder  # noqa: E402
from phase_cases import diploid_contig  # noqa: E402
import test_gpu_genome as tg  # noqa: E402


def _host(bam, body):
    t0 = time.perf_counter()
    out = []
    for ctg, rows in phasing.split_contigs(body).items():
        out.extend(phasing.phase_contig(rows, bam_io.read_bam(bam, ctg, fa_fields=True)[0])[0])
    return "".join(out), time.perf_counter() - t0


def genome_case(ws, models):
    with tempfile.TemporaryDirectory() as d:
        bam, fa = make(d, [("chr1", 2.0), ("chr2", 2.0)], 101)
        kw = dict(chunk_size=1_000_000, workspaces=ws, enable_phasing=True)
        genome.call_genome(bam, fa, models[0], models[1], os.path.join(d, "warm"), ctg_name="chr1", **kw)
        res = genome.call_genome(bam, fa, models[0], models[1], os.path.join(d, "out"), **kw)
        merged = res["texts"]["merge_output"].split("\n#CHROM", 1)[1].split("\n", 1)[1]
        phased = res["texts"]["phased_merge_output"].split("\n#CHROM", 1)[1].split("\n", 1)[1]
        host_body, host_s = _host(bam, merged)
        v = phasing.het_snvs(merged.splitlines(keepends=True))
        return {"rows": res["rows"], "het_snvs": len(v.pos), "phased_rows": phased.count("|"),
                "phase_stage_ms": {k: round(x, 3) for k, x in res["stages"]["phase"].items()},
                "call_genome_total_wall_ms": round(res["stages"]["total"]["wall_ms"], 3),
                "cpu_statement_ms": round(1e3 * host_s, 3), "equal_cpu_statement": host_body == phased}


def _timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, 1e3 * (time.perf_counter() - t0), a.elapsed_time(b)


def diploid_case(decoder, length=5_000_000):
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        rec, ref, rows, truth = diploid_contig(301, length, 30, 8000)
        bam = os.path.join(d, "p.bam")
        bam_io.write_bam(bam, rec, [("chr1", length)])
        bam_io.write_bai(bam)
        made = time.perf_counter() - t0
        phase_gpu.phase_contig(decoder, bam, "chr1", length, rows[:200], genome.CHUNK_SIZE)          # warm-up
        (got, *_), wall, dev = _timed(lambda: phase_gpu.phase_contig(decoder, bam, "chr1", length, rows, genome.CHUNK_SIZE))
        v = phasing.het_snvs(rows)
        frag, f_wall, f_dev = _timed(lambda: phase_gpu.contig_fragments(decoder, bam, "chr1", length, v, genome.CHUNK_SIZE))
        lay, l_wall, _ = _timed(lambda: phasing.layout(frag, len(v.pos)))
        (hap, cost), d_wall, d_dev = _timed(lambda: phase_gpu.solve(lay, decoder._device))
        t0 = time.perf_counter()
        host = phasing.phase_contig(rows, bam_io.read_bam(bam, "chr1", fa_fields=True)[0])
        host_s = time.perf_counter() - t0
        switch = sum(not ((hap[a:b] == truth[lay.col_var[a:b]]).all() or (hap[a:b] != truth[lay.col_var[a:b]]).all())
                     for a, b in zip(lay.blk_col_off[:-1], lay.blk_col_off[1:]))
        return {"length": length, "reads": int(len(rec["pos"])), "het_snvs": int(len(v.pos)), "entries": int(len(frag.read)),
                "admitted_reads": int(len(lay.read_id)), "blocks": int(lay.n_blocks), "columns": int(len(lay.col_var)),
                "largest_block_columns": int(max(b - a for a, b in zip(lay.blk_col_off[:-1], lay.blk_col_off[1:]))),
                "blocks_with_switch_errors": int(switch), "make_input_s": round(made, 3),
                "gpu_phase_contig": {"wall_ms": round(wall, 3), "device_ms": round(dev, 3)},
                "parts": {"fragments": {"wall_ms": round(f_wall, 3), "device_ms": round(f_dev, 3)},
                          "layout_host": {"wall_ms": round(l_wall, 3)},
                          "dp": {"wall_ms": round(d_wall, 3), "device_ms": round(d_dev, 3)}},
                "cpu_statement_ms": round(1e3 * host_s, 3), "equal_cpu_statement": host[0] == got and bool((host[4] == hap).all())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    models = tg._models()
    ws = cascade.Workspaces(0)
    dec = BamDecoder(0)
    try:
        rows = {"genome_call_case": genome_case(ws, models), "diploid_5mb": diploid_case(dec)}
    finally:
        ws.close()
        dec.close()
    line = {"bench": "phase", "gpu": name, "power_limit": limit, "whatshap": "not measured (not available)",
            "dp_kernel": phase_gpu.dp_attributes(), "cases": rows}
    text = json.dumps(line)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
