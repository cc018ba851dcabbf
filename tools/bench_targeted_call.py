"""What calling only inside a BED or at known sites costs through the cascade, against calling the whole region.

    python tools/bench_targeted_call.py [--region 131072] [--iters 5] [--warmup 1] [--out FILE]

The workloads of ``tools/bench_cascade_call.py`` (depth 40, ``--region`` columns, 8 kb and 150 bp reads, seeded), each run
untargeted and with three seeded target sets:

* ``exome``: intervals of 150-300 bp whose extended spans (33 bases either side, as CheckEnvs extends them) cover about 2 % of
  the region's columns;
* ``half``: intervals of 1-2 kb covering about 50 % of the columns;
* ``known_sites``: 2,000 known sites at random positions (genotyping mode, with the add-back).

For each run it reports the candidates the counter found and kept, the device ms of each ``call_region`` stage (CUDA events at
the stage boundaries, medians over ``--iters``) and, inside the pileup stage, the count and the text stage from their own event
pairs (the rest of that stage is Clair3_P and the decoder), and whether the targeted rows (and the genotyped body) equal
``call_region_host``'s.  Prints one JSON line with the card's name and power limit read in the same run.  Needs an H100.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_cascade_call import CFG, CFG_F, CFG_P, card, med  # noqa: E402
from clair3_b200 import bam_io, cascade, synth, synth_reads as sr, targets  # noqa: E402
from clair3_b200.model import Clair3_F, Clair3_P  # noqa: E402


def target_sets(start, end, seed=17):
    rng = np.random.default_rng(seed)
    width = end - start
    out = {}
    for name, share, lo, hi in (("exome", 0.02, 150, 300), ("half", 0.5, 1000, 2000)):
        n = max(1, int(round(share * width / ((lo + hi) / 2 + 2 * targets.EXPAND))))
        starts = np.sort(rng.choice(np.arange(start, end - hi, hi + 2 * targets.EXPAND + 1), n, replace=False))
        rows = "".join("ctg\t%d\t%d\n" % (s, s + int(rng.integers(lo, hi + 1))) for s in starts)
        out[name] = ("bed", targets.read_bed(rows), n)
    sites = np.sort(rng.choice(np.arange(start + 1, end + 1), 2000, replace=False))
    out["known_sites"] = ("known_sites", targets.read_vcf("".join("ctg\t%d\t.\tA\tC\t.\t.\t.\tGT\t0/1\n" % p for p in sites)), 2000)
    return out


def run(args, ws, iters, warmup, **kw):
    stages, count_ms, text_ms = [], [], []
    for i in range(warmup + iters):
        r = cascade.call_region(*args, workspaces=ws, **kw)
        torch.cuda.synchronize()
        if i >= warmup:
            stages.append(r["stages"])
            count_ms.append(ws.counter.last_ms()[0])
            text_ms.append(ws.counter.alt_text_last_ms()[0])
    per_stage = {s["stage"]: med([run_[j]["device_ms"] for run_ in stages]) for j, s in enumerate(stages[0])}
    return r, {"device_ms": per_stage, "count_ms": med(count_ms), "text_ms": med(text_ms),
               "forward_decode_ms": per_stage["pileup"] - med(count_ms) - med(text_ms)}


def workload(tmp, read_len, region, models, ws, iters, warmup):
    rec, ref, rs = sr.random_alignment(region, depth=CFG["depth"], read_len=read_len, seed=CFG["seed"], indel_rate=CFG["indel_rate"],
                                       origin=CFG["origin"])
    path = os.path.join(tmp, "w%d.bam" % read_len)
    bam_io.write_bam(path, rec, [("ctg", rs + len(ref))])
    bam_io.write_bai(path)
    idx = bam_io.read_bai(path + ".bai")
    start, end = CFG["origin"], CFG["origin"] + region
    args = (path, "ctg", start, end, ref, rs, models[0], models[1], CFG_P, CFG_F)
    full, t_full = run(args, ws, iters, warmup, index=idx)
    found = int(len(full["pileup"]["calls"]))
    out = {"read_len": read_len, "records": int(len(rec["pos"])), "candidates_found": found, "untargeted": t_full, "targeted": []}
    for name, (kind, tg, n) in target_sets(start, end).items():
        ct = tg.contig("ctg")
        covered = int(ct.keep(np.arange(start + 1, end + 1)).sum()) if kind == "bed" else None
        got, t = run(args, ws, iters, warmup, index=idx, **{kind: tg})
        want = cascade.call_region_host(*args, workspaces=ws, **{kind: tg})
        same = got["vcf"] == want["vcf"] and np.array_equal(got["pileup"]["calls"], want["pileup"]["calls"])
        if kind == "known_sites":
            same = same and got["genotyped"] == want["genotyped"]
        kept = int(len(got["pileup"]["calls"]))
        out["targeted"].append(dict(targets=name, entries=n, columns_in_targets=covered, candidates_kept=kept,
                                    kept_share=kept / max(found, 1), fa_candidates=int(len(got["candidates"])),
                                    vcf_rows=got["vcf"].count("\n"), identical_to_host_route=bool(same), **t))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--region", type=int, default=1 << 17)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_targeted_call: needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda:0")
    p = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    p.to(dev)
    p.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.pileup_state_dict(False, seed=1).items()})
    f = Clair3_F(add_indel_length=True, predict=True, input_channels=8)
    f.to(dev)
    f.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in synth.fa_state_dict(True, channels=8, seed=1).items()})
    ws = cascade.Workspaces(0)
    line = {"bench": "targeted_call", "region_columns": a.region, "depth": CFG["depth"], "iters": a.iters, "warmup": a.warmup}
    with tempfile.TemporaryDirectory() as tmp:
        line["workloads"] = [workload(tmp, n, a.region, (p, f), ws, a.iters, a.warmup) for n in (8000, 150)]
    ws.close()
    name, limit = card()
    line.update(gpu=name, power_limit=limit)
    out = json.dumps(line)
    print(out)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(out + "\n")
    if not all(t["identical_to_host_route"] for w in line["workloads"] for t in w["targeted"]):
        raise SystemExit("bench_targeted_call: the targeted device route and the host route disagree")


if __name__ == "__main__":
    main()
