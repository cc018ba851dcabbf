"""Throughput of the GPU full-alignment tensor builder (clair3_b200.fa_tensor) next to the reference's own C on the CPU.

    python tools/bench_fa_tensor.py [--region 200000] [--reps 5]

A synthetic ONT-like region (10 kb reads, one candidate per ~100 bp, one phased heterozygous SNP per ~1 kb) at depth ~50 and
~150 (the second exercises the shuffle).  For each: a parity check against the compiled reference (when oracle/_ref is built),
then CUDA-event timings after warm-up, rotating over six device copies of the records so that no build reads a copy that one of
the previous two reps read (the input comes from HBM, not from L2):
  gpu      candidates/s and aligned bases/s with device-resident records, two builders on two streams (joined to the timing
           stream before the closing event)
  e2e      pinned host records in, int8 matrix out (one builder)
  forward  records on the device -> Clair3_F probabilities on the device
  cpu      the reference's calculate_clair3_full_alignment from oracle/_ref on the same in-memory records, one process, and one
           process per chunk of candidates on every core, each with the records of its chunk only ("not measured" without
           oracle/_ref)
Prints one JSON line.  Writes nothing.
"""
import argparse
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from clair3_b200 import synth, synth_reads as sr                       # noqa: E402
from clair3_b200.fa_tensor import FullAlignmentBuilder                   # noqa: E402
from clair3_b200.model import Clair3_F                                   # noqa: E402
from clair3_b200.pileup_counts import BamRecords                         # noqa: E402

NOT_MEASURED = "not measured"
ROT = 6


def make_case(region, depth, seed):
    rec, ref, cand, var = sr.random_fa_case(seed, region_len=region, depth=depth, read_len=10000, n_cand=region // 100,
                                            n_var=region // 1000, dup_frac=0.0)
    return rec, ref, cand, var


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()
        return float(out[0])
    except Exception:
        return None


def timed(fn, reps, main, side=()):
    """Seconds per rep: CUDA events on the main stream around `reps` calls, after one warm-up call; the side streams the calls
    issue work on are joined to the main stream before the closing event."""
    fn(0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(main)
    for s in side:
        s.wait_stream(main)
    for i in range(reps):
        fn(i + 1)
    for s in side:
        main.wait_stream(s)
    e1.record(main)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps


FIELDS = ("pos", "flag", "mapq", "l_qseq", "cigar_off", "cigar", "seq_off", "seq", "qual_off", "qual", "qname_off", "qname")


def slice_records(rec, lo, hi):
    """The records overlapping [lo, hi) - what an indexed fetch of a chunk's region hands the reference - as a contiguous run."""
    ops = rec["cigar"] & 15
    refl = np.where(np.isin(ops, (0, 2, 3, 7, 8)), (rec["cigar"] >> 4).astype(np.int64), 0)
    csum = np.concatenate([[0], np.cumsum(refl)])
    span = csum[rec["cigar_off"][1:]] - csum[rec["cigar_off"][:-1]]
    keep = np.nonzero((rec["pos"] < hi) & (rec["pos"] + np.maximum(span, 1) > lo))[0]
    a, b = (int(keep[0]), int(keep[-1]) + 1) if len(keep) else (0, 0)
    out = {k: rec[k][a:b] for k in ("pos", "flag", "mapq", "l_qseq")}
    for k in ("cigar", "seq", "qual", "qname"):
        o = rec[k + "_off"]
        out[k] = rec[k][int(o[a]):int(o[b])]
        out[k + "_off"] = o[a:b + 1] - o[a]
    return out


_CPU = {}


def _cpu_chunk(i):
    from oracle import fa_ref
    rec, ref, cand, var = _CPU["chunks"][i]
    t = time.perf_counter()
    fa_ref.full_alignment(rec, cand, ref, variants=var, need_haplotagging=True, matrix_depth=89)
    return time.perf_counter() - t


def cpu_rates(case):
    """The compiled reference on the same records: one process over the whole region, then one process per chunk of candidates on
    every core, each chunk with only the records overlapping its candidates' windows (as a per-chunk region fetch returns them);
    the pool is started before the clock."""
    from oracle import fa_ref
    if not fa_ref.available():
        return NOT_MEASURED, NOT_MEASURED
    rec, ref, cand, var = case
    t = time.perf_counter()
    fa_ref.full_alignment(rec, cand, ref, variants=var, need_haplotagging=True, matrix_depth=89)
    single = len(cand) / (time.perf_counter() - t)
    n = os.cpu_count() or 1
    bounds = np.linspace(0, len(cand), n + 1).astype(int)
    _CPU["chunks"] = [(slice_records(rec, int(cand[a]) - 16, int(cand[b - 1]) + 17), ref, cand[a:b], var)
                      for a, b in zip(bounds[:-1], bounds[1:]) if b > a]
    with mp.get_context("fork").Pool(n) as pool:
        pool.map(abs, range(n))                              # workers are up before the clock starts
        t = time.perf_counter()
        pool.map(_cpu_chunk, range(len(_CPU["chunks"])), chunksize=1)
        allcores = len(cand) / (time.perf_counter() - t)
    return single, allcores


def bench_depth(depth, args, model):
    dev = torch.device("cuda:0")
    case = make_case(args.region, depth, seed=depth)
    rec, ref, cand, var = case
    bases = sr.aligned_bases(rec)
    parity = NOT_MEASURED
    b1, b2 = FullAlignmentBuilder(0), FullAlignmentBuilder(0)
    from oracle import fa_ref
    if fa_ref.available():
        want, want_alt, _ = fa_ref.full_alignment(rec, cand, ref, variants=var, need_haplotagging=True, matrix_depth=89)
        b1.build(rec, cand, ref, 0, variants=var)
        parity = bool(np.array_equal(b1.fetch(), want) and b1.alt_info_strings() == want_alt)
    host = BamRecords.from_dict(rec)
    # ROT copies of the records, used in turn: each build reads a copy no build of the previous two reps has touched, so the
    # inputs come from HBM, not from the 50 MB L2
    devs = [host.to_device(dev, ref) for _ in range(ROT)]
    s1, s2 = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    main = torch.cuda.current_stream(dev)

    def gpu(i):
        for j, (b, s) in enumerate(((b1, s1), (b2, s2))):
            d = devs[(2 * i + j) % ROT]
            with torch.cuda.stream(s):
                b.build(d, cand, d.ref, 0, variants=var)
    t_gpu = timed(gpu, args.reps, main, (s1, s2)) / 2

    pinned = [{k: torch.from_numpy(np.ascontiguousarray(getattr(host, k))).pin_memory().numpy() for k in FIELDS} for _ in range(2)]
    out = torch.empty((len(cand), 89, 33, 8), dtype=torch.int8).pin_memory().numpy()
    from clair3_b200._ffi import ffi, lib, check

    def e2e(i):
        b1.build(pinned[i % 2], cand, ref, 0, variants=var)
        check(lib().c3b_fa_fetch(b1._h, ffi.cast("int8_t *", out.ctypes.data), ffi.NULL, ffi.NULL))
    t_e2e = timed(e2e, args.reps, main)

    def fwd(i):
        d = devs[i % ROT]
        b1.build(d, cand, d.ref, 0, variants=var)
        b1.forward(model)
    t_fwd = timed(fwd, args.reps, main)
    cpu1, cpun = cpu_rates(case) if args.cpu else (NOT_MEASURED, NOT_MEASURED)
    n_kept = b1.sizes()[1]
    b1.close()
    b2.close()
    return {"depth": depth, "candidates": int(len(cand)), "kept_reads": n_kept, "aligned_bases": int(bases), "parity": parity,
            "gpu_cand_per_s": len(cand) / t_gpu, "gpu_bases_per_s": bases / t_gpu, "e2e_cand_per_s": len(cand) / t_e2e,
            "forward_cand_per_s": len(cand) / t_fwd, "cpu_cand_per_s_1proc": cpu1, "cpu_cand_per_s_all_cores": cpun,
            "cpu_cores": os.cpu_count()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--region", type=int, default=200000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-cpu", dest="cpu", action="store_false")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    sd = synth.fa_state_dict(True, channels=8, seed=1)
    model = Clair3_F(add_indel_length=True, predict=True, input_channels=8)
    model.to(dev)
    model.eval()
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    res = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "region_bp": args.region,
           "runs": [bench_depth(d, args, model) for d in (50, 150)]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
