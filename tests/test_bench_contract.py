"""bench.py contract checks that need no GPU: the reference arm runs on host cores only and must print ONE JSON line with
the keys the driver reads; under a multi-rank launch only rank 0 works and prints."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(extra_env, *args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", **extra_env)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", *args], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return [l for l in r.stdout.splitlines() if l.startswith("{")]


def test_reference_arm_prints_one_contract_line():
    lines = _run({}, "--steps", "1", "--warmup", "1", "--workload", "fa")
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "candidate-sites/sec" and d["unit"] == "sites/s"
    assert d["higher_is_better"] is True and d["steps"] == 1 and d["value"] > 0
    assert d["e2e"] == {"value": d["value"], "unit": "sites/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["value"] == d["value"] and cb["cores"] >= 1 and "sample" in cb
    assert cb["single_process"]["value"] > 0 and cb["deployment_shape"]["processes"] >= 1
    assert "Full-alignment" in d["config"]["workload"]


def test_reference_arm_other_ranks_exit_quietly():
    assert _run({"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"}, "--steps", "1", "--warmup", "1", "--gpus", "2") == []


def test_workload_selection():
    """Default line: everything on one GPU; under a multi-rank launch the feature counter (replicas only, no exchange) is left out
    unless asked for by name."""
    sys.path.insert(0, ROOT)
    import bench
    default = "pileup,fa,fa_dwell,cascade,pileup_counts"
    assert bench.select_workloads(default, False, 1) == default.split(",")
    assert bench.select_workloads(default, False, 8) == ["pileup", "fa", "fa_dwell", "cascade"]
    assert bench.select_workloads("pileup_counts", True, 2) == ["pileup_counts"]


def test_counter_cpu_baseline_in_the_reference_deployment_shape():
    """bench.cpu_counts_all_cores: one single-threaded oracle process per chunk of the region, rates summed; together the workers
    count exactly the bases the one-process oracle counts."""
    sys.path.insert(0, ROOT)
    import bench
    from clair3_b200 import synth_reads as sr
    from oracle import pileup_oracle as po
    rec, ref, rs = sr.random_alignment(6000, depth=20, read_len=700, seed=2)
    r = bench.cpu_counts_all_cores(rec, ref, rs, 1000, 7000, 3, min_seconds=0.0)
    assert r["processes"] == 3 and r["value"] > 0 and r["unit"] == "bases/s"
    sub = po._reads_overlapping(rec, 3000, 5000)
    whole = po.clair3_pileup(rec, 3000, 5000, ref, rs)
    part = po.clair3_pileup(sub, 3000, 5000, ref, rs)
    assert len(sub["pos"]) < len(rec["pos"])
    for k in ("matrix", "major", "stats", "cand_cols"):
        assert np.array_equal(whole[k], part[k]), k


def test_summary_tool_renders_the_committed_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_summary.py"), os.path.join(ROOT, "profiles", "h100_bench_line.json")],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-1000:]
    for needle in ("| pileup |", "| fa |", "| cascade |", "## pileup_counts", "bases/s"):
        assert needle in r.stdout, needle
