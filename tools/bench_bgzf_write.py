"""What writing BGZF costs on the GPU (``BamDecoder.write_bgzf``, ``c3b_bgzf_compress``) against the host writer
(``bam_io.write_bgzf``: zlib level 6 in one Python thread), and what it changes in the genome route's ``write`` stage.

    python tools/bench_bgzf_write.py [--repeats 5] [--vcf-mib 256] [--random-mib 64] [--out FILE]

Three inputs:

* ``genome_texts``: the pileup, full_alignment and merge_output texts of ``tools/bench_genome_call.py``'s first case (two
  2 Mb contigs, 1 Mb chunks), from one ``genome.call_genome`` run;
* ``vcf``: a ``--vcf-mib`` MiB VCF-like text (``tests/bgzf_corpus.vcf_text`` rows, a 16 MiB text repeated: BGZF blocks are
  independent and its window is 32 KiB, so the repeat changes nothing a block sees);
* ``random``: ``--random-mib`` MiB of seeded random bytes (every block stored).

For each: ``device_ms`` (the compression's three kernels between CUDA events, median of ``--repeats`` after a warm-up) and its
MiB/s; the host wall time from text in memory to file on disk for both writers in the same run (``device_writer_ms``,
``host_writer_ms``, medians); and whether the files are equal.  For the genome texts also the route's own ``write`` split:
``compress`` (both files of each text through the writer and to disk) and ``tbi`` (the Python index loop), once with the
host writer and once with the device writer, summed over the three files.  Prints one JSON line with the card's name and
power limit read in the same run.  Needs an H100.
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
import bgzf_corpus as bc  # noqa: E402
import test_gpu_genome as tg  # noqa: E402


def med(x):
    return float(np.median(x))


def writers(dec, d, data, repeats):
    """Device and host writer on one text: device ms, wall ms of each writer, equal files."""
    mib = len(data) / 2 ** 20
    dev_ms, dev_wall, host_wall = [], [], []
    dp, hp = os.path.join(d, "dev.gz"), os.path.join(d, "host.gz")
    dec.write_bgzf(dp, data)                              # warm-up: module load, buffer growth
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dec.write_bgzf(dp, data)
        dev_wall.append(1e3 * (time.perf_counter() - t0))
        dev_ms.append(dec.last_ms()[0])
        t0 = time.perf_counter()
        bam_io.write_bgzf(hp, data)
        host_wall.append(1e3 * (time.perf_counter() - t0))
    with open(dp, "rb") as f1, open(hp, "rb") as f2:
        equal = f1.read() == f2.read()
    return {"mib": round(mib, 3), "blocks": -(-len(data) // bam_io._BGZF_PAYLOAD), "device_ms": med(dev_ms),
            "device_mib_per_s": mib / (med(dev_ms) / 1e3) if med(dev_ms) > 0 else None, "device_writer_ms": med(dev_wall),
            "host_writer_ms": med(host_wall), "host_mib_per_s": mib / (med(host_wall) / 1e3), "equal_files": equal,
            "compressed_bytes": os.path.getsize(hp)}


def write_split(dec, d, texts, repeats):
    """The genome route's write of its texts (genome.write_vcf_gz), split into compress and tbi, host and device writer."""
    out = {}
    for label, decoder in (("host_writer", None), ("device_writer", dec)):
        runs = []
        for r in range(repeats + 1):
            st = cascade.Stages(dec._device)
            for n, t in texts.items():
                genome.write_vcf_gz(os.path.join(d, "%s_%s.vcf.gz" % (label, n)), t, decoder, st)
            s = st.summed()
            if r:
                runs.append({"compress_ms": s["compress"]["wall_ms"], "tbi_ms": s["write"]["wall_ms"],
                             "total_ms": s["total"]["wall_ms"]})
        out[label] = {k: med([x[k] for x in runs]) for k in runs[0]}
    equal = all(open(os.path.join(d, "host_writer_%s.vcf.gz%s" % (n, x)), "rb").read()
                == open(os.path.join(d, "device_writer_%s.vcf.gz%s" % (n, x)), "rb").read() for n in texts for x in ("", ".tbi"))
    out["equal_files"] = equal
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--vcf-mib", type=int, default=256)
    ap.add_argument("--random-mib", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    models = tg._models()
    ws = cascade.Workspaces(0)
    rows = {}
    try:
        with tempfile.TemporaryDirectory() as d:
            bam, fa = make(d, [("chr1", 2.0), ("chr2", 2.0)], 101)
            res = genome.call_genome(bam, fa, models[0], models[1], os.path.join(d, "out"), chunk_size=1_000_000, workspaces=ws)
            texts = res["texts"]
            rows["genome_route_stages_ms"] = {k: {x: round(y, 3) for x, y in v.items()} for k, v in res["stages"].items()}
            rows["genome_write_split"] = write_split(ws.decoder, d, texts, a.repeats)
            rows["genome_texts"] = {n: writers(ws.decoder, d, t.encode(), a.repeats) for n, t in texts.items()}
            unit = bc.vcf_text(200_000, 5).encode()[:16 << 20]
            vcf = (unit * (-(-(a.vcf_mib << 20) // len(unit))))[:a.vcf_mib << 20]
            rows["vcf"] = writers(ws.decoder, d, vcf, max(1, a.repeats // 2))
            del vcf
            rnd = np.random.default_rng(3).integers(0, 256, a.random_mib << 20, dtype=np.uint8).tobytes()
            rows["random"] = writers(ws.decoder, d, rnd, max(1, a.repeats // 2))
    finally:
        ws.close()
    line = {"bench": "bgzf_write", "gpu": name, "power_limit": limit, "cases": rows}
    text = json.dumps(line)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
