"""``python -m clair3_b200.run_clair3``: Clair3's ``run_clair3.py`` for the options this project runs (DESIGN.md 5g).

    python -m clair3_b200.run_clair3 --bam_fn in.bam --ref_fn ref.fa --model_path MODEL_DIR --platform ont \\
        --output OUT_DIR --no_phasing_for_fa True

Loads ``pileup.pt`` and ``full_alignment.pt`` from ``--model_path`` and writes ``pileup.vcf.gz``, ``full_alignment.vcf.gz`` and
``merge_output.vcf.gz`` with their ``.tbi`` into ``--output`` (``genome.call_genome``).  Several GPUs: start one process per GPU
with ``torchrun --nproc_per_node N -m clair3_b200.run_clair3 ...``; each rank takes the GPU of its ``LOCAL_RANK``.
``--threads`` is accepted and ignored.  Phasing (``--no_phasing_for_fa`` not True), ``--gvcf``, the haploid modes and
platform ``ilmn`` are refused.
"""
from __future__ import annotations

import argparse
import os
import shlex
import sys


def _bool(v):
    if isinstance(v, bool):
        return v
    if v.lower() in ("yes", "true", "t", "y", "1"):
        return True
    if v.lower() in ("no", "false", "f", "n", "0"):
        return False
    raise argparse.ArgumentTypeError("boolean value expected, got %r" % v)


def parser():
    p = argparse.ArgumentParser(prog="python -m clair3_b200.run_clair3",
                                description="Call variants from an indexed BAM and an indexed FASTA with Clair3's cascade on the GPU")
    p.add_argument("--bam_fn", required=True)
    p.add_argument("--ref_fn", required=True)
    p.add_argument("--model_path", required=True, help="folder with pileup.pt and full_alignment.pt")
    p.add_argument("--platform", required=True, choices=["ont", "hifi", "ilmn"])
    p.add_argument("--output", required=True)
    p.add_argument("--threads", type=int, default=1, help="accepted for compatibility; ignored")
    p.add_argument("--sample_name", default="SAMPLE")
    p.add_argument("--ctg_name", default="EMPTY")
    p.add_argument("--bed_fn", default="EMPTY")
    p.add_argument("--vcf_fn", default="EMPTY")
    p.add_argument("--chunk_size", type=int, default=5000000)
    p.add_argument("--min_contig_size", type=int, default=0)
    p.add_argument("--qual", type=int, default=2)
    p.add_argument("--var_pct_full", type=float, default=0)
    p.add_argument("--ref_pct_full", type=float, default=0)
    p.add_argument("--snp_min_af", type=float, default=0)
    p.add_argument("--indel_min_af", type=float, default=0)
    p.add_argument("--min_mq", type=int, default=5)
    p.add_argument("--min_coverage", type=int, default=2)
    for flag in ("--include_all_ctgs", "--call_snp_only", "--enable_long_indel", "--enable_variant_calling_at_sequence_head_and_tail",
                 "--print_ref_calls", "--pileup_only", "--no_phasing_for_fa", "--enable_dwell_time", "--gvcf", "--haploid_precise",
                 "--haploid_sensitive"):
        p.add_argument(flag, nargs="?", const=True, default=False, type=_bool)
    return p


def main(argv=None):
    argv = sys.argv[1:] if argv is None else list(argv)
    args = parser().parse_args(argv)
    import torch

    from . import genome, launcher
    from .model import Clair3_F, Clair3_P

    if args.platform == "ilmn":
        raise NotImplementedError("run_clair3: platform 'ilmn' is not implemented")
    if not args.no_phasing_for_fa:
        raise NotImplementedError("run_clair3: phasing for full alignment is not implemented; add --no_phasing_for_fa True")
    # run_clair3.py:283-288, 380-388: absolute input paths, and the floors of the read filters
    bam_fn, ref_fn = os.path.abspath(args.bam_fn), os.path.abspath(args.ref_fn)
    min_mq, min_coverage, min_contig_size = max(args.min_mq, 5), max(args.min_coverage, 2), max(args.min_contig_size, 0)
    group, local = None, 0
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        import torch.distributed as dist
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        dist.init_process_group("nccl" if torch.cuda.device_count() > 1 else "gloo")
        group = dist.group.WORLD
    dev = torch.device("cuda", torch.cuda.current_device())
    channels = 9 if args.enable_dwell_time else 8
    m_p = Clair3_P(add_indel_length=False, predict=True, input_channels=18)
    m_f = Clair3_F(add_indel_length=True, predict=True, input_channels=channels)
    for m, name in ((m_p, "pileup"), (m_f, "full_alignment")):
        m.to(dev)
        m.load_state_dict(launcher.load_checkpoint(os.path.join(args.model_path, name)))
        m.eval()
    try:
        out = genome.call_genome(
            bam_fn, ref_fn, m_p, m_f, os.path.abspath(args.output), platform=args.platform, sample_name=args.sample_name,
            cmdline=" ".join(shlex.quote(a) for a in [sys.argv[0]] + argv), ctg_name=args.ctg_name,
            include_all_ctgs=args.include_all_ctgs, min_contig_size=min_contig_size, chunk_size=args.chunk_size,
            bed_fn=None if args.bed_fn == "EMPTY" else os.path.abspath(args.bed_fn),
            vcf_fn=None if args.vcf_fn == "EMPTY" else os.path.abspath(args.vcf_fn), qual=args.qual,
            var_pct_full=args.var_pct_full, ref_pct_full=args.ref_pct_full, snp_min_af=args.snp_min_af,
            indel_min_af=args.indel_min_af, min_mq=min_mq, min_coverage=min_coverage, call_snp_only=args.call_snp_only,
            enable_long_indel=args.enable_long_indel,
            enable_variant_calling_at_sequence_head_and_tail=args.enable_variant_calling_at_sequence_head_and_tail,
            print_ref_calls=args.print_ref_calls, pileup_only=args.pileup_only, no_phasing_for_fa=args.no_phasing_for_fa,
            enable_dwell_time=args.enable_dwell_time, gvcf=args.gvcf, haploid_precise=args.haploid_precise,
            haploid_sensitive=args.haploid_sensitive, device=dev, group=group)
    finally:
        if group is not None:
            import torch.distributed as dist
            dist.destroy_process_group()
    if out is not None:
        for name, path in out["files"].items():
            print("[INFO] %s: %s (%d rows)" % (name, path, out["rows"][name]))
    return 0


if __name__ == "__main__":
    sys.exit(main())
