"""One-process-per-GPU driver for the network stage of Clair3's GPU mode (SURVEY.md 8f N2).

The reference's multi-GPU mode (``clair3/CallVariantsFromCffiGPU.py:75-333``) first stages every chunk's candidate tensors as
``<prefix>.npy`` + ``<prefix>.info`` files (``preprocess/CreateTensorPileupFromCffi.py:443-452``), sizes a number of "GPU
threads" from ``nvidia-smi`` free memory (``:13-43``), cuts the file list into contiguous per-slot lists (``:141-156`` /
``:268-283``) and starts one ``CallVariantsFromCffi`` OS process per slot with GNU parallel (``:163-199``), each of which
loads the checkpoint again and runs ``_torch_predict`` + ``batch_output`` serially.

This module replaces that launcher for the network stage:

    torchrun --nnodes=1 --nproc-per-node N -m clair3_b200.launcher \\
        --file_list tmp/pileup_file_list --chkpnt_fn model/pileup --pileup --out_prefix tmp/pileup_pred

* one rank per GPU (no memory-slot heuristic), the SAME contiguous cut of the file list as the reference (``split_file_list``),
  so every rank's output is in the reference's order;
* rank 0 reads the ``.pt`` (``_load_torch_checkpoint`` semantics: optional ``.pt`` suffix, bare or ``{"state_dict": ...}``) and
  the packed weight images reach the other ranks by ONE NCCL broadcast (``sharding.broadcast_weights``);
* each rank streams its files through ``predict_stream`` (pinned staging, H2D / kernels / D2H of consecutive batches overlapped)
  and writes ``<out_prefix>_<rank>.prediction / .position / .alt_info`` - exactly the memmaps the reference's own
  ``CallVariants --predict_fn`` writes (``clair3/CallVariants.py:1790-1796``) and its ``--input_probabilities`` replay reads
  (``:1624-1685``) - so the reference's unmodified decoder turns every shard into a VCF shard:
  ``python clair3.py CallVariants --input_probabilities --tensor_fn <out_prefix>_<rank> --call_fn <rank>.vcf ...``
  (the command is written to ``<out_prefix>_<rank>.decode_cmd``; ``--clair3_entry path/to/clair3.py`` runs it);
* ``--drop_ref_calls``: rows that the GPU-side first stage of the decoder (``c3b_decode_stage1``) marks as early-out
  homozygous-reference calls - which ``output_with`` drops unless ``--showRef`` (``clair3/CallVariants.py:1182-1186``) - are not
  written at all, so the per-site Python decoder only sees the sites that can become variants.
* ``--decode_rows``: each rank also decodes its shard in-process (``clair3_b200.decode.batch_output``: stage 1 and the
  outcome ranking of stage 2 on the GPU, the alt-info checks and row formatting on the host) and writes
  ``<out_prefix>_<rank>.vcf_rows`` - the VCF body (no header lines) that the replay command above writes for the shard with
  its default options.

The tensors keep the reference's wire dtypes (int8 ``.npy``, the GPU-mode narrowing of ``CreateTensorPileupFromCffi.py:447``).
Host-side logic (file split, batching, shard writing) has no CUDA dependency and is covered by the gloo CPU tests with a stub
model; the product path constructs the sm_90a modules and fails without an H100.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

FLANKING_BASE_NUM = 16                   # shared/param_p.py flankingBaseNum: the centre of the 33-base reference window
REF_GT21 = {"A": 0, "C": 4, "G": 7, "T": 9}      # gt21_enum_from_label(base + base), clair3/task/gt21.py:29-61
BATCH_SITES = {"pileup": 1024, "fa": 256}


def split_file_list(files, slots):
    """The reference's contiguous cut: ceil(len / slots) files per slot, empty slots dropped
    (``clair3/CallVariantsFromCffiGPU.py:141-156``).  Returns ``slots`` lists (possibly empty at the tail)."""
    files = list(files)
    if slots <= 0:
        raise ValueError("slots must be positive")
    each = len(files) // slots if len(files) % slots == 0 else len(files) // slots + 1
    return [files[i * each:(i + 1) * each] for i in range(slots)]


def read_file_list(path):
    """File-list format of ``--output_tensor_can_fn_list``: one tensor prefix per line, relative to the list's directory
    (``clair3/CallVariantsFromCffi.py:107-114``)."""
    parent = os.path.dirname(os.path.abspath(path))
    out = []
    for line in open(path).read().strip().split("\n"):
        if line:
            out.append(line if os.path.isabs(line) else os.path.join(parent, line))
    return out


def load_tensor_file(prefix):
    """``<prefix>.npy`` + ``<prefix>.info`` (``position\\talt_info`` per line) -> (tensor, positions, alt_infos)
    (``clair3/CallVariantsFromCffi.py:112-125``)."""
    tensor = np.load(prefix + ".npy")
    positions, alt_infos = [], []
    for row in open(prefix + ".info").read().strip().split("\n"):
        if not row:
            continue
        pos, alt = row.split("\t")
        positions.append(pos)
        alt_infos.append(alt)
    if not (len(tensor) == len(positions) == len(alt_infos)):
        raise ValueError("%s: %d tensors but %d info rows" % (prefix, len(tensor), len(positions)))
    return tensor, positions, alt_infos


def iter_batches(files, batch_sites):
    """Batches in file order; the last batch of every file is ragged (``tensor_generator_for_chunk``, ``:126-134``)."""
    for prefix in files:
        tensor, positions, alt_infos = load_tensor_file(prefix)
        for s in range(0, len(tensor), batch_sites):
            yield tensor[s:s + batch_sites], positions[s:s + batch_sites], alt_infos[s:s + batch_sites]


def center_ref_gt21(position_strings):
    """gt21 index of ref+ref per site from the ``ctg:pos:refseq`` strings (``output_with``, ``clair3/CallVariants.py:1133-1143``:
    the centre base of a 33-base window, or the only base); 255 where the base is not A/C/G/T (such rows are never dropped)."""
    out = np.full(len(position_strings), 255, dtype=np.uint8)
    for i, s in enumerate(position_strings):
        seq = s.rstrip().split(":")[-1]
        base = seq[FLANKING_BASE_NUM if len(seq) > 1 else 0].upper() if seq else "N"
        out[i] = REF_GT21.get(base, 255)
    return out


class ShardWriter:
    """``.prediction`` / ``.position`` / ``.alt_info`` in the reference's replay format (``clair3/CallVariants.py:1790-1796``)."""

    def __init__(self, prefix, capacity, out_dim):
        self.prefix, self.n = prefix, 0
        cap = max(int(capacity), 1)
        self.pred = np.lib.format.open_memmap(prefix + ".prediction.tmp", dtype=np.float32, mode="w+", shape=(cap, out_dim))
        self.pos = np.lib.format.open_memmap(prefix + ".position.tmp", dtype="S100", mode="w+", shape=(cap, 1))
        self.alt = np.lib.format.open_memmap(prefix + ".alt_info.tmp", dtype="S2000", mode="w+", shape=(cap, 1))

    def append(self, y, positions, alt_infos):
        k = len(y)
        self.pred[self.n:self.n + k] = y
        self.pos[self.n:self.n + k, 0] = np.array([p.encode() for p in positions], dtype="S100") if k else []
        self.alt[self.n:self.n + k, 0] = np.array([a.encode() for a in alt_infos], dtype="S2000") if k else []
        self.n += k

    def close(self):
        """Trim to the rows written (the reference's reader takes the array length as the dataset size)."""
        for name, arr in ((".prediction", self.pred), (".position", self.pos), (".alt_info", self.alt)):
            out = np.lib.format.open_memmap(self.prefix + name, dtype=arr.dtype, mode="w+", shape=(self.n,) + arr.shape[1:])
            out[:] = arr[:self.n]
            out.flush()
            del out
        del self.pred, self.pos, self.alt
        for name in (".prediction", ".position", ".alt_info"):
            os.remove(self.prefix + name + ".tmp")
        return self.n


def run_rank(model, files, out_prefix, kind, drop_ref_calls=False, streams=8, decode=None, decode_rows=None):
    """Network stage of one rank: files -> shard.  ``model`` follows the module protocol (``predict_stream`` and, for
    ``drop_ref_calls``, ``decode_stage1``); returns (sites read, rows written).  ``decode_rows``: an OutputConfig; the shard's
    rows are also decoded (``decode_stage1`` / ``decode_stage2`` of ``model``) into ``<out_prefix>.vcf_rows``."""
    batch_sites = BATCH_SITES[kind]
    metas = []
    vcf = None
    if decode_rows is not None:
        from . import decode as host_decode
        vcf = open(out_prefix + ".vcf_rows", "w")

    def tensors():
        for x, positions, alt_infos in iter_batches(files, batch_sites):
            metas.append((positions, alt_infos))
            yield x

    total = sum(len(np.load(f + ".npy", mmap_mode="r")) for f in files)
    writer = ShardWriter(out_prefix, total, model.out_dim)
    read = 0
    for y in model.predict_stream(tensors(), streams=streams):
        positions, alt_infos = metas.pop(0)
        read += len(y)
        if drop_ref_calls and len(y):
            gt = center_ref_gt21(positions)
            known = gt != 255
            d = (decode or model.decode_stage1)(y, np.where(known, gt, 0).astype(np.uint8))
            is_ref = np.asarray(d["is_ref"].cpu() if hasattr(d["is_ref"], "cpu") else d["is_ref"]).astype(bool) & known
            keep = np.nonzero(~is_ref)[0]
            y = y[keep]
            positions = [positions[i] for i in keep]
            alt_infos = [alt_infos[i] for i in keep]
        writer.append(y, positions, alt_infos)
        if vcf is not None and len(y):
            vcf.write(host_decode.batch_output(model, positions, alt_infos, y, decode_rows))
    if vcf is not None:
        vcf.close()
    return read, writer.close()


def load_checkpoint(path):
    """``_load_torch_checkpoint`` semantics (``clair3/CallVariantsFromCffi.py:19-28``) on the host."""
    import torch
    if not path.endswith(".pt"):
        path = path + ".pt"
    ckpt = torch.load(path, map_location="cpu")
    return ckpt["state_dict"] if isinstance(ckpt, dict) and "state_dict" in ckpt else ckpt


def decode_command(args, rank, shard):
    cmd = [args.python, args.clair3_entry or "clair3.py", "CallVariants", "--input_probabilities", "--tensor_fn", shard,
           "--call_fn", os.path.join(args.call_dir or os.path.dirname(shard), "%s_%d.vcf" % ("pileup" if args.pileup else "full_alignment", rank)),
           "--sampleName", args.sampleName, "--platform", args.platform]
    if args.ref_fn:
        cmd += ["--ref_fn", args.ref_fn]
    if args.pileup:
        cmd += ["--pileup"]
    if args.add_indel_length:
        cmd += ["--add_indel_length", "True"]
    return cmd


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--file_list", required=True, help="tensor prefixes, one per line (the reference's per-GPU list format)")
    ap.add_argument("--chkpnt_fn", required=True)
    ap.add_argument("--out_prefix", required=True)
    ap.add_argument("--pileup", action="store_true")
    ap.add_argument("--add_indel_length", action="store_true")
    ap.add_argument("--enable_dwell_time", action="store_true")
    ap.add_argument("--platform", default="ont")
    ap.add_argument("--drop_ref_calls", action="store_true")
    ap.add_argument("--decode_rows", action="store_true",
                    help="also decode every shard in-process into <out_prefix>_<rank>.vcf_rows (VCF body, no header)")
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--clair3_entry", default=None, help="path to the reference's clair3.py: run its decoder on every shard")
    ap.add_argument("--call_dir", default=None)
    ap.add_argument("--python", default=sys.executable)
    ap.add_argument("--sampleName", default="SAMPLE")
    ap.add_argument("--ref_fn", default=None)
    args = ap.parse_args(argv)

    import torch
    import torch.distributed as dist

    from . import sharding
    from .model import Clair3_F, Clair3_P

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    device = torch.device("cuda", local_rank)
    torch.cuda.set_device(device)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)

    kind = "pileup" if args.pileup else "fa"
    if args.pileup:
        m = Clair3_P(add_indel_length=args.add_indel_length, predict=True, input_channels=18)
    else:
        m = Clair3_F(add_indel_length=args.add_indel_length, predict=True, input_channels=8 + (1 if args.enable_dwell_time else 0))
    m.to(device)
    m.eval()
    sd = load_checkpoint(args.chkpnt_fn)                 # every rank reads the (small) key/shape table; only rank 0's values count
    if rank != 0:
        sd = {k: torch.zeros_like(v) for k, v in sd.items()}
    m.load_state_dict(sd)
    if world > 1:
        sharding.broadcast_weights(m, src=0)

    files = split_file_list(read_file_list(args.file_list), world)[rank]
    shard = "%s_%d" % (args.out_prefix, rank)
    rows_config = None
    if args.decode_rows:
        from .decode import replay_config
        rows_config = replay_config(args.pileup, args.add_indel_length)
    read, written = run_rank(m, files, shard, kind, drop_ref_calls=args.drop_ref_calls, streams=args.streams,
                             decode_rows=rows_config)
    cmd = decode_command(args, rank, shard)
    with open(shard + ".decode_cmd", "w") as f:
        f.write(" ".join(cmd) + "\n")
    print("[clair3_b200.launcher] rank %d/%d: %d files, %d sites, %d rows -> %s" % (rank, world, len(files), read, written, shard), flush=True)
    if args.clair3_entry and written:
        import subprocess
        subprocess.check_call(cmd)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
