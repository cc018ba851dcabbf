"""Read-based phasing on the GPU (``include/clair3_b200_phase.h``, ``csrc/phase.cu``; DESIGN.md 5g.3): ``clair3_b200.phasing``'s
statement, with the allele observations and the DP on the device.

* ``fragments`` reads the observations of device-resident records (``BamDecoder.decode(..., fa_fields=True)``) at a contig's
  variants: one warp per record, compacted by a block scan.  ``contig_fragments`` decodes a contig span by span and takes each
  read only in the span that holds its alignment start, so the observations equal ``phasing.fragments`` over the whole
  contig's records.
* Read selection and the blocks stay on the host (``phasing.layout``): the greedy selection admits one read at a time in a
  global order, each admission depending on every earlier one, and both run over the compact observations (a few per read),
  not over the records.
* ``solve`` runs every block's DP and backtrace on the device (``c3b_phase_dp``) and returns what ``phasing.solve`` returns.

No CPU fallback: everything here calls ``libclair3b200.so``.
"""
from __future__ import annotations

import numpy as np
import torch

from . import phasing
from ._ffi import PHASE_CONSTANTS, C3BError, check, ffi, lib
from .records import records_struct

SEGMENT = PHASE_CONSTANTS["C3B_PHASE_SEGMENT"]


def _stream(device):
    return ffi.cast("void *", torch.cuda.current_stream(device).cuda_stream)


def _ptr(ctype, t):
    return ffi.cast(ctype + " *", t.data_ptr())


def device_variants(variants, device):
    """``phasing.Variants`` as the device tensors ``c3b_phase_variants`` points at: (struct, tensors that own the memory)."""
    t = [torch.from_numpy(np.ascontiguousarray(a)).to(device) for a in (variants.pos, variants.ref, variants.alt)]
    s = ffi.new("c3b_phase_variants *")
    s.n = len(variants.pos)
    s.pos, s.ref, s.alt = (_ptr("const " + c, x) if x.numel() else ffi.NULL for c, x in zip(("int64_t", "uint8_t", "uint8_t"), t))
    return s, t


def fragments(rec, dvariants, lo, hi, read_base):
    """The observations of the records ``rec`` (``DeviceBamRecords`` with qualities) whose pos lies in [lo, hi), at the device
    variants ``dvariants`` (``device_variants``' result): ``phasing.Fragments`` on the host, read ids counted from
    ``read_base`` at the first record with pos >= lo, and the number of records with pos >= lo.  One host wait for the sizes."""
    if rec.t.get("qual") is None:
        raise C3BError("phase_gpu.fragments: the records need their qualities (decode with fa_fields=True)")
    dev, (vs, _) = rec.device, dvariants
    L = lib()
    st = records_struct(rec, optional=True)
    offsets = torch.empty(rec.n_reads + 1, dtype=torch.int64, device=dev)
    n_ent, first = ffi.new("int64_t *"), ffi.new("int64_t *")
    check(L.c3b_phase_count(st, int(lo), int(hi), vs, _ptr("int64_t", offsets), n_ent, first, _stream(dev)))
    n, first = int(n_ent[0]), int(first[0])
    out = [torch.empty(max(n, 1), dtype=d, device=dev)[:n] for d in (torch.int64, torch.int32, torch.uint8, torch.uint8)]
    if n:
        check(L.c3b_phase_write(st, int(lo), int(hi), vs, _ptr("const int64_t", offsets), first, int(read_base),
                                _ptr("int64_t", out[0]), _ptr("int32_t", out[1]), _ptr("uint8_t", out[2]), _ptr("uint8_t", out[3]),
                                _stream(dev)))
    return phasing.Fragments(*(x.cpu().numpy() for x in out)), rec.n_reads - first


def contig_fragments(decoder, bam_fn, ctg, length, variants, span, index=None):
    """``phasing.fragments`` of every record of contig ``ctg`` on the GPU: the contig decoded in spans of ``span`` bases, each
    record taken in the span that holds its pos (the last span reaches past the contig's end)."""
    if not len(variants.pos):
        return phasing.empty_fragments()
    dv = device_variants(variants, decoder._device)
    parts, base = [], 0
    starts = list(range(0, max(int(length), 1), int(span)))
    for i, lo in enumerate(starts):
        last = i == len(starts) - 1
        hi = None if last else lo + int(span)
        rec = decoder.decode(bam_fn, ctg, lo, hi, fa_fields=True, index=index)
        f, taken = fragments(rec, dv, lo, (1 << 62) if last else hi, base)
        base += taken
        parts.append(f)
        del rec
    return phasing.Fragments(*(np.concatenate(a) for a in zip(*parts)))


def solve(lay, device, n_ctas=None):
    """``phasing.solve`` on the device: (haplotype 0's allele per column, cost per block), from one ``c3b_phase_dp`` call."""
    nb, nc = lay.n_blocks, len(lay.col_var)
    if nb == 0:
        return np.zeros(0, np.uint8), np.zeros(0, np.int64)
    device = torch.device(device)
    m = np.diff(lay.blk_col_off)
    slot = np.left_shift(np.int64(1), lay.blk_kmax.astype(np.int64) - 1)
    n_ck = (m + SEGMENT - 1) // SEGMENT - 1
    ckpt_off = np.concatenate([[0], np.cumsum(n_ck * slot)])
    order = np.lexsort((np.arange(nb), -(m * slot))).astype(np.int64)          # the largest blocks first
    up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(device)   # noqa: E731
    t = {"col_off": up(lay.blk_col_off, np.int64), "read_off": up(lay.blk_read_off, np.int64), "kmax": up(lay.blk_kmax, np.int32),
         "ckpt_off": up(ckpt_off[:-1], np.int64), "read_first": up(lay.read_first, np.int32),
         "read_last": up(lay.read_last, np.int32), "ent_off": up(lay.col_ent_off, np.int64),
         "ent_read": up(lay.ent_read, np.int32), "ent_allele": up(lay.ent_allele, np.uint8),
         "ent_weight": up(lay.ent_weight, np.uint8), "order": up(order, np.int64)}
    s = ffi.new("c3b_phase_blocks *")
    s.n_blocks, s.n_cols = nb, nc
    ctypes = {"col_off": "int64_t", "read_off": "int64_t", "kmax": "int32_t", "ckpt_off": "int64_t", "read_first": "int32_t",
              "read_last": "int32_t", "ent_off": "int64_t", "ent_read": "int32_t", "ent_allele": "uint8_t",
              "ent_weight": "uint8_t", "order": "int64_t"}
    for k, v in t.items():
        setattr(s, k, _ptr("const " + ctypes[k], v) if v.numel() else ffi.cast("const %s *" % ctypes[k], 8))
    if n_ctas is None:
        n_ctas = torch.cuda.get_device_properties(device).multi_processor_count
    n_ctas = int(min(n_ctas, nb))
    seg_stride = int(slot.max())
    hap = torch.empty(nc, dtype=torch.uint8, device=device)
    cost = torch.empty(nb, dtype=torch.int64, device=device)
    ckpt = torch.empty(max(int(ckpt_off[-1]), 1), dtype=torch.int32, device=device)
    seg = torch.empty(n_ctas * SEGMENT * seg_stride, dtype=torch.int16, device=device)
    meta = torch.empty(4 * nc, dtype=torch.int16, device=device)
    ebit = torch.empty(max(len(lay.ent_read), 1), dtype=torch.uint8, device=device)
    status = torch.empty(1, dtype=torch.int64, device=device)
    check(lib().c3b_phase_dp(s, n_ctas, _ptr("uint8_t", hap), _ptr("int64_t", cost), _ptr("uint32_t", ckpt), _ptr("uint16_t", seg),
                             seg_stride, _ptr("uint16_t", meta), _ptr("uint8_t", ebit), _ptr("int64_t", status), _stream(device)))
    bad = int(status.item())
    if bad:
        raise C3BError("c3b_phase_dp: block %d breaks the layout's bounds (more than %d active reads, or a column no read links)"
                       % (bad - 1, phasing.MAX_COVERAGE))
    return hap.cpu().numpy(), cost.cpu().numpy()


def dp_attributes():
    """The DP kernel's registers, shared memory bytes, local memory bytes and thread limit."""
    r, sm, lm, mt = ffi.new("int *"), ffi.new("int64_t *"), ffi.new("int64_t *"), ffi.new("int *")
    check(lib().c3b_phase_dp_attributes(r, sm, lm, mt))
    return {"registers": int(r[0]), "shared_bytes": int(sm[0]), "local_bytes": int(lm[0]), "max_threads": int(mt[0])}


def phase_contig(decoder, bam_fn, ctg, length, rows, span, index=None):
    """``phasing.phase_contig`` on the GPU for contig ``ctg`` of ``length`` bases: its rows with the phased ones rewritten,
    and (variants, fragments, layout, haplotypes, costs)."""
    v = phasing.het_snvs(rows)
    frag = contig_fragments(decoder, bam_fn, ctg, length, v, span, index)
    lay = phasing.layout(frag, len(v.pos))
    hap, cost = solve(lay, decoder._device)
    return phasing.phase_rows(rows, v, lay, hap), v, frag, lay, hap, cost
