"""Host side of the GPU full-alignment tensor builder (``include/clair3_b200_fa.h``; SURVEY.md 8f row N4, full-alignment half).

Mirrors the reference's ``CreateTensorFullAlignment`` (HKU-BAL/Clair3 ``preprocess/CreateTensorFullAlignmentFromCffi.py:19-170``:
``lib.calculate_clair3_full_alignment`` -> int8 ``[candidates, depth, 33, 8|9]`` + ``all_alt_info`` strings) from the point where
htslib has decoded the alignment records: the caller hands over the ``bam1_t`` fields as ``BamRecords`` (with ``qual``, ``qname``
and, for dwell time, ``mv``), the tensor is built on the H100 and can go straight into Clair3_F without leaving HBM.  No CPU
fallback: everything here calls ``libclair3b200.so``.
"""
from __future__ import annotations

import gzip

import numpy as np
import torch

from ._ffi import C3BError, check, ffi, lib
from .pileup_counts import BamRecords, DeviceBamRecords, _insertion_bytes, khash_iteration_order

FLANKING = 16                   # shared/param_f.py flankingBaseNum
NO_OF_POSITIONS = 33
MATRIX_DEPTH = {"ont": 89, "hifi": 55, "ilmn": 55}      # shared/param_f.py matrix_depth_dict
_ACGT = "ACGT"
_ACGT2NUM = {"C": 1, "G": 2, "T": 3}                    # acgt2num (src/clair3_full_alignment_dwell.h:49-54): others -> 0


def _fa_struct(rec, on_dev):
    s = ffi.new("c3b_fa_records *")
    s.core = rec._struct()[0]
    for k, ct in (("qual", "uint8_t"), ("qname", "uint8_t"), ("mv", "int32_t")):
        if on_dev:
            v, o = rec.t.get(k), rec.t.get(k + "_off")
            vp, op = (ffi.NULL, ffi.NULL) if o is None else (v.data_ptr(), o.data_ptr())
        else:
            v, o = getattr(rec, k, None), getattr(rec, k + "_off", None)
            vp, op = (ffi.NULL, ffi.NULL) if o is None else (v.ctypes.data if v.size else ffi.NULL, o.ctypes.data)
        if o is not None and vp == ffi.NULL:
            vp = ffi.cast("void *", 8)          # an empty value array with valid offsets: never dereferenced
        setattr(s, k + "_off", ffi.cast("const int64_t *", op))
        setattr(s, k, ffi.cast("const %s *" % ct, vp))
    return s


def _variant_array(variants):
    """(position, ref_base, alt_base, genotype, phase_set) tuples -> c3b_fa_variant[] (``struct Variant``)."""
    n = len(variants)
    arr = ffi.new("c3b_fa_variant[]", max(n, 1))
    for i, (p, rb, ab, gt, ps) in enumerate(variants):
        arr[i].position = int(p)
        arr[i].ref_base = (rb.encode() if isinstance(rb, str) else bytes([rb]))[:1]
        arr[i].alt_base = (ab.encode() if isinstance(ab, str) else bytes([ab]))[:1]
        arr[i].genotype = int(gt)
        arr[i].phase_set = int(ps)
    return arr, n


class FullAlignmentBuilder:
    """One tensor-building workspace on one H100 (``c3b_fa``).  ``build()`` is asynchronous on the current torch stream of the
    device (apart from two short waits that size its scratch); ``fetch()`` / ``alt_info_strings()`` wait for it."""

    def __init__(self, device=0):
        dev = torch.device(device) if not isinstance(device, int) else torch.device("cuda", device)
        if dev.type != "cuda":
            raise C3BError("FullAlignmentBuilder needs a CUDA device (no CPU fallback)")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self._device = dev
        out = ffi.new("c3b_fa **")
        check(lib().c3b_fa_create(out, dev.index or 0))
        self._h = out[0]
        self._keep = None
        self._shape = None

    def build(self, records, candidates, ref_seq, ref_start, variants=None, matrix_depth=89, need_haplotagging=True, min_mq=5,
              max_indel_length=50, dwell=False, rand_seed=1, rand_skip=0):
        """``calculate_clair3_full_alignment`` (src/clair3_full_alignment_dwell.c:437) on decoded records.  ``candidates``: 0-based
        positions, strictly ascending.  ``ref_seq``: the reference bases from ``ref_start`` (str / bytes, or a uint8 tensor on the
        device with device records).  ``variants``: phased heterozygous SNPs as (position, ref_base, alt_base, genotype 1|2,
        phase_set) sorted by position (``phased_variants_from_vcf``).  ``dwell``: 9 channels, the last from the ``mv`` tag.
        The shuffle of candidates with more than ``matrix_depth`` reads draws from glibc ``rand()`` after ``srand(rand_seed)`` and
        ``rand_skip`` draws; ``rand_seed=1, rand_skip=0`` is what a fresh process sees (``draws`` in ``sizes()`` chains calls)."""
        on_dev = isinstance(records, DeviceBamRecords)
        rec = records if on_dev else BamRecords.from_dict(records)
        cand = np.ascontiguousarray(candidates, dtype=np.int64)
        if cand.ndim != 1 or (len(cand) and (cand[0] < 0 or (np.diff(cand) <= 0).any())):
            raise C3BError("build: candidates must be 0-based positions in strictly ascending order")
        var, nv = _variant_array(list(variants) if variants is not None else [])
        prm = ffi.new("c3b_fa_params *")
        prm.matrix_depth, prm.need_haplotagging, prm.min_mq = int(matrix_depth), int(bool(need_haplotagging)), int(min_mq)
        prm.dwell, prm.rand_seed, prm.rand_skip = int(bool(dwell)), int(rand_seed) & 0xFFFFFFFF, int(rand_skip)
        st = _fa_struct(rec, on_dev)
        stream = torch.cuda.current_stream(self._device).cuda_stream
        if on_dev:
            if ref_seq is None:
                ref_seq = rec.ref
            if not (isinstance(ref_seq, torch.Tensor) and ref_seq.dtype == torch.uint8 and ref_seq.device == rec.device):
                raise C3BError("build: device records need the reference bases as a uint8 tensor on the same device")
            ref, refbuf = ref_seq.contiguous(), None
            refptr, reflen = ffi.cast("const char *", ref.data_ptr()), ref.numel()
            host_ref = None
        else:
            ref = ref_seq.encode() if isinstance(ref_seq, str) else bytes(ref_seq)
            refbuf = ffi.from_buffer(ref)
            refptr, reflen = ffi.cast("const char *", refbuf), len(ref)
            host_ref = ref
        check(lib().c3b_fa_build(self._h, st, int(on_dev), ffi.cast("const int64_t *", cand.ctypes.data), len(cand), var, nv, refptr,
                                 int(ref_start), reflen, prm, ffi.cast("void *", stream)))
        self._keep = (rec, ref, refbuf, st, cand, var)      # buffers stay alive while the copies / kernels are in flight
        self._shape = (len(cand), int(matrix_depth), 9 if dwell else 8)
        self._alt = (host_ref, int(ref_start), int(max_indel_length))
        return self

    def sizes(self):
        """(candidates, kept reads, glibc rand() draws consumed)."""
        a, b, c = ffi.new("int64_t *"), ffi.new("int64_t *"), ffi.new("int64_t *")
        check(lib().c3b_fa_sizes(self._h, a, b, c))
        return int(a[0]), int(b[0]), int(c[0])

    def fetch(self):
        """The int8 matrix [n_cand, matrix_depth, 33, 8|9] (``fa_data.matrix``) as a numpy array."""
        n, depth, C = self._shape
        m = np.zeros((n, depth, NO_OF_POSITIONS, C), np.int8)
        check(lib().c3b_fa_fetch(self._h, ffi.cast("int8_t *", m.ctypes.data), ffi.NULL, ffi.NULL))
        return m

    def kept_reads(self):
        """(record index, haplotype 0/1/2) of every kept read, in the reference's read_array order (diagnosis)."""
        _, nk, _ = self.sizes()
        idx, hap = np.zeros(nk, np.int64), np.zeros(nk, np.int32)
        check(lib().c3b_fa_fetch(self._h, ffi.NULL, ffi.cast("int32_t *", hap.ctypes.data), ffi.cast("int64_t *", idx.ctypes.data)))
        return idx, hap

    def alt_info_strings(self):
        """The ``all_alt_info`` strings (src/clair3_full_alignment_dwell.c:950-1006), one per candidate: ``"<pos+1>-<depth>-<ref>-"``
        then ``X<b> n`` for the non-reference bases in A C G T order, ``I<ref><bases> n`` in the iteration order of the
        reference's khash string counter, ``D<ref bases> n`` in the order of its khash int counter, ``R<ref> n`` last."""
        host_ref, ref_start, max_indel = self._alt
        rec = self._keep[0]
        if host_ref is None or isinstance(rec, DeviceBamRecords):
            raise C3BError("alt_info_strings needs host records and reference (the inserted bases are read on the host)")
        n = self._shape[0]
        na = ffi.new("int64_t *")
        check(lib().c3b_fa_fetch_alleles(self._h, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, 0, na))
        k = int(na[0])
        depth, acgt = np.zeros(n, np.int32), np.zeros((n, 4), np.int32)
        al_off, al_n = np.zeros(n, np.int32), np.zeros(n, np.int32)
        meta, rd, qp, cn = (np.zeros(max(k, 1), np.uint32) for _ in range(4))
        c = ffi.cast
        check(lib().c3b_fa_fetch_alleles(self._h, c("int32_t *", depth.ctypes.data), c("int32_t *", acgt.ctypes.data),
                                         c("int32_t *", al_off.ctypes.data), c("int32_t *", al_n.ctypes.data),
                                         c("uint32_t *", meta.ctypes.data), c("uint32_t *", rd.ctypes.data),
                                         c("uint32_t *", qp.ctypes.data), c("uint32_t *", cn.ctypes.data), len(meta), na))
        cand = self._keep[4]
        out = []
        for i in range(n):
            sl = slice(int(al_off[i]), int(al_off[i]) + int(al_n[i]))
            out.append(format_alt_info(int(cand[i]), int(depth[i]), acgt[i], host_ref, ref_start, max_indel,
                                       meta[sl], rd[sl], qp[sl], cn[sl], rec))
        return out

    def forward(self, model):
        """Clair3_F over every candidate of the last build, straight from the device-resident matrix (``c3b_forward`` with
        ``x_on_device = 1``, int8).  Returns what ``model(x)`` returns for the same matrix, on the device."""
        if getattr(model, "_handle", None) is None:
            raise C3BError("forward: the model has no device / weights yet (.to(device), .load_state_dict())")
        n, depth, C = self._shape
        if model._kind != _const("C3B_FULL_ALIGNMENT") or model.input_channels != C:
            raise C3BError("forward: needs the full-alignment network (Clair3_F) with %d input channels" % C)
        if torch.device(model._device) != self._device:
            raise C3BError("forward: the model lives on %s, the builder on %s" % (model._device, self._device))
        self.sizes()
        y = torch.empty((n, model.out_dim), dtype=torch.float32, device=self._device)
        if n:
            pm = ffi.new("const int8_t **")
            check(lib().c3b_fa_device(self._h, pm))
            stream = torch.cuda.current_stream(self._device).cuda_stream
            check(lib().c3b_forward(model._handle, ffi.cast("void *", pm[0]), _const("C3B_DT_I8"), 1, n, depth,
                                    ffi.cast("float *", y.data_ptr()), 1, ffi.cast("void *", stream)))
        return model._split(y)

    def last_ms(self):
        ms, k = ffi.new("float *"), ffi.new("int *")
        check(lib().c3b_fa_last_ms(self._h, ms, k))
        return float(ms[0]), int(k[0])

    def close(self):
        if getattr(self, "_h", None) is not None:
            lib().c3b_fa_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _const(name):
    from ._ffi import CONSTANTS
    return CONSTANTS[name]


def format_alt_info(candidate, depth, acgt, ref, ref_start, max_indel_length, meta, read, qpos, cnt, rec):
    """One ``all_alt_info`` string (src/clair3_full_alignment_dwell.c:950-1006) from a candidate's depth, A/C/G/T counts and its
    distinct indel alleles in order of first occurrence."""
    off = candidate - ref_start
    raw = ref[off:off + 1] if 0 <= off < len(ref) else b"\0"
    rbc = raw.decode("latin-1").upper()
    rf = _ACGT2NUM.get(rbc, 0)
    ref_count = int(acgt[rf])
    parts = ["%d-%d-%s-" % (candidate + 1, depth, rbc)]
    for j in range(4):
        if j != rf and acgt[j] > 0:
            parts.append("X%s %d " % (_ACGT[j], int(acgt[j])))
    ins_keys, ins_cnt, del_keys, del_cnt, again = [], {}, [], {}, [False, False]
    for m, r, q, c in zip(meta.tolist(), read.tolist(), qpos.tolist(), cnt.tolist()):
        length = m & 0x3FFFFFFF
        again[m >> 31] |= bool(m >> 30 & 1)
        if m >> 31:
            key = _insertion_bytes(rec, r, q, length)
            ins_keys.append(key)
            ins_cnt[key] = c
        else:
            del_keys.append(length)
            del_cnt[length] = c
    for j in khash_iteration_order(ins_keys, put_after_last=again[1]):
        key = ins_keys[j]
        ref_count -= ins_cnt[key]
        if len(key) <= max_indel_length:
            parts.append("I%s%s %d " % (rbc, key.decode("latin-1"), ins_cnt[key]))
    for j in khash_iteration_order(del_keys, put_after_last=again[0]):
        length = del_keys[j]
        ref_count -= del_cnt[length]
        if length <= max_indel_length:
            tail = ref[off + 1:off + 1 + length]
            nul = tail.find(b"\0")
            parts.append("D%s %d " % ((tail if nul < 0 else tail[:nul]).decode("latin-1"), del_cnt[length]))
    if ref_count > 0:
        parts.append("R%s %d " % (rbc, ref_count))
    return "".join(parts)


def create_tensor_full_alignment(records, ctg_name, candidates, ref_seq, ref_start, variants=None, builder=None, device=0, **params):
    """``CreateTensorFullAlignment`` with ``tensor_can_fn == "PIPE"`` (preprocess/CreateTensorFullAlignmentFromCffi.py:136-170) on
    decoded records: returns (np_fa_data int8 [n, depth, 33, 8|9], all_position_info ["ctg:pos:ref"], all_alt_info
    ["depth-alt text"]).  Keyword arguments as ``FullAlignmentBuilder.build``."""
    own = builder is None
    builder = builder or FullAlignmentBuilder(device)
    try:
        builder.build(records, candidates, ref_seq, ref_start, variants=variants, **params)
        np_fa_data = builder.fetch()
        strings = builder.alt_info_strings()
    finally:
        if own:
            builder.close()
    all_position_info, all_alt_info = [], []
    for s in strings:
        pos, depth, center_ref_base, alt = s.rstrip().split("-")[:4]
        all_position_info.append(ctg_name + ":" + pos + ":" + center_ref_base)
        all_alt_info.append(depth + "-" + alt)
    return np_fa_data, all_position_info, all_alt_info


def candidates_from_bed(path, ctg_name):
    """Candidate centres of a ``--full_aln_regions`` bed (preprocess/CreateTensorFullAlignmentFromCffi.py:51-78, :113): rows
    ``ctg start end`` give the centre ``start + 1 + (end - start) // 2 - 1`` (1-based; ``end - 18`` when ``start == 0``); rows with
    a fourth column (phased SNPs) only widen the region.  Returns (0-based sorted unique candidates, ctg_start, ctg_end) with the
    1-based region bounds the reference uses, or ([], None, None) when no row names the contig."""
    centres, lo, hi = set(), None, None
    with open(path) as f:
        for row in f:
            row = row.rstrip().split("\t")
            if row[0] != ctg_name:
                continue
            position, end = int(row[1]) + 1, int(row[2]) + 1
            lo = position if lo is None else min(lo, position)
            hi = end if hi is None else max(hi, end)
            if len(row) <= 3:
                centres.add(end - FLANKING - 2 if position == 1 else position + (end - position) // 2 - 1)
    if lo is None:
        return [], None, None
    return sorted({c - 1 for c in centres if lo <= c <= hi}), lo, hi


def phased_variants_from_vcf(path, ctg_name=None):
    """Phased heterozygous variants of a (gzip-compressed or plain) VCF as ``struct Variant`` tuples (position 0-based, ref_base,
    alt_base, genotype 1 for 0|1 and 2 otherwise, phase_set = the last FORMAT value): preprocess/CreateTensorFullAlignmentFromCffi.py
    :81-108.  Unphased genotypes are skipped."""
    with open(path, "rb") as f:
        magic = f.read(2)
    opener = gzip.open if magic == b"\x1f\x8b" else open
    out = []
    with opener(path, "rt") as f:
        for row in f:
            row = row.rstrip()
            if not row or row[0] == "#":
                continue
            cols = row.strip().split("\t")
            if ctg_name and cols[0] != ctg_name:
                continue
            info = cols[9].split(":")
            genotype, phase_set = info[0], info[-1]
            if "|" not in genotype:
                continue
            out.append((int(cols[1]) - 1, cols[3][:1], cols[4][:1], 1 if genotype == "0|1" else 2, int(phase_set)))
    return out


def glibc_rand(seed=1, skip=0, n=1):
    """``n`` values of glibc ``rand()`` after ``srand(seed)`` and ``skip`` draws: the TYPE_3 additive generator (r[i] = r[i-31] +
    r[i-3] mod 2^32, output r >> 1) restated, with the skip taken by squaring its 31x31 transition matrix - the same jump the GPU
    builder makes per candidate."""
    seed &= 0xFFFFFFFF
    if seed == 0:
        seed = 1
    r = [0] * 375
    word = seed - (1 << 32) if seed >= 1 << 31 else seed
    r[0] = word & 0xFFFFFFFF
    for i in range(1, 31):
        hi, lo = int(word / 127773), word - int(word / 127773) * 127773           # C division truncates toward zero
        word = (16807 * lo - 2836 * hi)
        word = ((word + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)                     # int32
        if word < 0:
            word += 2147483647
        r[i] = word & 0xFFFFFFFF
    for i in range(31, 34):
        r[i] = r[i - 31]
    for i in range(34, 375):
        r[i] = (r[i - 31] + r[i - 3]) & 0xFFFFFFFF
    state = np.array(r[344:375], dtype=np.uint64)
    M = np.zeros((31, 31), dtype=np.uint64)
    for i in range(30):
        M[i, i + 1] = 1
    M[30, 0] = M[30, 28] = 1
    k = int(skip)
    while k:                                          # uint64 products wrap mod 2^64, which keeps them exact mod 2^32
        if k & 1:
            state = (M @ state) & 0xFFFFFFFF
        M = (M @ M) & 0xFFFFFFFF
        k >>= 1
    ring = [int(x) for x in state]
    out = []
    for t in range(n):
        if t < 31:
            v = ring[t]
        else:
            v = (ring[t % 31] + ring[(t - 3) % 31]) & 0xFFFFFFFF
            ring[t % 31] = v
        out.append(v >> 1)
    return np.array(out, dtype=np.int64)
