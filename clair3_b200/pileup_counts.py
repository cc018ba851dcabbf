"""Host side of the GPU pileup feature counter (``include/clair3_b200_pileup.h``; SURVEY.md 8f row N4, pileup half).

Mirrors the reference's binding of ``calculate_clair3_pileup`` (HKU-BAL/Clair3 ``preprocess/CreateTensorPileupFromCffi.py:30-85,
127-180``: ``pileup_counts_clair3`` -> ``lib.calculate_clair3_pileup`` -> ``_plp_data_to_numpy``) from the point where htslib has
decoded the alignment records: the caller hands over the ``bam1_t`` fields as arrays (``BamRecords``), the counting, candidate
selection and - optionally - the Clair3_P forward over the candidates' windows run on the H100 without the count matrix ever
leaving HBM.  No CPU fallback: everything here calls ``libclair3b200.so``.
"""
from __future__ import annotations

import numpy as np
import torch

from ._ffi import C3BError, check, ffi, lib

FLANKING = 16                 # shared/param_p.py flankingBaseNum; pileup_flanking_base_num src/clair3_pileup.h:93
CHANNELS = 18

_FIELDS = (("pos", np.int64), ("flag", np.uint16), ("mapq", np.uint8), ("cigar_off", np.int64), ("cigar", np.uint32),
           ("seq_off", np.int64), ("seq", np.uint8), ("l_qseq", np.int32))


class BamRecords:
    """A coordinate-sorted run of alignment records of one contig in htslib's in-memory layout (``c3b_bam_records``):
    pos / flag / mapq / l_qseq per read, CIGAR words ``len << 4 | op`` and 4-bit packed sequences addressed through
    ``cigar_off`` / ``seq_off`` (n + 1 offsets each)."""

    def __init__(self, **arrays):
        missing = [k for k, _ in _FIELDS if k not in arrays]
        if missing:
            raise C3BError("BamRecords: missing %s" % ", ".join(missing))
        for k, dt in _FIELDS:
            setattr(self, k, np.ascontiguousarray(arrays[k], dtype=dt))
        n = len(self.pos)
        if not (len(self.flag) == len(self.mapq) == len(self.l_qseq) == n):
            raise C3BError("BamRecords: per-read arrays differ in length")
        if len(self.cigar_off) != n + 1 or len(self.seq_off) != n + 1:
            raise C3BError("BamRecords: cigar_off / seq_off need n_reads + 1 entries")
        if n:
            if self.cigar_off[0] != 0 or self.seq_off[0] != 0 or self.cigar_off[-1] != len(self.cigar) or self.seq_off[-1] != len(self.seq):
                raise C3BError("BamRecords: offsets do not span cigar / seq")
            if (np.diff(self.cigar_off) < 0).any() or (np.diff(self.seq_off) < 0).any():
                raise C3BError("BamRecords: offsets must not decrease")
            if (np.diff(self.pos) < 0).any():
                raise C3BError("BamRecords: records must be sorted by pos (a coordinate-sorted BAM)")
            if ((self.l_qseq.astype(np.int64) + 1) // 2 > np.diff(self.seq_off)).any():
                raise C3BError("BamRecords: a packed sequence is shorter than (l_qseq + 1) / 2 bytes")
        self.n_reads = n
        # optional fields read by the full-alignment tensor builder (clair3_b200.fa_tensor): values + n_reads + 1 offsets each
        for k, dt in _OPTIONAL:
            v, o = arrays.get(k), arrays.get(k + "_off")
            if (v is None) != (o is None):
                raise C3BError("BamRecords: %s and %s_off go together" % (k, k))
            if v is not None:
                v = np.frombuffer(v, dtype=np.uint8).copy() if isinstance(v, (bytes, bytearray)) else v
                v, o = np.ascontiguousarray(v, dtype=dt), np.ascontiguousarray(o, dtype=np.int64)
                if len(o) != n + 1 or o[0] != 0 or o[-1] != len(v) or (np.diff(o) < 0).any():
                    raise C3BError("BamRecords: %s_off must be n_reads + 1 non-decreasing offsets from 0 to len(%s)" % (k, k))
                if k == "qual" and (np.diff(o) != self.l_qseq).any():
                    raise C3BError("BamRecords: every read needs l_qseq base qualities")
            setattr(self, k, v)
            setattr(self, k + "_off", o)

    @classmethod
    def from_dict(cls, d):
        if isinstance(d, cls):
            return d
        names = [k for f, _ in _OPTIONAL for k in (f, f + "_off")]
        extra = {k: d[k] for k in names if d.get(k) is not None}
        return cls(**{k: d[k] for k, _ in _FIELDS}, **extra)

    def _struct(self):
        s = ffi.new("c3b_bam_records *")
        s.n_reads = self.n_reads
        for k, dt in _FIELDS:
            setattr(s, k, ffi.cast("const %s *" % _CTYPE[np.dtype(dt).name], getattr(self, k).ctypes.data))
        return s

    def nbytes(self):
        return int(sum(getattr(self, k).nbytes for k, _ in _FIELDS))

    def to_device(self, device, ref_seq=None):
        """The same records as device tensors (``c3b_plp_count(..., on_device = 1)``): for callers whose decoder already writes
        into HBM, and for timing the counter without the host copies."""
        return DeviceBamRecords(self, device, ref_seq)


_OPTIONAL = (("qual", np.uint8), ("qname", np.uint8), ("mv", np.int32))     # bam_get_qual, bam_get_qname (no NUL), the mv B-array
_CTYPE = {"int64": "int64_t", "uint16": "uint16_t", "uint8": "uint8_t", "uint32": "uint32_t", "int32": "int32_t"}
_TORCH_VIEW = {"uint16": np.int16, "uint32": np.int32}          # torch has no unsigned 16/32-bit tensors: same bits, signed view


class DeviceBamRecords:
    def __init__(self, rec, device, ref_seq=None):
        self.n_reads = rec.n_reads
        self.device = torch.device(device)
        self.t = {}
        for k, dt in _FIELDS:
            a = getattr(rec, k)
            v = a.view(_TORCH_VIEW.get(np.dtype(dt).name, a.dtype)) if a.size else a.astype(_TORCH_VIEW.get(np.dtype(dt).name, a.dtype))
            self.t[k] = torch.from_numpy(np.ascontiguousarray(v)).to(self.device)
        for k, dt in _OPTIONAL:
            for name in (k, k + "_off"):
                a = getattr(rec, name, None)
                self.t[name] = None if a is None else torch.from_numpy(np.ascontiguousarray(a if a.size else np.zeros(1, a.dtype))).to(self.device)
        self.ref = None
        if ref_seq is not None:
            b = ref_seq.encode() if isinstance(ref_seq, str) else bytes(ref_seq)
            self.ref = torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()).to(self.device)

    def _struct(self):
        s = ffi.new("c3b_bam_records *")
        s.n_reads = self.n_reads
        for k, dt in _FIELDS:
            setattr(s, k, ffi.cast("const %s *" % _CTYPE[np.dtype(dt).name], self.t[k].data_ptr()))
        return s


class PileupCounter:
    """One counting workspace on one H100 (``c3b_plp``).  ``count()`` is asynchronous on the current torch stream of the device;
    ``sizes()`` / ``fetch()`` wait for it."""

    def __init__(self, device=0):
        dev = torch.device(device) if not isinstance(device, int) else torch.device("cuda", device)
        if dev.type != "cuda":
            raise C3BError("PileupCounter needs a CUDA device (no CPU fallback)")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self._device = dev
        out = ffi.new("c3b_plp **")
        check(lib().c3b_plp_create(out, dev.index or 0))
        self._h = out[0]
        self._keep = None
        self._shape = None
        self._pin = {}

    def count(self, records, start, end, ref_seq, ref_start, min_depth=2, min_snp_af=0.08, min_indel_af=0.15, min_mq=5,
              call_snp_only=False, call_ht=False, gvcf=False, alt_info=False, max_indel_length=50):
        """Arguments as ``calculate_clair3_pileup`` takes them (src/clair3_pileup.c:142) with the region as 0-based
        [start, end) and the reference bases of [ref_start, ref_start + len(ref_seq)).  ``alt_info=True`` also exports the
        candidates' allele lists so that ``alt_info_strings()`` can format the reference's ``all_alt_info`` text."""
        on_dev = isinstance(records, DeviceBamRecords)
        rec = records if on_dev else BamRecords.from_dict(records)
        prm = ffi.new("c3b_plp_params *")
        prm.min_depth, prm.min_snp_af, prm.min_indel_af, prm.min_mq = int(min_depth), float(min_snp_af), float(min_indel_af), int(min_mq)
        prm.call_snp_only, prm.call_ht, prm.gvcf = int(bool(call_snp_only)), int(bool(call_ht)), int(bool(gvcf))
        prm.alt_info = int(bool(alt_info))
        st = rec._struct()
        stream = torch.cuda.current_stream(self._device).cuda_stream
        if on_dev:
            if ref_seq is None:
                ref_seq = rec.ref
            if not (isinstance(ref_seq, torch.Tensor) and ref_seq.dtype == torch.uint8 and ref_seq.device == rec.device):
                raise C3BError("count: device records need the reference bases as a uint8 tensor on the same device")
            ref, refbuf = ref_seq.contiguous(), None
            refptr, reflen = ffi.cast("const char *", ref.data_ptr()), ref.numel()
        else:
            ref = ref_seq.encode() if isinstance(ref_seq, str) else bytes(ref_seq)
            refbuf = ffi.from_buffer(ref)
            refptr, reflen = ffi.cast("const char *", refbuf), len(ref)
        check(lib().c3b_plp_count(self._h, st, int(on_dev), int(start), int(end), refptr, int(ref_start), reflen, prm,
                                  ffi.cast("void *", stream)))
        self._keep = (rec, ref, refbuf, st)          # buffers stay alive while the copies / kernels are in flight
        self._shape = (int(end) - int(start), bool(gvcf))
        self._alt = (bool(alt_info), int(start), int(end), int(ref_start), int(max_indel_length))
        return self

    def sizes(self):
        a, b = ffi.new("int64_t *"), ffi.new("int64_t *")
        check(lib().c3b_plp_sizes(self._h, a, b))
        return int(a[0]), int(b[0])

    def _pinned(self, name, shape, dtype):
        """A reusable page-locked host buffer (grown on demand): D2H into pinned memory runs at the PCIe rate, into a fresh
        pageable numpy array at a fraction of it (page faults + staging)."""
        n = int(np.prod(shape))
        t = self._pin.get(name)
        if t is None or t.numel() < n or t.dtype != dtype:
            t = torch.empty(max(n, 1) + max(n, 1) // 4, dtype=dtype).pin_memory()
            self._pin[name] = t
        return t[:n].view(*shape).numpy()

    def fetch(self, pinned=False):
        """dict: matrix [n_cols,18] int64, major [n_cols], stats [n_cols,6] int32 (depth, ref, alt, del, ins, flags), cand_cols,
        cand_ok (+ pos_ref_count / pos_total_count [end - start] after ``gvcf=True``).  ``pinned=True``: the arrays are views of
        the counter's page-locked staging buffers - no allocation, full PCIe rate - valid until the next ``fetch``."""
        nc, nk = self.sizes()
        W, gvcf = self._shape
        if pinned:
            out = {"matrix": self._pinned("matrix", (nc, CHANNELS), torch.int64), "major": self._pinned("major", (nc,), torch.int64),
                   "stats": self._pinned("stats", (nc, 6), torch.int32), "cand_cols": self._pinned("cand_cols", (nk,), torch.int64),
                   "cand_ok": self._pinned("cand_ok", (nk,), torch.uint8)}
        else:
            out = {"matrix": np.zeros((nc, CHANNELS), np.int64), "major": np.zeros(nc, np.int64), "stats": np.zeros((nc, 6), np.int32),
                   "cand_cols": np.zeros(nk, np.int64), "cand_ok": np.zeros(nk, np.uint8)}
        c = ffi.cast
        prc = ptc = ffi.NULL
        if gvcf:
            out["pos_ref_count"] = self._pinned("prc", (W,), torch.int64) if pinned else np.zeros(W, np.int64)
            out["pos_total_count"] = self._pinned("ptc", (W,), torch.int64) if pinned else np.zeros(W, np.int64)
            prc, ptc = c("int64_t *", out["pos_ref_count"].ctypes.data), c("int64_t *", out["pos_total_count"].ctypes.data)
        check(lib().c3b_plp_fetch(self._h, c("int64_t *", out["matrix"].ctypes.data), c("int64_t *", out["major"].ctypes.data),
                                  c("int32_t *", out["stats"].ctypes.data), c("int64_t *", out["cand_cols"].ctypes.data),
                                  c("uint8_t *", out["cand_ok"].ctypes.data), prc, ptc))
        return out

    def alt_info_strings(self, fetched=None):
        """The ``all_alt_info`` strings of ``calculate_clair3_pileup`` (src/clair3_pileup.c:391-450), one per candidate in
        candidate order: ``"<pos+1>-<depth>-<ref base>-X<b> n D<ref bases> n I<ref base><inserted bases> n R<ref base> n "`` -
        SNP alleles in A C G T order, deletions by length, insertions in the iteration order of the reference's khash string
        counter, the remaining reference depth last.  The GPU supplies the allele lists (``c3b_plp_fetch_alleles``), the text is
        formatted here from the HOST records of the count (the inserted bases are read from the representative reads)."""
        want, start, end, ref_start, max_indel = self._alt
        if not want:
            raise C3BError("alt_info_strings: count(..., alt_info=True) first")
        rec, ref = self._keep[0], self._keep[1]
        if isinstance(rec, DeviceBamRecords):
            raise C3BError("alt_info_strings needs host records (the inserted bases are read on the host)")
        r = fetched if fetched is not None else self.fetch()
        W = self._shape[0]
        n = ffi.new("int64_t *")
        check(lib().c3b_plp_fetch_alleles(self._h, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, 0, n))
        na = int(n[0])
        al_off, al_n, ins_last = np.zeros(W, np.int32), np.zeros(W, np.int32), np.zeros(W, np.int32)
        meta, rd, qp, cn = (np.zeros(max(na, 1), np.uint32) for _ in range(4))
        c = ffi.cast
        check(lib().c3b_plp_fetch_alleles(self._h, c("int32_t *", al_off.ctypes.data), c("int32_t *", al_n.ctypes.data),
                                          c("int32_t *", ins_last.ctypes.data),
                                          c("uint32_t *", meta.ctypes.data), c("uint32_t *", rd.ctypes.data),
                                          c("uint32_t *", qp.ctypes.data), c("uint32_t *", cn.ctypes.data), len(meta), n))
        out = []
        for ci in r["cand_cols"]:
            p = int(r["major"][ci])
            a0 = int(al_off[p - start])
            sl = slice(a0, a0 + int(al_n[p - start]))
            out.append(format_alt_info(p, r["matrix"][ci], r["stats"][ci], ref, ref_start, max_indel,
                                       meta[sl], rd[sl], qp[sl], cn[sl], rec, ins_last=int(ins_last[p - start]),
                                       fetch_end=end + FETCH_EXPAND + 1))
        return out

    def window_bounds(self):
        """int64 [n_cand, 2]: the rows [lo, hi) of each candidate's 33-row window (from ``cand_cols - 16``) that lie in its
        contiguous run of positions (``c3b_plp_window_bounds``); the reference's tensor is zero on the window's other rows
        (``preprocess/CreateTensorPileupFromCffi.py:374-391``)."""
        _, nk = self.sizes()
        out = np.zeros((nk, 2), np.int64)
        check(lib().c3b_plp_window_bounds(self._h, ffi.cast("int64_t *", out.ctypes.data), ffi.NULL))
        return out

    def forward(self, model):
        """Clair3_P over the 33-column window of EVERY candidate of the last count, straight from the device-resident matrix
        (``c3b_forward_windows_bounded`` with ``on_device = 1``): each window reads its candidate's contiguous run and zeros
        outside it, which is the tensor the reference builds (``preprocess/CreateTensorPileupFromCffi.py:356-396``).  Returns
        (probabilities float32 [n_cand, 24|90] on the device, cand_ok uint8 [n_cand] on the host): ``cand_ok == 0``: the
        reference drops that candidate, and its row must be ignored."""
        if getattr(model, "_handle", None) is None:
            raise C3BError("forward: the model has no device / weights yet (.to(device), .load_state_dict())")
        if getattr(model, "input_channels", CHANNELS) != CHANNELS or model._kind != lib_const("C3B_PILEUP"):
            raise C3BError("forward: needs the pileup network (Clair3_P, 18 channels)")
        if torch.device(model._device) != self._device:
            raise C3BError("forward: the model lives on %s, the counter on %s" % (model._device, self._device))
        nc, nk = self.sizes()
        y = torch.empty((nk, model.out_dim), dtype=torch.float32, device=self._device)
        ok = np.zeros(nk, np.uint8)
        if nk == 0:
            return y, ok
        pm, ps, pk, pb = (ffi.new("const int64_t **"), ffi.new("const int64_t **"), ffi.new("const uint8_t **"),
                          ffi.new("const int64_t **"))
        check(lib().c3b_plp_device(self._h, pm, ffi.NULL, ffi.NULL, ps, pk))
        check(lib().c3b_plp_window_bounds(self._h, ffi.NULL, pb))
        stream = torch.cuda.current_stream(self._device).cuda_stream
        check(lib().c3b_forward_windows_bounded(model._handle, ffi.cast("void *", pm[0]), lib_const("C3B_DT_I64"), nc, ps[0], pb[0],
                                                1, nk, ffi.cast("float *", y.data_ptr()), 1, 0, ffi.cast("void *", stream)))
        check(lib().c3b_plp_fetch(self._h, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.cast("uint8_t *", ok.ctypes.data), ffi.NULL, ffi.NULL))
        return y, ok

    def last_ms(self):
        ms, n = ffi.new("float *"), ffi.new("int *")
        check(lib().c3b_plp_last_ms(self._h, ms, n))
        return float(ms[0]), int(n[0])

    def close(self):
        if getattr(self, "_h", None) is not None:
            lib().c3b_plp_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_NT16 = "=ACMGRSVTWYHKDBN"                      # htslib seq_nt16_str
_B2I = {2: 1, 6: 2, 19: 3}                     # base2index (src/clair3_pileup.h:57-62): 'C' - 'A', 'G' - 'A', 'T' - 'A'


def khash_iteration_order(keys, put_after_last=False):
    """Bucket order of klib's khash (vendored by the reference as src/khash.h) after inserting the distinct keys ``keys`` in this
    order - the order in which the reference prints a column's insertion alleles (``kh_begin .. kh_end`` over
    ``ins_counts_all``, src/clair3_pileup.c:427-441).  Restated for an insert-only table: X31 string hash (khash.h:395-400) for
    byte strings, the identity (kh_int_hash_func, a 32-bit key) for ints, power-of-two buckets from 4, triangular probing (:329),
    growth whenever n_occupied >= 0.77 n_buckets at the start of a put (:312-320), and kh_resize's in-place kick-out rehash
    (:268-292).  ``put_after_last``: the table saw one more put (of a key already present) after the last new key - that put
    still grows a full table first."""
    hashes = []
    for k in keys:
        if isinstance(k, (int, np.integer)):
            hashes.append(int(k) & 0xFFFFFFFF)
            continue
        h = k[0] if k else 0
        for ch in k[1:]:
            h = (h * 31 + ch) & 0xFFFFFFFF
        hashes.append(h)
    n, size, upper, slot = 0, 0, 0, []

    def grow(n, slot):
        nn = 4
        while nn < n + 1:
            nn <<= 1
        if size >= int(nn * 0.77 + 0.5):
            return n, slot, int(n * 0.77 + 0.5)
        new, taken = slot + [-1] * (nn - n), [False] * nn
        occ = [s >= 0 for s in slot] + [False] * (nn - n)
        mask = nn - 1
        for j in range(n):
            if not occ[j]:
                continue
            cur, occ[j], new[j] = new[j], False, -1
            while True:
                i, step = hashes[cur] & mask, 0
                while taken[i]:
                    step += 1
                    i = (i + step) & mask
                taken[i] = True
                if i < n and occ[i]:
                    new[i], cur = cur, new[i]
                    occ[i] = False
                else:
                    new[i] = cur
                    break
        return nn, new, int(nn * 0.77 + 0.5)

    for key in range(len(keys)):
        if size >= upper:
            n, slot, upper = grow(n, slot)
        mask, step = n - 1, 0
        i = hashes[key] & mask
        while slot[i] >= 0:
            step += 1
            i = (i + step) & mask
        slot[i] = key
        size += 1
    if put_after_last and keys and size >= upper:
        n, slot, upper = grow(n, slot)
    return [s for s in slot if s >= 0]


def _insertion_bytes(rec, read, q0, length):
    so, lq = int(rec.seq_off[read]), int(rec.l_qseq[read])
    out = bytearray()
    for i in range(q0, q0 + length):
        nib = 0
        if 0 <= i < lq:
            b = int(rec.seq[so + (i >> 1)])
            nib = (b >> 4) if (i & 1) == 0 else (b & 15)
        out.append(ord(_NT16[nib]))
    return bytes(out)


FETCH_EXPAND = 1000      # mpileup_expand_reference_region (src/clair3_pileup.h:63): the reference fetches [start - 1000, end + 1000]


def format_alt_info(pos, row, stats, ref, ref_start, max_indel_length, meta, read, qpos, cnt, rec, ins_last=-1, fetch_end=None):
    """One ``all_alt_info`` string (src/clair3_pileup.c:391-450) from a candidate's matrix row, its stats and its allele records.
    ``ins_last``: the last read with an insertion on the column - when it comes after the first read of the last new insertion
    string, that put of a present string still grows a full khash table first (src/khash.h:310-318), which reorders the text.
    ``fetch_end``: the end (exclusive) of the reference's FASTA fetch, ``end + 1001`` (src/clair3_pileup.c:188-190) - the deletion
    text stops there; None = the end of ``ref``."""
    off = pos - ref_start
    rb = ref[off:off + 1].upper() if 0 <= off < len(ref) else b"N"
    rbc = rb.decode("latin-1")
    rf = _B2I.get(rb[0] - 65, 0)
    depth, ref_depth = int(stats[0]), int(stats[1])
    parts = ["%d-%d-%s-" % (pos + 1, depth, rbc)]
    for i in range(4):
        alt_sum = int(row[i]) + int(row[i + 9])
        if alt_sum > 0 and i != rf:
            parts.append("X%s %d " % ("ACGT"[i], alt_sum))
    dels, ins_order, ins_cnt = {}, [], {}
    for m, r, q, c in zip(meta.tolist(), read.tolist(), qpos.tolist(), cnt.tolist()):
        length = m & 0x3FFFFFFF
        if m >> 31:
            key = _insertion_bytes(rec, r, q, length)
            if key not in ins_cnt:
                ins_cnt[key] = [0, r]
                ins_order.append(key)
            ins_cnt[key][0] += c
            ins_cnt[key][1] = min(ins_cnt[key][1], r)
        else:
            dels[length] = dels.get(length, 0) + c
    for length in sorted(dels):
        d = dels[length]
        ref_depth -= d
        if d > 0 and length <= max_indel_length:
            stop = off + 1 + length if fetch_end is None else min(off + 1 + length, fetch_end - ref_start)
            tail = ref[off + 1:stop]
            nul = tail.find(b"\0")
            parts.append("D%s %d " % ((tail if nul < 0 else tail[:nul]).decode("latin-1"), d))
    ins_order.sort(key=lambda k: ins_cnt[k][1])           # first occurrence over both strands = the reference's insertion order
    again = bool(ins_order) and ins_last > ins_cnt[ins_order[-1]][1]
    for j in khash_iteration_order(ins_order, put_after_last=again):
        key = ins_order[j]
        val = ins_cnt[key][0]
        ref_depth -= val
        if len(key) <= max_indel_length:
            parts.append("I%s%s %d " % (rbc, key.decode("latin-1"), val))
    if ref_depth > 0:
        parts.append("R%s %d " % (rbc, ref_depth))
    return "".join(parts)


def chunk_region(contig_length, chunk_id, chunk_num):
    """The 1-based contig slice [ctg_start, ctg_end] of chunk ``chunk_id`` (1-based, as ``--chunk_id``) of ``chunk_num``:
    ``preprocess/CreateTensorPileupFromCffi.py:249,281-292`` (no BED / VCF restriction)."""
    if not 1 <= chunk_id <= chunk_num:
        raise C3BError("chunk_region: chunk_id %d outside 1..%d" % (chunk_id, chunk_num))
    cid = chunk_id - 1
    chunk_size = contig_length // chunk_num + 1 if contig_length % chunk_num else contig_length // chunk_num
    ctg_start = chunk_size * cid
    return ctg_start, ctg_start + chunk_size


def counting_region(ctg_start, ctg_end, no_of_positions=2 * FLANKING + 1):
    """The 0-based, end-exclusive [start, end) that reaches ``calculate_clair3_pileup`` for a 1-based contig slice: the slice is
    widened by ``no_of_positions`` (``:305-311``), written as the region string ``name:{max(0, start - 1)}-{end}`` (``:55``) and
    parsed by ``hts_parse_reg``, which turns the 1-based start into ``start - 1`` (clipped at 0) and keeps the end
    (``src/clair3_pileup.c:148-151``)."""
    ctg_start = max(1, ctg_start)
    extend_start = max(1, ctg_start - no_of_positions)
    extend_end = ctg_end + no_of_positions
    s = max(0, extend_start - 1)
    return max(0, s - 1), extend_end


def chunks_for_rank(chunk_num, rank, world):
    """The 1-based chunk ids rank ``rank`` of ``world`` counts: contiguous runs, like the reference's per-GPU file lists
    (``clair3/CallVariantsFromCffiGPU.py:141-156``), so every rank's candidates stay in contig order.  Regions are independent:
    the counter shards with no exchange step at all (one ``PileupCounter`` per process / GPU)."""
    from .sharding import site_range
    lo, hi = site_range(chunk_num, rank, world)
    return list(range(lo + 1, hi + 1))


def lib_const(name):
    from ._ffi import CONSTANTS
    return CONSTANTS[name]


def enforce_chunk_contiguity(counts, positions):
    """``__enforce_pileup_chunk_contiguity`` (preprocess/CreateTensorPileupFromCffi.py:180-236) for ONE region: the counter reports
    covered columns only, so a coverage hole shows up as a jump > 1 in ``positions['major']``; the reference cuts the matrix there
    and hands the caller a list of contiguous (counts, positions) chunks."""
    if len(positions) == 0:
        return []
    gaps = np.where(np.ediff1d(positions["major"]) > 1)[0] + 1
    out, first = [], 0
    for g in list(gaps) + [len(positions)]:
        if g > first:
            out.append((counts[first:g], positions[first:g]))
        first = g
    return out


def alt_info_list(strings, ref_name):
    """The tuples ``_process_region`` builds from the C strings (preprocess/CreateTensorPileupFromCffi.py:66-73):
    (1-based position, "ctg:pos:ref_base", "depth-alt text")."""
    out = []
    for s in strings:
        f = s.rstrip().split("-")
        if len(f) < 4:
            continue
        pos, depth, center_ref_base, alt = f[:4]
        out.append((int(pos), ref_name + ":" + pos + ":" + center_ref_base, depth + "-" + alt))
    return out


def pileup_counts_clair3(records, ref_name, start, end, ref_seq, ref_start, counter=None, device=0, **params):
    """``pileup_counts_clair3`` of the reference (preprocess/CreateTensorPileupFromCffi.py:30-85) on decoded records: returns
    (chunk_results, all_alt_info_list, gvcf_output) - contiguous (counts [n,18] int64, positions with 'major' / 'minor') chunks,
    the (pos, "ctg:pos:ref", "depth-alt") tuples of every candidate and, with ``gvcf=True``, [pos_ref_count, pos_total_count] -
    for the 0-based [start, end) that reaches ``calculate_clair3_pileup`` (see ``counting_region``).  Keyword arguments as
    ``PileupCounter.count``; the allele text needs host records."""
    own = counter is None
    counter = counter or PileupCounter(device)
    try:
        params = dict(params)
        params["alt_info"] = True
        r = counter.count(records, start, end, ref_seq, ref_start, **params).fetch()
        strings = counter.alt_info_strings(r)
    finally:
        if own:
            counter.close()
    positions = np.zeros(len(r["major"]), dtype=[("major", int), ("minor", int)])
    positions["major"] = r["major"]
    gvcf_output = [r["pos_ref_count"], r["pos_total_count"]] if "pos_ref_count" in r else []
    return enforce_chunk_contiguity(r["matrix"], positions), alt_info_list(strings, ref_name), gvcf_output
