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

from ._ffi import CONSTANTS, C3BError, check, ffi, lib
from ._workspace import _Workspace, _device_view
from .records import CORE, BamRecords, DeviceBamRecords, insertion_bytes, records_struct

FLANKING = 16                 # shared/param_p.py flankingBaseNum; pileup_flanking_base_num src/clair3_pileup.h:93
CHANNELS = 18

_FIELDS = tuple((f.name, f.dtype) for f in CORE)     # (name, dtype) of the core record fields, for bench.py's pinned copy


class PileupCounter(_Workspace):
    """One counting workspace on one H100 (``c3b_plp``).  ``count()`` is asynchronous on the current torch stream of the device;
    ``sizes()`` / ``fetch()`` wait for it."""

    _API = "c3b_plp"
    _OWNER = "counter"

    def __init__(self, device=0):
        super().__init__(device)
        self._keep = None
        self._shape = None
        self._alt = None
        self._sizes = None            # (n_cols, n_cand) once sizes() has waited for the work queued so far
        self._pin = {}

    def count(self, records, start, end, ref_seq, ref_start, min_depth=2, min_snp_af=0.08, min_indel_af=0.15, min_mq=5,
              call_snp_only=False, call_ht=False, gvcf=False, alt_info=False, max_indel_length=50, targets=None):
        """Arguments as ``calculate_clair3_pileup`` takes them (src/clair3_pileup.c:142) with the region as 0-based
        [start, end) and the reference bases of [ref_start, ref_start + len(ref_seq)).  ``alt_info=True`` also exports the
        candidates' allele lists, from which ``alt_text()`` formats the reference's ``all_alt_info`` text on the device
        (``alt_info_strings()``: the same on the host) and ``call()`` decodes every candidate.  ``targets``: a
        ``targets.ContigTargets`` (a BED's or a known-sites VCF's targets on this contig); the candidates outside them are
        dropped on the device before anything keyed by candidate (``c3b_plp_count_targeted``), the matrix, ``major`` and
        ``stats`` stay as they are."""
        on_dev = isinstance(records, DeviceBamRecords)
        rec = records if on_dev else BamRecords.from_dict(records)
        prm = ffi.new("c3b_plp_params *")
        prm.min_depth, prm.min_snp_af, prm.min_indel_af, prm.min_mq = int(min_depth), float(min_snp_af), float(min_indel_af), int(min_mq)
        prm.call_snp_only, prm.call_ht, prm.gvcf = int(bool(call_snp_only)), int(bool(call_ht)), int(bool(gvcf))
        prm.alt_info = int(bool(alt_info))
        st = records_struct(rec)
        refptr, reflen, ref = self._reference(ref_seq, rec, "count")
        tg, tg_keep = None, None
        if targets is None:
            check(lib().c3b_plp_count(self._h, st, int(on_dev), int(start), int(end), refptr, int(ref_start), reflen, prm, self._stream()))
        else:
            tg, tg_keep = targets.struct(self._device)
            check(lib().c3b_plp_count_targeted(self._h, st, int(on_dev), int(start), int(end), refptr, int(ref_start), reflen, prm,
                                               tg, self._stream()))
        self._keep = (rec, ref, st, tg, tg_keep)     # buffers stay alive while the copies / kernels are in flight
        self._shape = (int(end) - int(start), bool(gvcf))
        self._alt = (bool(alt_info), int(start), int(end), int(ref_start), int(max_indel_length))
        self._sizes = None
        return self

    def sizes(self):
        a, b = ffi.new("int64_t *"), ffi.new("int64_t *")
        check(lib().c3b_plp_sizes(self._h, a, b))
        self._sizes = int(a[0]), int(b[0])
        return self._sizes

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
        counter, the remaining reference depth last.  With host records the GPU supplies the allele lists
        (``c3b_plp_fetch_alleles``) and the text is formatted here (``format_alt_info``: the inserted bases are read from the
        representative reads), which is the statement the device text is tested against; with device-resident records the
        strings are the device's (``alt_text()``)."""
        if not (self._alt and self._alt[0]):
            raise C3BError("alt_info_strings: count(..., alt_info=True) first")
        want, start, end, ref_start, max_indel = self._alt
        rec, ref = self._keep[0], self._keep[1]
        if isinstance(rec, DeviceBamRecords):
            return self.alt_text().alt_text_fetch()["text"]
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

    def _lib(self):
        return lib()

    def _text_max_indel(self):
        if not self._alt:
            raise C3BError("alt_text: count(..., alt_info=True) first")
        if not self._alt[0]:
            raise C3BError("alt_text: the count ran without alt_info=True")
        return self._alt[4]

    def _text_queued(self):
        self._sizes = None

    def _n_cand(self):
        return (self._sizes or self.sizes())[1]

    def _call_fields(self):
        """``cand_ok`` uint8 [n_cand]: 0 where the reference drops the candidate; ``call`` decodes it all the same, so ignore its
        row.  ``device``: ``cand_ok`` where the count left it."""
        nk = self._sizes[1]
        ok = np.zeros(nk, np.uint8)
        check(lib().c3b_plp_fetch(self._h, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.cast("uint8_t *", ok.ctypes.data), ffi.NULL, ffi.NULL))
        pk = ffi.new("const uint8_t **")
        check(lib().c3b_plp_device(self._h, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, pk))
        return {"cand_ok": ok, "device": {"cand_ok": _device_view(int(ffi.cast("uintptr_t", pk[0])), nk, torch.uint8, self._device)}}

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
        self._check_model(model, "forward")
        nc, nk = self.sizes()
        y = torch.empty((nk, model.out_dim), dtype=torch.float32, device=self._device)
        ok = np.zeros(nk, np.uint8)
        if nk == 0:
            return y, ok
        self._forward_into(model, y)
        check(lib().c3b_plp_fetch(self._h, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.cast("uint8_t *", ok.ctypes.data), ffi.NULL, ffi.NULL))
        return y, ok

    def _network(self):
        return CONSTANTS["C3B_PILEUP"], CHANNELS, "the pileup network (Clair3_P, 18 channels)"

    def _queue_forward(self, model, y):
        """Clair3_P over the candidates' bounded windows."""
        nc, nk = self._sizes
        pm, ps, pk, pb = (ffi.new("const int64_t **"), ffi.new("const int64_t **"), ffi.new("const uint8_t **"),
                          ffi.new("const int64_t **"))
        check(lib().c3b_plp_device(self._h, pm, ffi.NULL, ffi.NULL, ps, pk))
        check(lib().c3b_plp_window_bounds(self._h, ffi.NULL, pb))
        check(lib().c3b_forward_windows_bounded(model._handle, ffi.cast("void *", pm[0]), CONSTANTS["C3B_DT_I64"], nc, ps[0], pb[0],
                                                1, nk, ffi.cast("float *", y.data_ptr()), 1, 0, self._stream()))


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
            key = insertion_bytes(rec, r, q, length)
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
    ``preprocess/CreateTensorPileupFromCffi.py:249,281-292``, for a run without ``--bed_fn`` / ``--vcf_fn`` (with them:
    ``bed_chunk_region`` / ``known_sites_chunk``)."""
    if not 1 <= chunk_id <= chunk_num:
        raise C3BError("chunk_region: chunk_id %d outside 1..%d" % (chunk_id, chunk_num))
    cid = chunk_id - 1
    chunk_size = contig_length // chunk_num + 1 if contig_length % chunk_num else contig_length // chunk_num
    ctg_start = chunk_size * cid
    return ctg_start, ctg_start + chunk_size


def bed_chunk_region(bed_start, bed_end, chunk_id, chunk_num):
    """The 1-based contig slice [ctg_start, ctg_end] of chunk ``chunk_id`` of ``chunk_num`` over the span of an extended BED
    (``targets.ContigTargets.bed_region``): ``preprocess/CreateTensorPileupFromCffi.py:295-298``."""
    if not 1 <= chunk_id <= chunk_num:
        raise C3BError("bed_chunk_region: chunk_id %d outside 1..%d" % (chunk_id, chunk_num))
    span = bed_end - bed_start
    chunk_size = span // chunk_num + 1 if span % chunk_num else span // chunk_num
    ctg_start = bed_start + 1 + chunk_size * (chunk_id - 1)
    return ctg_start, ctg_start + chunk_size


def known_sites_chunk(sites, chunk_id, chunk_num):
    """Chunk ``chunk_id`` of ``chunk_num`` in genotyping mode (``preprocess/CreateTensorPileupFromCffi.py:300-308``): the
    contig's sorted unique known 1-based positions cut into equal slices.  Returns (ctg_start, ctg_end, the slice) - the
    1-based slice from its smallest to its largest site - or None for an empty slice, which the reference skips."""
    if not 1 <= chunk_id <= chunk_num:
        raise C3BError("known_sites_chunk: chunk_id %d outside 1..%d" % (chunk_id, chunk_num))
    sites = np.asarray(sites, np.int64)
    n = len(sites)
    size = n // chunk_num if n % chunk_num == 0 else n // chunk_num + 1
    part = sites[(chunk_id - 1) * size:chunk_id * size]
    if not len(part):
        return None
    return int(part.min()), int(part.max()), part


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
    ``PileupCounter.count``."""
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
