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
    """Alignment records in device memory (``c3b_plp_count`` / ``c3b_fa_build`` with ``on_device = 1``): the tensors ``t`` by field
    name (unsigned fields as same-width signed tensors; an optional field absent is None) and, optionally, the reference bases
    ``ref`` as a uint8 tensor on the same device.  Made from host records (``BamRecords.to_device``) or from tensors a device
    decoder wrote (``from_tensors``)."""

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
        self.ref = _device_ref(ref_seq, self.device)

    @classmethod
    def from_tensors(cls, tensors, device, ref_seq=None):
        """Records from device tensors, taken over without a copy: ``tensors`` maps every ``BamRecords`` field to a contiguous
        tensor on ``device`` of that field's width (int16 for ``flag``, int32 for ``cigar``), and each optional field and its
        ``_off`` to tensors or None.  The tensors must satisfy what ``BamRecords`` checks on the host."""
        self = cls.__new__(cls)
        self.device = torch.device(device)
        self.n_reads = int(tensors["pos"].numel())
        self.t = {k: tensors[k] for k, _ in _FIELDS}
        for k, _ in _OPTIONAL:
            for name in (k, k + "_off"):
                self.t[name] = tensors.get(name)
        for k, v in self.t.items():
            if v is not None and (v.device != self.device or not v.is_contiguous()):
                raise C3BError("DeviceBamRecords: %s must be a contiguous tensor on %s" % (k, self.device))
        self.ref = _device_ref(ref_seq, self.device)
        return self

    def host(self):
        """The records as ``bam_io.read_bam`` returns them (numpy arrays of its dtypes; the optional fields where present)."""
        out = {}
        for k, dt in _FIELDS + _OPTIONAL + tuple((k + "_off", np.int64) for k, _ in _OPTIONAL):
            v = self.t.get(k)
            if v is not None:
                out[k] = v.cpu().numpy().view(dt) if np.dtype(dt).itemsize == v.element_size() else v.cpu().numpy().astype(dt)
        return out


def _device_ref(ref_seq, device):
    """Reference bases (str / bytes, or a uint8 tensor) as a uint8 tensor on ``device``; None stays None."""
    if ref_seq is None:
        return None
    if isinstance(ref_seq, torch.Tensor):
        return ref_seq.to(device=device, dtype=torch.uint8).contiguous()
    b = ref_seq.encode() if isinstance(ref_seq, str) else bytes(ref_seq)
    return torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()).to(device)


def _records_struct(rec, optional=False):
    """The ``c3b_bam_records`` of a ``BamRecords`` or a ``DeviceBamRecords`` (``optional=True``: the ``c3b_fa_records`` around it,
    with qual / qname / mv where the records carry them, null where they do not).  The struct holds raw addresses: the records
    must outlive the call that reads it."""
    on_dev = isinstance(rec, DeviceBamRecords)
    arrays = rec.t if on_dev else vars(rec)
    addr = (lambda a: a.data_ptr()) if on_dev else (lambda a: a.ctypes.data)
    s = ffi.new("c3b_fa_records *" if optional else "c3b_bam_records *")
    core = s.core if optional else s
    core.n_reads = rec.n_reads
    for k, dt in _FIELDS:
        setattr(core, k, ffi.cast("const %s *" % _CTYPE[np.dtype(dt).name], addr(arrays[k])))
    for k, dt in _OPTIONAL if optional else ():
        v, o = arrays.get(k), arrays.get(k + "_off")
        if o is not None:
            setattr(s, k + "_off", ffi.cast("const int64_t *", addr(o)))
            vp = addr(v) if len(v) else 8      # an empty value array with valid offsets: non-null, never dereferenced
            setattr(s, k, ffi.cast("const %s *" % _CTYPE[np.dtype(dt).name], vp))
    return s


class _Handle:
    """A library workspace on one CUDA device, created by ``<_API>_create`` and released by ``<_API>_destroy``, whose calls run
    on the device's current torch stream (``PileupCounter``, ``FullAlignmentBuilder``, ``bam_decode.BamDecoder``)."""

    _API = None                      # "c3b_plp" / "c3b_fa" / "c3b_bam"

    def __init__(self, device):
        dev = torch.device(device) if not isinstance(device, int) else torch.device("cuda", device)
        if dev.type != "cuda":
            raise C3BError("%s needs a CUDA device (no CPU fallback)" % type(self).__name__)
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self._device = dev
        out = ffi.new(self._API + " **")
        check(self._entry("_create")(out, dev.index or 0))
        self._h = out[0]

    def _lib(self):
        """The library as the module that defines the workspace's class binds it: a subclass defined in another module returns
        that module's ``lib``, so every call a workspace makes goes through one binding."""
        return lib()

    def _entry(self, name):
        """The workspace's entry point ``<_API><name>``."""
        return getattr(self._lib(), self._API + name)

    def _stream(self):
        return ffi.cast("void *", torch.cuda.current_stream(self._device).cuda_stream)

    def _timing(self, fn):
        ms, n = ffi.new("float *"), ffi.new("int *")
        check(fn(self._h, ms, n))
        return float(ms[0]), int(n[0])

    def last_ms(self):
        """(device milliseconds, kernel launches) of the last call, between CUDA events on its stream."""
        return self._timing(self._entry("_last_ms"))

    def close(self):
        if getattr(self, "_h", None) is not None:
            self._entry("_destroy")(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _Workspace(_Handle):
    """What ``PileupCounter`` and ``FullAlignmentBuilder`` share beyond the workspace itself: the reference bases of a call, and
    the all_alt_info text stage with the call path behind it."""

    @staticmethod
    def _reference(ref_seq, rec, who):
        """(pointer, length, object that owns the bytes) of a call's reference bases: str / bytes on the host, or with device
        records a uint8 tensor on their device (default: the one ``to_device`` was given)."""
        if isinstance(rec, DeviceBamRecords):
            if ref_seq is None:
                ref_seq = rec.ref
            if not (isinstance(ref_seq, torch.Tensor) and ref_seq.dtype == torch.uint8 and ref_seq.device == rec.device):
                raise C3BError("%s: device records need the reference bases as a uint8 tensor on the same device" % who)
            ref = ref_seq.contiguous()
            return ffi.cast("const char *", ref.data_ptr()), ref.numel(), ref
        ref = ref_seq.encode() if isinstance(ref_seq, str) else bytes(ref_seq)
        return ffi.cast("const char *", ffi.from_buffer(ref)), len(ref), ref

    # The all_alt_info text stage and the call path behind it, the same for both workspaces.  Each class states what differs:
    # _text_max_indel (whether a text stage can follow the last call, and its default max_indel_length), _text_queued (what a
    # queued text stage makes stale), _n_cand (the candidate count without a wait beyond the one ``sizes()`` makes), _network
    # (the network its candidates go through), _queue_forward (how that network is queued) and _call_fields (what ``call``
    # returns beside the decoder's results).
    _OWNER = None                    # "counter" / "builder", in the errors

    def alt_text(self, max_indel_length=None):
        """Enqueues the text stage (``<_API>_alt_text``) behind the last count / build, on its stream and without a host wait:
        the ``all_alt_info`` string of every candidate and what the decoder takes of it, formatted on the device.
        ``max_indel_length``: as the reference's (default: what the count / build was given).  Device-resident records must stay
        alive until the text has been fetched."""
        default = self._text_max_indel()
        if max_indel_length is None:
            max_indel_length = default
        if isinstance(max_indel_length, bool) or not isinstance(max_indel_length, (int, np.integer)):
            raise C3BError("alt_text: max_indel_length must be an integer, got %r" % (max_indel_length,))
        check(self._entry("_alt_text")(self._h, int(max_indel_length)))
        self._text_queued()
        return self

    def _text_queued(self):
        pass

    def alt_text_sizes(self):
        """(bytes of all text strings, bytes of all decoder strings) of the last ``alt_text``."""
        a, b = ffi.new("int64_t *"), ffi.new("int64_t *")
        check(self._entry("_alt_text_sizes")(self._h, a, b))
        return int(a[0]), int(b[0])

    def alt_text_fetch(self):
        """dict: ``text`` (the ``all_alt_info`` strings, one per candidate), ``decoder`` (the ``"depth-alt"`` strings the
        reference passes on with each candidate), ``ref_base`` uint8 [n_cand], ``position`` int64 [n_cand] (1-based).  Waits for
        the text stage."""
        nk = self._n_cand()
        nt, nd = self.alt_text_sizes()
        text, dec = np.zeros(max(nt, 1), np.uint8), np.zeros(max(nd, 1), np.uint8)
        toff, doff = np.zeros(nk + 1, np.int64), np.zeros(nk + 1, np.int64)
        rb, pos = np.zeros(nk, np.uint8), np.zeros(nk, np.int64)
        c = ffi.cast
        check(self._entry("_fetch_alt_text")(self._h, c("char *", text.ctypes.data), c("int64_t *", toff.ctypes.data),
                                             c("char *", dec.ctypes.data), c("int64_t *", doff.ctypes.data),
                                             c("uint8_t *", rb.ctypes.data), c("int64_t *", pos.ctypes.data)))
        tb, db = text.tobytes(), dec.tobytes()
        return {"text": [tb[toff[j]:toff[j + 1]].decode("latin-1") for j in range(nk)],
                "decoder": [db[doff[j]:doff[j + 1]].decode("latin-1") for j in range(nk)], "ref_base": rb, "position": pos}

    def alt_text_device(self):
        """The text stage's results as tensors that alias the workspace (valid until the next count / build / ``alt_text``):
        ``text`` uint8 [n_text_bytes], ``text_off`` int64 [n_cand + 1], ``decoder`` uint8 [n_decoder_bytes], ``decoder_off``
        int64 [n_cand + 1], ``ref_base`` uint8 [n_cand], ``position`` int64 [n_cand]; ``decoder`` / ``decoder_off`` /
        ``ref_base`` are ``decode_calls``' ``alt_bytes`` / ``alt_offsets`` / ``ref_base``.  Waits (``sizes()``) only when
        nothing has waited since the last count / build / ``alt_text``; after that wait it touches the stream no more."""
        nk = self._n_cand()
        nt, nd = self.alt_text_sizes()
        p = [ffi.new("const char **"), ffi.new("const int64_t **"), ffi.new("const char **"), ffi.new("const int64_t **"),
             ffi.new("const uint8_t **"), ffi.new("const int64_t **")]
        check(self._entry("_alt_text_device")(self._h, *p))
        shapes = (("text", nt, torch.uint8), ("text_off", nk + 1, torch.int64), ("decoder", nd, torch.uint8),
                  ("decoder_off", nk + 1, torch.int64), ("ref_base", nk, torch.uint8), ("position", nk, torch.int64))
        return {name: _device_view(int(ffi.cast("uintptr_t", q[0])), n, dt, self._device) for (name, n, dt), q in zip(shapes, p)}

    def alt_text_last_ms(self):
        """Device time and kernel launches of the last ``alt_text`` (``last_ms`` reports the count / build alone)."""
        return self._timing(self._entry("_alt_text_last_ms"))

    def call(self, model, output_config, ctg_name, k=16):
        """The candidates of the last count / build from records to call records on the current stream: the text stage, the
        network over every candidate and ``model.decode_calls`` on the device views, with one host wait (the sizes) before the
        network is queued.  Returns ``decode.batch_calls``' dict (``chromosome``, ``position``, ``calls``, ``text``, ``ad``,
        ``start``; ``decode.calls_text`` formats it) plus ``Y``, the probabilities, on the device, and for the counter
        ``cand_ok`` uint8 [n_cand].  Every candidate is decoded, as the reference decodes every full-alignment candidate;
        ``cand_ok == 0``: the reference drops that pileup candidate, ignore its row.  Raises what ``batch_calls`` raises on an
        alt_info string the decoder rejects."""
        from . import decode
        decode._check_config(output_config)
        self._check_model(model, "call")
        if bool(output_config.add_indel_length) != model.add_indel_length:
            raise C3BError("call: output_config.add_indel_length must match the model")
        self.alt_text()
        self.sizes()                                       # the one wait: the count / build and the text together
        v = self.alt_text_device()
        nk = self._n_cand()
        y = torch.empty((nk, model.out_dim), dtype=torch.float32, device=self._device)
        self._forward_into(model, y)
        out = model.decode_calls(y, v["ref_base"], v["decoder"], v["decoder_off"], output_config, k=k)
        fields = self._call_fields()
        res = decode.calls_result(decode._numpy(out), [ctg_name] * nk, v["position"].cpu().numpy(), v["decoder_off"].cpu().numpy())
        res.update(fields, Y=y)
        return res

    def _call_fields(self):
        return {}

    def _check_model(self, model, who):
        if getattr(model, "_handle", None) is None:
            raise C3BError("%s: the model has no device / weights yet (.to(device), .load_state_dict())" % who)
        kind, channels, name = self._network()
        if getattr(model, "input_channels", channels) != channels or model._kind != kind:
            raise C3BError("%s: needs %s" % (who, name))
        if torch.device(model._device) != self._device:
            raise C3BError("%s: the model lives on %s, the %s on %s" % (who, model._device, self._OWNER, self._device))

    def _forward_into(self, model, y):
        """The network over every candidate into y, stream-ordered."""
        if len(y):
            self._queue_forward(model, y)


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
              call_snp_only=False, call_ht=False, gvcf=False, alt_info=False, max_indel_length=50):
        """Arguments as ``calculate_clair3_pileup`` takes them (src/clair3_pileup.c:142) with the region as 0-based
        [start, end) and the reference bases of [ref_start, ref_start + len(ref_seq)).  ``alt_info=True`` also exports the
        candidates' allele lists, from which ``alt_text()`` formats the reference's ``all_alt_info`` text on the device
        (``alt_info_strings()``: the same on the host) and ``call()`` decodes every candidate."""
        on_dev = isinstance(records, DeviceBamRecords)
        rec = records if on_dev else BamRecords.from_dict(records)
        prm = ffi.new("c3b_plp_params *")
        prm.min_depth, prm.min_snp_af, prm.min_indel_af, prm.min_mq = int(min_depth), float(min_snp_af), float(min_indel_af), int(min_mq)
        prm.call_snp_only, prm.call_ht, prm.gvcf = int(bool(call_snp_only)), int(bool(call_ht)), int(bool(gvcf))
        prm.alt_info = int(bool(alt_info))
        st = _records_struct(rec)
        refptr, reflen, ref = self._reference(ref_seq, rec, "count")
        check(lib().c3b_plp_count(self._h, st, int(on_dev), int(start), int(end), refptr, int(ref_start), reflen, prm, self._stream()))
        self._keep = (rec, ref, st)                  # buffers stay alive while the copies / kernels are in flight
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
        row."""
        ok = np.zeros(self._sizes[1], np.uint8)
        check(lib().c3b_plp_fetch(self._h, ffi.NULL, ffi.NULL, ffi.NULL, ffi.NULL, ffi.cast("uint8_t *", ok.ctypes.data), ffi.NULL, ffi.NULL))
        return {"cand_ok": ok}

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


class _DeviceArray:
    def __init__(self, ptr, n, dtype):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": {torch.uint8: "|u1", torch.int64: "<i8"}[dtype],
                                         "data": (ptr, False), "version": 2}


def _device_view(ptr, n, dtype, device):
    """A tensor over n elements of workspace memory at ptr (no copy; the workspace owns the memory)."""
    if n == 0:
        return torch.empty(0, dtype=dtype, device=device)
    return torch.as_tensor(_DeviceArray(ptr, n, dtype), device=device)


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
