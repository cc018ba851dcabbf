"""The alignment-record layout that the pileup counter, the full-alignment builder and the GPU BAM reader share.

A run of records is htslib's ``bam1_t`` fields as arrays: ``c3b_bam_records`` (``include/clair3_b200_pileup.h``) and the optional
fields of ``c3b_fa_records`` (``include/clair3_b200_fa.h``).  ``FIELDS`` states each array once; ``BamRecords`` holds a run on the
host, ``DeviceBamRecords`` in device memory, and ``records_struct`` gives the C struct of either.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

from ._ffi import C3BError, ffi

PER_READ, OFFSETS, VALUES = "n", "n + 1", "values"       # a field's length: n_reads, n_reads + 1, or its offsets' last entry


class Field(NamedTuple):
    name: str
    dtype: type             # numpy
    ctype: str              # C element type
    length: str             # PER_READ, OFFSETS or VALUES
    optional: bool          # c3b_fa_records' qual / qname / mv: absent when its offsets are null

    @property
    def view(self):
        """The numpy dtype of the field's tensors: torch's tensors of uint16 / uint32 bits are the signed twins."""
        return {np.uint16: np.int16, np.uint32: np.int32}.get(self.dtype, self.dtype)

    @property
    def torch_dtype(self):
        return {np.int64: torch.int64, np.int32: torch.int32, np.int16: torch.int16, np.uint8: torch.uint8}[self.view]

    def size(self, n_reads, n_values=None):
        """The field's entries for n_reads reads; n_values for a value field."""
        return {PER_READ: n_reads, OFFSETS: n_reads + 1}.get(self.length, n_values)


FIELDS = (
    Field("pos", np.int64, "int64_t", PER_READ, False),
    Field("flag", np.uint16, "uint16_t", PER_READ, False),
    Field("mapq", np.uint8, "uint8_t", PER_READ, False),
    Field("cigar_off", np.int64, "int64_t", OFFSETS, False),
    Field("cigar", np.uint32, "uint32_t", VALUES, False),
    Field("seq_off", np.int64, "int64_t", OFFSETS, False),
    Field("seq", np.uint8, "uint8_t", VALUES, False),
    Field("l_qseq", np.int32, "int32_t", PER_READ, False),
    Field("qual_off", np.int64, "int64_t", OFFSETS, True),          # bam_get_qual
    Field("qual", np.uint8, "uint8_t", VALUES, True),
    Field("qname_off", np.int64, "int64_t", OFFSETS, True),         # bam_get_qname, without the NUL
    Field("qname", np.uint8, "uint8_t", VALUES, True),
    Field("mv_off", np.int64, "int64_t", OFFSETS, True),            # the mv B-array
    Field("mv", np.int32, "int32_t", VALUES, True),
)
CORE = tuple(f for f in FIELDS if not f.optional)
OPTIONAL = tuple(f for f in FIELDS if f.optional and f.length == VALUES)     # each goes with its offsets, name + "_off"


def _decreases(a):
    """Whether a step of ``a`` goes down.  Compared, not differenced: ``np.diff`` wraps at 2^63, so an offset near -2^63 between
    two small ones would pass as two steps up."""
    return bool((a[1:] < a[:-1]).any())


class BamRecords:
    """A coordinate-sorted run of alignment records of one contig in htslib's in-memory layout (``c3b_bam_records``):
    pos / flag / mapq / l_qseq per read, CIGAR words ``len << 4 | op`` and 4-bit packed sequences addressed through
    ``cigar_off`` / ``seq_off`` (n + 1 offsets each)."""

    def __init__(self, **arrays):
        missing = [f.name for f in CORE if f.name not in arrays]
        if missing:
            raise C3BError("BamRecords: missing %s" % ", ".join(missing))
        for f in CORE:
            setattr(self, f.name, np.ascontiguousarray(arrays[f.name], dtype=f.dtype))
        n = len(self.pos)
        if not (len(self.flag) == len(self.mapq) == len(self.l_qseq) == n):
            raise C3BError("BamRecords: per-read arrays differ in length")
        if len(self.cigar_off) != n + 1 or len(self.seq_off) != n + 1:
            raise C3BError("BamRecords: cigar_off / seq_off need n_reads + 1 entries")
        if n:
            if self.cigar_off[0] != 0 or self.seq_off[0] != 0 or self.cigar_off[-1] != len(self.cigar) or self.seq_off[-1] != len(self.seq):
                raise C3BError("BamRecords: offsets do not span cigar / seq")
            if _decreases(self.cigar_off) or _decreases(self.seq_off):
                raise C3BError("BamRecords: offsets must not decrease")
            if _decreases(self.pos):
                raise C3BError("BamRecords: records must be sorted by pos (a coordinate-sorted BAM)")
            if ((self.l_qseq.astype(np.int64) + 1) // 2 > np.diff(self.seq_off)).any():
                raise C3BError("BamRecords: a packed sequence is shorter than (l_qseq + 1) / 2 bytes")
        self.n_reads = n
        # optional fields read by the full-alignment tensor builder (clair3_b200.fa_tensor): values + n_reads + 1 offsets each
        for f in OPTIONAL:
            k = f.name
            v, o = arrays.get(k), arrays.get(k + "_off")
            if (v is None) != (o is None):
                raise C3BError("BamRecords: %s and %s_off go together" % (k, k))
            if v is not None:
                v = np.frombuffer(v, dtype=np.uint8).copy() if isinstance(v, (bytes, bytearray)) else v
                v, o = np.ascontiguousarray(v, dtype=f.dtype), np.ascontiguousarray(o, dtype=np.int64)
                if len(o) != n + 1 or o[0] != 0 or o[-1] != len(v) or _decreases(o):
                    raise C3BError("BamRecords: %s_off must be n_reads + 1 non-decreasing offsets from 0 to len(%s)" % (k, k))
                if k == "qual" and (np.diff(o) != self.l_qseq).any():
                    raise C3BError("BamRecords: every read needs l_qseq base qualities")
            setattr(self, k, v)
            setattr(self, k + "_off", o)

    @classmethod
    def from_dict(cls, d):
        if isinstance(d, cls):
            return d
        extra = {f.name: d[f.name] for f in FIELDS if f.optional and d.get(f.name) is not None}
        return cls(**{f.name: d[f.name] for f in CORE}, **extra)

    def nbytes(self):
        return int(sum(getattr(self, f.name).nbytes for f in CORE))

    def to_device(self, device, ref_seq=None):
        """The same records as device tensors (``c3b_plp_count(..., on_device = 1)``): for callers whose decoder already writes
        into HBM, and for timing the counter without the host copies."""
        return DeviceBamRecords(self, device, ref_seq)


class DeviceBamRecords:
    """Alignment records in device memory (``c3b_plp_count`` / ``c3b_fa_build`` with ``on_device = 1``): the tensors ``t`` by field
    name (unsigned fields as same-width signed tensors; an optional field absent is None) and, optionally, the reference bases
    ``ref`` as a uint8 tensor on the same device.  Made from host records (``BamRecords.to_device``) or from tensors a device
    decoder wrote (``from_tensors``)."""

    def __init__(self, rec, device, ref_seq=None):
        self.n_reads = rec.n_reads
        self.device = torch.device(device)
        self.t = {}
        for f in FIELDS:
            a = getattr(rec, f.name, None)
            self.t[f.name] = None if a is None else torch.from_numpy(a.view(f.view)).to(self.device)
        self.ref = _device_ref(ref_seq, self.device)

    @classmethod
    def from_tensors(cls, tensors, device, ref_seq=None):
        """Records from device tensors, taken over without a copy: ``tensors`` maps every core field of ``FIELDS`` to a
        contiguous integer tensor on ``device`` of that field's width (2 bytes for ``flag``, 4 for ``cigar``: torch's signed
        views serve), and each optional field and its ``_off`` to tensors or None.  Checked here, from the tensors' metadata
        alone: device, contiguity, width, ``n_reads`` entries per read, ``n_reads + 1`` offsets, and each optional field with
        its offsets.  The values are checked by every call that takes the records, before any kernel indexes through an
        offset: one kernel (``clair3_b200/csrc/records_check.cuh``) holds the offsets, ``pos`` and ``l_qseq`` to everything
        ``BamRecords`` checks on the host, each last offset to its value array's length (``records_struct`` passes the
        lengths), and the call raises ``C3BError`` naming the field and the first read that breaks it."""
        self = cls.__new__(cls)
        self.device = torch.device(device)
        self.n_reads = n = int(tensors["pos"].numel())
        self.t = {}
        for f in FIELDS:
            v = self.t[f.name] = tensors.get(f.name) if f.optional else tensors[f.name]
            if v is None:
                continue
            if v.device != self.device or not v.is_contiguous():
                raise C3BError("DeviceBamRecords: %s must be a contiguous tensor on %s" % (f.name, self.device))
            if v.dtype.is_floating_point or v.dtype.is_complex or v.element_size() != np.dtype(f.dtype).itemsize:
                raise C3BError("DeviceBamRecords: %s needs %d-byte integers (%s), got %s"
                               % (f.name, np.dtype(f.dtype).itemsize, f.torch_dtype, v.dtype))
            want = f.size(n)
            if want is not None and v.numel() != want:
                raise C3BError("DeviceBamRecords: %s has %d entries, not %s = %d" % (f.name, v.numel(), f.length, want))
        for f in OPTIONAL:
            if (self.t[f.name] is None) != (self.t[f.name + "_off"] is None):
                raise C3BError("DeviceBamRecords: %s and %s_off go together" % (f.name, f.name))
        self.ref = _device_ref(ref_seq, self.device)
        return self

    def host(self):
        """The records as ``bam_io.read_bam`` returns them (numpy arrays of its dtypes; the optional fields where present)."""
        return {f.name: self.t[f.name].cpu().numpy().view(f.dtype) for f in FIELDS if self.t[f.name] is not None}


def _device_ref(ref_seq, device):
    """Reference bases (str / bytes, or a uint8 tensor) as a uint8 tensor on ``device``; None stays None."""
    if ref_seq is None:
        return None
    if isinstance(ref_seq, torch.Tensor):
        return ref_seq.to(device=device, dtype=torch.uint8).contiguous()
    b = ref_seq.encode() if isinstance(ref_seq, str) else bytes(ref_seq)
    return torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()).to(device)


def records_struct(rec, optional=False):
    """The ``c3b_bam_records`` of a ``BamRecords`` or a ``DeviceBamRecords`` (``optional=True``: the ``c3b_fa_records`` around it,
    with qual / qname / mv where the records carry them, null where they do not), with the length of each value array.  The
    struct holds raw addresses: the records must outlive the call that reads it."""
    on_dev = isinstance(rec, DeviceBamRecords)
    arrays = rec.t if on_dev else vars(rec)
    addr = (lambda a: a.data_ptr()) if on_dev else (lambda a: a.ctypes.data)
    s = ffi.new("c3b_fa_records *" if optional else "c3b_bam_records *")
    core = s.core if optional else s
    core.n_reads = rec.n_reads
    for f in FIELDS if optional else CORE:
        a = arrays.get(f.name)
        if a is not None:
            p = 8 if f.optional and f.length == VALUES and not len(a) else addr(a)    # an empty value array: non-null, never read
            setattr(s if f.optional else core, f.name, ffi.cast("const %s *" % f.ctype, p))
            if f.length == VALUES:
                setattr(s if f.optional else core, "n_" + f.name, len(a))
    return s


_NT16 = "=ACMGRSVTWYHKDBN"                      # htslib seq_nt16_str


def insertion_bytes(rec, read, q0, length):
    """Bases [q0, q0 + length) of read ``read``'s packed sequence as nt16 letters, '=' outside the read."""
    so, lq = int(rec.seq_off[read]), int(rec.l_qseq[read])
    out = bytearray()
    for i in range(q0, q0 + length):
        nib = 0
        if 0 <= i < lq:
            b = int(rec.seq[so + (i >> 1)])
            nib = (b >> 4) if (i & 1) == 0 else (b & 15)
        out.append(ord(_NT16[nib]))
    return bytes(out)
