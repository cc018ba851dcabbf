"""The BAM reader on the GPU (``include/clair3_b200_bam.h``): a region's alignment records straight from the file into device memory.

The host reads what it must to find the bytes - the header and the first record's virtual offset (``bam_io.read_bam_header``),
and with a ``.bai`` index the compressed byte range of the region (``bam_io.read_bai`` / ``bam_io.bai_range``) - and checks the
BGZF block headers.  The GPU inflates the blocks, finds the record chain, parses and filters the records exactly as
``bam_io.read_bam(path, contig, start, end)`` does and scatters them into packed arrays.  The result is a
``records.DeviceBamRecords`` that ``PileupCounter.count`` and ``FullAlignmentBuilder.build`` take as they are: a region goes
from compressed bytes to call records on the device.  ``fetch_fasta`` does the same for a window of a bgzip-compressed
reference FASTA: the host finds the covering blocks through the ``.fai`` and ``.gzi``, the GPU inflates them and gathers the
bases.  ``write_bgzf`` runs the other direction: it compresses a text into a BGZF file on the GPU, byte for byte as
``bam_io.write_bgzf`` writes it.  No CPU fallback: everything here calls ``libclair3b200.so``.
"""
from __future__ import annotations

import os

import torch

from . import bam_io
from ._ffi import C3BError, check, ffi, lib
from ._workspace import _Handle
from .records import FIELDS, VALUES, DeviceBamRecords

_NO_START, _NO_END = -1, 1 << 62            # read_bam's bounds when start / end are not given


class BamDecoder(_Handle):
    """One decoding workspace on one H100 (``c3b_bam``).  ``decode`` / ``decode_bytes`` queue the decode on the device's current
    torch stream, wait once for the sizes, and return records in tensors the decoder allocated: a later decode does not touch
    them."""

    _API = "c3b_bam"

    def __init__(self, device=0):
        super().__init__(device)
        self._headers = {}
        self._fasta = {}

    def _lib(self):
        return lib()

    def _header(self, path):
        key = (os.path.abspath(path), os.path.getmtime(path), os.path.getsize(path))
        if key not in self._headers:
            self._headers[key] = bam_io.read_bam_header(path)
        return self._headers[key]

    def decode(self, path, ctg, start=None, end=None, fa_fields=False, ref_seq=None, index=None):
        """The records of contig ``ctg`` overlapping [start, end) (0-based, end-exclusive; None = unbounded) of the BAM at
        ``path``, as ``bam_io.read_bam(path, ctg, start, end, fa_fields=fa_fields)`` returns them, in device memory.
        ``index``: a ``.bai`` path or a ``bam_io.read_bai`` result; by default ``path + ".bai"`` when that file exists.  With an
        index only the region's byte range is read; without one, every block after the header.  ``ref_seq``: reference bases to
        keep with the records (``DeviceBamRecords.ref``)."""
        refs, first = self._header(path)
        names = [n for n, _ in refs]
        if ctg not in names:
            raise ValueError("contig %r is not in the BAM header" % ctg)
        tid = names.index(ctg)
        if index is None and os.path.exists(str(path) + ".bai"):
            index = str(path) + ".bai"
        with open(path, "rb") as f:
            if index is not None:
                idx = bam_io.read_bai(index) if isinstance(index, (str, os.PathLike)) else index
                lo = 0 if start is None else int(start)
                hi = (1 << 29) if end is None else int(end)
                c0, c1, u0, u1 = bam_io.bai_range(idx, tid, lo, hi, path)
                f.seek(c0)
                data = f.read(c1 - c0)
            else:
                f.seek(first >> 16)
                data = f.read()
                u0, u1 = first & 0xFFFF, -1
        return self.decode_bytes(data, u0, u1, tid, start, end, fa_fields=fa_fields, ref_seq=ref_seq)

    def decode_bytes(self, data, first_uoff, end_uoff, tid, start=None, end=None, fa_fields=False, ref_seq=None):
        """``decode`` on whole BGZF blocks already in memory: ``data`` (bytes-like), the first record's offset in the first
        block's data and the uncompressed offset where the records end (-1: the end of the data), and the contig's index in the
        header."""
        data = memoryview(data).cast("B") if not isinstance(data, (bytes, bytearray)) else data
        lo = _NO_START if start is None else int(start)
        hi = _NO_END if end is None else int(end)
        L = self._lib()
        buf = ffi.from_buffer(data) if len(data) else ffi.NULL
        check(L.c3b_bam_decode(self._h, buf, len(data), int(first_uoff), int(end_uoff), int(tid), lo, hi, int(bool(fa_fields)),
                               self._stream()))
        n = [ffi.new("int64_t *") for _ in range(6)]
        check(L.c3b_bam_sizes(self._h, *n))
        n_reads = int(n[0][0])          # then the length of each value field, in table order
        n_values = dict(zip((f.name for f in FIELDS if f.length == VALUES), (int(x[0]) for x in n[1:])))
        t, out = {}, ffi.new("c3b_bam_out *")
        for f in FIELDS:
            if f.optional and not fa_fields:
                continue
            count = f.size(n_reads, n_values.get(f.name))
            t[f.name] = v = torch.empty(max(count, 1), dtype=f.torch_dtype, device=self._device)[:count]    # never null, even empty
            setattr(out, f.name, ffi.cast(f.ctype + " *", v.data_ptr()))
        check(L.c3b_bam_fetch(self._h, out, 1))
        return DeviceBamRecords.from_tensors(t, self._device, ref_seq)

    def _fasta_index(self, path, fai, gzi):
        """({name: .fai row}, .gzi table) of a BGZF FASTA, read once per file."""
        key = (os.path.abspath(path), os.path.getmtime(path), os.path.getsize(path), fai, gzi)
        if key not in self._fasta:
            gzi_path = bam_io.fasta_bgzf_gzi(path, gzi)
            if gzi_path is None:
                raise ValueError("%s: not a bgzip-compressed FASTA; read a plain FASTA with bam_io.fetch_fasta" % path)
            self._fasta[key] = ({r[0]: r for r in bam_io.read_fai(fai or str(path) + ".fai")}, bam_io.read_gzi(gzi_path))
        return self._fasta[key]

    def fetch_fasta(self, path, name, start=0, end=None, fai=None, gzi=None, wait=True):
        """Bases [start, end) of sequence ``name`` of a bgzip-compressed FASTA, clipped to the sequence, as a uint8 tensor on the
        decoder's device whose bytes equal ``bam_io.fetch_fasta(path, name, start, end)``.  The host reads the ``.fai`` (default
        ``path + ".fai"``), the ``.gzi`` (default ``path + ".gzi"``) and the compressed blocks that cover the window; the GPU
        inflates them and gathers the bases (``c3b_fasta_fetch``), on the device's current torch stream.  ``wait=False``
        returns without waiting for the status of the blocks: the caller then calls ``fasta_status`` after its own next wait
        (``decode`` makes one), before it trusts the bases."""
        rows, gzi_table = self._fasta_index(path, fai, gzi)
        if name not in rows:
            raise ValueError("sequence %r not found in the index of %s" % (name, path))
        _, length, _, lb, lw = row = rows[name]
        start = max(0, int(start))
        end = length if end is None else min(int(end), length)
        if end <= start:
            return torch.empty(0, dtype=torch.uint8, device=self._device)
        _, _, c0, c1, u0 = bam_io.fasta_span(row, start, end, gzi_table)
        with open(path, "rb") as f:
            f.seek(c0)
            data = f.read() if c1 is None else f.read(c1 - c0)
        return self.fetch_fasta_bytes(data, u0, start, lb, lw, end - start, wait=wait)

    def fetch_fasta_bytes(self, data, first_uoff, start, line_bases, line_bytes, n_bases, wait=True):
        """``fetch_fasta`` on whole BGZF blocks already in memory: ``data`` (bytes-like), the window's offset in the first
        block's data, its first base on the sequence, the sequence's line geometry from the ``.fai`` and the number of bases."""
        data = memoryview(data).cast("B") if not isinstance(data, (bytes, bytearray)) else data
        out = torch.empty(max(int(n_bases), 1), dtype=torch.uint8, device=self._device)[:int(n_bases)]
        buf = ffi.from_buffer(data) if len(data) else ffi.NULL
        check(self._lib().c3b_fasta_fetch(self._h, buf, len(data), int(first_uoff), int(start), int(line_bases), int(line_bytes),
                                          int(n_bases), ffi.cast("uint8_t *", out.data_ptr()), self._stream()))
        if wait:
            self.fasta_status()
        return out

    def fasta_status(self):
        """Raises when a block of the last ``fetch_fasta`` did not inflate (C3BError naming the block and the reason); waits for
        that fetch's kernels unless the stream has passed them."""
        check(self._lib().c3b_fasta_status(self._h))


    def compress_bgzf(self, data):
        """``data`` as BGZF blocks of 0xFF00 bytes, compressed on the GPU (``c3b_bgzf_compress``) to exactly the bytes
        ``bam_io.write_bgzf`` writes before its end-of-file block: (the file image as bytes, the offset of every block in it
        and then the image's length).  ``data``: bytes-like or str on the host, or a uint8 tensor on the decoder's device.  One
        host wait, on the device's current torch stream."""
        L = self._lib()
        if isinstance(data, torch.Tensor):
            if data.dtype != torch.uint8 or data.device != self._device:
                raise C3BError("compress_bgzf: a tensor must be uint8 on the decoder's device %s" % self._device)
            data = data.contiguous()
            n, ptr, on_device = data.numel(), ffi.cast("const uint8_t *", data.data_ptr()), 1
        else:
            data = data.encode() if isinstance(data, str) else data
            data = memoryview(data).cast("B") if not isinstance(data, (bytes, bytearray)) else data
            n, ptr, on_device = len(data), ffi.from_buffer(data) if len(data) else ffi.NULL, 0
        check(L.c3b_bgzf_compress(self._h, ptr, n, on_device, self._stream()))
        nb = -(-n // bam_io._BGZF_PAYLOAD)
        size, off = ffi.new("int64_t *"), ffi.new("int64_t[]", nb + 1)
        check(L.c3b_bgzf_sizes(self._h, size, off))
        image = bytearray(int(size[0]))
        check(L.c3b_bgzf_fetch(self._h, ffi.from_buffer(image) if image else ffi.NULL, 0))
        return bytes(image), [int(off[i]) for i in range(nb + 1)]

    def write_bgzf(self, path, data):
        """``bam_io.write_bgzf`` on the GPU: writes ``data`` (as ``compress_bgzf`` takes it) to ``path`` as a BGZF file with
        the end-of-file block, the same bytes, and returns the same ``voffset(u)``, which ``bam_io.write_tbi`` indexes with."""
        image, off = self.compress_bgzf(data)
        with open(path, "wb") as f:
            f.write(image)
            f.write(bam_io._EOF)
        return bam_io.bgzf_voffset(off[:-1], off[-1])
