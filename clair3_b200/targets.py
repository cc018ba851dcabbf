"""Where a run calls: a BED of target regions (``--bed_fn``) or a VCF of known sites (``--vcf_fn``, genotyping mode).

The reference turns either file into one extended BED per contig (HKU-BAL/Clair3 ``preprocess/CheckEnvs.py``:
``split_extend_bed`` :136-164 and ``split_extend_vcf`` :99-133) and its pileup step keeps a candidate only when that BED's
interval tree holds it and, in genotyping mode, when it is one of the chunk's known sites
(``preprocess/CreateTensorPileupFromCffi.py:347-355``).  ``read_bed`` / ``read_vcf`` read and extend the files the same way;
``ContigTargets`` holds one contig's result as sorted int64 arrays, states the reference's test on the host (``keep``) and
uploads the arrays once per device for the counter's test on the GPU (``c3b_plp_count_targeted``, DESIGN.md 5f).
"""
from __future__ import annotations

import gzip
from collections import OrderedDict

import numpy as np
import torch

from ._ffi import ffi

EXPAND = 33          # shared/param_p.py no_of_positions = 2 * flankingBaseNum + 1: the extension on either side


def _lines(source):
    """The text lines of a path (gzip or plain, as ``gzip -fdc`` reads both), of bytes / str contents, or of an iterable of
    lines."""
    if isinstance(source, (bytes, bytearray)):
        data = bytes(source)
    elif isinstance(source, str) and "\n" not in source:
        with open(source, "rb") as fh:
            data = fh.read()
    elif isinstance(source, str):
        return source.splitlines(keepends=True)
    else:
        return list(source)
    if data[:2] == b"\x1f\x8b":
        data = gzip.decompress(data)
    return data.decode().splitlines(keepends=True)


class Targets:
    """The extended targets of every contig of one BED (``kind == "bed"``) or one known-sites VCF (``kind == "vcf"``):
    ``intervals[ctg]`` = (starts, ends) in file order, 0-based and end-exclusive as the extended BED holds them; for a VCF also
    ``sites[ctg]`` (sorted unique 1-based positions, ``shared/utils.py:vcf_candidates_from``) and ``rows`` ((ctg, pos) -> the
    row's text, the last row of a duplicate key, in first-seen key order: what AddBackMissingVariantsInGenotyping reads)."""

    def __init__(self, kind, intervals, sites=None, rows=None):
        self.kind, self.intervals, self.sites, self.rows = kind, intervals, sites, rows
        self._contigs = {}

    def contigs(self):
        return list(self.intervals) if self.kind == "bed" else list(self.sites)

    def contig(self, ctg, chunk=None):
        """``ContigTargets`` of contig ``ctg`` (empty when the file has none of it).  ``chunk`` = (chunk_id, chunk_num): in
        genotyping mode, keep only that chunk's slice of the known sites (``pileup_counts.known_sites_chunk``)."""
        key = (ctg, chunk)
        if key not in self._contigs:
            s, e = self.intervals.get(ctg, (np.zeros(0, np.int64), np.zeros(0, np.int64)))
            known, rows = None, None
            if self.kind == "vcf":
                known = self.sites.get(ctg, np.zeros(0, np.int64))
                if chunk is not None:
                    from .pileup_counts import known_sites_chunk
                    c = known_sites_chunk(known, *chunk)
                    known = np.zeros(0, np.int64) if c is None else c[2]
                mine = set(known.tolist())
                rows = {p: r for (c, p), r in self.rows.items() if c == ctg and p in mine}
            self._contigs[key] = ContigTargets(ctg, s, e, known, rows)
        return self._contigs[key]


def read_bed(source):
    """A BED (path, gzip or plain; or its contents) as CheckEnvs' ``split_extend_bed`` extends it: ``#`` rows skipped, every
    other row ``ctg s e ...`` becomes [max(0, s - 33), max(0, e + 33)); a row with e < s or a negative coordinate is refused
    (ValueError), as the reference exits on it."""
    iv = OrderedDict()
    for i, row in enumerate(_lines(source)):
        if row[:1] == "#":
            continue
        cols = row.strip().split()
        try:
            ctg, s, e = cols[0], int(cols[1]), int(cols[2])
        except (IndexError, ValueError):
            raise ValueError("read_bed: row %d is not 'contig start end': %r" % (i + 1, row)) from None
        if e < s or s < 0 or e < 0:
            raise ValueError("read_bed: invalid BED input in row %d: %s %d %d" % (i + 1, ctg, s, e))
        iv.setdefault(ctg, ([], []))
        iv[ctg][0].append(max(0, s - EXPAND))
        iv[ctg][1].append(max(0, e + EXPAND))
    return Targets("bed", {c: (np.array(a, np.int64), np.array(b, np.int64)) for c, (a, b) in iv.items()})


def read_vcf(source):
    """A known-sites VCF (path, gzip or plain; or its contents): CheckEnvs' ``split_extend_vcf`` gives each site at 1-based
    ``pos`` the interval [pos - 34, pos + 33) and leaves out the sites with pos - 1 < 33, which stay known sites all the same
    (``vcf_candidates_from``); a position below 1 is refused (ValueError)."""
    iv, sites, rows = OrderedDict(), OrderedDict(), OrderedDict()
    for i, row in enumerate(_lines(source)):
        if row[:1] == "#":
            continue
        cols = row.strip().split(maxsplit=3)
        try:
            ctg, pos = cols[0], int(cols[1])
        except (IndexError, ValueError):
            raise ValueError("read_vcf: row %d is not 'contig pos ...': %r" % (i + 1, row)) from None
        if pos - 1 < 0:
            raise ValueError("read_vcf: invalid VCF input in row %d: %s %d" % (i + 1, ctg, pos))
        sites.setdefault(ctg, set()).add(pos)
        rows.pop((ctg, pos), None)
        rows[(ctg, pos)] = row if row.endswith("\n") else row + "\n"
        if pos - 1 - EXPAND < 0:
            continue
        iv.setdefault(ctg, ([], []))
        iv[ctg][0].append(pos - 1 - EXPAND)
        iv[ctg][1].append(pos + EXPAND)
    return Targets("vcf", {c: (np.array(a, np.int64), np.array(b, np.int64)) for c, (a, b) in iv.items()},
                   {c: np.array(sorted(v), np.int64) for c, v in sites.items()}, rows)


class ContigTargets:
    """One contig's targets as the counter's test reads them (``c3b_plp_targets``): the intervals sorted by start (a zero-length
    row stored as [s, s + 1), as the reference's interval tree stores it), the running maximum of their ends, and in genotyping
    mode the known 1-based positions (``known`` None: no known-site test) with their rows (``rows``: position -> text)."""

    def __init__(self, ctg, starts, ends, known=None, rows=None):
        s, e = np.asarray(starts, np.int64), np.asarray(ends, np.int64)
        self._span = (int(s.min()), int(e.max())) if len(s) else None
        e = np.where(e == s, s + 1, e)
        order = np.argsort(s, kind="stable")
        self.ctg = ctg
        self.starts, self.ends = s[order], e[order]
        self.end_max = np.maximum.accumulate(self.ends) if len(self.ends) else self.ends.copy()
        self.known = None if known is None else np.unique(np.asarray(known, np.int64))
        self.rows = rows
        self._dev = {}

    def bed_region(self):
        """(bed_start, bed_end) of ``bed_tree_from(..., return_bed_region=True)``: the smallest start and largest end, which
        ``pileup_counts.bed_chunk_region`` cuts into chunks; None when the contig has no interval."""
        return self._span

    def keep(self, positions):
        """bool per 1-based position: ``is_region_in(tree, ctg, pos - 1, pos + 1)`` (some interval with s <= pos <= e) and, in
        genotyping mode, pos is a known site: the reference's two tests, restated on the host."""
        q = np.asarray(positions, np.int64)
        i = np.searchsorted(self.starts, q, side="right") - 1
        ok = (i >= 0) & (self.end_max[np.maximum(i, 0)] >= q) if len(self.starts) else np.zeros(q.shape, bool)
        if self.known is not None:
            ok &= np.isin(q, self.known)
        return ok

    def struct(self, device):
        """A ``c3b_plp_targets`` over device copies of the arrays, made once per device; the returned tuple keeps them alive."""
        key = str(device)
        if key not in self._dev:
            t = [torch.from_numpy(a.copy()).to(device) for a in (self.starts, self.ends, self.end_max)]
            known = None if self.known is None else torch.from_numpy(self.known.copy()).to(device)
            self._dev[key] = (t, known)
        t, known = self._dev[key]
        return device_struct(*t, known)


def device_struct(starts, ends, end_max, known=None):
    """A ``c3b_plp_targets`` over int64 device tensors (``known`` None: no known-site test).  Returns (struct, tensors): the
    tensors must outlive the count."""
    st = ffi.new("c3b_plp_targets *")
    st.n_intervals = int(starts.numel())
    p = lambda t: ffi.cast("const int64_t *", t.data_ptr()) if t.numel() else ffi.NULL  # noqa: E731
    st.starts, st.ends, st.end_max = p(starts), p(ends), p(end_max)
    st.n_sites = -1 if known is None else int(known.numel())
    st.sites = ffi.NULL if known is None else p(known)
    st.on_device = 1
    return st, (starts, ends, end_max, known)
