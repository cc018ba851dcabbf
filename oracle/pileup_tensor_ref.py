"""TEST INFRASTRUCTURE ONLY: the reference's own candidate-window loop, run live, as a checker.

Between the pileup counter and Clair3_P the reference decides which candidates get a 33-row tensor and what that tensor holds:
``CreateTensorPileup`` (HKU-BAL/Clair3 ``preprocess/CreateTensorPileupFromCffi.py:239-454``) slices every candidate's window out
of the contiguous chunks that ``__enforce_pileup_chunk_contiguity`` (``:180-236``) cuts from ``calculate_clair3_pileup``'s
matrix (``:343-397``).  ``create_tensor_pileup()`` runs that Python, unmodified, from the reference checkout that
``oracle.fa_ref.reference_src()`` finds.  It imports the checkout at run time and copies nothing from it.  The reference binds its
C through cffi as the module ``libclair3``; a small ctypes stand-in (``_LibClair3``) takes its place here and forwards
``calculate_clair3_pileup``, ``create_bam_fset``, ``destroy_bam_fset`` and ``destroy_plp_data`` to the compiled reference counter
of ``oracle/pileup_ref.py``, so ``pileup_counts_clair3``, ``_plp_data_to_numpy``, ``__enforce_pileup_chunk_contiguity`` and the
candidate loop all run as they are.  CPU only.  Only tests/ and tools/ may import this module; the product never does.
"""
from __future__ import annotations

import argparse
import ctypes
import os
import sys
import tempfile
import types

import numpy as np

from oracle import pileup_ref
from oracle.fa_ref import CONTIG, reference_src

FEATURES = 18
WINDOW = 33

_module = None


class _Owned:
    """What ``ffi.gc(handle, destructor)`` returns: the handle, released when the last reference goes."""

    def __init__(self, handle, destructor):
        self._as_parameter_ = handle
        self._destructor = destructor

    def __del__(self):
        if self._destructor is not None and self._as_parameter_:
            self._destructor(self)
            self._destructor = None


class _PlpData:
    """The ``plp_data`` cffi proxy: field access reads through the pointer."""

    def __init__(self, ptr):
        self._ptr = ptr

    def __getattr__(self, name):
        return getattr(self._ptr.contents, name)


class _Ffi:
    @staticmethod
    def buffer(ptr, size):
        return ctypes.string_at(ptr, size) if size else b""

    @staticmethod
    def string(s):
        return s if isinstance(s, bytes) else ctypes.string_at(s)

    @staticmethod
    def gc(handle, destructor):
        return _Owned(handle, destructor)


class _Lib:
    featlenclair3 = FEATURES

    def __init__(self, L):
        self._L = L

    def calculate_clair3_pileup(self, region, fset, fasta, *args):
        return _PlpData(self._L.calculate_clair3_pileup(region, fset, fasta, *args))

    def create_bam_fset(self, bam, fasta):
        return self._L.create_bam_fset(bam, fasta)

    def destroy_bam_fset(self, fset):
        self._L.destroy_bam_fset(fset)

    def destroy_plp_data(self, plp, gvcf):
        self._L.destroy_plp_data(plp._ptr, bool(gvcf))


def available():
    """The reference checkout (for its Python) and the compiled reference counter are both present."""
    src = reference_src()
    return src is not None and os.path.exists(os.path.join(os.path.dirname(src), "preprocess", "CreateTensorPileupFromCffi.py")) \
        and pileup_ref.build() is not None


def _load():
    global _module
    if _module is None:
        src = reference_src()
        if src is None:
            raise FileNotFoundError("no reference checkout found (set CLAIR3_REFERENCE)")
        root = os.path.dirname(src)
        stub = types.ModuleType("libclair3")
        stub.lib, stub.ffi = _Lib(pileup_ref._load()), _Ffi()
        saved_path, saved_mod = list(sys.path), sys.modules.get("libclair3")
        sys.path.insert(0, root)
        sys.modules["libclair3"] = stub
        try:
            import importlib
            mod = importlib.import_module("preprocess.CreateTensorPileupFromCffi")
        finally:
            sys.path[:] = saved_path
            if saved_mod is None:
                sys.modules.pop("libclair3", None)
            else:
                sys.modules["libclair3"] = saved_mod
        if not os.path.abspath(mod.__file__).startswith(os.path.abspath(root) + os.sep):
            raise ImportError("preprocess.CreateTensorPileupFromCffi did not come from the reference checkout %s" % root)
        _module = mod
    return _module


def create_tensor_pileup(records, ref_seq, ref_start, ctg_start, ctg_end, min_depth=2, min_snp_af=0.08, min_indel_af=0.15,
                         min_mq=5, call_snp_only=False, call_ht=False):
    """The reference's ``CreateTensorPileup(args)`` with ``tensor_can_fn="PIPE"`` on in-memory records: contig ``CONTIG`` =
    ``'N' * ref_start + ref_seq``, the 1-based slice [ctg_start, ctg_end], platform ilmn, no fast mode, no BED, no VCF, no gVCF.
    The keyword arguments are those of ``PileupCounter.count``.  The counter region of the same call is
    ``clair3_b200.pileup_counts.counting_region(ctg_start, ctg_end)``.  Returns (tensors int32 [k, 33, 18], position strings
    ``"ctg:pos:ref_base"``, alt strings ``"depth-alt"``), k = the windows the reference keeps, in its order."""
    mod = _load()
    keep = pileup_ref.register(records, ref_seq, ref_start, min_mq)     # noqa: F841 - alive until the pileup has run
    with tempfile.TemporaryDirectory(prefix="c3b_plp_tensor_") as tmp:
        fasta = os.path.join(tmp, "ref.fa")
        contig = keep[1]
        with open(fasta, "wb") as f:
            f.write(b">" + CONTIG.encode() + b"\n" + contig + b"\n")
        with open(fasta + ".fai", "w") as f:
            f.write("%s\t%d\t%d\t%d\t%d\n" % (CONTIG, len(contig), len(CONTIG) + 2, len(contig), len(contig) + 1))
        args = argparse.Namespace(
            platform="ilmn", bam_fn=os.path.join(tmp, "in-memory.bam"), ref_fn=fasta, tensor_can_fn="PIPE", vcf_fn=None,
            min_af=float(min_snp_af), snp_min_af=float(min_snp_af), indel_min_af=float(min_indel_af), ctgName=CONTIG,
            ctgStart=int(ctg_start), ctgEnd=int(ctg_end), bed_fn=None, gvcf=False, sampleName="SAMPLE", samtools="samtools",
            fast_mode=False, enable_variant_calling_at_sequence_head_and_tail=bool(call_ht), minCoverage=int(min_depth),
            minMQ=int(min_mq), minBQ=0, max_depth=144, call_snp_only=bool(call_snp_only), extend_bed=None, temp_file_dir=tmp,
            indel_fn=None, enable_long_indel=False, chunk_num=None, chunk_id=None, test_pos=0)
        tensors, pos_info, alt_info = mod.CreateTensorPileup(args)
    tensors = np.asarray(tensors, dtype=np.int32)
    if tensors.size == 0:
        tensors = tensors.reshape(0, WINDOW, FEATURES)
    return tensors, list(pos_info), list(alt_info)


def kept_positions(pos_info):
    """1-based positions of the kept windows, from the reference's ``"ctg:pos:ref_base"`` strings."""
    return np.array([int(s.split(":")[1]) for s in pos_info], dtype=np.int64)
