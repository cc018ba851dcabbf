"""ORACLE — test infrastructure only (never imported by the product path).

The records of ``c3b_decode_calls`` (``clair3_b200/csrc/decode.cu``, stage 3) built on the CPU from the host decoder in
``clair3_b200/decode.py``: ``parse_alt_info``, the numpy stages (``decode_oracle``, ``decode_stage2_oracle``, ranked in full),
``output_from_ranked`` and ``row_fields``, which ``tests/golden/decode_stage2.npz`` and ``tests/golden/decode_calls.npz`` pin to
the reference's own ``output_from`` and ``batch_output``.  An exception of the host path becomes the record's status.
"""
from __future__ import annotations

import numpy as np

from clair3_b200 import decode
from clair3_b200.model import CALL_DTYPE

from . import decode_oracle as dec1
from . import decode_stage2_oracle as dec2

GENOTYPE_CODE = {v: k for k, v in decode.GENOTYPES.items()}
HET = (2, 4, 5, 7, 8, 9)


def _genotype(flags, multi, config):
    g = None
    if flags[0]:
        g = "0/0"
    elif flags[1] or flags[3] or flags[6]:
        g = "1/1"
    elif flags[2] or flags[4] or flags[5] or flags[7] or flags[8]:
        g = "0/1"
    if multi:
        g = "1/2"
    if g is not None and (config.is_haploid_precise_mode_enabled or config.is_haploid_sensitive_mode_enabled):
        g = "1" if "1" in g else "0"
    return g


def site_record(depth, alt, info, config):
    """(record fields, REF, ALT, allele counts) of one decoded site, or raises what the host path raises."""
    flags, (ref, alt_b), p = info
    is_ref = bool(flags[0])
    multi = "," in str(alt_b)
    printed = not ((not config.is_show_reference and is_ref) or (not is_ref and ref == alt_b))
    if config.is_haploid_precise_mode_enabled and any(flags[c] for c in HET):
        printed = False
    if config.is_haploid_sensitive_mode_enabled and multi:
        printed = False
    if printed:
        genotype, ref_t, alt_t, ref_count, counts, support = decode.row_fields(depth, alt, info, config)
    else:                                   # format_row returns early: no counts; the text and genotype as it would print them
        genotype, counts, support = _genotype(flags, multi, config), [], 0
        ref_count = 0
        for key, count in alt.items():
            if key[:1] == "R":
                ref_count = int(count)
        ref_count = max(0, ref_count)
        ref_t, alt_t = ref, ("." if is_ref else alt_b)
        if not config.keep_iupac_bases:
            ref_t, alt_t = decode.convert_iupac_to_n(ref_t), decode.convert_iupac_to_n(alt_t)
    rec = {"dp": depth, "support": support, "ref_count": ref_count, "prob": np.float32(p), "ref_len": len(ref_t),
           "alt_len": len(alt_t), "n_ad": len(counts), "flags": sum(int(bool(f)) << b for b, f in enumerate(flags)),
           "genotype": GENOTYPE_CODE[genotype], "printed": int(printed), "status": 0}
    return rec, ref_t, alt_t, counts


def decode_calls(y, ref_base, alt_bytes, alt_offsets, config):
    """What ``Clair3_X.decode_calls`` returns (numpy): ``calls`` (CALL_DTYPE [B]), ``text`` uint8 and ``ad`` int64 pools."""
    y = np.asarray(y, dtype=np.float32)
    ref_base = np.asarray(ref_base, dtype=np.uint8)
    alt_bytes = np.asarray(alt_bytes, dtype=np.uint8)
    off = np.asarray(alt_offsets, dtype=np.int64)
    B, out_dim = y.shape
    pool = 2 * len(alt_bytes) + 8 * B
    calls = np.zeros(B, CALL_DTYPE)
    text = np.zeros(pool, np.uint8)
    ad = np.zeros(pool, np.int64)
    if B == 0:
        return {"calls": calls, "text": text, "ad": ad}
    bases = [chr(b) for b in ref_base]
    gt21 = np.array([decode.GT21_OF_BASE.get(decode.BASE2ACGT.get(b, "A"), 0) for b in bases], np.uint8)
    s1 = dec1.decode_stage1(y, gt21)
    ranked = dec2.decode_stage2(y, gt21, k=decode.ENTRIES[out_dim])
    max_len = config.maximum_variant_length_that_need_infer
    for s in range(B):
        c = calls[s]
        c["genotype"] = 255
        if not (0 <= off[s] <= off[s + 1] <= len(alt_bytes)) or bases[s] not in decode.BASE2ACGT:
            c["status"] = 5
            continue
        raw = alt_bytes[off[s]:off[s + 1]].tobytes()
        if any(b >= 0x80 for b in raw):
            c["status"] = 4
            continue
        try:
            depth, alt = decode.parse_alt_info(raw.decode())
        except ValueError:
            c["status"] = 1
            continue
        if any(abs(v) > 1 << 62 for v in [depth] + list(alt.values())):
            c["status"] = 4
            continue
        try:
            if s1["is_ref"][s]:
                acgt = decode.BASE2ACGT[bases[s]]
                info = decode.REFERENCE_FLAGS, (acgt, acgt), np.float32(s1["ref_prob"][s])
            else:
                info = decode.output_from_ranked(bases[s], 0, ranked["cat"][s], ranked["idx"][s], ranked["prob"][s],
                                                 ranked["tie_mask"][s], ranked["count"][s], alt, out_dim == 90, max_len)
            rec, ref_t, alt_t, counts = site_record(depth, alt, info, config)
        except IndexError:
            c["status"] = 2
            continue
        except TypeError:
            c["status"] = 3
            continue
        for name, v in rec.items():
            c[name] = v
        start = 2 * off[s] + 8 * s
        t = (ref_t + alt_t).encode()
        text[start:start + len(t)] = np.frombuffer(t, np.uint8)
        ad[start:start + len(counts)] = counts
    return {"calls": calls, "text": text, "ad": ad}


class OracleCalls:
    """Module-protocol stand-in whose ``decode_calls`` is this oracle (``decode.batch_output`` then takes the records route)."""

    def __init__(self, out_dim):
        self.out_dim = out_dim

    def decode_calls(self, y, ref_base, alt_bytes, alt_offsets, config, k=16):
        out = decode_calls(y, ref_base, alt_bytes, alt_offsets, config)
        out["calls"] = out["calls"].view(np.uint8).reshape(len(out["calls"]), CALL_DTYPE.itemsize)
        return out
