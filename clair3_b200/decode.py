"""Host side of the GPU decoder: turns ranked outcome lists into the reference's VCF rows.

The reference decodes one site at a time in Python (``batch_output`` -> ``output_with`` -> ``output_from`` ->
``possible_outcome_probabilites_from``, ``clair3/CallVariants.py:1069-1116, 1118-1394, 676-1012, 406-659``), building up to 804
float32 outcome probabilities per site and running ``max()`` / ``in`` over them once per retry.  Here the GPU does that part:

* ``c3b_decode_stage1`` drops the early-out homozygous-reference sites;
* ``c3b_decode_stage2`` ranks every other site's outcomes in the order ``output_from`` tries them, with the ``is_*`` flags
  each attempt would return (the tie mask);

and this module only walks the ranked entries, checking each against the site's ``alt_info`` (``output_from_ranked``), and
formats the row (``output_with``'s rules).  ``batch_output`` is the drop-in for the reference's function of the same name.

Not implemented (``NotImplementedError``): ``gvcf`` (the ``compute_PL`` column), ``is_debug`` and ``is_output_for_ensemble``.
"""
from __future__ import annotations

from collections import namedtuple
from math import e, log

import numpy as np

PHRED_TRANS = -10 * log(e, 10)                          # clair3/CallVariants.py:27
FLANKING_BASE_NUM = 16                                  # shared/param_{p,f}.py flankingBaseNum
VL_MAX = 16                                             # clair3/task/variant_length.py: VariantLength.max
MAX_INFER_LENGTH = 50                                   # shared/param_p.py maximum_variant_length_that_need_infer
LONG_INDEL_DISTANCE = 0.1                               # shared/param_p.py long_indel_distance_proportion
BASE2ACGT = dict(zip("ACGTURYSWKMBDHVN", "ACGTTACCAGACAAAA"))    # shared/utils.py IUPAC_base_to_ACGT_base_dict
GT21_OF_BASE = {"A": 0, "C": 4, "G": 7, "T": 9}         # gt21_enum_from_label(base + base)
HOMO_SNP_LABELS = ("AA", "CC", "GG", "TT")
HETERO_SNP_LABELS = ("AC", "AG", "AT", "CG", "CT", "GT")
ACGT = "ACGT"

# the reference's OutputConfig field names (clair3/CallVariants.py:29-44); batch_output accepts any object that has them
OutputConfig = namedtuple("OutputConfig", [
    "is_show_reference", "is_debug", "is_haploid_precise_mode_enabled", "is_haploid_sensitive_mode_enabled",
    "is_output_for_ensemble", "quality_score_for_pass", "tensor_fn", "input_probabilities", "add_indel_length", "gvcf", "pileup",
    "enable_long_indel", "maximum_variant_length_that_need_infer", "keep_iupac_bases"])


def replay_config(pileup, add_indel_length):
    """The OutputConfig of ``CallVariants --input_probabilities`` with only ``--pileup`` / ``--add_indel_length`` given
    (every other option at its default: ``--qual 2``, no showRef, no haploid mode, no long indels)."""
    return OutputConfig(is_show_reference=False, is_debug=False, is_haploid_precise_mode_enabled=False,
                        is_haploid_sensitive_mode_enabled=False, is_output_for_ensemble=False, quality_score_for_pass=2,
                        tensor_fn=None, input_probabilities=True, add_indel_length=bool(add_indel_length), gvcf=False,
                        pileup=bool(pileup), enable_long_indel=False, maximum_variant_length_that_need_infer=MAX_INFER_LENGTH,
                        keep_iupac_bases=False)


# categories in output_from's elif order, homo_Ref first (the bit order of the tie mask and of the returned flag tuple)
REF, HOMO_SNP, HETERO_SNP, HOMO_INS, HETERO_ACGT_INS, HETERO_INSINS, HOMO_DEL, HETERO_ACGT_DEL, HETERO_DELDEL, INSDEL = range(10)
ENTRIES = {90: 804, 24: 24}
INSINS_PAIRS = [(i, j) for i in range(1, 17) for j in range(i, 17)]
DELDEL_PAIRS = [(min(i, j), max(i, j)) for i in range(1, 17) for j in range(1, 17) if not (i == j and i != 16)]
INSDEL_PAIRS = [(i, j) for i in range(1, 17) for j in range(1, 17)]
REFERENCE_FLAGS = (True,) + (False,) * 9


# ------------------------------------------------------------------------------------------------ alt-info rules
def find_alt_base(alt_info_dict, alternate_base=None):
    """SNP alleles seen in the reads, most supported first (ties keep alt_info order); the proposed base is replaced by the
    best-supported one when it is absent or trails it by 9 or more reads.  Returns (bases, base)."""
    snps = [(key[1], count) for key, count in alt_info_dict.items() if key[0] == "X"]
    snps.sort(key=lambda kv: kv[1], reverse=True)
    if not snps:
        return [], None
    proposed = [count for base, count in snps if base == alternate_base]
    if not proposed or snps[0][1] - proposed[0] >= 9:
        alternate_base = snps[0][0]
    return [base for base, _ in snps], alternate_base


def _indel_bases(alt_info_dict, kind, propose_length, minimum, maximum, ignore, return_multi):
    if not alt_info_dict:
        return ""
    proposed, others = {}, {}
    for key, count in alt_info_dict.items():
        if key[0] != kind:
            continue
        bases = key[1:]
        if propose_length and len(bases) == propose_length and bases != ignore:
            proposed[bases] = count
        elif minimum <= len(bases) <= maximum and bases != ignore:
            others[bases] = count
    if propose_length and proposed:
        return max(proposed, key=proposed.get)
    if return_multi:
        ranked = [b for b, _ in sorted(others.items(), key=lambda kv: kv[1])[::-1]]
        if kind == "I":
            return ranked[:2] if ranked else ""
        if len(ranked) <= 1:
            return ""
        return [ranked[0], ranked[1]] if len(ranked[0]) > len(ranked[1]) else [ranked[1], ranked[0]]
    return max(others, key=others.get) if others else ""


def insertion_bases_using_alt_info_from(alt_info_dict, propose_insertion_length=None, minimum_insertion_length=1,
                                        maximum_insertion_length=50, insertion_bases_to_ignore="", return_multi=False):
    """Inserted sequence (reference base included) with the most reads: of the proposed length when any has it, else within
    [minimum, maximum]; ``return_multi``: the two best, most reads first."""
    return _indel_bases(alt_info_dict, "I", propose_insertion_length + 1 if propose_insertion_length else None,
                        minimum_insertion_length, maximum_insertion_length, insertion_bases_to_ignore, return_multi)


def deletion_bases_using_alt_info_from(alt_info_dict, propose_deletion_length=None, minimum_deletion_length=1,
                                       maximum_deletion_length=50, deletion_bases_to_ignore="", return_multi=False):
    """Deleted sequence with the most reads (same selection as insertions); ``return_multi``: the two best, longer first."""
    return _indel_bases(alt_info_dict, "D", propose_deletion_length, minimum_deletion_length, maximum_deletion_length,
                        deletion_bases_to_ignore, return_multi)


def _proposed(length):
    return length if length and length < VL_MAX else None


def _try_outcome(cat, idx, ref_seq_base, alt_info_dict, add_indel_length, max_len):
    """One attempt of output_from: (reference_base, alternate_base) for outcome ``idx`` of category ``cat``, or None when the
    reads do not support it (the reference then zeroes that probability and retries).

    output_from's loop runs while either allele is None, and every attempt starts with alternate_base None.  Some failing
    attempts set both before their ``continue`` and so end the loop all the same; they return that pair here too:
    a homozygous / heterozygous SNP whose best read-supported base is the reference base (ref, ref), a SNP+insertion without
    SNP reads (ref, insertion), two equal insertions (ref, insertion) and two deletions of equal length (ref+del, ref)."""
    ins = lambda length=None, **kw: insertion_bases_using_alt_info_from(                          # noqa: E731
        alt_info_dict, propose_insertion_length=_proposed(length), maximum_insertion_length=max_len, **kw)
    dele = lambda length=None, **kw: deletion_bases_using_alt_info_from(                          # noqa: E731
        alt_info_dict, propose_deletion_length=_proposed(length), maximum_deletion_length=max_len, **kw)
    ref = ref_seq_base
    if cat == HOMO_SNP:
        b1, b2 = HOMO_SNP_LABELS[idx]
        _, alt = find_alt_base(alt_info_dict, b1 if b1 != ref else b2)
        return None if alt is None else (ref, alt)
    if cat == HETERO_SNP:
        b1, b2 = HETERO_SNP_LABELS[idx]
        if b1 != ref and b2 != ref:
            bases, _ = find_alt_base(alt_info_dict)
            return None if len(bases) < 2 else (ref, ",".join(bases[:2]))
        _, alt = find_alt_base(alt_info_dict, b1 if b1 != ref else b2)
        return None if alt is None else (ref, alt)
    if cat == HOMO_INS:
        bases = ins(idx + 1 if add_indel_length else None)
        return (ref, bases) if bases else None
    if cat == HETERO_ACGT_INS:
        base, length = (ACGT[idx % 4], idx // 4 + 1) if add_indel_length else (ACGT[idx], None)
        bases = ins(length)
        if not bases:
            return None
        if base != ref:
            snps, _ = find_alt_base(alt_info_dict)
            return (ref, "%s,%s" % (snps[0], bases)) if snps else (ref, bases)
        return ref, bases
    if cat == HETERO_INSINS:
        pair = []
        if add_indel_length:
            l1, l2 = INSINS_PAIRS[idx]
            b1 = ins(l1)
            if b1:
                b2 = ins(l2, insertion_bases_to_ignore=b1)
                if b2:
                    pair = [b1, b2]
        if len(pair) < 2:
            pair = ins(return_multi=True)
        if len(pair) < 2:
            return None
        return (ref, "%s,%s" % (pair[1], pair[0])) if pair[0] != pair[1] else (ref, pair[0])
    if cat in (HOMO_DEL, HETERO_ACGT_DEL):
        if cat == HOMO_DEL:
            base, length = None, (idx + 1 if add_indel_length else None)
        else:
            base, length = (ACGT[idx % 4], idx // 4 + 1) if add_indel_length else (ACGT[idx], None)
        bases = dele(length)
        if not bases:
            return None
        ref_allele = ref + bases
        if base is not None and base != ref_allele[0]:
            return ref_allele, "%s,%s" % (ref_allele[0], base + ref_allele[1:])
        return ref_allele, ref_allele[0]
    if cat == HETERO_DELDEL:
        pair = []
        if add_indel_length:
            l1, l2 = sorted(DELDEL_PAIRS[idx], reverse=True)
            b1 = dele(l1)
            if b1:
                b2 = dele(l2, deletion_bases_to_ignore=b1)
                if b2:
                    pair = [b1, b2] if len(b1) > len(b2) else [b2, b1]
        if len(pair) < 2:
            pair = dele(return_multi=True)
        if len(pair) < 2:
            return None
        ref_allele = ref + pair[0]
        a1, a2 = ref_allele[0], ref_allele[0] + ref_allele[len(pair[1]) + 1:]
        if a1 != a2 and ref_allele != a1 and ref_allele != a2:
            return ref_allele, "%s,%s" % (a1, a2)
        return ref_allele, a1
    if cat == INSDEL:
        l_del, l_ins = INSDEL_PAIRS[idx] if add_indel_length else (None, None)
        ins_bases, del_bases = ins(l_ins), dele(l_del)
        if not ins_bases or not del_bases:
            return None
        ref_allele = ref + del_bases
        return ref_allele, "%s,%s" % (ref_allele[0], ins_bases + ref_allele[1:])
    raise ValueError("unknown outcome category %r" % (cat,))


def output_from_ranked(reference_sequence, tensor_position_center, cat, idx, prob, tie_mask, count, alt_info_dict,
                       add_indel_length, maximum_variant_length_that_need_infer):
    """``output_from`` (CallVariants.py:676-1012) over one site's ranked entries (the first ``count`` of ``cat`` / ``idx`` /
    ``prob`` / ``tie_mask``, from ``decode_stage2``).  Returns what the reference returns - (flags, (ref, alt), probability) -
    or None when the entries run out before an attempt succeeds or homo_Ref is reached (re-rank with a larger ``k``)."""
    ref_base = reference_sequence[tensor_position_center]
    ref_acgt = BASE2ACGT[ref_base]
    for t in range(int(count)):
        c = int(cat[t])
        p = np.float32(prob[t])
        if c == REF:
            return REFERENCE_FLAGS, (ref_acgt, ref_acgt), p
        got = _try_outcome(c, int(idx[t]), ref_base, alt_info_dict, add_indel_length, maximum_variant_length_that_need_infer)
        if got is not None:
            m = int(tie_mask[t])
            return tuple(bool(m >> b & 1) for b in range(10)), got, p
    return None


# ------------------------------------------------------------------------------------------------ row formatting
def quality_score_from(p):
    """QUAL of probability ``p`` (a numpy float32: the ratio is float32 arithmetic, the log double)."""
    return float(round(max(PHRED_TRANS * log(((1.0 - p) + 1e-10) / (p + 1e-10)) + 10, 0), 2))


def convert_iupac_to_n(s):
    if s == ".":
        return s
    return "".join(ch if ch.upper() in "ACGTN,." else "N" for ch in s)


def _long_indel_reads(alt, proposed_ins_base="", propose_del_base_length=0):
    """get_long_indel_read_count as output_with calls it (never with is_del): reads of other long insertions within 10 % of the
    proposed length.  A deletion's proposed length only enables the count, which then spans [50, -1.1] and is always 0."""
    if not (len(proposed_ins_base) > MAX_INFER_LENGTH or propose_del_base_length > MAX_INFER_LENGTH):
        return 0
    length = len(proposed_ins_base) - 1
    lo, hi = max(length * (1.0 - LONG_INDEL_DISTANCE), MAX_INFER_LENGTH), length * (1.0 + LONG_INDEL_DISTANCE)
    return sum(count for bases, count in alt.items() if bases != proposed_ins_base and lo <= len(bases) <= hi)


def parse_alt_info(alt_info):
    """``depth-KEY count KEY count ...`` -> (depth, {key: count})   (output_with, CallVariants.py:1146-1155)."""
    if isinstance(alt_info, np.ndarray):
        alt_info = alt_info.reshape(-1)[0]
    if isinstance(alt_info, (bytes, np.bytes_)):
        alt_info = alt_info.decode()
    parts = alt_info.rstrip().split("-")
    seqs = (parts[1] if len(parts) > 1 else "").split(" ")
    return int(parts[0]), dict(zip(seqs[::2], [int(c) for c in seqs[1::2]]))


def parse_chr_pos_seq(chr_pos_seq):
    if isinstance(chr_pos_seq, np.ndarray):
        chr_pos_seq = chr_pos_seq.reshape(-1)[0]
    if isinstance(chr_pos_seq, (bytes, np.bytes_)):
        chr_pos_seq = chr_pos_seq.decode()
    info = chr_pos_seq.rstrip().split(":")
    chromosome = info[0] if len(info) == 3 else ":".join(info[:-2])
    return chromosome, int(info[-2]), info[-1]


def format_row(chromosome, position, read_depth, alt_info_dict, output_info, output_config):
    """``output_with``'s filters and VCF row (CallVariants.py:1180-1394) for one ``output_from`` result; None = no row."""
    flags, (reference_base, alternate_base), probability = output_info
    (is_ref, is_homo_snp, is_het_snp, is_homo_ins, is_het_acgt_ins, is_het_insins, is_homo_del, is_het_acgt_del,
     is_het_deldel, is_insdel) = flags
    if (not output_config.is_show_reference and is_ref) or (not is_ref and reference_base == alternate_base):
        return None
    if reference_base is None or alternate_base is None:
        return None
    is_multi = "," in str(alternate_base)
    if output_config.is_haploid_precise_mode_enabled and (is_het_snp or is_het_acgt_ins or is_het_insins or is_het_acgt_del
                                                          or is_het_deldel or is_insdel):
        return None
    if output_config.is_haploid_sensitive_mode_enabled and is_multi:
        return None
    fields = row_fields(read_depth, alt_info_dict, output_info, output_config)
    return row_text(chromosome, position, read_depth, probability, is_ref, fields, output_config)


def row_fields(read_depth, alt_info_dict, output_info, output_config):
    """The data of ``output_with``'s row for a call ``format_row`` prints: (genotype, REF, ALT, ref_count, allele counts,
    support), REF / ALT as the row prints them.  Only for a printed call (the filters of ``format_row`` passed)."""
    flags, (reference_base, alternate_base), probability = output_info
    (is_ref, is_homo_snp, is_het_snp, is_homo_ins, is_het_acgt_ins, is_het_insins, is_homo_del, is_het_acgt_del,
     is_het_deldel, is_insdel) = flags
    is_multi = "," in str(alternate_base)
    genotype = None
    if is_ref:
        genotype = "0/0"
    elif is_homo_snp or is_homo_ins or is_homo_del:
        genotype = "1/1"
    elif is_het_snp or is_het_acgt_ins or is_het_insins or is_het_acgt_del or is_het_deldel:
        genotype = "0/1"
    if is_multi:
        genotype = "1/2"

    snp, ins, dels, ref_count = {}, {}, {}, 0
    for key, count in alt_info_dict.items():
        if key[0] == "X":
            snp[key[1]] = int(count)
        elif key[0] == "I":
            ins[key[1:]] = int(count)
        elif key[0] == "D":
            dels[key[1:]] = int(count)
        elif key[0] == "R":
            ref_count = int(count)
    ref_count = max(0, ref_count)
    long_indel = output_config.enable_long_indel
    support, counts = 0, []
    if is_ref:
        support = ref_count
        alternate_base = "."
    elif is_homo_snp or is_het_snp:
        for base in str(alternate_base):
            if base != ",":
                counts.append(snp.get(base, 0))
                support += counts[-1]
    elif is_homo_ins or is_het_insins:
        for bases in alternate_base.split(","):
            n = ins.get(bases, 0) + (_long_indel_reads(ins, proposed_ins_base=bases) if long_indel else 0)
            support += n
            counts.append(n)
    elif is_het_acgt_ins:
        snp_base = alternate_base.split(",")[0][0] if is_multi else None
        bases = alternate_base.split(",")[1] if is_multi else alternate_base
        n_snp = snp.get(snp_base, 0) if is_multi else 0
        n_ins = ins.get(bases, 0) + (_long_indel_reads(ins, proposed_ins_base=bases) if long_indel else 0)
        support = n_ins + n_snp
        if snp_base:
            counts.append(n_snp)
        counts.append(n_ins)
    elif is_homo_del or is_het_deldel:
        if dels:
            if is_homo_del:
                del_bases = reference_base[1:] if len(reference_base) > 1 else None
                extra = _long_indel_reads(dels, propose_del_base_length=len(del_bases)) if long_indel else 0
                support = dels.get(del_bases, 0) + extra
                counts.append(support)
            elif len(dels) > 1:
                for bases in alternate_base.split(","):
                    n = _deletion_reads(dels, len(reference_base) - len(bases), long_indel)
                    counts.append(n)
                    support += n
    elif is_het_acgt_del:
        alleles = alternate_base.split(",")
        snp_base = (alleles[1][0] if len(alleles) > 1 else None) if is_multi else None
        n_snp = snp.get(snp_base, 0) if is_multi else 0
        del_bases = reference_base[1:] if len(reference_base) > 1 else None
        extra = _long_indel_reads(dels, propose_del_base_length=len(del_bases)) if long_indel else 0
        n_del = dels.get(del_bases, 0) + extra
        support = n_del + n_snp
        if snp_base:
            counts.append(n_snp)
        counts.append(n_del)
    elif is_insdel:
        for bases in alternate_base.split(","):
            alt_len = len(reference_base) - len(bases)
            if alt_len < 0:
                ins_bases = bases[:-(len(reference_base) - 1)] if len(reference_base) > 1 else bases
                n = ins.get(ins_bases, 0) + (_long_indel_reads(ins, proposed_ins_base=ins_bases) if long_indel else 0)
            else:
                n = _deletion_reads(dels, alt_len, long_indel)
            counts.append(n)
            support += n

    if output_config.is_haploid_precise_mode_enabled or output_config.is_haploid_sensitive_mode_enabled:
        genotype = "1" if "1" in genotype else "0"
    if not output_config.keep_iupac_bases:
        reference_base = convert_iupac_to_n(reference_base)
        alternate_base = convert_iupac_to_n(alternate_base)
    return genotype, reference_base, alternate_base, ref_count, counts, support


def row_text(chromosome, position, read_depth, probability, is_ref, fields, output_config):
    """The VCF row of a printed call from its ``row_fields``: QUAL, FILTER and AF are computed here."""
    genotype, reference_base, alternate_base, ref_count, counts, support = fields
    af = ((support + 0.0) / read_depth) if read_depth != 0 else 0.0
    af = 1 if af > 1 else af
    qual = quality_score_from(probability)
    if is_ref:
        filt = "RefCall"
    elif output_config.quality_score_for_pass is None or qual >= output_config.quality_score_for_pass:
        filt = "PASS"
    else:
        filt = "LowQual"
    ad = str(ref_count) + ("," + ",".join(str(c) for c in counts) if counts else "")
    af_s = "%.4f" % af if len(counts) <= 1 else ",".join("%.4f" % min(1.0, 1.0 * c / read_depth) for c in counts)
    return "%s\t%d\t.\t%s\t%s\t%.2f\t%s\t%s\tGT:GQ:DP:AD:AF\t%s:%d:%d:%s:%s\n" % (
        chromosome, position, reference_base, alternate_base, qual, filt, "P" if output_config.pileup else "F", genotype, qual,
        read_depth, ad, af_s)


def _deletion_reads(dels, length, long_indel):
    """Reads of the first deletion of that length in alt_info order (plus the always-zero long-deletion term)."""
    same = [c for bases, c in dels.items() if len(bases) == length]
    return (same[0] if same else 0) + (_long_indel_reads(dels, propose_del_base_length=length) if long_indel else 0)


# ------------------------------------------------------------------------------------------------ batch
def _check_config(output_config):
    for name in ("gvcf", "is_debug", "is_output_for_ensemble"):
        if getattr(output_config, name, False):
            raise NotImplementedError("clair3_b200.decode.batch_output does not implement %s output; use the reference's "
                                      "decoder for it" % name)


def _numpy(d):
    return {k: (v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)) for k, v in d.items()}


def batch_output(model, batch_chr_pos_seq, alt_info_list, Y, output_config, k=16):
    """The reference's ``batch_output`` (CallVariants.py:1069-1116) for one batch: returns the VCF rows as one string.
    ``model`` provides ``decode_calls`` (a ``Clair3_P`` / ``Clair3_F``: the walk runs on the GPU, ``batch_calls``) or only
    ``decode_stage1`` / ``decode_stage2`` (the walk runs here, ``output_from_ranked``); ``Y`` float32 [B, 24|90];
    ``output_config`` any object with the reference's ``OutputConfig`` field names."""
    _check_config(output_config)
    Y = np.ascontiguousarray(np.asarray(Y.cpu() if hasattr(Y, "cpu") else Y, dtype=np.float32))
    B = len(batch_chr_pos_seq)
    if len(Y) != B:
        raise ValueError("Inconsistent shape between input tensor and output predictions %d/%d" % (B, len(Y)))
    if B == 0:
        return ""
    if hasattr(model, "decode_calls"):
        return calls_text(batch_calls(model, batch_chr_pos_seq, alt_info_list, Y, output_config, k=k), output_config)
    add_indel_length = bool(output_config.add_indel_length)
    if Y.shape[1] != (90 if add_indel_length else 24):
        raise ValueError("Y has %d columns but add_indel_length=%s" % (Y.shape[1], add_indel_length))
    max_len = output_config.maximum_variant_length_that_need_infer
    sites = []
    for chr_pos_seq, alt_info in zip(batch_chr_pos_seq, alt_info_list):
        chromosome, position, seq = parse_chr_pos_seq(chr_pos_seq)
        center = FLANKING_BASE_NUM if len(seq) > 1 else 0
        depth, alt = parse_alt_info(alt_info)
        sites.append((chromosome, position, seq, center, depth, alt))
    ref_gt21 = np.array([GT21_OF_BASE[BASE2ACGT[s[2][s[3]]]] for s in sites], dtype=np.uint8)

    s1 = _numpy(model.decode_stage1(Y, ref_gt21))
    nonref = s1["nonref_idx"][:int(s1["n_nonref"][0])]
    results = [None] * B
    for b in np.nonzero(s1["is_ref"])[0]:
        base = BASE2ACGT[sites[b][2][sites[b][3]]]
        results[b] = (REFERENCE_FLAGS, (base, base), np.float32(s1["ref_prob"][b]))
    if len(nonref):
        rerank = []
        s2 = _numpy(model.decode_stage2(Y, ref_gt21, sites=nonref.astype(np.int32), k=k))
        for j, b in enumerate(nonref):
            _, _, seq, center, _, alt = sites[b]
            results[b] = output_from_ranked(seq, center, s2["cat"][j], s2["idx"][j], s2["prob"][j], s2["tie_mask"][j],
                                            s2["count"][j], alt, add_indel_length, max_len)
            if results[b] is None:
                rerank.append(b)
        if rerank:                                 # the walk ran past the first k entries: rank those sites in full
            s2 = _numpy(model.decode_stage2(Y, ref_gt21, sites=np.array(rerank, dtype=np.int32), k=ENTRIES[Y.shape[1]]))
            for j, b in enumerate(rerank):
                _, _, seq, center, _, alt = sites[b]
                results[b] = output_from_ranked(seq, center, s2["cat"][j], s2["idx"][j], s2["prob"][j], s2["tie_mask"][j],
                                                s2["count"][j], alt, add_indel_length, max_len)
                assert results[b] is not None, "a full-length ranking always ends at homo_Ref"
    rows = []
    for (chromosome, position, _, _, depth, alt), info in zip(sites, results):
        row = format_row(chromosome, position, depth, alt, info, output_config)
        if row is not None:
            rows.append(row)
    return "".join(rows)


# ------------------------------------------------------------------------------------------------ calls as data
GENOTYPES = {0: "0/0", 1: "0/1", 2: "1/1", 3: "1/2", 4: "0", 5: "1", 255: None}
_STATUS_ERRORS = {1: ValueError, 2: IndexError, 3: TypeError, 4: ValueError, 5: ValueError}
_STATUS_TEXT = {1: "alt_info does not parse as 'depth-KEY count ...' (int() raises)",
                2: "alt_info holds an empty or a bare 'X' key, which output_from / output_with index",
                3: "the row takes len() of a missing deletion (enable_long_indel with a one-base REF under a deletion flag)",
                4: "alt_info holds a non-ASCII byte or a count beyond +-2**62",
                5: "bad alt_info offsets or reference base"}


def _as_bytes(s):
    if isinstance(s, np.ndarray):
        s = s.reshape(-1)[0]
    if isinstance(s, (bytes, np.bytes_)):
        return bytes(s)
    return str(s).encode()


def batch_calls(model, batch_chr_pos_seq, alt_info_list, Y, output_config, k=16):
    """Every site's call as arrays (``model.decode_calls``: the walk, the re-rank and the row's counts on the GPU).  Returns a
    dict: ``chromosome`` (list of str), ``position`` int64 [B], ``calls`` (``model.CALL_DTYPE`` records [B]: probability,
    flags, genotype code (``GENOTYPES``), printed, DP, AD's ref count, AF support, REF / ALT lengths, allele-count count),
    ``text`` / ``ad`` (the pools) and ``start`` int64 [B] (site s's REF, then ALT, at ``text[start[s]:]``, its allele counts
    at ``ad[start[s]:]``).  Raises what ``batch_output``'s host walk raises on an alt_info string it cannot decode."""
    _check_config(output_config)
    Y = np.ascontiguousarray(np.asarray(Y.cpu() if hasattr(Y, "cpu") else Y, dtype=np.float32))
    B = len(batch_chr_pos_seq)
    if len(Y) != B:
        raise ValueError("Inconsistent shape between input tensor and output predictions %d/%d" % (B, len(Y)))
    if Y.shape[1] != (90 if output_config.add_indel_length else 24):
        raise ValueError("Y has %d columns but add_indel_length=%s" % (Y.shape[1], bool(output_config.add_indel_length)))
    chromosomes, positions, ref_base = [], np.zeros(B, np.int64), np.zeros(B, np.uint8)
    for i, chr_pos_seq in enumerate(batch_chr_pos_seq):
        chromosome, position, seq = parse_chr_pos_seq(chr_pos_seq)
        base = seq[FLANKING_BASE_NUM if len(seq) > 1 else 0]
        BASE2ACGT[base]                                  # the host path's KeyError on a base outside the IUPAC table
        chromosomes.append(chromosome)
        positions[i] = position
        ref_base[i] = ord(base)
    alts = [_as_bytes(a) for a in alt_info_list]
    offsets = np.zeros(B + 1, np.int64)
    np.cumsum([len(a) for a in alts], out=offsets[1:])
    alt_bytes = np.frombuffer(bytearray(b"".join(alts)), dtype=np.uint8)
    return calls_result(_numpy(model.decode_calls(Y, ref_base, alt_bytes, offsets, output_config, k=k)), chromosomes, positions,
                        offsets)


def calls_result(out, chromosomes, positions, offsets):
    """``batch_calls``' dict from ``model.decode_calls``' arrays (on the host) of sites whose alt_info starts at ``offsets``, or
    the exception the host walk raises for the first site whose alt_info the decoder rejected."""
    from .model import CALL_DTYPE
    B = len(positions)
    calls = out["calls"].view(CALL_DTYPE).reshape(B)
    status = calls["status"]
    if status.any():
        early = np.isin(status, (1, 4, 5))                      # what the host path rejects before it decodes any site
        s = int(np.argmax(early)) if early.any() else int(np.argmax(status != 0))
        raise _STATUS_ERRORS[int(status[s])]("site %d (%s:%d): %s" % (s, chromosomes[s], positions[s], _STATUS_TEXT[int(status[s])]))
    return {"chromosome": chromosomes, "position": positions, "calls": calls, "text": out["text"], "ad": out["ad"],
            "start": 2 * offsets[:-1] + 8 * np.arange(B, dtype=np.int64)}


def calls_text(res, output_config):
    """The VCF rows of ``batch_calls``' printed calls (QUAL, FILTER and AF formatted here)."""
    return "".join(call_row(res, s, output_config) for s in np.nonzero(res["calls"]["printed"])[0])


def call_row(res, s, output_config):
    """The VCF row of ``batch_calls``' printed call ``s``."""
    c, text, ad = res["calls"][s], res["text"], res["ad"]
    o, rl, al, na = int(res["start"][s]), int(c["ref_len"]), int(c["alt_len"]), int(c["n_ad"])
    fields = (GENOTYPES[int(c["genotype"])], text[o:o + rl].tobytes().decode(), text[o + rl:o + rl + al].tobytes().decode(),
              int(c["ref_count"]), [int(v) for v in ad[o:o + na]], int(c["support"]))
    return row_text(res["chromosome"][s], int(res["position"][s]), int(c["dp"]), c["prob"], bool(c["flags"] & 1), fields,
                    output_config)
