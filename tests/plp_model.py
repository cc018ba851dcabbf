"""Test helper: a slow pure-Python, RANDOM-ACCESS model of the pileup counter (every (read, position) pair resolved on its own from
prefix sums over the CIGAR, the way clair3_b200/csrc/plp_counts.cu works) - an independent second statement of
oracle/pileup_oracle.c (which walks an incremental cursor column by column like htslib).  Small inputs only."""
import numpy as np

REFC = {0, 2, 3, 7, 8}
QRYC = {0, 1, 4, 7, 8}
MATCH = {0, 7, 8}
N2C = [-1, 0, 1, -1, 2, -1, -1, -1, 3, -1, -1, -1, -1, -1, -1, -1, -1, 9, 10, -1, 11, -1, -1, -1, 12, -1, -1, -1, -1, -1, -1, -1]
B2I = [0, 0, 1, 0, 0, 0, 2, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0]


def _nib(seq, so, lq, i):
    if i < 0 or i >= lq:
        return 0
    b = int(seq[so + (i >> 1)])
    return (b >> 4) & 15 if (i & 1) == 0 else b & 15


def model_pileup(rec, start, end, ref_seq, ref_start, min_depth=2, min_snp_af=0.08, min_indel_af=0.15, min_mq=5,
                 call_snp_only=False, call_ht=False):
    W = end - start
    cnt = np.zeros((W, 18), np.int64)
    quirk = np.zeros(W, np.int64)
    depth = np.zeros(W, np.int64)
    covered = np.zeros(W, bool)
    dels = [dict() for _ in range(W)]          # (strand, length) -> count
    ins = [dict() for _ in range(W)]           # (strand, string) -> count
    alle = [dict() for _ in range(W)]          # allele -> [first read, first inserted base in it, count], in order of first occurrence
    ins_last = np.full(W, -1, np.int64)        # the last read with an insertion on the column (c3b_plp_fetch_alleles: ins_last)
    n = len(rec["pos"])
    for r in range(n):
        fl = int(rec["flag"][r])
        if fl & (4 | 256 | 512 | 1024 | 2048) or int(rec["mapq"][r]) < min_mq:
            continue
        cig = rec["cigar"][rec["cigar_off"][r]:rec["cigar_off"][r + 1]]
        ops = [int(c) & 15 for c in cig]
        lens = [int(c) >> 4 for c in cig]
        xend, y0, x, y = [], [], 0, 0
        for o, l in zip(ops, lens):
            y0.append(y)
            if o in REFC:
                x += l
            if o in QRYC:
                y += l
            xend.append(x)
        beg = int(rec["pos"][r])
        if x == 0:
            continue
        rev = 1 if fl & 16 else 0
        so, lq = int(rec["seq_off"][r]), int(rec["l_qseq"][r])
        for p in range(max(beg, start), min(beg + x, end)):
            off = p - beg
            k = next(i for i in range(len(ops)) if xend[i] > off)
            op, l = ops[k], lens[k]
            covered[p - start] = True
            if op == 3:
                continue
            indel = 0
            if off == xend[k] - 1 and k + 1 < len(ops):
                o2 = ops[k + 1]
                if o2 == 2 and op != 2:
                    j = k + 1
                    while j < len(ops) and ops[j] == 2:
                        indel -= lens[j]
                        j += 1
                elif o2 == 1:
                    j = k + 1
                    while j < len(ops) and ops[j] in (1, 6):
                        if ops[j] == 1:
                            indel += lens[j]
                        j += 1
                elif o2 == 6 and k + 2 < len(ops):
                    j = k + 2
                    while j < len(ops) and ops[j] not in REFC:
                        if ops[j] == 1:
                            indel += lens[j]
                        j += 1
            is_del = op == 2
            qpos = y0[k] if is_del else y0[k] + (off - (xend[k] - l))
            c = p - start
            if indel < 0:
                dels[c][(rev, -indel)] = dels[c].get((rev, -indel), 0) + 1
                alle[c].setdefault((0, rev, -indel, None), [r, 0, 0])[2] += 1
            bi = (17 if rev else 8) if is_del else N2C[_nib(rec["seq"], so, lq, qpos) + 16 * rev]
            depth[c] += 1
            if bi >= 0:
                cnt[c, bi] += 1
            else:
                quirk[c] += 1
            if indel > 0:
                f0 = 0 if is_del else 1
                s = tuple(_nib(rec["seq"], so, lq, qpos + f0 + i) for i in range(indel))
                ins[c][(rev, s)] = ins[c].get((rev, s), 0) + 1
                alle[c].setdefault((1, rev, indel, s), [r, qpos + f0, 0])[2] += 1
                ins_last[c] = r
    rows, major, stats, alleles, last = [], [], [], [], []
    prev_emitted = None
    for c in range(W):
        if not covered[c]:
            continue
        p = start + c
        m = cnt[c].copy()
        for rev, (fa, fb) in ((0, (6, 7)), (1, (15, 16))):
            v = [x for (s, _), x in dels[c].items() if s == rev]
            m[fa], m[fb] = sum(v), max(v, default=0)
        for rev, (fa, fb) in ((0, (4, 5)), (1, (13, 14))):
            v = [x for (s, _), x in ins[c].items() if s == rev]
            m[fa], m[fb] = sum(v), max(v, default=0)
        del_count, ins_count = int(m[6] + m[15]), int(m[4] + m[13])
        off = p - ref_start
        rb = ref_seq[off].upper() if 0 <= off < len(ref_seq) else "N"
        bi = ord(rb) - 65
        rf = B2I[bi] if 0 <= bi < 32 else 0
        fsum, rsum = int(m[0:4].sum()), int(m[9:13].sum())
        ref_count = alt = 0
        major_alt = "\0"
        for i in range(4):
            if i == rf:
                ref_count = int(m[i] + m[i + 9])
            else:
                cc = int(m[i] + m[i + 9])
                if cc > alt:
                    alt, major_alt = cc, "ACGT"[i]
        m[rf], m[rf + 9] = -fsum, -rsum
        d = max(1, int(depth[c]))
        f32 = np.float32
        snp = f32(alt) / f32(d) >= f32(min_snp_af)
        if call_snp_only:
            ok = snp
        else:
            ok = (ref_count < alt or ref_count < ins_count or ref_count < del_count
                  or (ref_count > 0 and ref_count == alt and ord(rb) - ord(major_alt) < 0) or snp
                  or f32(del_count) / f32(d) >= f32(min_indel_af) or f32(ins_count) / f32(d) >= f32(min_indel_af))
        ok = ok and d >= min_depth and rb in "ACGT"
        if not call_ht:
            lo = p - 16
            ok = ok and lo >= max(start, 1) and bool(covered[lo - start:c].all())
        if quirk[c] and rows:
            rows[-1][17] += quirk[c]
        rows.append(m)
        major.append(p)
        alleles.append([((k[0] << 31) | (k[1] << 30) | k[2], v[0], v[1], v[2]) for k, v in alle[c].items()])
        last.append(int(ins_last[c]))
        stats.append([d, ref_count, alt, del_count, ins_count, 1 if ok else 0])
    matrix = np.array(rows, np.int64).reshape(-1, 18)
    stats = np.array(stats, np.int32).reshape(-1, 6)
    if len(stats):
        stats[:, 5] |= np.where((matrix == 0).all(axis=1), 2, 0).astype(np.int32)
    major = np.array(major, np.int64)
    cand = np.nonzero(stats[:, 5] & 1)[0].astype(np.int64) if len(stats) else np.zeros(0, np.int64)
    okw, bounds = [], []
    for c in cand:            # preprocess/CreateTensorPileupFromCffi.py:356-396 (see oracle/pileup_oracle.c)
        lo, hi = c, c
        while lo > max(c - 16, 0) and major[lo - 1] == major[lo] - 1:
            lo -= 1
        while hi < min(c + 18, len(major) - 1) and major[hi + 1] == major[hi] + 1:
            hi += 1
        if lo == c - 16 and hi == c + 18:
            g = not (stats[c - 16:c + 17, 5] & 2).any()
        else:
            g = call_ht and hi > c and (lo == c - 16 or hi >= c + 16)
        okw.append(1 if g else 0)
        bounds.append((lo, min(hi, c + 16) + 1))
    return {"matrix": matrix, "major": major, "stats": stats, "cand_cols": cand, "cand_ok": np.array(okw, np.uint8),
            "window_bounds": np.array(bounds, np.int64).reshape(-1, 2),
            "alleles": alleles,        # per emitted column: (meta, first read, query offset, count) as c3b_plp_fetch_alleles exports them
            "ins_last": np.array(last, np.int64)}
