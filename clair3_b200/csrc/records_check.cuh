// records_check.cuh - the check of a run of alignment records (c3b_bam_records, c3b_fa_records' optional fields) that every
// consumer's record intake makes before any kernel indexes through an offset: exactly the conditions BamRecords
// (clair3_b200/records.py) enforces on the host.  __host__ __device__: intake runs it on the host for host records and as
// records_check_kernel (c3b_api.cu) for device records, and tests/records_check_host.cpp builds it for the host with
// AddressSanitizer and UBSan.
//
// It reads the n_reads per-read entries of pos and l_qseq and the n_reads + 1 entries of each offset array, never a value array,
// so it stays in range whatever the offsets hold.  A fault is a 64-bit key, reason << 40 | read: the smallest key of a run is
// the first condition BamRecords tests that fails, at the first read that fails it, and the device check min-reduces it.
#pragma once
#include <stdint.h>

#include "../../include/clair3_b200_fa.h"

#ifndef C3B_HD
#if defined(__CUDACC__)
#define C3B_HD __host__ __device__ __forceinline__
#else
#define C3B_HD inline
#endif
#endif

// The reasons, in the order BamRecords tests them.
enum {
    C3B_REC_CIGAR_SPAN = 1,     // cigar_off[0] != 0 or cigar_off[n] != n_cigar
    C3B_REC_SEQ_SPAN,           // seq_off[0] != 0 or seq_off[n] != n_seq
    C3B_REC_CIGAR_DEC,          // cigar_off decreases
    C3B_REC_SEQ_DEC,            // seq_off decreases
    C3B_REC_POS,                // pos decreases
    C3B_REC_SEQ_SHORT,          // seq_off[i + 1] - seq_off[i] < (l_qseq + 1) / 2
    C3B_REC_QUAL_PAIR,          // qual without qual_off or qual_off without qual
    C3B_REC_QUAL_OFF,           // qual_off not non-decreasing from 0 to n_qual
    C3B_REC_QUAL_LEN,           // qual_off[i + 1] - qual_off[i] != l_qseq
    C3B_REC_QNAME_PAIR,
    C3B_REC_QNAME_OFF,
    C3B_REC_MV_PAIR,
    C3B_REC_MV_OFF,
    C3B_REC_REASONS
};
#define C3B_REC_OK (~0ull)

// What the check reads: the per-read arrays, the offset arrays (cigar, seq, qual, qname, mv; null = absent) and the length of
// each value array.
struct C3bRecordsView {
    int64_t n;
    const int64_t *pos;
    const int32_t *l_qseq;
    const int64_t *off[5];
    int64_t len[5];
};

inline C3bRecordsView c3b_records_view(const c3b_bam_records *core, const c3b_fa_records *opt) {
    C3bRecordsView v = {core->n_reads, core->pos, core->l_qseq, {core->cigar_off, core->seq_off}, {core->n_cigar, core->n_seq}};
    if (opt) {
        v.off[2] = opt->qual_off; v.len[2] = opt->n_qual;
        v.off[3] = opt->qname_off; v.len[3] = opt->n_qname;
        v.off[4] = opt->mv_off; v.len[4] = opt->n_mv;
    }
    return v;
}

C3B_HD uint64_t c3b_records_key(int reason, int64_t read) { return (uint64_t)reason << 40 | (uint64_t)read; }

// The pairing of the optional fields: an offset array without its values or values without their offsets.
inline uint64_t c3b_records_pairs(const c3b_fa_records *opt) {
    if (!opt) return C3B_REC_OK;
    if (!opt->qual != !opt->qual_off) return c3b_records_key(C3B_REC_QUAL_PAIR, 0);
    if (!opt->qname != !opt->qname_off) return c3b_records_key(C3B_REC_QNAME_PAIR, 0);
    if (!opt->mv != !opt->mv_off) return c3b_records_key(C3B_REC_MV_PAIR, 0);
    return C3B_REC_OK;
}

// The smallest fault key that entry i (0 <= i <= n) of the offset arrays and read i (i < n) show; C3B_REC_OK for none.  The core
// fields are checked only when there are reads, the optional ones always, as BamRecords does.  Differences of offsets wrap as
// numpy's do: a run whose offsets could overflow one already fails an earlier reason.
C3B_HD uint64_t c3b_records_fault_at(const C3bRecordsView &v, int64_t i) {
    const int span[5] = {C3B_REC_CIGAR_SPAN, C3B_REC_SEQ_SPAN, C3B_REC_QUAL_OFF, C3B_REC_QNAME_OFF, C3B_REC_MV_OFF};
    const int dec[5] = {C3B_REC_CIGAR_DEC, C3B_REC_SEQ_DEC, C3B_REC_QUAL_OFF, C3B_REC_QNAME_OFF, C3B_REC_MV_OFF};
    const int64_t n = v.n, last = n > 0 ? n - 1 : 0;
    uint64_t key = C3B_REC_OK;
    auto hit = [&](int reason, int64_t read) {
        const uint64_t k = c3b_records_key(reason, read);
        if (k < key) key = k;
    };
    for (int f = 0; f < 5; ++f) {
        const int64_t *o = v.off[f];
        if (!o || (f < 2 && n == 0)) continue;
        if (i == 0 && o[0] != 0) hit(span[f], 0);
        if (i == n && o[n] != v.len[f]) hit(span[f], last);
        if (i > 0 && o[i] < o[i - 1]) hit(dec[f], i - 1);
    }
    if (i < n) {
        if (i > 0 && v.pos[i] < v.pos[i - 1]) hit(C3B_REC_POS, i);
        const int64_t lq = v.l_qseq[i];
        const int64_t bytes = (int64_t)((uint64_t)v.off[1][i + 1] - (uint64_t)v.off[1][i]);
        if (((lq + 1) >> 1) > bytes) hit(C3B_REC_SEQ_SHORT, i);        // floor division, as numpy's //
        if (v.off[2] && (int64_t)((uint64_t)v.off[2][i + 1] - (uint64_t)v.off[2][i]) != lq) hit(C3B_REC_QUAL_LEN, i);
    }
    return key;
}

// The whole check on the host: the pairing and every entry.  The entries are checked whatever the pairing: an offset array
// without values is still read only within its n + 1 entries.
inline uint64_t c3b_records_check(const c3b_bam_records *core, const c3b_fa_records *opt) {
    uint64_t key = c3b_records_pairs(opt);
    const C3bRecordsView v = c3b_records_view(core, opt);
    for (int64_t i = 0; i <= v.n; ++i) {
        const uint64_t k = c3b_records_fault_at(v, i);
        if (k < key) key = k;
    }
    return key;
}

// The field a fault names and what is wrong with it.
inline const char *c3b_records_fault_text(uint64_t key) {
    static const char *const text[C3B_REC_REASONS] = {
        "",
        "cigar_off does not run from 0 to n_cigar",
        "seq_off does not run from 0 to n_seq",
        "cigar_off decreases",
        "seq_off decreases",
        "pos is below the previous read's (records must be sorted by pos)",
        "seq holds fewer than (l_qseq + 1) / 2 bytes",
        "qual and qual_off go together",
        "qual_off does not run from 0 to n_qual without decreasing",
        "qual holds other than l_qseq base qualities",
        "qname and qname_off go together",
        "qname_off does not run from 0 to n_qname without decreasing",
        "mv and mv_off go together",
        "mv_off does not run from 0 to n_mv without decreasing",
    };
    const uint64_t r = key >> 40;
    return r > 0 && r < C3B_REC_REASONS ? text[r] : "unknown fault";
}

C3B_HD int64_t c3b_records_fault_read(uint64_t key) { return (int64_t)(key & ((1ull << 40) - 1)); }
