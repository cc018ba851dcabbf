// fa_tensor.cu - the full-alignment tensor builder on the GPU (include/clair3_b200_fa.h; SURVEY.md 8f row N4, full-alignment half).
//
// Reference: calculate_clair3_full_alignment(), HKU-BAL/Clair3 src/clair3_full_alignment_dwell.c:437-1054 - one pass over the
// reads with a khash lookup per (read, position), then one pass per candidate over all kept reads, a glibc-rand() shuffle and a
// qsort.  Here:
//
//   K1 fa_flank_count / K2 fa_flank_fill   the sorted, de-duplicated union F of the candidate windows [c-16, c+16] (clipped at
//                        0).  Candidates ascend, so the union is a concatenation and flanking index = position order (:501-533).
//   K3 fa_read_scan      one thread per read: filter (flag & 2316, mapq < min_mq), read_end (M D N = X), the run of F inside
//                        [pos, read_end) by two binary searches, and the read's name into an open-addressing hash table whose
//                        slots keep the smallest record index of each name (exact byte compare, atomicMin).
//   K4 fa_read_keep      first-of-name test (a read without overlap still claims its name, :547-626) and overlap > 0.
//   K5 fa_read_compact   kept reads in file order (the reference's read_array; the compacted index is its read_index).
//   K6 fa_signal         (dwell) per-base signal lengths from the mv tag (:20-74) into a per-kept-read pool.
//   K7 fa_haplotag       (haplotagging) one thread per kept read with mapq >= 20: haplotag_read / realign_read /
//                        cigar_prefix_length restated literally (:158-422); Levenshtein on one DP row over the <= 22-base
//                        reference side; per-phase-set costs in a small per-thread list.
//   K8 fa_pos_info       one thread per kept read: the CIGAR walk of :654-765 writing the read's Pos_info run (alt code or -1,
//                        bq, deletion length, insertion query offset + length, dwell signal) with the same overwrite order.
//   K9 fa_select_count   one warp per candidate: the kept reads with read_start < c+17 and read_end > c-16 (prefix max of the
//                        read ends bounds the search); their number decides the shuffle and its rand() draws.
//   K10 (block_scan)     draw offset of every candidate = prefix sum of n-1 over earlier shuffling candidates.  The same
//                        one-CTA scan (block_scan.cuh) sizes F, numbers the kept reads and lays out their pools, and takes the
//                        running maximum of the kept reads' ends.
//   K11 fa_candidate     one CTA per candidate: counters over ALL kept reads on the candidate (depth, A/C/G/T, distinct
//                        deletion lengths and insertion strings in first-occurrence order, exported for the text stage),
//                        Fisher-Yates with the glibc TYPE_3 stream generated at the candidate's offset (jump-ahead by
//                        precomputed matrix powers: the stream is linear mod 2^32), rank sort by (haplotype, index), padding,
//                        and the int8 [depth][33][C] block in Clair3_F's wire layout.
//
// Bound: latency of dependent global loads (integer work, no tensor cores).  Bytes per call: the records once per pass (K3, K7,
// K8), 20 B of Pos_info per (kept read, flanking position) written once and read by K11, and the matrix (depth x 33 x C B per
// candidate) written once.  DESIGN.md 5b.
//
// The all_alt_info text is a second stage (fa_alt_text.cu, c3b_fa_alt_text) that reads K11's export where the build left it.
#include <limits.h>
#include <stdlib.h>

#include <vector>

#include "block_scan.cuh"
#include "c3b_internal.h"
#include "../../include/clair3_b200_fa.h"

namespace {

constexpr int FLANK = 16;           // flanking_base_num, src/clair3_full_alignment_dwell.h:22
constexpr int NPOS = 33;            // no_of_positions
constexpr int MAXSEL = 1536;        // reads overlapping one candidate window that K11 can hold
constexpr int CAND_THREADS = 256;
constexpr int MAX_PS = 64;          // distinct phase sets one read may touch (K7)
constexpr int MAX_OVERWRITTEN = 64; // insertions on one candidate that a later insertion of the same read and anchor overwrote (K11)
constexpr int JUMP_BITS = 63;       // rand() offsets below 2^63

struct PosInfo {                    // Pos_info (src/clair3_full_alignment_dwell.h:138-146); alt 0 = not covered by M / D
    int8_t alt;                     // nt16 code, -1 deleted
    int8_t bq;
    int16_t n_ins;                  // insertion operations anchored on this base (2I1I, 1I1P1I: 2); ins_q / ins_len hold the last
    int32_t del_len;
    int32_t ins_q;
    int32_t ins_len;
    int32_t sig;
};

struct Kept {                       // per kept read, compacted in file order
    int64_t *orig;                  // record index
    int64_t *start, *end, *pmax;    // read_start, read_end, running max of read_end
    int64_t *fs;                    // index in F of the first flanking position >= read_start (flanking_start)
    int32_t *ov;                    // overlap_candidates_num
    int64_t *pi;                    // first Pos_info of the read in the pool
    int64_t *sig;                   // first per-base signal of the read in the signal pool, -1 = none
    int32_t *hap;
};

__device__ __forceinline__ int nib(const uint8_t *sq, int64_t i) { return (sq[i >> 1] >> ((~i & 1) << 2)) & 15; }

__device__ __constant__ char NT16[17] = "=ACMGRSVTWYHKDBN";

// num2countbase_fa (src/clair3_full_alignment_dwell.h:39-44) indexed by (char - 'A'); 0 outside 'A'..'`'
__device__ __forceinline__ int8_t fa_val(char ch) {
    switch (ch) {
    case 'A': return 100; case 'C': return 25; case 'D': return -100; case 'G': return 75; case 'I': return -50;
    case 'N': return 100; case 'T': return 50; default: return 0;
    }
}
// acgt2num (:49-54): C 1, G 2, T 3, anything else 0
__device__ __forceinline__ int acgt_idx(char ch) { return ch == 'C' ? 1 : ch == 'G' ? 2 : ch == 'T' ? 3 : 0; }
__device__ __forceinline__ char upper(char c) { return (c >= 'a' && c <= 'z') ? (char)(c - 32) : c; }

__device__ __forceinline__ int64_t lower_bound64(const int64_t *a, int64_t lo, int64_t hi, int64_t v) {
    while (lo < hi) {
        const int64_t m = (lo + hi) >> 1;
        if (a[m] < v) lo = m + 1; else hi = m;
    }
    return lo;
}

__device__ __forceinline__ bool ref_op(uint32_t op) { return op == 0 || op == 2 || op == 3 || op == 7 || op == 8; }

// ---------------------------------------------------------------------------------------------------------------- K1 / K2
// n_dev: with device candidates, the launch covers the capacity and the count is read here; slots past it add nothing to F.
__global__ void fa_flank_count_kernel(const int64_t *__restrict__ cand, int64_t n_cand, const int64_t *__restrict__ n_dev,
                                      int64_t *__restrict__ fstart, int64_t *__restrict__ fcnt) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_cand) return;
    if (n_dev && k >= *n_dev) { fcnt[k] = 0; return; }
    const int64_t c = cand[k];
    const int64_t lo = c - FLANK < 0 ? 0 : c - FLANK;
    const int64_t prev_hi = k > 0 ? cand[k - 1] + FLANK : -1;
    const int64_t s = lo > prev_hi + 1 ? lo : prev_hi + 1;
    fstart[k] = s;
    fcnt[k] = c + FLANK - s + 1;
}

__global__ void fa_flank_fill_kernel(const int64_t *__restrict__ fstart, const int64_t *__restrict__ fcnt,
                                     const int64_t *__restrict__ foff, int64_t n_cand, const int64_t *__restrict__ n_dev,
                                     int64_t *__restrict__ F) {
    const int64_t k = blockIdx.x;
    if (k >= n_cand || (n_dev && k >= *n_dev)) return;
    for (int64_t i = threadIdx.x; i < fcnt[k]; i += blockDim.x) F[foff[k] + i] = fstart[k] + i;
}

// K0 (device candidates): candidates[first .. first + n) into the workspace, n = the device count less first, clipped to
// [0, cap]; n and the device count go to counters 10 / 11, which the first sizing wait reads.  The host path's checks stay:
// a position that is negative, at or above 2^31 - 17, or not above its predecessor sets status bit 16.
__global__ void fa_cand_intake_kernel(const int64_t *__restrict__ cand, const int64_t *__restrict__ n_total, int64_t first,
                                      int64_t cap, int64_t *__restrict__ out, int64_t *__restrict__ cnt, int *status) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t n = *n_total - first;
    n = n < 0 ? 0 : n > cap ? cap : n;
    if (k == 0) { cnt[10] = n; cnt[11] = *n_total; }
    if (k >= n) return;
    const int64_t c = cand[first + k];
    out[k] = c;
    if (c < 0 || c >= (int64_t)INT_MAX - FLANK || (k > 0 && c <= cand[first + k - 1])) atomicOr(status, 16);
}

// ---------------------------------------------------------------------------------------------------------------- K3 / K4
__device__ __forceinline__ uint32_t name_hash(const uint8_t *s, int64_t n) {
    uint32_t h = 2166136261u;                       // FNV-1a
    for (int64_t i = 0; i < n; ++i) h = (h ^ s[i]) * 16777619u;
    return h;
}

__device__ __forceinline__ bool same_name(const C3bReads &R, int64_t a, int64_t b) {
    const int64_t a0 = R.qname_off[a], la = R.qname_off[a + 1] - a0, b0 = R.qname_off[b], lb = R.qname_off[b + 1] - b0;
    if (la != lb) return false;
    for (int64_t i = 0; i < la; ++i)
        if (R.qname[a0 + i] != R.qname[b0 + i]) return false;
    return true;
}

__global__ void fa_read_scan_kernel(C3bReads R, int min_mq, const int64_t *__restrict__ F, int64_t nF, int64_t *__restrict__ rend,
                                    int64_t *__restrict__ rlo, int32_t *__restrict__ rov, uint8_t *__restrict__ pass,
                                    int64_t *__restrict__ table, uint32_t tmask) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R.n) return;
    const bool ok = !(R.flag[r] & 2316) && (int)R.mapq[r] >= min_mq;      // SAMTOOLS_VIEW_FILTER_FLAG, :539-545
    pass[r] = ok ? 1 : 0;
    const int64_t p = R.pos[r];
    int64_t e = p;
    for (int64_t k = R.cigar_off[r]; k < R.cigar_off[r + 1]; ++k) {
        const uint32_t c = R.cigar[k];
        if (ref_op(c & 15u)) e += (int64_t)(c >> 4);
    }
    rend[r] = e;
    const int64_t lo = lower_bound64(F, 0, nF, p);
    const int64_t hi = lower_bound64(F, lo, nF, e);
    rlo[r] = lo;
    rov[r] = (int32_t)(hi > lo ? hi - lo : 0);
    if (!ok || !R.qname_off) return;
    const int64_t n0 = R.qname_off[r];
    uint32_t i = name_hash(R.qname + n0, R.qname_off[r + 1] - n0) & tmask;
    for (uint32_t step = 1;; ++step) {
        unsigned long long *slot = reinterpret_cast<unsigned long long *>(table + i);
        const long long cur = (long long)atomicCAS(slot, (unsigned long long)-1ll, (unsigned long long)r);
        if (cur == -1) return;
        if (same_name(R, cur, r)) {
            atomicMin(reinterpret_cast<long long *>(slot), (long long)r);
            return;
        }
        i = (i + step) & tmask;
    }
}

__global__ void fa_read_keep_kernel(C3bReads R, const uint8_t *__restrict__ pass, const int32_t *__restrict__ rov,
                                    const int64_t *__restrict__ table, uint32_t tmask, int64_t *__restrict__ keep,
                                    int64_t *__restrict__ kov) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R.n) return;
    bool k = pass[r] && rov[r] > 0;
    if (k && R.qname_off) {
        const int64_t n0 = R.qname_off[r];
        uint32_t i = name_hash(R.qname + n0, R.qname_off[r + 1] - n0) & tmask;
        for (uint32_t step = 1;; ++step) {
            const int64_t cur = table[i];
            if (cur == r || cur < 0) break;
            if (same_name(R, cur, r)) { k = false; break; }
            i = (i + step) & tmask;
        }
    }
    keep[r] = k ? 1 : 0;
    kov[r] = k ? rov[r] : 0;
}

// ---------------------------------------------------------------------------------------------------------------- K5
__global__ void fa_read_compact_kernel(C3bReads R, int dwell, const int64_t *__restrict__ keep, const int64_t *__restrict__ kidx,
                                       const int64_t *__restrict__ kov_ex, const int64_t *__restrict__ rend,
                                       const int64_t *__restrict__ rlo, const int32_t *__restrict__ rov, Kept K,
                                       int64_t *__restrict__ sig_len) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R.n || !keep[r]) return;
    const int64_t k = kidx[r];
    K.orig[k] = r;
    K.start[k] = R.pos[r];
    K.end[k] = rend[r];
    K.fs[k] = rlo[r];
    K.ov[k] = rov[r];
    K.pi[k] = kov_ex[r];
    K.hap[k] = 0;
    // compute_signal_lengths_from_mv_tag returns NULL for no tag, <= 1 element or l_qseq 0 (:25-35)
    const bool has = dwell && R.mv_off && R.mv_off[r + 1] - R.mv_off[r] > 1 && R.l_qseq[r] > 0;
    sig_len[k] = has ? R.l_qseq[r] : 0;
}

// ---------------------------------------------------------------------------------------------------------------- K6
__global__ void fa_signal_kernel(C3bReads R, Kept K, const int64_t *__restrict__ sig_len, const int64_t *__restrict__ sig_ex,
                                 int64_t n_kept, int32_t *__restrict__ sig) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_kept) return;
    if (!sig_len[k]) { K.sig[k] = -1; return; }
    const int64_t r = K.orig[k], off = sig_ex[k];
    K.sig[k] = off;
    const int64_t L = R.l_qseq[r];
    const bool rev = (R.flag[r] & 16) != 0;
    const int32_t *mv = R.mv + R.mv_off[r];
    const int64_t n = R.mv_off[r + 1] - R.mv_off[r];
    int64_t b = -1;
    for (int64_t i = 1; i < n; ++i) {                // :41-61
        if (mv[i] != 0) {
            if (++b >= L) break;
        } else if (b < 0) {
            continue;
        }
        sig[off + (rev ? L - 1 - b : b)] += 1;       // the reverse strand's array is flipped (:63-71)
    }
}

// ---------------------------------------------------------------------------------------------------------------- K7
struct HapArgs {
    C3bReads R;
    Kept K;
    int64_t n_kept;
    const c3b_fa_variant *var;
    int64_t n_var;
    const char *ref;
    int64_t ref_start, ref_len;
    int *status;
};

// cigar_prefix_length (:158-205); leaves ref_bases / query_bases untouched when the CIGAR runs out first
__device__ void cigar_prefix_length(const uint32_t *cig, uint64_t reference_bases, uint64_t &ref_bases, uint64_t &query_bases,
                                    uint64_t left, uint64_t right, uint64_t consumed, bool reverse) {
    uint64_t ref_pos = 0, query_pos = 0;
    for (uint64_t i = left; i < right; ++i) {
        const uint64_t index = reverse ? left + right - i - 1 : i;
        const uint32_t op = cig[index] & 15u;
        uint64_t length = cig[index] >> 4;
        length = i == left ? consumed : length;
        if (length == 0) continue;
        if (op == 0 || op == 7 || op == 8) {
            query_pos += length;
            ref_pos += length;
            if (ref_pos >= reference_bases) {
                ref_bases = reference_bases;
                query_bases = query_pos + reference_bases - ref_pos;
                return;
            }
        } else if (op == 2) {
            ref_pos += length;
            if (ref_pos >= reference_bases) {
                ref_bases = reference_bases;
                query_bases = query_pos;
                return;
            }
        } else if (op == 1) {
            query_pos += length;
        } else if (op == 3) {
            ref_bases = reference_bases;
            query_bases = query_pos;
            return;
        }
    }
}

constexpr int OVERHANG = 10;                 // overhang, src/clair3_full_alignment_dwell.h:19
constexpr int RMAX = 2 * OVERHANG + 3;       // longest reference / alt string of realign_read (+1 for the appended alt base)

// Levenshtein distance between the query (read bases [qst, qen)) and a short string b: one DP row over b.
__device__ int levenshtein_q(const uint8_t *sq, uint64_t qst, uint64_t qen, const char *b, int bl) {
    const uint64_t al = qen - qst;
    if (al == 0) return bl;
    if (bl == 0) return (int)al;
    int row[RMAX + 1];
    for (int j = 0; j <= bl; ++j) row[j] = j;
    for (uint64_t i = 1; i <= al; ++i) {
        const char ca = NT16[nib(sq, (int64_t)(qst + i - 1))];
        int diag = row[0];
        row[0] = (int)i;
        for (int j = 1; j <= bl; ++j) {
            const int up = row[j];
            int v = diag + (ca == b[j - 1] ? 0 : 1);
            if (up + 1 < v) v = up + 1;
            if (row[j - 1] + 1 < v) v = row[j - 1] + 1;
            row[j] = v;
            diag = up;
        }
    }
    return row[bl];
}

// realign_read (:262-313)
__device__ int realign_read(const HapArgs &A, const c3b_fa_variant &v, const uint32_t *cig, uint64_t n_cigar, const uint8_t *sq,
                            uint64_t i, uint64_t consumed, uint64_t query_pos) {
    const uint64_t middle_length = cig[i] >> 4;
    const uint64_t left_consumed = consumed > 0 ? consumed : 0;
    const uint64_t right_consumed = consumed < middle_length ? middle_length - consumed : 0;
    uint64_t lrb = 0, lqb = 0, rrb = 0, rqb = 0;
    cigar_prefix_length(cig, OVERHANG, lrb, lqb, 0, i + 1, left_consumed, true);
    cigar_prefix_length(cig, OVERHANG + 1, rrb, rqb, i, n_cigar, right_consumed, false);
    const uint64_t qst = query_pos - lqb, qen = query_pos + rqb;
    if (qen == qst) return 0;
    const int64_t rst = (int64_t)v.position - (int64_t)lrb - A.ref_start;
    const int64_t ren = (int64_t)v.position + (int64_t)rrb - A.ref_start;
    // get_ref_seq copies with strncpy: it stops at the end of the fetched reference
    char ref[RMAX], alt[RMAX];
    int rl = 0;
    for (int64_t p = rst; p < ren && rl < RMAX - 1; ++p) {
        if (p < 0 || p >= A.ref_len) break;
        ref[rl++] = A.ref[p];
    }
    for (int j = 0; j < rl; ++j) alt[j] = ref[j];
    int al = rl;
    if ((int64_t)lrb < rl) alt[lrb] = v.alt_base;
    else if ((int64_t)lrb == rl) alt[al++] = v.alt_base;       // right_ref_bases == 0: alt[left_ref_bases] appends
    const int dr = levenshtein_q(sq, qst, qen, ref, rl);
    const int da = levenshtein_q(sq, qst, qen, alt, al);
    return dr < da ? 1 : dr > da ? 2 : 0;
}

__global__ void fa_haplotag_kernel(HapArgs A) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= A.n_kept) return;
    const int64_t r = A.K.orig[k];
    if ((int)A.R.mapq[r] < 20) return;                                    // min_haplotag_mq
    const uint32_t *cig = A.R.cigar + A.R.cigar_off[r];
    const uint64_t n_cigar = (uint64_t)(A.R.cigar_off[r + 1] - A.R.cigar_off[r]);
    const uint8_t *sq = A.R.seq + A.R.seq_off[r];
    int ps_key[MAX_PS], ps_val[MAX_PS], nps = 0;
    const uint64_t n = (uint64_t)A.n_var;
    uint64_t ref_pos = (uint64_t)A.R.pos[r], query_pos = 0, v_position = 0;
    // variant_current_pos after the reads before this one, then the skip of :329-330: the first variant at or after read_start
    uint64_t j = 0, hi = n;
    while (j < hi) {
        const uint64_t m = (j + hi) >> 1;
        if ((uint64_t)(int64_t)A.var[m].position < ref_pos) j = m + 1; else hi = m;
    }
    auto cost = [&](int allele, const c3b_fa_variant &v) {             // update_haplotype_cost (:246-260)
        if (allele == 0) return;
        const int d = allele == v.genotype ? 1 : -1;
        for (int t = 0; t < nps; ++t)
            if (ps_key[t] == v.phase_set) { ps_val[t] += d; return; }
        if (nps == MAX_PS) { atomicOr(A.status, 4); return; }
        ps_key[nps] = v.phase_set;
        ps_val[nps++] = d;
    };
    for (uint64_t i = 0; i < n_cigar; ++i) {
        const uint32_t op = cig[i] & 15u;
        const uint64_t length = cig[i] >> 4;
        if (j < n) v_position = (uint64_t)(int64_t)A.var[j].position;
        if (op == 0 || op == 7 || op == 8) {
            while (j < n && v_position < ref_pos + length) {
                cost(realign_read(A, A.var[j], cig, n_cigar, sq, i, v_position - ref_pos, query_pos + v_position - ref_pos), A.var[j]);
                ++j;
                if (j < n) v_position = (uint64_t)(int64_t)A.var[j].position;
            }
            query_pos += length;
            ref_pos += length;
        } else if (op == 1) {
            if (j < n && v_position == ref_pos) {
                cost(realign_read(A, A.var[j], cig, n_cigar, sq, i, 0, query_pos), A.var[j]);
                ++j;
                if (j < n) v_position = (uint64_t)(int64_t)A.var[j].position;
            }
            query_pos += length;
        } else if (op == 2) {
            while (j < n && v_position < ref_pos + length) {
                cost(realign_read(A, A.var[j], cig, n_cigar, sq, i, v_position - ref_pos, query_pos), A.var[j]);
                ++j;
                if (j < n) v_position = (uint64_t)(int64_t)A.var[j].position;
            }
            ref_pos += length;
        } else if (op == 3) {
            while (j < n && v_position < ref_pos + length) {
                ++j;
                if (j < n) v_position = (uint64_t)(int64_t)A.var[j].position;
            }
            ref_pos += length;
        } else if (op == 4) {
            query_pos += length;
        }
    }
    int mx = 0, mn = 0;
    for (int t = 0; t < nps; ++t) {
        if (ps_val[t] > mx) mx = ps_val[t];
        if (ps_val[t] < mn) mn = ps_val[t];
    }
    A.K.hap[k] = (nps == 0 || (mx == 0 && mn == 0)) ? 0 : (mx > (mn < 0 ? -mn : mn) ? 1 : 2);
}

// ---------------------------------------------------------------------------------------------------------------- K8
__device__ __forceinline__ int8_t norm_bq(int q) { return (int8_t)(int)(q < 40 ? 100 * q / 40.0 : 100); }   // normalize_bq

__global__ void fa_pos_info_kernel(C3bReads R, Kept K, int64_t n_kept, const int64_t *__restrict__ F, const int32_t *__restrict__ sig,
                                   PosInfo *__restrict__ pool) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_kept) return;
    const int64_t r = K.orig[k];
    const uint32_t *cig = R.cigar + R.cigar_off[r];
    const int64_t nc = R.cigar_off[r + 1] - R.cigar_off[r];
    const uint8_t *sq = R.seq + R.seq_off[r];
    const uint8_t *ql = R.qual_off ? R.qual + R.qual_off[r] : nullptr;
    const int64_t lq = R.l_qseq[r];
    const int64_t fs = K.fs[k], fe = fs + K.ov[k];
    const int32_t *sg = K.sig[k] >= 0 ? sig + K.sig[k] : nullptr;
    PosInfo *pi = pool + K.pi[k] - fs;              // pi[flanking index]
    int64_t ref_pos = K.start[k], query_pos = 0, cur = fs;
    auto find = [&](int64_t p) -> int64_t {         // flanking index of p inside the read's run, or -1
        const int64_t i = lower_bound64(F, fs, fe, p);
        return (i < fe && F[i] == p) ? i : -1;
    };
    for (int64_t i = 0; i < nc; ++i) {
        const uint32_t op = cig[i] & 15u;
        const int64_t length = cig[i] >> 4;
        if (op == 0 || op == 7 || op == 8) {
            while (cur < fe && F[cur] < ref_pos) ++cur;
            for (; cur < fe && F[cur] < ref_pos + length; ++cur) {
                const int64_t q = query_pos + (F[cur] - ref_pos);
                PosInfo &e = pi[cur];
                e.alt = (int8_t)nib(sq, q);
                e.bq = norm_bq(ql ? ql[q] : 255);
                if (sg && q < lq) e.sig = sg[q];
            }
            query_pos += length;
            ref_pos += length;
        } else if (op == 2) {
            const int64_t a = find(ref_pos - 1);
            if (a >= 0) pi[a].del_len = (int32_t)length;
            while (cur < fe && F[cur] < ref_pos) ++cur;
            for (; cur < fe && F[cur] < ref_pos + length; ++cur) pi[cur].alt = -1;
            ref_pos += length;
        } else if (op == 1) {
            const int64_t a = find(ref_pos - 1);
            if (a >= 0) {
                pi[a].ins_q = (int32_t)query_pos;
                pi[a].ins_len = (int32_t)length;
                if (pi[a].n_ins < SHRT_MAX) ++pi[a].n_ins;
                if (sg) {
                    int32_t s = 0;
                    for (int64_t t = 0; t < length; ++t)
                        if (query_pos + t < lq) s += sg[query_pos + t];
                    pi[a].sig += s;
                }
            }
            query_pos += length;
        } else if (op == 3) {
            ref_pos += length;
        } else if (op == 4) {
            query_pos += length;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------- K9
__global__ void fa_select_count_kernel(const int64_t *__restrict__ cand, int64_t n_cand, Kept K, int64_t n_kept, int depth,
                                       int64_t *__restrict__ ra, int64_t *__restrict__ rb, int64_t *__restrict__ nsel,
                                       int64_t *__restrict__ draws) {
    const int lane = threadIdx.x & 31;
    const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= n_cand) return;
    const int64_t c = cand[w];
    // reads are sorted by start; pmax (running max of read_end) is non-decreasing
    int64_t a = 0, hi = n_kept;
    while (a < hi) {
        const int64_t m = (a + hi) >> 1;
        if (K.pmax[m] > c - FLANK) hi = m; else a = m + 1;
    }
    const int64_t b = lower_bound64(K.start, a, n_kept, c + FLANK + 1);
    int64_t cnt = 0;
    for (int64_t j = a + lane; j < b; j += 32) cnt += K.end[j] > c - FLANK ? 1 : 0;
#pragma unroll
    for (int d = 16; d; d >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
    if (lane == 0) {
        ra[w] = a;
        rb[w] = b;
        nsel[w] = cnt;
        // the reference's start_pos = candidate - 16 is a size_t: below 16 it wraps and no read is selected (:790, :810)
        const int64_t nm = c < FLANK ? 0 : cnt;
        draws[w] = nm > depth ? nm - 1 : 0;
    }
}

// ---------------------------------------------------------------------------------------------------------------- K11
struct CandArgs {
    C3bReads R;
    Kept K;
    const int64_t *cand;
    const int64_t *F;
    int64_t nF;
    const PosInfo *pool;
    const char *ref;
    int64_t ref_start, ref_len;
    const int64_t *ra, *rb, *nsel, *draw_off;
    int64_t rand_skip;
    const uint32_t *jump;         // [JUMP_BITS][31][31]: M^(2^b) of the TYPE_3 state recurrence
    const uint32_t *state0;       // [31] state at the first output after srand
    int depth, C;
    int8_t *matrix;
    int32_t *c_depth, *c_acgt, *al_off, *al_n;
    uint32_t *al_meta, *al_read, *al_qpos, *al_cnt;
    unsigned long long *al_used;
    int *status;
};

__device__ __forceinline__ bool same_ins(const C3bReads &R, const Kept &K, int64_t ka, int qa, int64_t kb, int qb, int len) {
    const uint8_t *sa = R.seq + R.seq_off[K.orig[ka]], *sb = R.seq + R.seq_off[K.orig[kb]];
    for (int t = 0; t < len; ++t)
        if (nib(sa, qa + t) != nib(sb, qb + t)) return false;
    return true;
}


// normalize_af(count / (float)depth) (.h:13, :926): the macro does not parenthesise its argument, so its `100 * x` is
// `100 * count / (float)depth` - (float)(100 count) / depth in float32, not 100 * (count / depth) (53 / 100: 53, not 52)
__device__ __forceinline__ int8_t norm_af(int64_t count, int depth) {
    const float x = __fdiv_rn((float)count, (float)depth);
    return (int8_t)(int)(x < 1.0f ? __fdiv_rn((float)(100 * count), (float)depth) : 100.0f);
}

__global__ void __launch_bounds__(CAND_THREADS) fa_candidate_kernel(CandArgs A) {
    __shared__ int32_t sel[MAXSEL];       // kept-read index of every read in the window, kept order
    __shared__ int32_t ord[MAXSEL];       // the same, shuffled (read_hap_array of :812-816)
    __shared__ int32_t ev_del[MAXSEL];    // deletion length anchored at the candidate, 0 none
    __shared__ int32_t ev_ins[MAXSEL];    // insertion length anchored at the candidate, 0 none
    __shared__ int32_t ev_q[MAXSEL];      // its query offset
    __shared__ int16_t ev_dcnt[MAXSEL];   // first occurrence of a deletion length: reads showing it, else 0
    __shared__ int16_t ev_icnt[MAXSEL];   // first occurrence of an insertion string: reads showing it, else 0
    __shared__ int32_t rows[256];         // kept-read index of every matrix row, -1 padding
    __shared__ int8_t row_af[256];
    __shared__ int8_t spill[256 * NPOS];  // channel 6 of every row
    // the insertions that Pos_info lost to a later one on the same read and anchor (2I1I, 1I1P1I): the reference's counter still
    // saw them (:746-752), before the kept one.  Sorted by read (stable: each read's run is in CIGAR order).
    __shared__ int32_t ow_i[MAX_OVERWRITTEN];       // index in sel
    __shared__ int32_t ow_len[MAX_OVERWRITTEN], ow_q[MAX_OVERWRITTEN];
    __shared__ int16_t ow_cnt[MAX_OVERWRITTEN];     // first occurrence of its string: reads showing it, else 0
    __shared__ int32_t wsum[CAND_THREADS / 32];
    __shared__ int s_depth, s_acgt[4], s_now;
    __shared__ uint32_t st[32];
    const int64_t ci = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t c = A.cand[ci];
    const int64_t a = A.ra[ci], b = A.rb[ci];
    const int n_all = (int)A.nsel[ci];
    const int depth = A.depth, C = A.C;
    if (n_all > MAXSEL) {                 // reported by c3b_fa_sizes
        if (tid == 0) atomicOr(A.status, 1);
        return;
    }
    if (tid == 0) { s_depth = 0; s_acgt[0] = s_acgt[1] = s_acgt[2] = s_acgt[3] = 0; s_now = 0; }
    // ordered compaction of the window's reads (the reference's loop at :805-814)
    int base = 0;
    for (int64_t j0 = a; j0 < b; j0 += CAND_THREADS) {
        const int64_t j = j0 + tid;
        const bool in = j < b && A.K.end[j] > c - FLANK;
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (lane == 0) wsum[warp] = __popc(m);
        __syncthreads();
        int off = base;
        for (int w = 0; w < warp; ++w) off += wsum[w];
        if (in) sel[off + __popc(m & ((1u << lane) - 1u))] = ord[off + __popc(m & ((1u << lane) - 1u))] = (int32_t)j;
        int tot = 0;
        for (int w = 0; w < CAND_THREADS / 32; ++w) tot += wsum[w];
        base += tot;
        __syncthreads();
    }
    // counters over every kept read on the candidate (:661-753): the Pos_info at c's flanking index in each read's run
    const int64_t fc = lower_bound64(A.F, 0, A.nF, c);
    for (int i = tid; i < n_all; i += CAND_THREADS) {
        const int64_t k = sel[i];
        const int64_t off = fc - A.K.fs[k];
        ev_del[i] = 0;
        ev_ins[i] = 0;
        ev_q[i] = 0;
        if (off < 0 || off >= A.K.ov[k]) continue;
        const PosInfo e = A.pool[A.K.pi[k] + off];
        if (e.alt > 0) {
            atomicAdd(&s_depth, 1);
            atomicAdd(&s_acgt[acgt_idx(NT16[e.alt])], 1);
        } else if (e.alt < 0) {
            atomicAdd(&s_depth, 1);
        }
        ev_del[i] = e.del_len;
        ev_ins[i] = e.ins_len;
        ev_q[i] = e.ins_q;
        if (e.n_ins > 1) {                // walk the read's CIGAR again for the insertions anchored on c before the kept one
            const int64_t r = A.K.orig[k];
            const int n_ow = e.n_ins - 1;
            const int slot = atomicAdd(&s_now, n_ow);
            if (slot + n_ow > MAX_OVERWRITTEN) {
                atomicOr(A.status, 8);
                continue;
            }
            int64_t ref_pos = A.K.start[k], query_pos = 0;
            int w = 0;
            for (int64_t x = A.R.cigar_off[r]; x < A.R.cigar_off[r + 1] && w < n_ow; ++x) {
                const uint32_t op = A.R.cigar[x] & 15u;
                const int64_t length = A.R.cigar[x] >> 4;
                if (op == 0 || op == 7 || op == 8) { ref_pos += length; query_pos += length; }
                else if (op == 2 || op == 3) ref_pos += length;
                else if (op == 4) query_pos += length;
                else if (op == 1) {
                    if (ref_pos - 1 == c) {
                        ow_i[slot + w] = i;
                        ow_len[slot + w] = (int32_t)length;
                        ow_q[slot + w++] = (int32_t)query_pos;
                    }
                    query_pos += length;
                }
            }
        }
    }
    __syncthreads();
    const int n_ow = s_now <= MAX_OVERWRITTEN ? s_now : 0;   // beyond the capacity: an error from c3b_fa_sizes, nothing exported
    if (tid == 0) {
        for (int x = 1; x < n_ow; ++x) {  // stable insertion sort by read: put order
            const int32_t vi = ow_i[x], vl = ow_len[x], vq = ow_q[x];
            int y = x;
            for (; y > 0 && ow_i[y - 1] > vi; --y) {
                ow_i[y] = ow_i[y - 1];
                ow_len[y] = ow_len[y - 1];
                ow_q[y] = ow_q[y - 1];
            }
            ow_i[y] = vi;
            ow_len[y] = vl;
            ow_q[y] = vq;
        }
    }
    __syncthreads();
    // the insertion puts in order: for each read (kept order) its overwritten insertions, then its kept one (key i << 16 | 0xFFFF);
    // overwritten insertion x of read i has key i << 16 | x
    auto count_ins = [&](int64_t key, int64_t kr, int q, int len) -> int {   // reads showing the string, 0 unless key is its first
        int cnt = 0;
        for (int t = 0; t < n_all; ++t)
            if (ev_ins[t] == len && same_ins(A.R, A.K, sel[t], ev_q[t], kr, q, len)) {
                if ((((int64_t)t << 16) | 0xFFFF) < key) return 0;
                ++cnt;
            }
        for (int x = 0; x < n_ow; ++x)
            if (ow_len[x] == len && same_ins(A.R, A.K, sel[ow_i[x]], ow_q[x], kr, q, len)) {
                if ((((int64_t)ow_i[x] << 16) | x) < key) return 0;
                ++cnt;
            }
        return cnt;
    };
    // distinct alleles and their counts; first occurrence in put order = the order in which the reference's counters saw them
    for (int i = tid; i < n_all; i += CAND_THREADS) {
        int dc = 0, ic = 0;
        if (ev_del[i] > 0) {
            for (int t = 0; t < n_all; ++t)
                if (ev_del[t] == ev_del[i]) {
                    if (t < i) { dc = 0; break; }
                    ++dc;
                }
        }
        if (ev_ins[i] > 0) ic = count_ins(((int64_t)i << 16) | 0xFFFF, sel[i], ev_q[i], ev_ins[i]);
        ev_dcnt[i] = (int16_t)dc;
        ev_icnt[i] = (int16_t)ic;
    }
    for (int x = tid; x < n_ow; x += CAND_THREADS) ow_cnt[x] = (int16_t)count_ins(((int64_t)ow_i[x] << 16) | x, sel[ow_i[x]], ow_q[x], ow_len[x]);
    __syncthreads();
    if (tid == 0) {
        int nal = 0;
        for (int i = 0; i < n_all; ++i) nal += (ev_dcnt[i] > 0) + (ev_icnt[i] > 0);
        for (int x = 0; x < n_ow; ++x) nal += ow_cnt[x] > 0;
        const unsigned long long o = nal ? atomicAdd(A.al_used, (unsigned long long)nal) : 0ull;
        if (o + (unsigned long long)nal > (unsigned long long)C3B_AL_CAP) {
            atomicOr(A.status, 2);
            A.al_off[ci] = 0;
            A.al_n[ci] = 0;
        } else {
            A.al_off[ci] = o;
            A.al_n[ci] = nal;
            // bit 30 of the last allele of a kind: a later read showed an allele of that kind again - that put grows a full
            // khash before it finds the key, which changes the table's bucket order (khash.h:310-318)
            // insertion puts are numbered in put order (p); deletions by read
            int last_d = -1, last_p = -1, n_put = 0;
            for (int i = 0, x = 0; i < n_all; ++i) {
                if (ev_dcnt[i] > 0) last_d = i;
                for (; x < n_ow && ow_i[x] == i; ++x, ++n_put)
                    if (ow_cnt[x] > 0) last_p = n_put;
                if (ev_ins[i] > 0) {
                    if (ev_icnt[i] > 0) last_p = n_put;
                    ++n_put;
                }
            }
            bool tail_d = false;
            for (int i = 0; i < n_all; ++i) tail_d |= i > last_d && ev_del[i] > 0;
            const bool tail_i = last_p < n_put - 1;
            int w = (int)o;
            auto put_ins = [&](int p, int i, int len, int q, int cnt) {
                A.al_meta[w] = 0x80000000u | (uint32_t)len | (p == last_p && tail_i ? 0x40000000u : 0u);
                A.al_read[w] = (uint32_t)A.K.orig[sel[i]];
                A.al_qpos[w] = (uint32_t)q;
                A.al_cnt[w++] = (uint32_t)cnt;
            };
            for (int i = 0, x = 0, p = 0; i < n_all; ++i) {
                if (ev_dcnt[i] > 0) {
                    A.al_meta[w] = (uint32_t)ev_del[i] | (i == last_d && tail_d ? 0x40000000u : 0u);
                    A.al_read[w] = (uint32_t)A.K.orig[sel[i]];
                    A.al_qpos[w] = 0;
                    A.al_cnt[w++] = (uint32_t)ev_dcnt[i];
                }
                for (; x < n_ow && ow_i[x] == i; ++x, ++p)
                    if (ow_cnt[x] > 0) put_ins(p, i, ow_len[x], ow_q[x], ow_cnt[x]);
                if (ev_ins[i] > 0) {
                    if (ev_icnt[i] > 0) put_ins(p, i, ev_ins[i], ev_q[i], ev_icnt[i]);
                    ++p;
                }
            }
        }
        A.c_depth[ci] = s_depth;
        for (int t = 0; t < 4; ++t) A.c_acgt[ci * 4 + t] = s_acgt[t];
    }
    // the reads of the matrix: none below position 16 (the reference's size_t start_pos wraps there, :790 / :810)
    const int n = c < FLANK ? 0 : n_all;
    if (n > depth) {
        // sort_read_name_by_haplotype's Fisher-Yates (:121-134) on the glibc TYPE_3 stream at this candidate's offset
        if (warp == 0) {
            if (lane < 31) st[lane] = A.state0[lane];
            __syncwarp();
            const uint64_t off = (uint64_t)A.rand_skip + (uint64_t)A.draw_off[ci];
            for (int bit = 0; bit < JUMP_BITS; ++bit) {
                if (!((off >> bit) & 1u)) continue;
                const uint32_t *M = A.jump + (size_t)bit * 31 * 31;
                uint32_t acc = 0;
                if (lane < 31)
                    for (int j = 0; j < 31; ++j) acc += M[lane * 31 + j] * st[j];
                __syncwarp();
                if (lane < 31) st[lane] = acc;
                __syncwarp();
            }
        }
        __syncthreads();
        if (tid == 0) {
            for (int i = 0; i < n - 1; ++i) {
                uint32_t r;
                if (i < 31) {
                    r = st[i];
                } else {                                 // r[m] = r[m-31] + r[m-3] in a ring of the last 31 values
                    r = st[i % 31] + st[(i - 3) % 31];
                    st[i % 31] = r;
                }
                const uint64_t rnd = r >> 1;
                const uint64_t j = (uint64_t)i + rnd / (2147483647ull / (uint64_t)(n - i) + 1ull);
                const int32_t t = ord[j];
                ord[j] = ord[i];
                ord[i] = t;
            }
        }
    }
    __syncthreads();
    // qsort of the first min(n, depth) by (haplotype, read index) - the keys are distinct, so a rank sort gives the same order -
    // and the padding split of :139-150
    const int m = n < depth ? n : depth;
    const int top = n < depth ? (depth - m) >> 1 : 0;
    for (int d = tid; d < depth; d += CAND_THREADS) rows[d] = -1;
    __syncthreads();
    for (int i = tid; i < m; i += CAND_THREADS) {
        const int64_t ki = ord[i];
        const int64_t key = ((int64_t)A.K.hap[ki] << 32) | ki;
        int rank = 0;
        for (int t = 0; t < m; ++t) {
            const int64_t kt = ord[t];
            rank += (((int64_t)A.K.hap[kt] << 32) | kt) < key;
        }
        rows[top + rank] = (int32_t)ki;
    }
    __syncthreads();
    auto ref_at = [&](int64_t p) -> char {
        const int64_t o = p - A.ref_start;
        return (o >= 0 && o < A.ref_len) ? upper(A.ref[o]) : '\0';
    };
    // the allele-frequency channel of every row, from its centre column (:852-896, :915-948)
    const char cref = ref_at(c);
    for (int d = tid; d < depth; d += CAND_THREADS) {
        int8_t af = 0;
        const int64_t k = rows[d];
        const int64_t off = k >= 0 ? fc - A.K.fs[k] : -1;
        if (k >= 0 && off >= 0 && off < A.K.ov[k]) {
            const PosInfo e = A.pool[A.K.pi[k] + off];
            const char altc = NT16[e.alt > 0 ? e.alt : 0];
            if (e.alt <= 0) {
            } else if (e.ins_len > 0) {         // the counter's value for the kept string, overwritten insertions included
                bool found = false;
                for (int i = 0; i < n_all && !found; ++i)
                    if (ev_icnt[i] > 0 && ev_ins[i] == e.ins_len && same_ins(A.R, A.K, sel[i], ev_q[i], k, e.ins_q, e.ins_len)) {
                        af = norm_af(ev_icnt[i], s_depth);
                        found = true;
                    }
                for (int x = 0; x < n_ow && !found; ++x)
                    if (ow_cnt[x] > 0 && ow_len[x] == e.ins_len && same_ins(A.R, A.K, sel[ow_i[x]], ow_q[x], k, e.ins_q, e.ins_len)) {
                        af = norm_af(ow_cnt[x], s_depth);
                        found = true;
                    }
            } else if (e.del_len > 0) {
                for (int i = 0; i < n_all; ++i)
                    if (ev_dcnt[i] > 0 && ev_del[i] == e.del_len) {
                        af = norm_af(ev_dcnt[i], s_depth);
                        break;
                    }
            } else if (cref != altc) {
                af = norm_af(s_acgt[acgt_idx(altc)], s_depth);
            }
        }
        row_af[d] = af > 0 ? af : 0;
    }
    // channel 6, one thread per row: the insertion bases of column p (p < 32, a covered and not deleted column) spill to the
    // right; the row is walked in column order, so a later column overwrites an earlier one as in the reference (:855-870)
    const int64_t fw = fc - FLANK;                  // flanking index of c - 16: the window is contiguous in F
    for (int d = tid; d < depth; d += CAND_THREADS) {
        int8_t *sp = spill + d * NPOS;
        for (int q = 0; q < NPOS; ++q) sp[q] = 0;
        const int64_t k = rows[d];
        if (k < 0) continue;
        const int64_t fs = A.K.fs[k], ov = A.K.ov[k];
        const PosInfo *pi = A.pool + A.K.pi[k];
        const uint8_t *sq = A.R.seq + A.R.seq_off[A.K.orig[k]];
        for (int p = 0; p < NPOS - 1; ++p) {
            const int64_t o = fw + p - fs;
            if (o < 0 || o >= ov) continue;
            const PosInfo e = pi[o];
            if (e.alt <= 0 || e.ins_len <= 0) continue;
            const int n_sp = e.ins_len < NPOS - p ? e.ins_len : NPOS - p;
            for (int t = 0; t < n_sp; ++t) sp[p + t] = fa_val(NT16[nib(sq, (int64_t)e.ins_q + t)]);
        }
    }
    __syncthreads();
    // the block: one thread per (row, column), every byte of it written (:819-912)
    int8_t *blk = A.matrix + (size_t)ci * depth * NPOS * C;
    for (int t = tid; t < depth * NPOS; t += CAND_THREADS) {
        const int d = t / NPOS, q = t - d * NPOS;
        int8_t v[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        const int64_t k = rows[d];
        if (k >= 0) {
            const int64_t r = A.K.orig[k];
            const int64_t fs = A.K.fs[k], ov = A.K.ov[k];
            const PosInfo *pi = A.pool + A.K.pi[k];
            const int64_t off = fw + q - fs;
            if (off >= 0 && off < ov) {
                const PosInfo e = pi[off];
                if (e.alt > 0) {                        // deleted (-1) columns are skipped (:837-842); 0: not covered by M / D
                    const char rb = ref_at(c - FLANK + q), altc = NT16[e.alt];
                    const int8_t ref_v = fa_val(rb);
                    int8_t alt_v = 0;
                    if (e.ins_len > 0) alt_v = fa_val('I');
                    else if (e.del_len > 0) alt_v = fa_val('D');
                    else if (rb != altc) alt_v = fa_val(altc);
                    const int mq = A.R.mapq[r];
                    v[0] = ref_v;
                    v[1] = alt_v;
                    v[2] = (A.R.flag[r] & 16) ? 50 : 100;                                     // normalize_strand
                    v[3] = (int8_t)(int)(mq < 60 ? 100 * mq / 60.0 : 100);                     // normalize_mq
                    v[4] = e.bq;
                    v[5] = ref_v != 0 ? row_af[d] : 0;
                    v[7] = A.K.hap[k] == 1 ? 30 : A.K.hap[k] == 2 ? 90 : 60;                  // HAP_TYPE
                    v[8] = (int8_t)e.sig;
                }
            }
            v[6] = spill[d * NPOS + q];
        }
        int8_t *dst = blk + ((size_t)d * NPOS + q) * C;
        for (int ch = 0; ch < C; ++ch) dst[ch] = v[ch];
    }
}

// glibc's TYPE_3 generator (random_r.c): srandom_r fills r[0..30] with 16807 * r[i-1] mod (2^31 - 1) (Schrage's method on
// int32), r[i] = r[i-31] + r[i-3] mod 2^32 from i = 34 on (r[31..33] = r[0..2]), and rand() number k is r[344 + k] >> 1.
void glibc_state(uint32_t seed, uint32_t out[31]) {
    if (seed == 0) seed = 1;
    std::vector<uint32_t> r(375);
    int32_t word = (int32_t)seed;
    r[0] = (uint32_t)word;
    for (int i = 1; i < 31; ++i) {
        const long hi = word / 127773, lo = word % 127773;
        word = (int32_t)(16807 * lo - 2836 * hi);
        if (word < 0) word += 2147483647;
        r[i] = (uint32_t)word;
    }
    for (int i = 31; i < 34; ++i) r[i] = r[i - 31];
    for (int i = 34; i < 375; ++i) r[i] = r[i - 31] + r[i - 3];
    for (int i = 0; i < 31; ++i) out[i] = r[344 + i];
}

// M^(2^b), b < JUMP_BITS, for the state (r[n], ..., r[n+30]) -> (r[n+1], ..., r[n+31]), r[n+31] = r[n] + r[n+28]
void glibc_jump_matrices(std::vector<uint32_t> &out) {
    out.assign((size_t)JUMP_BITS * 961, 0u);
    uint32_t *M = out.data();
    for (int i = 0; i < 30; ++i) M[i * 31 + i + 1] = 1u;
    M[30 * 31 + 0] = 1u;
    M[30 * 31 + 28] = 1u;
    for (int b = 1; b < JUMP_BITS; ++b) {
        const uint32_t *P = out.data() + (size_t)(b - 1) * 961;
        uint32_t *Q = out.data() + (size_t)b * 961;
        for (int i = 0; i < 31; ++i)
            for (int j = 0; j < 31; ++j) {
                uint32_t s = 0;
                for (int t = 0; t < 31; ++t) s += P[i * 31 + t] * P[t * 31 + j];
                Q[i * 31 + j] = s;
            }
    }
}

}  // namespace

// Timed stages: 0 the build (c3b_fa_build), 1 the text (c3b_fa_alt_text).  counters: int64 0 nF, 1 n_kept, 2 pool entries,
// 3 signal entries, 4 draws, 5 status, 6 al_used, 7 the text stage's status, 8 n_text_bytes, 9 n_decoder_bytes, and with device
// candidates 10 the build's candidate count, 11 the device count it was cut from.
constexpr int N_COUNTERS = 12, TEXT_WORD = 7;

struct c3b_fa : C3bRegionWorkspace {
    C3bBuf in_cand, in_var, jump, state0;
    C3bBuf fstart, fcnt, foff, F;
    C3bBuf rend, rlo, rov, pass, table, keep, kidx, kovr, kov_ex;
    C3bBuf k_orig, k_start, k_end, k_pmax, k_fs, k_ov, k_pi, k_sig, k_hap, sig_len, sig_ex;
    C3bBuf pool, sig;
    C3bBuf ra, rb, nsel, draws, draw_off;
    C3bBuf matrix, c_depth, c_acgt;
    int64_t n_cand = 0, depth = 0, C = 8, n_kept = 0;
    bool built = false;
    bool synced = false;                 // c3b_fa_sizes has waited for everything queued since the last build or text stage
};

// The text stage's results need an issued c3b_fa_alt_text and, to read its counter words, the build's wait.  `who` names the
// entry point in the error.
static int fa_texted(c3b_fa *w, const char *who, bool wait) {
    if (!w || !w->texted) { c3b_set_error("%s: no c3b_fa_alt_text has been issued", who); return 1; }
    return wait && !w->synced && c3b_fa_sizes(w, nullptr, nullptr, nullptr);
}
static const char *const FA_TEXT_HINT = "build fewer candidates";

extern "C" {

int c3b_fa_create(c3b_fa **out, int device_ordinal) {
    if (c3b_region_create(out, device_ordinal, 2, N_COUNTERS, TEXT_WORD, "c3b_fa_create")) return 1;
    c3b_fa *w = *out;
    std::vector<uint32_t> J;
    glibc_jump_matrices(J);
    if (w->jump.ensure(J.size() * 4, nullptr, "c3b_fa") || w->state0.ensure(31 * 4, nullptr, "c3b_fa") ||
        cudaMemcpy(w->jump.p, J.data(), J.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
        c3b_set_error("c3b_fa_create: allocation failed");
        c3b_fa_destroy(w);
        *out = nullptr;
        return 1;
    }
    return 0;
}

static inline unsigned blocks_for(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

// The build behind both entry points.  Host candidates: candidates[0 .. n_cand).  Device candidates (dcand != nullptr):
// dcand[first ..] up to n_cand of them, as many as *dn allows; the count is read at the first sizing wait.
static int fa_build(c3b_fa *w, const char *who, const c3b_fa_records *records, int on_device, const int64_t *candidates,
                    int64_t n_cand, const int64_t *dcand, const int64_t *dn, int64_t first, int64_t *n_cand_out, int64_t *n_total,
                    const c3b_fa_variant *variants, int64_t n_var, const char *ref_seq, int64_t ref_start, int64_t ref_len,
                    const c3b_fa_params *params, void *cuda_stream) {
    if (!w || !records || !params) { c3b_set_error("%s: null argument", who); return 1; }
    if (params->matrix_depth < 1 || params->matrix_depth > 256) {
        c3b_set_error("%s: matrix_depth %d outside 1..256", who, params->matrix_depth);
        return 1;
    }
    if (dcand) {
        if (!dn || first < 0 || n_cand < 0 || n_cand >= (int64_t)INT_MAX / 33) { c3b_set_error("%s: bad candidates", who); return 1; }
    } else {
        if (n_cand < 0 || n_cand >= (int64_t)INT_MAX / 33 || (n_cand > 0 && !candidates)) { c3b_set_error("%s: bad candidates", who); return 1; }
        for (int64_t i = 0; i < n_cand; ++i)
            if (candidates[i] < 0 || candidates[i] >= (int64_t)INT_MAX - FLANK || (i && candidates[i] <= candidates[i - 1])) {
                c3b_set_error("%s: candidates must be 0-based positions below 2^31 - 17, strictly ascending (index %lld)", who,
                              (long long)i);
                return 1;
            }
    }
    if (n_var < 0 || (n_var > 0 && !variants)) { c3b_set_error("%s: bad variants", who); return 1; }
    for (int64_t i = 1; i < n_var; ++i)
        if (variants[i].position < variants[i - 1].position) {
            c3b_set_error("%s: variants must be sorted by position (index %lld)", who, (long long)i);
            return 1;
        }
    C3B_CUDA(cudaSetDevice(w->device));
    cudaStream_t s = (cudaStream_t)cuda_stream;
    w->stream = s;
    w->built = w->synced = w->texted = false;
    w->n_cand = n_cand;
    w->depth = params->matrix_depth;
    w->C = params->dwell ? 9 : 8;
    w->n_kept = 0;
    const int depth = params->matrix_depth;

    if (w->intake(who, &records->core, records, params->dwell != 0, INT_MAX, on_device, ref_seq, ref_start, ref_len)) return 1;
    const C3bReads &R = w->R;
    const int64_t n = R.n;
    const char *dref = w->dref;
    const size_t Kz = (size_t)(n_cand > 0 ? n_cand : 1), Nz = (size_t)(n > 0 ? n : 1);
    auto grow = [&](C3bBuf &b, size_t bytes) { return b.ensure(bytes, s, "c3b_fa"); };
    if (grow(w->in_cand, Kz * 8) || grow(w->in_var, (size_t)(n_var > 0 ? n_var : 1) * sizeof(c3b_fa_variant))) return 1;
    if (n_cand && !dcand) C3B_CUDA(cudaMemcpyAsync(w->in_cand.p, candidates, (size_t)n_cand * 8, cudaMemcpyHostToDevice, s));
    if (n_var) C3B_CUDA(cudaMemcpyAsync(w->in_var.p, variants, (size_t)n_var * sizeof(c3b_fa_variant), cudaMemcpyHostToDevice, s));
    uint32_t st0[31];
    glibc_state(params->rand_seed, st0);
    C3B_CUDA(cudaMemcpyAsync(w->state0.p, st0, sizeof(st0), cudaMemcpyHostToDevice, s));

    // scratch and outputs
    const size_t Fz = Kz * 33;
    uint64_t T = 2;                                 // name table: a power of two >= 2 n (n < 2^31, so T - 1 fits 32 bits)
    while ((int64_t)T < 2 * n) T <<= 1;
    if (grow(w->fstart, Kz * 8) || grow(w->fcnt, Kz * 8) || grow(w->foff, Kz * 8) || grow(w->F, Fz * 8) ||
        grow(w->rend, Nz * 8) || grow(w->rlo, Nz * 8) || grow(w->rov, Nz * 4) || grow(w->pass, Nz) ||
        grow(w->table, (size_t)T * 8) || grow(w->keep, Nz * 8) || grow(w->kidx, Nz * 8) || grow(w->kovr, Nz * 8) ||
        grow(w->kov_ex, Nz * 8) || grow(w->k_orig, Nz * 8) || grow(w->k_start, Nz * 8) || grow(w->k_end, Nz * 8) ||
        grow(w->k_pmax, Nz * 8) || grow(w->k_fs, Nz * 8) || grow(w->k_ov, Nz * 4) || grow(w->k_pi, Nz * 8) ||
        grow(w->k_sig, Nz * 8) || grow(w->k_hap, Nz * 4) || grow(w->sig_len, Nz * 8) || grow(w->sig_ex, Nz * 8) ||
        grow(w->ra, Kz * 8) || grow(w->rb, Kz * 8) || grow(w->nsel, Kz * 8) || grow(w->draws, Kz * 8) ||
        grow(w->draw_off, Kz * 8) || (!dcand && grow(w->matrix, Kz * (size_t)depth * 33 * (size_t)w->C)) || grow(w->c_depth, Kz * 4) ||
        grow(w->c_acgt, Kz * 16) || grow(w->al_off, Kz * 4) || grow(w->al_n, Kz * 4) || grow(w->al_meta, (size_t)C3B_AL_CAP * 4) ||
        grow(w->al_read, (size_t)C3B_AL_CAP * 4) || grow(w->al_qpos, (size_t)C3B_AL_CAP * 4) || grow(w->al_cnt, (size_t)C3B_AL_CAP * 4))
        return 1;
    int64_t *cnt = w->counters.as<int64_t>();
    C3B_CUDA(cudaMemsetAsync(cnt, 0, 64, s));
    int *status = reinterpret_cast<int *>(cnt + 5);
    unsigned long long *al_used = reinterpret_cast<unsigned long long *>(cnt + 6);

    Kept K;
    K.orig = w->k_orig.as<int64_t>(); K.start = w->k_start.as<int64_t>(); K.end = w->k_end.as<int64_t>();
    K.pmax = w->k_pmax.as<int64_t>(); K.fs = w->k_fs.as<int64_t>(); K.ov = w->k_ov.as<int32_t>(); K.pi = w->k_pi.as<int64_t>();
    K.sig = w->k_sig.as<int64_t>(); K.hap = w->k_hap.as<int32_t>();
    w->launches[0] = 0;
    C3B_CUDA(cudaEventRecord(w->ev[0][0], s));
    const int64_t *n_dev = nullptr;                 // device candidates: their count, known to the host after the first wait
    if (dcand) {
        fa_cand_intake_kernel<<<blocks_for(n_cand > 0 ? n_cand : 1, 256), 256, 0, s>>>(dcand, dn, first, n_cand,
                                                                                        w->in_cand.as<int64_t>(), cnt, status);
        w->launches[0] += 1;
        n_dev = cnt + 10;
    }
    int64_t nF = 0, n_kept = 0, n_pool = 0, n_sig = 0;
    if (n_cand > 0) {
        fa_flank_count_kernel<<<blocks_for(n_cand, 256), 256, 0, s>>>(w->in_cand.as<int64_t>(), n_cand, n_dev,
                                                                       w->fstart.as<int64_t>(), w->fcnt.as<int64_t>());
        block_scan_sum(w->fcnt.as<int64_t>(), w->foff.as<int64_t>(), n_cand, nullptr, cnt + 0, s);
        fa_flank_fill_kernel<<<(unsigned)n_cand, 64, 0, s>>>(w->fstart.as<int64_t>(), w->fcnt.as<int64_t>(), w->foff.as<int64_t>(),
                                                             n_cand, n_dev, w->F.as<int64_t>());
        w->launches[0] += 3;
    }
    if (n_cand > 0 || dcand) {
        // the size of F bounds the binary searches of K3 and K11; device candidates: their count sizes everything after
        C3B_CUDA(cudaMemcpyAsync(&w->host_counters[0], cnt + 0, dcand ? N_COUNTERS * 8 : 8, cudaMemcpyDeviceToHost, s));
        C3B_CUDA(cudaStreamSynchronize(s));
        nF = w->host_counters[0];
        if (dcand) {
            if ((int)w->host_counters[5] & 16) {
                c3b_set_error("%s: candidates must be 0-based positions below 2^31 - 17, strictly ascending", who);
                return 1;
            }
            w->n_cand = n_cand = w->host_counters[10];
            if (n_total) *n_total = w->host_counters[11];
            // the matrix, the one large per-candidate buffer, for the candidates the build has rather than its capacity
            if (grow(w->matrix, (size_t)(n_cand > 0 ? n_cand : 1) * (size_t)depth * 33 * (size_t)w->C)) return 1;
        }
        if (n > 0 && n_cand > 0) {
            C3B_CUDA(cudaMemsetAsync(w->table.p, 0xff, (size_t)T * 8, s));
            C3B_CUDA(cudaMemsetAsync(w->sig_len.p, 0, Nz * 8, s));
            fa_read_scan_kernel<<<blocks_for(n, 256), 256, 0, s>>>(R, params->min_mq, w->F.as<int64_t>(), nF, w->rend.as<int64_t>(),
                                                                   w->rlo.as<int64_t>(), w->rov.as<int32_t>(), w->pass.as<uint8_t>(),
                                                                   w->table.as<int64_t>(), (uint32_t)(T - 1));
            fa_read_keep_kernel<<<blocks_for(n, 256), 256, 0, s>>>(R, w->pass.as<uint8_t>(), w->rov.as<int32_t>(), w->table.as<int64_t>(),
                                                                   (uint32_t)(T - 1), w->keep.as<int64_t>(), w->kovr.as<int64_t>());
            block_scan_sum(w->keep.as<int64_t>(), w->kidx.as<int64_t>(), n, nullptr, cnt + 1, s);
            block_scan_sum(w->kovr.as<int64_t>(), w->kov_ex.as<int64_t>(), n, nullptr, cnt + 2, s);
            fa_read_compact_kernel<<<blocks_for(n, 256), 256, 0, s>>>(R, params->dwell, w->keep.as<int64_t>(), w->kidx.as<int64_t>(),
                                                                      w->kov_ex.as<int64_t>(), w->rend.as<int64_t>(), w->rlo.as<int64_t>(),
                                                                      w->rov.as<int32_t>(), K, w->sig_len.as<int64_t>());
            block_scan_sum(w->sig_len.as<int64_t>(), w->sig_ex.as<int64_t>(), n, nullptr, cnt + 3, s);
            w->launches[0] += 6;
            // the kept-read count and the pool sizes
            C3B_CUDA(cudaMemcpyAsync(w->host_counters, cnt, 32, cudaMemcpyDeviceToHost, s));
            C3B_CUDA(cudaStreamSynchronize(s));
            n_kept = w->host_counters[1];
            n_pool = w->host_counters[2];
            n_sig = w->host_counters[3];
        }
    }
    w->n_kept = n_kept;
    if (n_kept > 0) {
        if (grow(w->pool, (size_t)n_pool * sizeof(PosInfo)) || grow(w->sig, (size_t)(n_sig > 0 ? n_sig : 1) * 4)) return 1;
        C3B_CUDA(cudaMemsetAsync(w->pool.p, 0, (size_t)n_pool * sizeof(PosInfo), s));
        block_scan_max(K.end, K.pmax, n_kept, s);
        w->launches[0] += 1;
        if (n_sig > 0) C3B_CUDA(cudaMemsetAsync(w->sig.p, 0, (size_t)n_sig * 4, s));
        fa_signal_kernel<<<blocks_for(n_kept, 256), 256, 0, s>>>(R, K, w->sig_len.as<int64_t>(), w->sig_ex.as<int64_t>(), n_kept,
                                                                 w->sig.as<int32_t>());
        w->launches[0] += 1;
        if (params->need_haplotagging && n_var > 0) {
            HapArgs H;
            H.R = R; H.K = K; H.n_kept = n_kept; H.var = w->in_var.as<c3b_fa_variant>(); H.n_var = n_var;
            H.ref = dref; H.ref_start = ref_start; H.ref_len = ref_len > 0 ? ref_len : 0; H.status = status;
            fa_haplotag_kernel<<<blocks_for(n_kept, 128), 128, 0, s>>>(H);
            w->launches[0] += 1;
        }
        fa_pos_info_kernel<<<blocks_for(n_kept, 128), 128, 0, s>>>(R, K, n_kept, w->F.as<int64_t>(), w->sig.as<int32_t>(),
                                                                   w->pool.as<PosInfo>());
        w->launches[0] += 1;
    }
    if (n_cand > 0) {
        fa_select_count_kernel<<<blocks_for(n_cand * 32, 256), 256, 0, s>>>(w->in_cand.as<int64_t>(), n_cand, K, n_kept, depth,
                                                                          w->ra.as<int64_t>(), w->rb.as<int64_t>(),
                                                                          w->nsel.as<int64_t>(), w->draws.as<int64_t>());
        block_scan_sum(w->draws.as<int64_t>(), w->draw_off.as<int64_t>(), n_cand, nullptr, cnt + 4, s);
        CandArgs A;
        A.R = R; A.K = K; A.cand = w->in_cand.as<int64_t>(); A.F = w->F.as<int64_t>(); A.nF = nF; A.pool = w->pool.as<PosInfo>();
        A.ref = dref; A.ref_start = ref_start; A.ref_len = ref_len > 0 ? ref_len : 0;
        A.ra = w->ra.as<int64_t>(); A.rb = w->rb.as<int64_t>(); A.nsel = w->nsel.as<int64_t>(); A.draw_off = w->draw_off.as<int64_t>();
        A.rand_skip = params->rand_skip; A.jump = w->jump.as<uint32_t>(); A.state0 = w->state0.as<uint32_t>();
        A.depth = depth; A.C = (int)w->C; A.matrix = w->matrix.as<int8_t>();
        A.c_depth = w->c_depth.as<int32_t>(); A.c_acgt = w->c_acgt.as<int32_t>(); A.al_off = w->al_off.as<int32_t>();
        A.al_n = w->al_n.as<int32_t>(); A.al_meta = w->al_meta.as<uint32_t>(); A.al_read = w->al_read.as<uint32_t>();
        A.al_qpos = w->al_qpos.as<uint32_t>(); A.al_cnt = w->al_cnt.as<uint32_t>(); A.al_used = al_used; A.status = status;
        fa_candidate_kernel<<<(unsigned)n_cand, CAND_THREADS, 0, s>>>(A);
        w->launches[0] += 2;
    }
    C3B_CUDA(cudaEventRecord(w->ev[0][1], s));
    C3B_CUDA(cudaGetLastError());
    C3B_CUDA(cudaMemcpyAsync(w->host_counters, cnt, N_COUNTERS * 8, cudaMemcpyDeviceToHost, s));
    w->built = true;
    if (n_cand_out) *n_cand_out = n_cand;
    return 0;
}

int c3b_fa_build(c3b_fa *w, const c3b_fa_records *records, int on_device, const int64_t *candidates, int64_t n_cand,
                 const c3b_fa_variant *variants, int64_t n_var, const char *ref_seq, int64_t ref_start, int64_t ref_len,
                 const c3b_fa_params *params, void *cuda_stream) {
    return fa_build(w, "c3b_fa_build", records, on_device, candidates, n_cand, nullptr, nullptr, 0, nullptr, nullptr, variants,
                    n_var, ref_seq, ref_start, ref_len, params, cuda_stream);
}

int c3b_fa_build_device_candidates(c3b_fa *w, const c3b_fa_records *records, int on_device, const int64_t *candidates,
                                   const int64_t *n_candidates, int64_t first, int64_t max_cand, const c3b_fa_variant *variants,
                                   int64_t n_var, const char *ref_seq, int64_t ref_start, int64_t ref_len,
                                   const c3b_fa_params *params, void *cuda_stream, int64_t *n_cand, int64_t *n_total) {
    if ((!candidates && max_cand > 0) || !n_candidates) { c3b_set_error("c3b_fa_build_device_candidates: null argument"); return 1; }
    return fa_build(w, "c3b_fa_build_device_candidates", records, on_device, nullptr, max_cand, candidates, n_candidates, first,
                    n_cand, n_total, variants, n_var, ref_seq, ref_start, ref_len, params, cuda_stream);
}

int c3b_fa_sizes(c3b_fa *w, int64_t *n_cand, int64_t *n_kept, int64_t *rand_draws) {
    if (!w || !w->built) { c3b_set_error("c3b_fa_sizes: no c3b_fa_build has been issued"); return 1; }
    C3B_CUDA(cudaSetDevice(w->device));
    C3B_CUDA(cudaStreamSynchronize(w->stream));
    const int status = (int)w->host_counters[5];
    if (status & 1) { c3b_set_error("c3b_fa_build: more than %d reads overlap one candidate window", MAXSEL); return 1; }
    if (status & 2) { c3b_set_error("c3b_fa_build: more than %d distinct indel alleles to export; build fewer candidates per call", C3B_AL_CAP); return 1; }
    if (status & 4) { c3b_set_error("c3b_fa_build: a read touches variants of more than %d phase sets", MAX_PS); return 1; }
    if (status & 8) {
        c3b_set_error("c3b_fa_build: more than %d insertions on one candidate are overwritten by a later insertion on the same anchor",
                      MAX_OVERWRITTEN);
        return 1;
    }
    w->synced = true;
    if (n_cand) *n_cand = w->n_cand;
    if (n_kept) *n_kept = w->n_kept;
    if (rand_draws) *rand_draws = w->host_counters[4];
    return 0;
}

int c3b_fa_fetch(c3b_fa *w, int8_t *matrix, int32_t *kept_haplotype, int64_t *kept_read) {
    if (c3b_fa_sizes(w, nullptr, nullptr, nullptr)) return 1;
    const size_t nm = (size_t)w->n_cand * (size_t)w->depth * 33 * (size_t)w->C, nk = (size_t)w->n_kept;
    return w->get(matrix, w->matrix, nm) || w->get(kept_haplotype, w->k_hap, nk * 4) || w->get(kept_read, w->k_orig, nk * 8) ||
           w->wait();
}

int c3b_fa_fetch_alleles(c3b_fa *w, int32_t *depth, int32_t *acgt, int32_t *al_off, int32_t *al_n, uint32_t *meta, uint32_t *read,
                         uint32_t *qpos, uint32_t *cnt, int64_t capacity, int64_t *n_alleles) {
    if (c3b_fa_sizes(w, nullptr, nullptr, nullptr)) return 1;
    const int64_t used = w->host_counters[6], n = used < C3B_AL_CAP ? used : C3B_AL_CAP;
    if (n_alleles) *n_alleles = n;
    const size_t k = (size_t)w->n_cand;
    return w->get(depth, w->c_depth, k * 4) || w->get(acgt, w->c_acgt, k * 16) || w->get(al_off, w->al_off, k * 4) ||
           w->get(al_n, w->al_n, k * 4) || w->get_alleles("c3b_fa_fetch_alleles", n, capacity, meta, read, qpos, cnt) || w->wait();
}

int c3b_fa_device(c3b_fa *w, const int8_t **matrix) {
    if (!w || !w->built) { c3b_set_error("c3b_fa_device: no c3b_fa_build has been issued"); return 1; }
    if (matrix) *matrix = w->matrix.as<int8_t>();
    return 0;
}

int c3b_fa_alt_text(c3b_fa *w, int64_t max_indel_length) {
    if (!w || !w->built) { c3b_set_error("c3b_fa_alt_text: no c3b_fa_build has been issued"); return 1; }
    w->synced = false;                    // the status word and the totals travel with the next c3b_fa_sizes
    FaAltTextArgs A;
    if (w->text_prepare(w->n_cand, max_indel_length, "c3b_fa", A)) return 1;
    A.cand = w->in_cand.as<int64_t>(); A.c_depth = w->c_depth.as<int32_t>(); A.c_acgt = w->c_acgt.as<int32_t>();
    return w->text_enqueue(A, c3b_launch_fa_alt_text);
}

int c3b_fa_alt_text_sizes(c3b_fa *w, int64_t *n_text_bytes, int64_t *n_decoder_bytes) {
    const char *who = "c3b_fa_alt_text_sizes";
    return fa_texted(w, who, true) || w->text_sizes(who, FA_TEXT_HINT, n_text_bytes, n_decoder_bytes);
}

int c3b_fa_fetch_alt_text(c3b_fa *w, char *text, int64_t *text_off, char *decoder, int64_t *decoder_off, uint8_t *ref_base,
                          int64_t *position) {
    const char *who = "c3b_fa_fetch_alt_text";
    return fa_texted(w, who, true) ||
           w->text_fetch(who, FA_TEXT_HINT, w->n_cand, text, text_off, decoder, decoder_off, ref_base, position);
}

int c3b_fa_alt_text_device(c3b_fa *w, const char **text, const int64_t **text_off, const char **decoder,
                           const int64_t **decoder_off, const uint8_t **ref_base, const int64_t **position) {
    if (fa_texted(w, "c3b_fa_alt_text_device", false)) return 1;
    w->text_device(text, text_off, decoder, decoder_off, ref_base, position);
    return 0;
}

int c3b_fa_alt_text_last_ms(c3b_fa *w, float *ms, int *launches) {
    return fa_texted(w, "c3b_fa_alt_text_last_ms", false) || w->elapsed(1, ms, launches);
}

int c3b_fa_last_ms(c3b_fa *w, float *ms, int *launches) {
    if (!w || !w->built) { c3b_set_error("c3b_fa_last_ms: no c3b_fa_build has been issued"); return 1; }
    return w->elapsed(0, ms, launches);
}

void c3b_fa_destroy(c3b_fa *w) { c3b_region_destroy(w); }

}  // extern "C"
