/*
 * pileup_oracle.c - TEST INFRASTRUCTURE ONLY (checker for clair3_b200/csrc/plp_counts.cu; never linked into the product).
 *
 * Plain-C, single-threaded restatement of the reference's pileup feature counter
 *     calculate_clair3_pileup()            HKU-BAL/Clair3 src/clair3_pileup.c:142-476
 * on DECODED alignment records (the fields htslib's bam1_t carries), in the reference's own order of work: one pileup column at a
 * time, every overlapping read resolved with an incremental per-read CIGAR cursor, a per-column deletion-length table and
 * insertion-string counters, then the column's statistics and candidate test.
 *
 * The per-read / per-column resolution lives in a THIRD-PARTY dependency that the reference does not vendor: htslib 1.15.1
 * (downloaded by the reference's Makefile:32-46; only its public header src/sam.h is in the tree).  Restated here from htslib's
 * published behaviour:
 *     bam_plp_push / bam_plp_next (sam.c): a read is on column pos iff beg <= pos < beg + reference length of its CIGAR; columns
 *         nobody covers are not reported; records with (UNMAP|SECONDARY|QCFAIL|DUP) are dropped (the reference's own reader,
 *         src/medaka_bamiter.c:21-24, additionally drops SUPPLEMENTARY and mapq < min_mq before the pileup sees them);
 *     resolve_cigar2 (sam.c): cursor (k, x, y) on the current reference-consuming operation; qpos = y + (pos - x) on M/=/X; on D/N
 *         is_del = 1, qpos = y, is_refskip = (op == N); on the LAST reference position of an operation the next operation is
 *         peeked: D (when the current one is not D) -> indel = -(its length, adjacent D runs merged), I -> indel = +(length,
 *         further I's merged across P), P -> the I's that follow the pads.
 * The reference's own code is followed line by line for everything else, including its quirks:
 *     - a read base that is not A/C/G/T maps to feature index -1 (num2countbaseclair3, src/clair3_pileup.h:96-101), so
 *       `matrix[major_col + base_i] += 1` (src/clair3_pileup.c:280) lands on the PREVIOUS emitted column's last feature (index 17);
 *       on the very first column it is an out-of-bounds write that no output shows - dropped here;
 *     - contiguous_flanking_num restarts whenever pre_pos == 0 (src/clair3_pileup.c:227-230);
 *     - all_alt_count accumulates the running maximum (src/clair3_pileup.c:356-360).
 *
 * Pinned against the reference's own C: oracle/pileup_ref.py compiles src/clair3_pileup.c and src/medaka_bamiter.c against the
 * in-memory htslib stand-in of oracle/hts_stub/ (its pileup engine written independently of resolve() below), and
 * tests/test_pileup_reference_cpu.py requires this restatement to equal it bit for bit on the cases of tests/plp_ref_cases.py.
 *
 * Build: oracle/build_oracle.py (gcc -O2 -shared) -> oracle/_build/libpileup_oracle.so
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define OP_M 0
#define OP_I 1
#define OP_D 2
#define OP_N 3
#define OP_S 4
#define OP_H 5
#define OP_P 6
#define OP_EQ 7
#define OP_X 8

#define FEAT 18
#define FLANK 16              /* pileup_flanking_base_num, src/clair3_pileup.h:93 */
#define FETCH_EXPAND 1000     /* mpileup_expand_reference_region, src/clair3_pileup.h:63 */

/* src/clair3_pileup.h:96-101 */
static const int num2countbaseclair3[32] = {
    -1, 0, 1, -1, 2, -1, -1, -1, 3, -1, -1, -1, -1, -1, -1, -1,
    -1, 9, 10, -1, 11, -1, -1, -1, 12, -1, -1, -1, -1, -1, -1, -1,
};
/* src/clair3_pileup.h:57-62 */
static const int base2index[32] = {
    0, 0, 1, 0, 0, 0, 2, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
};
static const char plp_bases[] = "ACGT";

typedef struct {
    int k;              /* current reference-consuming operation, -1 = never processed */
    int64_t x;          /* reference position of its first base */
    int64_t y;          /* query position of its first base */
} cursor_t;

typedef struct {
    int is_del, is_refskip;
    int64_t indel;
    int64_t qpos;
} plp1_t;

static inline int consumes_ref(int op) { return op == OP_M || op == OP_D || op == OP_N || op == OP_EQ || op == OP_X; }
static inline int is_match(int op) { return op == OP_M || op == OP_EQ || op == OP_X; }

static int64_t ref_length(const uint32_t *cig, int64_t n) {
    int64_t l = 0;
    for (int64_t k = 0; k < n; ++k)
        if (consumes_ref(cig[k] & 15)) l += cig[k] >> 4;
    return l;
}

/* htslib resolve_cigar2: advance the cursor to `pos` (called for consecutive positions from the read's first one) and describe
 * what the read shows there. */
static void resolve(const uint32_t *cig, int64_t n, int64_t beg, int64_t pos, cursor_t *s, plp1_t *p) {
    int64_t k;
    if (s->k == -1) {
        s->x = beg;
        s->y = 0;
        for (k = 0; k < n; ++k) {
            int op = cig[k] & 15;
            int64_t l = cig[k] >> 4;
            if (consumes_ref(op)) break;
            if (op == OP_I || op == OP_S) s->y += l;
        }
        s->k = (int)k;
    } else {
        int64_t l = cig[s->k] >> 4;
        if (pos - s->x >= l) {
            if (is_match(cig[s->k] & 15)) s->y += l;
            s->x += l;
            for (k = s->k + 1; k < n; ++k) {
                int op = cig[k] & 15;
                int64_t l2 = cig[k] >> 4;
                if (consumes_ref(op)) break;
                if (op == OP_I || op == OP_S) s->y += l2;
            }
            s->k = (int)k;
        }
    }
    {
        int op = cig[s->k] & 15;
        int64_t l = cig[s->k] >> 4;
        p->is_del = 0;
        p->is_refskip = 0;
        p->indel = 0;
        if (s->x + l - 1 == pos && s->k + 1 < n) {
            int op2 = cig[s->k + 1] & 15;
            int64_t l2 = cig[s->k + 1] >> 4;
            if (op2 == OP_D && op != OP_D) {
                p->indel = -l2;
                for (k = s->k + 2; k < n; ++k) {
                    if ((cig[k] & 15) == OP_D) p->indel -= cig[k] >> 4;
                    else break;
                }
            } else if (op2 == OP_I) {
                p->indel = l2;
                for (k = s->k + 2; k < n; ++k) {
                    int o = cig[k] & 15;
                    if (o == OP_I) p->indel += cig[k] >> 4;
                    else if (o != OP_P) break;
                }
            } else if (op2 == OP_P && s->k + 2 < n) {
                int64_t l3 = 0;
                for (k = s->k + 2; k < n; ++k) {
                    int o = cig[k] & 15;
                    if (o == OP_I) l3 += cig[k] >> 4;
                    else if (o == OP_D || consumes_ref(o)) break;
                }
                if (l3 > 0) p->indel = l3;
            }
        }
        if (is_match(op)) {
            p->qpos = s->y + (pos - s->x);
        } else {
            p->is_del = 1;
            p->qpos = s->y;
            p->is_refskip = (op == OP_N);
        }
    }
}

static inline int nib_at(const uint8_t *seq, int64_t lq, int64_t i) {
    if (i < 0 || i >= lq) return 0;
    return (seq[i >> 1] >> ((~i & 1) << 2)) & 15;
}

/* a column's insertion-string counter (the reference uses three khash string counters, src/clair3_pileup.c:245-247) */
typedef struct {
    int64_t len;
    uint8_t *nibs;
    int64_t cnt_f, cnt_r;
} ins_t;


/* ---- all_alt_info text (src/clair3_pileup.c:391-450) ----------------------------------------------------------------------------
 * The insertion alleles are printed in the ITERATION ORDER of the reference's khash string counter ins_counts_all, i.e. by bucket.
 * khash (klib, vendored as src/khash.h) restated for an insert-only table: X31 string hash (:395-400), n_buckets a power of two >= 4,
 * triangular probing i = (i + ++step) & mask (:329), growth to the next power of two whenever n_occupied >= 0.77 * n_buckets at the
 * START of EVERY put (:310-318), and the in-place "kick-out" rehash of kh_resize (:268-292).  What matters is the order of first
 * occurrence of the distinct keys, and whether a put of a present key came after the last new one: that put does not move a key
 * itself, but it still grows a full table first (3, 6, 12, 25, 49 ... keys). */
typedef struct {
    uint32_t n, size, upper;
    int *slot;              /* bucket -> key index, -1 = empty */
} khs_t;

static uint32_t x31(const uint8_t *nibs, int64_t len) {
    static const char nt16[] = "=ACMGRSVTWYHKDBN";
    if (len == 0) return 0;
    uint32_t h = (uint32_t)nt16[nibs[0]];
    for (int64_t i = 1; i < len; ++i) h = (h << 5) - h + (uint32_t)nt16[nibs[i]];
    return h;
}

static void khs_resize(khs_t *h, uint32_t want, const uint32_t *hashes) {
    uint32_t nn = want;
    --nn; nn |= nn >> 1; nn |= nn >> 2; nn |= nn >> 4; nn |= nn >> 8; nn |= nn >> 16; ++nn;
    if (nn < 4) nn = 4;
    if (h->size >= (uint32_t)(nn * 0.77 + 0.5)) return;
    int *slot = (int *)malloc(sizeof(int) * nn);
    uint8_t *newf = (uint8_t *)calloc(nn, 1);                 /* new_flags: 1 = taken */
    uint8_t *oldocc = (uint8_t *)calloc(nn, 1);               /* old flags: 1 = still holds an element to move */
    for (uint32_t j = 0; j < nn; ++j) slot[j] = -1;
    for (uint32_t j = 0; j < h->n; ++j) { slot[j] = h->slot[j]; oldocc[j] = h->slot[j] >= 0; }
    uint32_t mask = nn - 1;
    for (uint32_t j = 0; j < h->n; ++j) {
        if (!oldocc[j]) continue;
        int key = slot[j];
        oldocc[j] = 0;
        slot[j] = -1;
        for (;;) {
            uint32_t i = hashes[key] & mask, step = 0;
            while (newf[i]) i = (i + (++step)) & mask;
            newf[i] = 1;
            if (i < h->n && oldocc[i]) {                      /* kick out the element that still sits there */
                int tmp = slot[i];
                slot[i] = key;
                key = tmp;
                oldocc[i] = 0;
            } else {
                slot[i] = key;
                break;
            }
        }
    }
    free(h->slot); free(newf); free(oldocc);
    h->slot = slot;
    h->n = nn;
    h->upper = (uint32_t)(nn * 0.77 + 0.5);
}

/* order[0..n_keys): the key indices (first-occurrence order in, bucket order out).  put_after_last: a put of a present key came
 * after the last new one - kh_put still grows a full table first (:310-318), which changes the bucket order. */
static void khash_iteration_order(const uint32_t *hashes, int n_keys, int put_after_last, int *order) {
    khs_t h = {0, 0, 0, NULL};
    for (int key = 0; key < n_keys; ++key) {
        if (h.size >= h.upper) khs_resize(&h, h.n + 1, hashes);
        uint32_t mask = h.n - 1, i = hashes[key] & mask, step = 0;
        while (h.slot[i] >= 0) i = (i + (++step)) & mask;     /* distinct keys: never equal to a present one */
        h.slot[i] = key;
        ++h.size;
    }
    if (put_after_last && h.size >= h.upper) khs_resize(&h, h.n + 1, hashes);
    int k = 0;
    for (uint32_t j = 0; j < h.n; ++j)
        if (h.slot[j] >= 0) order[k++] = h.slot[j];
    free(h.slot);
}

typedef struct {
    char *buf;
    int64_t len, cap;
} text_t;

static void text_add(text_t *t, const char *s, int64_t n) {
    if (!t->buf) return;
    if (t->len + n + 1 > t->cap) { t->len = t->cap + 1; return; }        /* overflow: reported through the returned length */
    memcpy(t->buf + t->len, s, (size_t)n);
    t->len += n;
    t->buf[t->len] = 0;
}

typedef struct {
    int64_t min_depth;
    float min_snp_af, min_indel_af;
    int32_t min_mq, call_snp_only, call_ht, gvcf;
    int64_t max_indel_length;       /* only shapes the all_alt_info text (:411, :428) */
} plp_params_t;

/* Outputs (caller-allocated for W = end - start columns): matrix [W][18], major [W], stats [W][6] = depth, ref_count, alt_count,
 * del_count, ins_count, flags (bit 0 = candidate, bit 1 = all 18 features zero); cand_cols / cand_ok [W]; pos_ref_count /
 * pos_total_count [W] (only written with gvcf); win_bounds [W][2] (optional: each candidate's window rows [lo, hi) inside its
 * contiguous run).  Returns 0, or 1 on an allocation failure. */
int oracle_clair3_pileup(int64_t n_reads, const int64_t *rpos, const uint16_t *flag, const uint8_t *mapq,
                         const int64_t *cigar_off, const uint32_t *cigar, const int64_t *seq_off, const uint8_t *seq,
                         const int32_t *l_qseq, int64_t start, int64_t end, const char *ref_seq, int64_t ref_start, int64_t ref_len,
                         const plp_params_t *prm, int64_t *n_cols_out, int64_t *matrix, int64_t *major, int32_t *stats,
                         int64_t *cand_cols, uint8_t *cand_ok, int64_t *n_cand_out, int64_t *pos_ref_count,
                         int64_t *pos_total_count, char *alt_text, int64_t alt_cap, int64_t *alt_len, int64_t *win_bounds) {
    /* alt_text (optional): the all_alt_info strings of the candidates, one per line, in candidate order */
    text_t txt = {alt_text, 0, alt_cap};
    if (alt_text && alt_cap > 0) alt_text[0] = 0;
    int64_t W = end - start;
    *n_cols_out = 0;
    *n_cand_out = 0;
    if (W <= 0 || n_reads <= 0) return 0;
    cursor_t *cur = (cursor_t *)malloc(sizeof(cursor_t) * (size_t)n_reads);
    int64_t *rend = (int64_t *)malloc(sizeof(int64_t) * (size_t)n_reads);
    uint8_t *keep = (uint8_t *)malloc((size_t)n_reads);
    if (!cur || !rend || !keep) return 1;
    int64_t first = INT64_MAX;
    for (int64_t r = 0; r < n_reads; ++r) {
        cur[r].k = -1;
        /* src/medaka_bamiter.c:21-24: UNMAP 4 | SECONDARY 256 | QCFAIL 512 | DUP 1024 | SUPPLEMENTARY 2048, then mapq */
        keep[r] = !(flag[r] & (4 | 256 | 512 | 1024 | 2048)) && (int)mapq[r] >= prm->min_mq;
        rend[r] = rpos[r] + ref_length(cigar + cigar_off[r], cigar_off[r + 1] - cigar_off[r]);
        if (rend[r] <= rpos[r]) keep[r] = 0;
        if (keep[r] && rpos[r] < first) first = rpos[r];
    }
    int64_t n_cols = 0, n_cand = 0;
    int64_t pre_pos = 0, contiguous = 0;
    int64_t lo = 0; /* reads before lo ended before the current column */
    if (prm->gvcf) {
        memset(pos_ref_count, 0, sizeof(int64_t) * (size_t)W);
        memset(pos_total_count, 0, sizeof(int64_t) * (size_t)W);
    }
    for (int64_t pos = first; pos < end && first != INT64_MAX; ++pos) {
        int64_t n_plp = 0;
        int64_t m[FEAT];
        memset(m, 0, sizeof(m));
        int64_t depth = 0, quirk = 0;
        int64_t del_cap = 32, *dels_f = NULL, *dels_r = NULL;
        ins_t *ins = NULL;
        int64_t n_ins = 0, cap_ins = 0;
        int ins_again = 0;          /* the latest insertion put was of a string already present */
        int in_region = pos >= start;
        if (in_region) {
            dels_f = (int64_t *)calloc((size_t)del_cap, sizeof(int64_t));
            dels_r = (int64_t *)calloc((size_t)del_cap, sizeof(int64_t));
        }
        while (lo < n_reads && (!keep[lo] || rend[lo] <= pos)) ++lo;
        for (int64_t r = lo; r < n_reads && rpos[r] <= pos; ++r) {
            if (!keep[r] || rend[r] <= pos) continue;
            plp1_t p;
            const uint32_t *cig = cigar + cigar_off[r];
            resolve(cig, cigar_off[r + 1] - cigar_off[r], rpos[r], pos, &cur[r], &p);
            ++n_plp;
            if (!in_region) continue;
            if (p.is_refskip) continue;                                        /* src/clair3_pileup.c:251 */
            int rev = (flag[r] & 16) != 0;
            if (p.indel < 0) {                                                   /* :253-272 */
                int64_t d = -p.indel;
                if (d >= del_cap) {
                    int64_t nc = d > 2 * del_cap ? d : 2 * del_cap;
                    dels_f = (int64_t *)realloc(dels_f, sizeof(int64_t) * (size_t)nc);
                    dels_r = (int64_t *)realloc(dels_r, sizeof(int64_t) * (size_t)nc);
                    memset(dels_f + del_cap, 0, sizeof(int64_t) * (size_t)(nc - del_cap));
                    memset(dels_r + del_cap, 0, sizeof(int64_t) * (size_t)(nc - del_cap));
                    del_cap = nc;
                }
                if (rev) dels_r[d - 1] += 1; else dels_f[d - 1] += 1;
            }
            const uint8_t *sq = seq + seq_off[r];
            int base_i;
            if (p.is_del) {                                                      /* :276-289 */
                base_i = rev ? 17 : 8;
            } else {
                int j = nib_at(sq, l_qseq[r], p.qpos) + (rev ? 16 : 0);
                base_i = num2countbaseclair3[j];
            }
            ++depth;
            if (base_i >= 0) m[base_i] += 1; else ++quirk;
            if (p.indel > 0) {                                                   /* :293-307 */
                int64_t f0 = p.is_del ? 0 : 1;
                int64_t L = p.indel, i;
                uint8_t *s = (uint8_t *)malloc((size_t)L);
                for (i = 0; i < L; ++i) s[i] = (uint8_t)nib_at(sq, l_qseq[r], p.qpos + f0 + i);
                for (i = 0; i < n_ins; ++i)
                    if (ins[i].len == L && memcmp(ins[i].nibs, s, (size_t)L) == 0) break;
                if (i == n_ins) {
                    if (n_ins == cap_ins) {
                        cap_ins = cap_ins ? 2 * cap_ins : 8;
                        ins = (ins_t *)realloc(ins, sizeof(ins_t) * (size_t)cap_ins);
                    }
                    ins[n_ins].len = L;
                    ins[n_ins].nibs = s;
                    ins[n_ins].cnt_f = ins[n_ins].cnt_r = 0;
                    ++n_ins;
                    ins_again = 0;
                } else {
                    free(s);
                    ins_again = 1;
                }
                if (rev) ins[i].cnt_r += 1; else ins[i].cnt_f += 1;
            }
        }
        if (!in_region || n_plp == 0) {        /* htslib reports only covered columns; the reference skips pos < start (:221) */
            for (int64_t i = 0; i < n_ins; ++i) free(ins[i].nibs);
            free(ins); free(dels_f); free(dels_r);
            continue;
        }
        if (pre_pos + 1 != pos || pre_pos == 0) contiguous = 0; else ++contiguous;      /* :227-231 */
        pre_pos = pos;
        /* the -1 quirk: this column's non-ACGT read bases were added to the previous emitted column's feature 17 */
        if (quirk && n_cols > 0) matrix[(n_cols - 1) * FEAT + 17] += quirk;
        int64_t del_count = 0, ins_count = 0, all, best;
        all = best = 0;
        for (int64_t i = 0; i < del_cap; ++i) { all += dels_f[i]; if (dels_f[i] > best) best = dels_f[i]; }   /* :312-322 */
        m[6] = all; m[7] = best; del_count += all;
        all = best = 0;
        for (int64_t i = 0; i < del_cap; ++i) { all += dels_r[i]; if (dels_r[i] > best) best = dels_r[i]; }   /* :324-333 */
        m[15] = all; m[16] = best; del_count += all;
        all = best = 0;
        for (int64_t i = 0; i < n_ins; ++i) { all += ins[i].cnt_f; if (ins[i].cnt_f > best) best = ins[i].cnt_f; }   /* :337-341 */
        m[4] = all; m[5] = best; ins_count += all;
        all = best = 0;
        for (int64_t i = 0; i < n_ins; ++i) { all += ins[i].cnt_r; if (ins[i].cnt_r > best) best = ins[i].cnt_r; }   /* :344-348 */
        m[13] = all; m[14] = best; ins_count += all;

        int64_t off = pos - ref_start;
        char ref_base = (off >= 0 && off < ref_len) ? ref_seq[off] : 'N';
        if (ref_base >= 'a' && ref_base <= 'z') ref_base = (char)(ref_base - 32);
        int bi = ref_base - 'A';
        int rf = (bi >= 0 && bi < 32) ? base2index[bi] : 0;
        int rr = rf + 9;
        char major_alt = '\0';
        int64_t fsum = 0, rsum = 0, ref_count = 0, alt_count = 0, all_alt = 0;
        for (int i = 0; i < 4; ++i) {                                            /* :353-366 */
            fsum += m[i];
            rsum += m[i + 9];
            if (i == rf) {
                ref_count = m[i] + m[i + 9];
            } else {
                int64_t c = m[i] + m[i + 9];
                if (c > alt_count) { alt_count = c; major_alt = plp_bases[i]; all_alt += alt_count; }
            }
        }
        m[rf] = -fsum;                                                           /* :368-369 */
        m[rr] = -rsum;
        if (depth < 1) depth = 1;
        int pass_min_depth = depth >= prm->min_depth;
        int ref_acgt = ref_base == 'A' || ref_base == 'C' || ref_base == 'G' || ref_base == 'T';
        int nonref_major = ref_count < alt_count || ref_count < ins_count || ref_count < del_count;
        int equal_major = ref_count > 0 && ref_count == alt_count && (ref_base - major_alt) < 0;
        int pass_af;
        if (prm->call_snp_only) {
            pass_af = alt_count / (float)depth >= prm->min_snp_af;
        } else {
            pass_af = nonref_major || equal_major || (alt_count / (float)depth >= prm->min_snp_af);
            pass_af = pass_af || (del_count / (float)depth >= prm->min_indel_af) || (ins_count / (float)depth >= prm->min_indel_af);
        }
        pass_af = pass_af && pass_min_depth && ref_acgt;
        if (!prm->call_ht) pass_af = pass_af && contiguous >= FLANK;
        if (pass_af && txt.buf) {                                               /* :391-450 */
            char tmp[96];
            int64_t ref_depth = ref_count;
            int n = snprintf(tmp, sizeof tmp, "%lld-%lld-%c-", (long long)(pos + 1), (long long)depth, ref_base);
            text_add(&txt, tmp, n);
            for (int i = 0; i < 4; ++i) {
                int64_t alt_sum = m[i] + m[i + 9];
                if (alt_sum > 0 && i != rf) { n = snprintf(tmp, sizeof tmp, "X%c %lld ", plp_bases[i], (long long)alt_sum); text_add(&txt, tmp, n); }
            }
            for (int64_t i = 0; i < del_cap; ++i) {
                int64_t d = dels_f[i] + dels_r[i];
                ref_depth -= d;
                if (d > 0 && i + 1 <= prm->max_indel_length) {
                    text_add(&txt, "D", 1);
                    for (int64_t q = 0; q <= i; ++q) {                          /* "%.*s" of ref_seq + offset + 1: raw case, stops at the end */
                        int64_t o = off + 1 + q;                                /* of the contig or of the fetch, end + 1000 inclusive (:188-190) */
                        if (o < 0 || o >= ref_len || ref_seq[o] == 0 || ref_start + o > end + FETCH_EXPAND) break;
                        text_add(&txt, ref_seq + o, 1);
                    }
                    n = snprintf(tmp, sizeof tmp, " %lld ", (long long)d);
                    text_add(&txt, tmp, n);
                }
            }
            if (n_ins > 0) {
                uint32_t *hs = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)n_ins);
                int *order = (int *)malloc(sizeof(int) * (size_t)n_ins);
                for (int64_t i = 0; i < n_ins; ++i) hs[i] = x31(ins[i].nibs, ins[i].len);
                khash_iteration_order(hs, (int)n_ins, ins_again, order);
                for (int64_t q = 0; q < n_ins; ++q) {
                    const ins_t *e = &ins[order[q]];
                    int64_t val = e->cnt_f + e->cnt_r;
                    ref_depth -= val;
                    if (e->len <= prm->max_indel_length) {
                        static const char nt16[] = "=ACMGRSVTWYHKDBN";
                        tmp[0] = 'I'; tmp[1] = ref_base;
                        text_add(&txt, tmp, 2);
                        for (int64_t b = 0; b < e->len; ++b) text_add(&txt, &nt16[e->nibs[b]], 1);
                        n = snprintf(tmp, sizeof tmp, " %lld ", (long long)val);
                        text_add(&txt, tmp, n);
                    }
                }
                free(hs); free(order);
            }
            if (ref_depth > 0) { n = snprintf(tmp, sizeof tmp, "R%c %lld ", ref_base, (long long)ref_depth); text_add(&txt, tmp, n); }
            text_add(&txt, "\n", 1);
        }
        int zero = 1;
        for (int i = 0; i < FEAT; ++i) { matrix[n_cols * FEAT + i] = m[i]; if (m[i]) zero = 0; }
        major[n_cols] = pos;
        stats[n_cols * 6 + 0] = (int32_t)depth;
        stats[n_cols * 6 + 1] = (int32_t)ref_count;
        stats[n_cols * 6 + 2] = (int32_t)alt_count;
        stats[n_cols * 6 + 3] = (int32_t)del_count;
        stats[n_cols * 6 + 4] = (int32_t)ins_count;
        stats[n_cols * 6 + 5] = (pass_af ? 1 : 0) | (zero ? 2 : 0);
        if (pass_af) cand_cols[n_cand++] = n_cols;
        if (prm->gvcf) {
            pos_ref_count[pos - start] = ref_count;
            pos_total_count[pos - start] = ref_count + all_alt + del_count + ins_count;
        }
        ++n_cols;
        for (int64_t i = 0; i < n_ins; ++i) free(ins[i].nibs);
        free(ins); free(dels_f); free(dels_r);
    }
    /* the quirk may have made a previously all-zero row non-zero (or the reverse cannot happen): recompute the zero flags */
    for (int64_t c = 0; c < n_cols; ++c) {
        int zero = 1;
        for (int i = 0; i < FEAT; ++i) if (matrix[c * FEAT + i]) zero = 0;
        stats[c * 6 + 5] = (stats[c * 6 + 5] & 1) | (zero ? 2 : 0);
    }
    /* The candidate loop of preprocess/CreateTensorPileupFromCffi.py:356-396 over the contiguous chunks of :180-236 (runs of
     * consecutive positions).  The candidate is on matrix row c, 1-based position pos = major[c] + 1; its run is looked at from
     * row c - 16 (lo) to row c + 18 (hi) at most.
     *   :358  start - 1 >= first and end <= last: the run covers row c - 16 and reaches row c + 18, two rows past the window;
     *   :365  ... and none of the 33 rows is all-zero.
     * With call_ht (:370-396), when that fails:
     *   :371  pos > last: a candidate on the run's last row is skipped;
     *   :374  head: the run starts after row c - 16 and reaches row c + 16 - zero rows in front, no all-zero test;
     *   :384  tail: the run covers row c - 16 and ends before row c + 18 - zero rows behind (from row c + 16 on, none), no test.
     * win_bounds (optional) [n_cand][2]: the window rows [lo, hi) that belong to the run; the others are the reference's zeros. */
    for (int64_t j = 0; j < n_cand; ++j) {
        int64_t c = cand_cols[j], lo = c, hi = c;
        while (lo > c - FLANK && lo > 0 && major[lo - 1] == major[lo] - 1) --lo;
        while (hi < c + FLANK + 2 && hi + 1 < n_cols && major[hi + 1] == major[hi] + 1) ++hi;
        int head_full = lo == c - FLANK;
        int ok;
        if (head_full && hi == c + FLANK + 2) {
            ok = 1;
            for (int64_t q = c - FLANK; ok && q <= c + FLANK; ++q)
                if (stats[q * 6 + 5] & 2) ok = 0;
        } else if (prm->call_ht) {
            ok = hi > c && (head_full || hi >= c + FLANK);
        } else {
            ok = 0;
        }
        cand_ok[j] = (uint8_t)ok;
        if (win_bounds) {
            win_bounds[2 * j] = lo;
            win_bounds[2 * j + 1] = (hi < c + FLANK ? hi : c + FLANK) + 1;
        }
    }
    *n_cols_out = n_cols;
    *n_cand_out = n_cand;
    if (alt_len) *alt_len = txt.len;
    free(cur); free(rend); free(keep);
    return 0;
}
