/*
 * In-memory stand-in for the htslib calls of the reference's full-alignment tensor builder and pileup feature counter (see
 * htslib/sam.h, htslib/faidx.h and fa_ref_shim.h next to this file).  Written from the SAM/BAM specification and htslib's documented
 * pileup behaviour; no htslib code.  TEST INFRASTRUCTURE ONLY.
 *
 * The bindings (oracle/fa_ref.py, oracle/pileup_ref.py) register one contig (fa_ref_set_contig) and the decoded records of that
 * contig (fa_ref_set_records) before each call of calculate_clair3_full_alignment / calculate_clair3_pileup; every file / index /
 * header handle is a dummy that refers to them.
 */
#include <errno.h>
#include <limits.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "htslib/faidx.h"
#include "htslib/sam.h"

/* this file implements the shim, it must not be redirected by it */
#undef malloc
#undef calloc
#undef realloc
#undef free
#undef strdup
#undef rand

const char seq_nt16_str[] = "=ACMGRSVTWYHKDBN";

/* ------------------------------------------------------------------------------------------------ guarded allocator */
#define GUARD 4096

void *fa_ref_malloc(size_t n) {
    uint8_t *p = (uint8_t *)calloc(1, n + 2 * GUARD);
    if (!p) return NULL;
    memcpy(p, &n, sizeof(n));                 /* the size sits at the far end of the front guard */
    return p + GUARD;
}

void *fa_ref_calloc(size_t n, size_t size) { return fa_ref_malloc(n * size); }

void fa_ref_free(void *p) {
    if (p) free((uint8_t *)p - GUARD);
}

void *fa_ref_realloc(void *p, size_t n) {
    void *q = fa_ref_malloc(n);
    if (p && q) {
        size_t old;
        memcpy(&old, (uint8_t *)p - GUARD, sizeof(old));
        memcpy(q, p, old < n ? old : n);
        fa_ref_free(p);
    }
    return q;
}

char *fa_ref_strdup(const char *s) {
    size_t n = strlen(s) + 1;
    char *q = (char *)fa_ref_malloc(n);
    if (q) memcpy(q, s, n);
    return q;
}

static long long g_rand_draws = 0;

int fa_ref_rand(void) {
    ++g_rand_draws;
    return rand();
}

long long fa_ref_rand_draws(void) { return g_rand_draws; }
void fa_ref_reset_rand_draws(void) { g_rand_draws = 0; }

/* ------------------------------------------------------------------------------------------------ registered data */
static struct {
    int64_t n;
    const int64_t *pos;
    const uint16_t *flag;
    const uint8_t *mapq;
    const int64_t *cigar_off;
    const uint32_t *cigar;
    const int64_t *seq_off;
    const uint8_t *seq;
    const int32_t *l_qseq;
    const int64_t *qual_off;   /* may be NULL: qualities absent (0xFF, as the specification stores them) */
    const uint8_t *qual;
    const int64_t *qname_off;  /* may be NULL: read i is named "r<i>" */
    const char *qname;
    const int64_t *mv_off;     /* may be NULL: no read has an mv tag */
    const int32_t *mv;
} R;

static char *g_contig_name = NULL;
static const char *g_contig = NULL;
static int64_t g_contig_len = 0;

int fa_ref_set_contig(const char *name, const char *seq, int64_t len) {
    free(g_contig_name);
    g_contig_name = (char *)malloc(strlen(name) + 1);
    if (!g_contig_name) return 1;
    strcpy(g_contig_name, name);
    g_contig = seq;
    g_contig_len = len;
    return 0;
}

void fa_ref_set_records(int64_t n, const int64_t *pos, const uint16_t *flag, const uint8_t *mapq, const int64_t *cigar_off,
                        const uint32_t *cigar, const int64_t *seq_off, const uint8_t *seq, const int32_t *l_qseq,
                        const int64_t *qual_off, const uint8_t *qual, const int64_t *qname_off, const char *qname,
                        const int64_t *mv_off, const int32_t *mv) {
    R.n = n;
    R.pos = pos; R.flag = flag; R.mapq = mapq; R.cigar_off = cigar_off; R.cigar = cigar; R.seq_off = seq_off; R.seq = seq;
    R.l_qseq = l_qseq; R.qual_off = qual_off; R.qual = qual; R.qname_off = qname_off; R.qname = qname; R.mv_off = mv_off; R.mv = mv;
}

/* ------------------------------------------------------------------------------------------------ handles */
struct htsFile { int dummy; };
struct hts_idx_t { int dummy; };
struct faidx_t { int dummy; };
struct hts_itr_t { int64_t next; hts_pos_t beg, end; int tid; };

htsFile *sam_open(const char *fn, const char *mode) { (void)fn; (void)mode; return (htsFile *)calloc(1, sizeof(htsFile)); }
htsFile *hts_open(const char *fn, const char *mode) { return sam_open(fn, mode); }
int hts_set_opt(htsFile *fp, enum hts_fmt_option opt, ...) { (void)fp; (void)opt; return 0; }
hts_idx_t *sam_index_load(htsFile *fp, const char *fn) { (void)fp; (void)fn; return (hts_idx_t *)calloc(1, sizeof(hts_idx_t)); }

sam_hdr_t *sam_hdr_read(htsFile *fp) {
    (void)fp;
    sam_hdr_t *h = (sam_hdr_t *)calloc(1, sizeof(sam_hdr_t));
    if (!h) return NULL;
    const char *nm = g_contig_name ? g_contig_name : "";
    h->target_name = (char **)calloc(1, sizeof(char *));
    if (h->target_name) h->target_name[0] = (char *)malloc(strlen(nm) + 1);
    if (!h->target_name || !h->target_name[0]) { free(h->target_name); free(h); return NULL; }
    strcpy(h->target_name[0], nm);
    h->n_targets = 1;
    return h;
}

int bam_name2id(sam_hdr_t *h, const char *ref) { (void)h; return g_contig_name && strcmp(ref, g_contig_name) == 0 ? 0 : -1; }
void hts_itr_destroy(hts_itr_t *itr) { free(itr); }

void sam_hdr_destroy(sam_hdr_t *h) {
    if (!h) return;
    for (int32_t i = 0; i < h->n_targets; ++i) free(h->target_name[i]);
    free(h->target_name);
    free(h);
}
void hts_idx_destroy(hts_idx_t *idx) { free(idx); }
int hts_close(htsFile *fp) { free(fp); return 0; }

hts_itr_t *sam_itr_queryi(const hts_idx_t *idx, int tid, hts_pos_t beg, hts_pos_t end) {
    (void)idx;
    hts_itr_t *it = (hts_itr_t *)calloc(1, sizeof(hts_itr_t));
    if (!it) return NULL;
    it->tid = tid; it->beg = beg; it->end = end; it->next = 0;
    return it;
}

static hts_pos_t ref_span(int64_t i) {
    hts_pos_t s = 0;
    for (int64_t k = R.cigar_off[i]; k < R.cigar_off[i + 1]; ++k) {
        const uint32_t op = R.cigar[k] & 0xf;
        if (op == BAM_CMATCH || op == BAM_CDEL || op == BAM_CREF_SKIP || op == BAM_CEQUAL || op == BAM_CDIFF) s += R.cigar[k] >> 4;
    }
    return s;
}

/* The specification's record layout: read name (NUL-terminated, NUL-padded to a multiple of 4 so that the CIGAR is aligned),
 * CIGAR words, packed sequence, qualities, auxiliary fields (here only "mv", type B, subtype i). */
static int fill_record(bam1_t *b, int64_t i) {
    char name[32];
    const char *nm;
    size_t nlen;
    if (R.qname_off) {
        nm = R.qname + R.qname_off[i];
        nlen = (size_t)(R.qname_off[i + 1] - R.qname_off[i]);
    } else {
        nlen = (size_t)snprintf(name, sizeof(name), "r%lld", (long long)i);
        nm = name;
    }
    const size_t l_qname = (nlen + 1 + 3) & ~(size_t)3;
    const uint32_t n_cigar = (uint32_t)(R.cigar_off[i + 1] - R.cigar_off[i]);
    const int32_t lq = R.l_qseq[i];
    const size_t l_seq = (size_t)(lq + 1) / 2;
    const int64_t n_mv = R.mv_off ? R.mv_off[i + 1] - R.mv_off[i] : 0;
    const size_t l_aux = n_mv > 0 ? 2 + 1 + 1 + 4 + 4 * (size_t)n_mv : 0;
    const size_t need = l_qname + 4 * (size_t)n_cigar + l_seq + (size_t)lq + l_aux;
    if (need > b->m_data) {
        uint8_t *d = (uint8_t *)realloc(b->data, need);
        if (!d) return -1;
        b->data = d;
        b->m_data = (uint32_t)need;
    }
    uint8_t *p = b->data;
    memset(p, 0, l_qname);
    memcpy(p, nm, nlen);
    p += l_qname;
    memcpy(p, R.cigar + R.cigar_off[i], 4 * (size_t)n_cigar);
    p += 4 * (size_t)n_cigar;
    memcpy(p, R.seq + R.seq_off[i], l_seq);
    p += l_seq;
    if (R.qual_off) memcpy(p, R.qual + R.qual_off[i], (size_t)lq);
    else memset(p, 0xff, (size_t)lq);
    p += lq;
    if (n_mv > 0) {
        const uint32_t cnt = (uint32_t)n_mv;
        *p++ = 'm'; *p++ = 'v'; *p++ = 'B'; *p++ = 'i';
        memcpy(p, &cnt, 4);
        p += 4;
        memcpy(p, R.mv + R.mv_off[i], 4 * (size_t)n_mv);
        p += 4 * (size_t)n_mv;
    }
    b->l_data = (int)need;
    b->core.tid = 0;
    b->core.pos = R.pos[i];
    b->core.qual = R.mapq[i];
    b->core.flag = R.flag[i];
    b->core.l_qname = (uint16_t)l_qname;
    b->core.l_extranul = (uint8_t)(l_qname - nlen - 1);
    b->core.n_cigar = n_cigar;
    b->core.l_qseq = lq;
    b->core.mtid = -1;
    b->core.mpos = -1;
    b->core.isize = 0;
    return 0;
}

int sam_itr_next(htsFile *fp, hts_itr_t *itr, bam1_t *b) {
    (void)fp;
    if (!itr || itr->tid != 0) return -1;
    while (itr->next < R.n) {
        const int64_t i = itr->next++;
        if (R.pos[i] >= itr->end) return -1;                 /* coordinate-sorted: nothing further overlaps */
        hts_pos_t span = ref_span(i);
        if (span < 1) span = 1;                              /* a record without reference-consuming operations covers one base */
        if (R.pos[i] + span <= itr->beg) continue;
        if (fill_record(b, i)) return -2;
        return 0;
    }
    return -1;
}

bam1_t *bam_init1(void) { return (bam1_t *)calloc(1, sizeof(bam1_t)); }

void bam_destroy1(bam1_t *b) {
    if (!b) return;
    free(b->data);
    free(b);
}

int sam_read1(htsFile *fp, sam_hdr_t *h, bam1_t *b) { (void)fp; (void)h; (void)b; return -1; }
int64_t bam_aux2i(const uint8_t *s) { (void)s; errno = EINVAL; return 0; }
char *bam_aux2Z(const uint8_t *s) { (void)s; errno = EINVAL; return NULL; }

hts_itr_t *sam_itr_querys(const hts_idx_t *idx, sam_hdr_t *hdr, const char *region) {
    (void)hdr;
    const char *colon = strrchr(region, ':');
    const size_t nlen = colon ? (size_t)(colon - region) : strlen(region);
    int beg, end;
    if (!g_contig_name || strlen(g_contig_name) != nlen || strncmp(region, g_contig_name, nlen) != 0) return NULL;
    hts_parse_reg(region, &beg, &end);
    return sam_itr_queryi(idx, 0, beg, end);
}

/* ------------------------------------------------------------------------------------------------ pileup engine
 * bam_mplp_* over ONE input, restated from htslib's documented pileup semantics (no htslib code):
 *   - records are pulled one at a time through the caller's callback (the reference's read_bam, which applies its own flag and
 *     MAPQ filters); they must come coordinate-sorted, and a record whose raw reference length (M/D/N/=/X) is 0 is dropped;
 *   - a read is on column pos iff beg <= pos < beg + raw reference length; only columns with at least one read are reported, in
 *     position order, reads in the order they were pulled; a column whose reads are all reference skips is still reported;
 *   - overlapping mates are NOT removed (the reference never calls bam_mplp_init_overlaps);
 *   - the operation under a column is located afresh from the start of the CIGAR: x / y = reference / query offset of its first
 *     base (I and S advance y before it, M/=/X advance both, D/N only x);
 *   - on M/=/X: qpos = y + (pos - x); on D or N: is_del = 1 and qpos = y; is_refskip = 1 on N;
 *   - on the LAST base of an operation the next one is peeked: D, when the current one is not a D, gives indel = -(the run of
 *     adjacent D's); I gives indel = +(the I's that follow, merged across P); P gives +(the I's after the pads, up to the next
 *     reference-consuming operation), or 0 when there are none;
 *   - the depth cap (bam_mplp_set_maxcnt) is asserted, not modelled: reaching it is an error.
 * CIGAR operations of length 0 are rejected (htslib's incremental cursor can stop on them; a fresh location steps over them). */
typedef struct {
    bam1_t b;
    hts_pos_t beg, end;
} plp_read_t;

struct bam_mplp_s {
    bam_plp_auto_f func;
    void *data;
    int maxcnt;
    plp_read_t *rd;            /* reads that may still cover the next column, in the order they were pulled */
    int n, cap;
    bam1_t next;               /* one record of lookahead */
    int have_next, eof, error;
    hts_pos_t pos, last_beg;
    bam_pileup1_t *plp;
    int plp_cap;
};

static int consumes_ref(int op) { return op == BAM_CMATCH || op == BAM_CDEL || op == BAM_CREF_SKIP || op == BAM_CEQUAL || op == BAM_CDIFF; }
static int is_match_op(int op) { return op == BAM_CMATCH || op == BAM_CEQUAL || op == BAM_CDIFF; }

bam_mplp_t bam_mplp_init(int n, bam_plp_auto_f func, void **data) {
    if (n != 1) { fprintf(stderr, "hts_stub: bam_mplp_init supports one input, not %d\n", n); return NULL; }
    bam_mplp_t m = (bam_mplp_t)calloc(1, sizeof(struct bam_mplp_s));
    if (!m) return NULL;
    m->func = func;
    m->data = data[0];
    m->maxcnt = 8000;
    m->last_beg = -1;
    return m;
}

void bam_mplp_set_maxcnt(bam_mplp_t m, int maxcnt) { m->maxcnt = maxcnt; }

void bam_mplp_destroy(bam_mplp_t m) {
    if (!m) return;
    for (int i = 0; i < m->n; ++i) free(m->rd[i].b.data);
    free(m->rd);
    free(m->next.data);
    free(m->plp);
    free(m);
}

/* pull the next record with a non-zero reference length into the lookahead; 0 = none left, -1 = error */
static int pull(bam_mplp_t m) {
    while (!m->eof) {
        int ret = m->func(m->data, &m->next);
        if (ret < 0) { m->eof = 1; break; }
        const uint32_t *cig = bam_get_cigar(&m->next);
        hts_pos_t rlen = 0;
        for (uint32_t k = 0; k < m->next.core.n_cigar; ++k) {
            if (bam_cigar_oplen(cig[k]) == 0) { fprintf(stderr, "hts_stub: zero-length CIGAR operation\n"); return -1; }
            if (consumes_ref(bam_cigar_op(cig[k]))) rlen += bam_cigar_oplen(cig[k]);
        }
        if (m->next.core.pos < m->last_beg) { fprintf(stderr, "hts_stub: records are not coordinate-sorted\n"); return -1; }
        m->last_beg = m->next.core.pos;
        if (rlen == 0) continue;
        m->have_next = 1;
        return 1;
    }
    return 0;
}

/* move the lookahead record into the set of active reads */
static int admit(bam_mplp_t m) {
    if (m->n == m->cap) {
        int nc = m->cap ? 2 * m->cap : 64;
        plp_read_t *r = (plp_read_t *)realloc(m->rd, sizeof(plp_read_t) * (size_t)nc);
        if (!r) return -1;
        m->rd = r;
        m->cap = nc;
    }
    plp_read_t *r = &m->rd[m->n];
    memset(r, 0, sizeof(*r));
    r->b = m->next;
    r->b.data = (uint8_t *)malloc(m->next.l_data > 0 ? (size_t)m->next.l_data : 1);
    if (!r->b.data) return -1;
    memcpy(r->b.data, m->next.data, (size_t)m->next.l_data);
    r->b.m_data = (uint32_t)(m->next.l_data > 0 ? m->next.l_data : 1);
    r->beg = m->next.core.pos;
    r->end = r->beg;
    const uint32_t *cig = bam_get_cigar(&r->b);
    for (uint32_t k = 0; k < r->b.core.n_cigar; ++k)
        if (consumes_ref(bam_cigar_op(cig[k]))) r->end += bam_cigar_oplen(cig[k]);
    ++m->n;
    m->have_next = 0;
    return 0;
}

/* what read b shows on column pos (beg <= pos < end) */
static void describe(bam1_t *b, hts_pos_t pos, bam_pileup1_t *p) {
    const uint32_t *cig = bam_get_cigar(b);
    const int n = (int)b->core.n_cigar;
    hts_pos_t x = b->core.pos, y = 0;
    int k;
    for (k = 0; k < n; ++k) {
        const int op = bam_cigar_op(cig[k]);
        const hts_pos_t l = bam_cigar_oplen(cig[k]);
        if (consumes_ref(op)) {
            if (pos < x + l) break;
            x += l;
            if (is_match_op(op)) y += l;
        } else if (op == BAM_CINS || op == BAM_CSOFT_CLIP) {
            y += l;
        }
    }
    const int op = bam_cigar_op(cig[k]);
    const hts_pos_t l = bam_cigar_oplen(cig[k]);
    memset(p, 0, sizeof(*p));
    p->b = b;
    p->cigar_ind = k;
    if (pos == x + l - 1 && k + 1 < n) {
        const int op2 = bam_cigar_op(cig[k + 1]);
        int j;
        if (op2 == BAM_CDEL && op != BAM_CDEL) {
            for (j = k + 1; j < n && bam_cigar_op(cig[j]) == BAM_CDEL; ++j) p->indel -= (int)bam_cigar_oplen(cig[j]);
        } else if (op2 == BAM_CINS) {
            for (j = k + 1; j < n && (bam_cigar_op(cig[j]) == BAM_CINS || bam_cigar_op(cig[j]) == BAM_CPAD); ++j)
                if (bam_cigar_op(cig[j]) == BAM_CINS) p->indel += (int)bam_cigar_oplen(cig[j]);
        } else if (op2 == BAM_CPAD) {
            for (j = k + 1; j < n && !consumes_ref(bam_cigar_op(cig[j])); ++j)
                if (bam_cigar_op(cig[j]) == BAM_CINS) p->indel += (int)bam_cigar_oplen(cig[j]);
        }
    }
    if (is_match_op(op)) {
        p->qpos = (int32_t)(y + (pos - x));
    } else {
        p->is_del = 1;
        p->qpos = (int32_t)y;
        p->is_refskip = op == BAM_CREF_SKIP;
    }
    p->is_head = pos == b->core.pos;
}

int bam_mplp_auto(bam_mplp_t m, int *tid, int *pos, int *n_plp, const bam_pileup1_t **plp) {
    if (m->error) return -1;
    for (;;) {
        if (!m->have_next && pull(m) < 0) { m->error = 1; return -1; }
        if (m->n == 0) {
            if (!m->have_next) return 0;
            if (m->pos < m->next.core.pos) m->pos = m->next.core.pos;         /* jump over the uncovered columns */
        }
        while (m->have_next && m->next.core.pos <= m->pos) {
            if (admit(m)) { m->error = 1; return -1; }
            if (pull(m) < 0) { m->error = 1; return -1; }
        }
        int w = 0;                                                            /* retire reads that ended before this column */
        for (int i = 0; i < m->n; ++i) {
            if (m->rd[i].end <= m->pos) free(m->rd[i].b.data);
            else m->rd[w++] = m->rd[i];
        }
        m->n = w;
        if (m->n == 0) continue;
        if (m->n >= m->maxcnt) { fprintf(stderr, "hts_stub: depth %d reaches the pileup cap %d\n", m->n, m->maxcnt); m->error = 1; return -1; }
        if (m->n > m->plp_cap) {
            bam_pileup1_t *q = (bam_pileup1_t *)realloc(m->plp, sizeof(bam_pileup1_t) * (size_t)m->n);
            if (!q) { m->error = 1; return -1; }
            m->plp = q;
            m->plp_cap = m->n;
        }
        for (int i = 0; i < m->n; ++i) describe(&m->rd[i].b, m->pos, &m->plp[i]);
        *tid = 0;
        *pos = (int)m->pos;
        *n_plp = m->n;
        plp[0] = m->plp;
        ++m->pos;
        return 1;
    }
}

const char *hts_parse_reg(const char *s, int *beg, int *end) {
    const char *colon = strrchr(s, ':');
    *beg = 0;
    *end = INT_MAX;
    if (!colon) return s + strlen(s);
    long long a = 0, z = 0;
    const char *p = colon + 1;
    int have_a = 0, have_z = 0;
    for (; *p && *p != '-'; ++p)
        if (*p >= '0' && *p <= '9') { a = a * 10 + (*p - '0'); have_a = 1; }
    if (*p == '-')
        for (++p; *p; ++p)
            if (*p >= '0' && *p <= '9') { z = z * 10 + (*p - '0'); have_z = 1; }
    *beg = have_a && a > 0 ? (int)(a - 1) : 0;
    *end = have_z ? (int)z : INT_MAX;
    return colon;
}

/* ------------------------------------------------------------------------------------------------ auxiliary fields */
static size_t aux_type_size(uint8_t t) {
    switch (t) {
    case 'A': case 'c': case 'C': return 1;
    case 's': case 'S': return 2;
    case 'i': case 'I': case 'f': return 4;
    default: return 0;
    }
}

uint8_t *bam_aux_get(const bam1_t *b, const char tag[2]) {
    uint8_t *p = bam_get_aux(b), *e = b->data + b->l_data;
    while (p + 3 <= e) {
        const uint8_t t = p[2];
        if (p[0] == (uint8_t)tag[0] && p[1] == (uint8_t)tag[1]) return p + 2;
        if (t == 'B') {
            uint32_t cnt;
            memcpy(&cnt, p + 4, 4);
            p += 8 + (size_t)cnt * aux_type_size(p[3]);
        } else if (t == 'Z' || t == 'H') {
            p += 3;
            while (p < e && *p) ++p;
            ++p;
        } else {
            p += 3 + aux_type_size(t);
        }
    }
    return NULL;
}

uint32_t bam_auxB_len(const uint8_t *s) {
    uint32_t cnt;
    if (s[0] != 'B') return 0;
    memcpy(&cnt, s + 2, 4);
    return cnt;
}

int64_t bam_auxB2i(const uint8_t *s, uint32_t idx) {
    const uint8_t *d = s + 6;
    switch (s[1]) {
    case 'c': return (int8_t)d[idx];
    case 'C': return d[idx];
    case 's': { int16_t v; memcpy(&v, d + 2 * (size_t)idx, 2); return v; }
    case 'S': { uint16_t v; memcpy(&v, d + 2 * (size_t)idx, 2); return v; }
    case 'i': { int32_t v; memcpy(&v, d + 4 * (size_t)idx, 4); return v; }
    case 'I': { uint32_t v; memcpy(&v, d + 4 * (size_t)idx, 4); return v; }
    default: return 0;
    }
}

/* ------------------------------------------------------------------------------------------------ FASTA */
faidx_t *fai_load(const char *fn) { (void)fn; return (faidx_t *)calloc(1, sizeof(faidx_t)); }
void fai_destroy(faidx_t *fai) { free(fai); }

/* The caller frees the result with the reference's free(), i.e. through the shim: allocate it there too. */
char *faidx_fetch_seq(const faidx_t *fai, const char *c_name, int p_beg_i, int p_end_i, int *len) {
    (void)fai;
    if (!g_contig_name || strcmp(c_name, g_contig_name) != 0) { *len = -2; return NULL; }
    int64_t b = p_beg_i < 0 ? 0 : p_beg_i, e = p_end_i;
    if (e >= g_contig_len) e = g_contig_len - 1;
    int64_t n = e >= b ? e - b + 1 : 0;
    char *s = (char *)fa_ref_malloc((size_t)n + 1);
    if (!s) { *len = -1; return NULL; }
    if (n) memcpy(s, g_contig + b, (size_t)n);
    s[n] = '\0';
    *len = (int)n;
    return s;
}
