/*
 * Minimal stand-in for the slice of htslib's SAM/BAM API that the reference's full-alignment tensor builder and pileup feature
 * counter use, written from the SAM/BAM format specification (section 4.2: the in-memory record is read name, CIGAR, 4-bit packed
 * sequence, qualities and auxiliary fields, back to back).  Alignment records are not read from a file: the Python bindings
 * (oracle/fa_ref.py, oracle/pileup_ref.py) register decoded records in memory, and the iterator hands back those that overlap the
 * queried region, in order.
 *
 * TEST INFRASTRUCTURE ONLY: this header exists so that the reference's own C can be compiled into oracle/_ref/ as a checker.
 */
#ifndef FA_REF_HTS_STUB_SAM_H
#define FA_REF_HTS_STUB_SAM_H

#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

typedef int64_t hts_pos_t;

typedef struct htsFile htsFile;
typedef struct hts_idx_t hts_idx_t;
typedef struct hts_itr_t hts_itr_t;
typedef struct sam_hdr_t sam_hdr_t;
typedef sam_hdr_t bam_hdr_t;
typedef htsFile samFile;

/* the header names the one registered contig (target id 0) */
struct sam_hdr_t {
    int32_t n_targets;
    char **target_name;
};

typedef struct bam1_core_t {
    hts_pos_t pos;
    int32_t tid;
    uint16_t bin;
    uint8_t qual;
    uint8_t l_extranul;
    uint16_t flag;
    uint16_t l_qname;
    uint32_t n_cigar;
    int32_t l_qseq;
    int32_t mtid;
    hts_pos_t mpos;
    hts_pos_t isize;
} bam1_core_t;

typedef struct bam1_t {
    bam1_core_t core;
    uint64_t id;
    uint8_t *data;
    int l_data;
    uint32_t m_data;
} bam1_t;

/* CIGAR operations, in the order of the specification's "MIDNSHP=X" */
#define BAM_CMATCH 0
#define BAM_CINS 1
#define BAM_CDEL 2
#define BAM_CREF_SKIP 3
#define BAM_CSOFT_CLIP 4
#define BAM_CHARD_CLIP 5
#define BAM_CPAD 6
#define BAM_CEQUAL 7
#define BAM_CDIFF 8
/* FLAG bits (specification section 1.4, column 2) */
#define BAM_FPAIRED 1
#define BAM_FPROPER_PAIR 2
#define BAM_FUNMAP 4
#define BAM_FMUNMAP 8
#define BAM_FREVERSE 16
#define BAM_FMREVERSE 32
#define BAM_FREAD1 64
#define BAM_FREAD2 128
#define BAM_FSECONDARY 256
#define BAM_FQCFAIL 512
#define BAM_FDUP 1024
#define BAM_FSUPPLEMENTARY 2048

#define bam_cigar_op(c) ((c) & 0xf)
#define bam_cigar_oplen(c) ((c) >> 4)
#define bam_is_rev(b) (((b)->core.flag & BAM_FREVERSE) != 0)
#define bam_get_qname(b) ((char *)(b)->data)
#define bam_get_cigar(b) ((uint32_t *)((b)->data + (b)->core.l_qname))
#define bam_get_seq(b) ((b)->data + (b)->core.l_qname + ((b)->core.n_cigar << 2))
#define bam_get_qual(b) ((b)->data + (b)->core.l_qname + ((b)->core.n_cigar << 2) + (((b)->core.l_qseq + 1) >> 1))
#define bam_get_aux(b) (bam_get_qual(b) + (b)->core.l_qseq)
#define bam_seqi(s, i) ((s)[(i) >> 1] >> ((~(i) & 1) << 2) & 0xf)

extern const char seq_nt16_str[];

enum hts_fmt_option { CRAM_OPT_REFERENCE = 1 };

htsFile *sam_open(const char *fn, const char *mode);
int hts_set_opt(htsFile *fp, enum hts_fmt_option opt, ...);
hts_idx_t *sam_index_load(htsFile *fp, const char *fn);
sam_hdr_t *sam_hdr_read(htsFile *fp);
int bam_name2id(sam_hdr_t *h, const char *ref);
hts_itr_t *sam_itr_queryi(const hts_idx_t *idx, int tid, hts_pos_t beg, hts_pos_t end);
int sam_itr_next(htsFile *fp, hts_itr_t *itr, bam1_t *b);
bam1_t *bam_init1(void);
void bam_destroy1(bam1_t *b);
void hts_itr_destroy(hts_itr_t *itr);
void sam_hdr_destroy(sam_hdr_t *h);
void hts_idx_destroy(hts_idx_t *idx);
int hts_close(htsFile *fp);
const char *hts_parse_reg(const char *s, int *beg, int *end);

uint8_t *bam_aux_get(const bam1_t *b, const char tag[2]);
uint32_t bam_auxB_len(const uint8_t *s);
int64_t bam_auxB2i(const uint8_t *s, uint32_t idx);

/* Link stubs for the reference's reader (src/medaka_bamiter.c): records only come through the region iterator, so sam_read1
 * reports end of file; the reference calls the aux conversions only when it filters by tag or read group, which it never does
 * here. */
htsFile *hts_open(const char *fn, const char *mode);
int sam_read1(htsFile *fp, sam_hdr_t *h, bam1_t *b);
int64_t bam_aux2i(const uint8_t *s);
char *bam_aux2Z(const uint8_t *s);

hts_itr_t *sam_itr_querys(const hts_idx_t *idx, sam_hdr_t *hdr, const char *region);
#define bam_itr_querys(idx, hdr, region) sam_itr_querys(idx, hdr, region)
#define bam_itr_destroy(iter) hts_itr_destroy(iter)

/* ---- the pileup engine (bam_mplp_*), one input only; the rules it follows are listed in hts_stub.c ---- */
typedef struct bam_pileup1_t {
    bam1_t *b;
    int32_t qpos;
    int indel, level;
    uint32_t is_del : 1, is_head : 1, is_tail : 1, is_refskip : 1, : 1, aux : 27;
    int cigar_ind;
} bam_pileup1_t;

typedef int (*bam_plp_auto_f)(void *data, bam1_t *b);
typedef struct bam_mplp_s *bam_mplp_t;

bam_mplp_t bam_mplp_init(int n, bam_plp_auto_f func, void **data);
void bam_mplp_set_maxcnt(bam_mplp_t iter, int maxcnt);
int bam_mplp_auto(bam_mplp_t iter, int *tid, int *pos, int *n_plp, const bam_pileup1_t **plp);
void bam_mplp_destroy(bam_mplp_t iter);

#endif
