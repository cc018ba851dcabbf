/*
 * clair3_b200_fa.h - C-ABI of the GPU full-alignment tensor builder in libclair3b200.so (SURVEY.md 8f, row N4, full-alignment
 * half): Clair3_F's int8 input tensor, built on the GPU from DECODED alignment records.
 *
 * Replaces (paths relative to HKU-BAL/Clair3)
 *     fa_data calculate_clair3_full_alignment(region, bam_path, fasta_path, variants, variant_num, candidates, candidate_num,
 *                                             need_haplotagging, min_mq, min_bq, matrix_depth, max_indel_length,
 *                                             enable_dwell_time)                         src/clair3_full_alignment_dwell.c:437-1054
 * as bound by preprocess/CreateTensorFullAlignmentFromCffi.py:120-134, from the point where htslib has decoded the records.  The
 * matrix is bit-exact with the reference on the same records (DESIGN.md 5b lists the inputs on which the reference itself is
 * undefined).  The all_alt_info strings are text: the GPU exports each candidate's depth, A/C/G/T counts and distinct indel
 * alleles (c3b_fa_fetch_alleles) and the host formats them (clair3_b200/fa_tensor.py).
 *
 * Same conventions as clair3_b200.h: int status, 0 = ok, message via c3b_last_error(); no CPU fallback.
 */
#ifndef CLAIR3_B200_FA_H
#define CLAIR3_B200_FA_H

#include <stddef.h>
#include <stdint.h>

#include "clair3_b200_pileup.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct c3b_fa c3b_fa;

/* The pileup record layout (c3b_bam_records, coordinate-sorted, one contig) plus the fields the full-alignment tensor reads.
 * Each pair is an [n+1] offset array and the concatenated values; a NULL offset array means the field is absent for every read. */
typedef struct c3b_fa_records {
    c3b_bam_records core;
    const int64_t *qual_off;    /* bam_get_qual(): l_qseq phred values per read; absent = 0xFF (no qualities, as BAM stores it)  */
    const uint8_t *qual;
    const int64_t *qname_off;   /* bam_get_qname() without the NUL; the reference keeps the first read of each name (:547-559);
                                   absent = every read has its own name                                                        */
    const uint8_t *qname;
    const int64_t *mv_off;      /* the "mv" B-array values, leading stride element included; an empty range = no tag          */
    const int32_t *mv;
} c3b_fa_records;

/* struct Variant (src/clair3_full_alignment_dwell.h:111-118): a phased heterozygous SNP; genotype 1 = 0|1, 2 = 1|0. */
typedef struct c3b_fa_variant {
    int32_t position;           /* 0-based */
    char ref_base;
    char alt_base;
    int32_t genotype;
    int32_t phase_set;
} c3b_fa_variant;

typedef struct c3b_fa_params {
    int32_t matrix_depth;       /* rows per candidate: 89 (ONT), 55 (HiFi / Illumina)                                         */
    int32_t need_haplotagging;  /* 1: tag reads with mapq >= 20 against the variants (:629-632)                               */
    int32_t min_mq;             /* reads below are dropped (:542)                                                            */
    int32_t dwell;              /* 1: 9 channels, channel 8 = per-base signal length from the mv tag (enable_dwell_time)      */
    uint32_t rand_seed;         /* the shuffle of candidates with more than matrix_depth reads uses glibc rand() (:117-134):   */
    int32_t reserved;           /* the stream after srand(rand_seed) and rand_skip draws; 1 / 0 = an unseeded process          */
    int64_t rand_skip;
} c3b_fa_params;

/* A workspace on one device (scratch grows on demand; one call in flight per workspace). */
int c3b_fa_create(c3b_fa **out, int device_ordinal);

/* Builds the tensor of n_cand candidates (0-based positions, strictly ascending).  variants: n_var phased SNPs sorted by position
 * (host memory, may be NULL when n_var = 0).  ref_seq holds the reference bases [ref_start, ref_start + ref_len).  on_device: the
 * record arrays and ref_seq are device pointers; otherwise host memory, copied on cuda_stream.  candidates and variants are
 * always host memory.  Asynchronous on cuda_stream, except for two waits that size the scratch: after the union of the candidate windows and
 * after the read pass. */
int c3b_fa_build(c3b_fa *w, const c3b_fa_records *records, int on_device, const int64_t *candidates, int64_t n_cand,
                 const c3b_fa_variant *variants, int64_t n_var, const char *ref_seq, int64_t ref_start, int64_t ref_len,
                 const c3b_fa_params *params, void *cuda_stream);

/* Waits for the last c3b_fa_build: candidates, reads kept (passed the filters, first of their name, overlapping a candidate
 * window: the reference's read_array) and glibc rand() draws consumed.  Fails if the call overflowed a capacity. */
int c3b_fa_sizes(c3b_fa *w, int64_t *n_cand, int64_t *n_kept, int64_t *rand_draws);

/* Copies results to host buffers (any pointer may be NULL):
 *   matrix          [n_cand][matrix_depth][33][8 | 9] int8   the full-alignment tensor (fa_data.matrix)
 *   kept_haplotype  [n_kept] int32   0 unphased, 1 / 2 haplotype, per kept read (diagnosis)
 *   kept_read       [n_kept] int64   record index of each kept read                                                         */
int c3b_fa_fetch(c3b_fa *w, int8_t *matrix, int32_t *kept_haplotype, int64_t *kept_read);

/* Per candidate, what the all_alt_info text (:950-1006) is made of:
 *   depth [n_cand] int32, acgt [n_cand][4] int32   reads covering the candidate (M or D) and their A/C/G/T counts (N counts as A)
 *   al_off / al_n [n_cand] int32                   first allele record and number of records of each candidate
 *   meta [n] uint32  insertion << 31 | again << 30 | length, again (set on the last allele of a kind only): a later read showed
 *                    an allele of that kind again, which still grows a full khash (khash.h:310-318);
 *   read [n] uint32  record index of the first read that showed the allele;
 *   qpos [n] uint32  query offset of its first inserted base (insertions);  cnt [n] uint32  reads showing it
 * Alleles are in order of first occurrence (deletions and insertions interleaved).  n_alleles alone sizes the buffers. */
int c3b_fa_fetch_alleles(c3b_fa *w, int32_t *depth, int32_t *acgt, int32_t *al_off, int32_t *al_n, uint32_t *meta, uint32_t *read,
                         uint32_t *qpos, uint32_t *cnt, int64_t capacity, int64_t *n_alleles);

/* The device matrix, valid until the next c3b_fa_build on w: pass it to c3b_forward(model, matrix, C3B_DT_I8, 1, n_cand,
 * matrix_depth, ...) so the tensor never leaves HBM on its way into Clair3_F. */
int c3b_fa_device(c3b_fa *w, const int8_t **matrix);

/* Device time of the last c3b_fa_build (CUDA events around its kernels, input copies excluded) and its kernel launches. */
int c3b_fa_last_ms(c3b_fa *w, float *ms, int *launches);

void c3b_fa_destroy(c3b_fa *w);

#ifdef __cplusplus
}
#endif
#endif /* CLAIR3_B200_FA_H */
