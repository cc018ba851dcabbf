/*
 * clair3_b200_phase.h - C-ABI of read-based phasing in libclair3b200.so (DESIGN.md 5g.3): the allele observations of device-
 * resident alignment records at a contig's heterozygous SNPs, and the all-heterozygous weighted minimum-error-correction DP over
 * phase blocks, with its backtrace, on the GPU.  clair3_b200/phasing.py states both; clair3_b200/phase_gpu.py drives them.
 *
 * No workspace: every array is device memory the caller allocated, and each call is queued on cuda_stream.  Same conventions
 * as clair3_b200.h: int status, 0 = ok, message via c3b_last_error(); no CPU fallback.
 */
#ifndef CLAIR3_B200_PHASE_H
#define CLAIR3_B200_PHASE_H

#include <stddef.h>
#include <stdint.h>

#include "clair3_b200_fa.h"

#ifdef __cplusplus
extern "C" {
#endif

#define C3B_PHASE_MAX_READS 15      /* reads active at one column: the read selection's coverage cap                           */
#define C3B_PHASE_SEGMENT 128       /* DP columns per backtrace segment                                                         */

/* The variants of one contig, device memory: 0-based positions ascending, REF and ALT as nt16 codes (A 1, C 2, G 4, T 8). */
typedef struct c3b_phase_variants {
    int64_t n;
    const int64_t *pos;
    const uint8_t *ref;
    const uint8_t *alt;
} c3b_phase_variants;

/* Counts the allele observations of the records whose pos lies in [lo, hi): one warp per record, walking its CIGAR against
 * the variant positions by binary search.  Records must carry their qualities (qual / qual_off).  The records are checked
 * first (records_check.cuh) and the call waits for that check.  A record that is unmapped, secondary, QC-fail, duplicate or
 * supplementary, or has MAPQ < 20, or shows fewer than two alleles, counts 0.
 *   offsets   [n_reads + 1] int64 device: each record's first entry, exclusive sum of the counts
 * Waits for the stream and returns the entry total in *n_entries and the index of the first record with pos >= lo in *first. */
int c3b_phase_count(const c3b_fa_records *records, int64_t lo, int64_t hi, const c3b_phase_variants *variants, int64_t *offsets,
                    int64_t *n_entries, int64_t *first, void *cuda_stream);

/* Writes the entries c3b_phase_count counted, ascending by record and variant, to out_read (record index - first + read_base,
 * int64), out_var (variant index, int32), out_allele (0 REF / 1 ALT) and out_weight (base quality).  Same records, lo, hi,
 * variants and offsets as the count; no host wait. */
int c3b_phase_write(const c3b_fa_records *records, int64_t lo, int64_t hi, const c3b_phase_variants *variants,
                    const int64_t *offsets, int64_t first, int64_t read_base, int64_t *out_read, int32_t *out_var,
                    uint8_t *out_allele, uint8_t *out_weight, void *cuda_stream);

/* The blocks of a contig (clair3_b200/phasing.py Layout), device memory.  Block b: columns [col_off[b], col_off[b + 1]) and
 * reads [read_off[b], read_off[b + 1]) ordered by (first column, id), each with its first / last column within the block;
 * column c: entries [ent_off[c], ent_off[c + 1]) with the block-local read, allele and weight.  Checkpoint slots: block b
 * keeps one DP column per C3B_PHASE_SEGMENT columns but its last in ckpt[ckpt_off[b] ..], 2^(kmax_b - 1) words each, with
 * kmax_b its most active reads at one column. */
typedef struct c3b_phase_blocks {
    int64_t n_blocks;
    int64_t n_cols;
    const int64_t *col_off;       /* [n_blocks + 1]                                                                           */
    const int64_t *read_off;      /* [n_blocks + 1]                                                                           */
    const int32_t *kmax;          /* [n_blocks]                                                                               */
    const int64_t *ckpt_off;      /* [n_blocks]                                                                               */
    const int32_t *read_first;    /* [n_reads]                                                                                */
    const int32_t *read_last;     /* [n_reads]                                                                                */
    const int64_t *ent_off;       /* [n_cols + 1]                                                                             */
    const int32_t *ent_read;      /* [n_entries]                                                                              */
    const uint8_t *ent_allele;    /* [n_entries]                                                                              */
    const uint8_t *ent_weight;    /* [n_entries]                                                                              */
    const int64_t *order;         /* [n_blocks] the order in which the CTAs take the blocks (largest first)                   */
} c3b_phase_blocks;

/* Solves every block, one CTA per block at a time over n_ctas persistent CTAs, and backtracks on the device:
 *   hap       [n_cols] uint8: haplotype 0's allele at each column (0 at each block's first column)
 *   cost      [n_blocks] int64: each block's optimal cost
 *   ckpt      uint32: the checkpoint slots (ckpt_off's total)
 *   seg       uint16 [n_ctas * C3B_PHASE_SEGMENT * seg_stride]: each CTA's predecessor table of one segment, seg_stride >=
 *             2^(kmax - 1) for every block
 *   meta      uint16 [4 * n_cols], ebit uint8 [n_entries]: each column's active-set shape and each entry's bit
 *   status    int64 [1]: 0, or the (block + 1) of a block whose columns break the stated bounds
 * No host wait. */
int c3b_phase_dp(const c3b_phase_blocks *blocks, int n_ctas, uint8_t *hap, int64_t *cost, uint32_t *ckpt, uint16_t *seg,
                 int64_t seg_stride, uint16_t *meta, uint8_t *ebit, int64_t *status, void *cuda_stream);

/* Registers, shared memory and local memory of the DP kernel (cudaFuncGetAttributes), for its report. */
int c3b_phase_dp_attributes(int *registers, int64_t *shared_bytes, int64_t *local_bytes, int *max_threads);

#ifdef __cplusplus
}
#endif
#endif /* CLAIR3_B200_PHASE_H */
