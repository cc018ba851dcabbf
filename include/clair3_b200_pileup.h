/*
 * clair3_b200_pileup.h - C-ABI of the GPU pileup feature counter in libclair3b200.so (SURVEY.md 8f, row N4, pileup half): the
 * per-column count matrix that feeds Clair3_P, built on the GPU from DECODED alignment records.
 *
 * Replaces (paths relative to HKU-BAL/Clair3)
 *     plp_data calculate_clair3_pileup(region, bam_set, fasta_path, min_depth, min_snp_af, min_indel_af, min_mq,
 *                                      max_indel_length, call_snp_only, max_depth, gvcf, call_ht)      src/clair3_pileup.c:142-476
 * as bound by preprocess/CreateTensorPileupFromCffi.py:60-75 and unpacked by _plp_data_to_numpy (:127-180) - from the point where
 * htslib has decoded the BAM records on: BGZF / BAM / CRAM decoding and the FASTA fetch stay on the CPU with htslib (not in this
 * image), the caller hands over what bam1_t carries.  What is counted, column by column, is exactly what the reference's loop
 * over bam_mplp_auto() counts (see oracle/pileup_oracle.c for the line-by-line restatement, quirks included).
 *
 * The all_alt_info strings (src/clair3_pileup.c:391-450) are text: the GPU exports the per-candidate allele lists
 * (c3b_plp_fetch_alleles) and the host shim formats them, byte for byte as the reference does.
 *
 * Same conventions as clair3_b200.h: int status, 0 = ok, message via c3b_last_error(); no CPU fallback.
 */
#ifndef CLAIR3_B200_PILEUP_H
#define CLAIR3_B200_PILEUP_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct c3b_plp c3b_plp;

/* A coordinate-sorted run of alignment records of ONE contig, fields as htslib lays them out in bam1_t
 * (the vendored public header src/sam.h: bam1_core_t, bam_get_cigar, bam_get_seq).  The library trusts the offsets: cigar_off and
 * seq_off must be non-decreasing, start at 0 and address cigar[] / seq[] in bounds, every packed sequence must hold
 * (l_qseq + 1) / 2 bytes (clair3_b200/pileup_counts.py: BamRecords checks all of this on the host). */
typedef struct c3b_bam_records {
    int64_t n_reads;
    const int64_t *pos;         /* [n]   bam1_core_t.pos: 0-based leftmost coordinate, ascending                         */
    const uint16_t *flag;       /* [n]   bam1_core_t.flag (0x10 = reverse strand; 0x4|0x100|0x200|0x400|0x800 are dropped,
                                         src/medaka_bamiter.c:21-22)                                                     */
    const uint8_t *mapq;        /* [n]   bam1_core_t.qual (dropped below min_mq, src/medaka_bamiter.c:24)                */
    const int64_t *cigar_off;   /* [n+1] first CIGAR word of read i in cigar[]                                            */
    const uint32_t *cigar;      /*       bam_get_cigar(): len << 4 | op, op = MIDNSHP=X                                   */
    const int64_t *seq_off;     /* [n+1] first BYTE of read i's packed sequence in seq[]                                  */
    const uint8_t *seq;         /*       bam_get_seq(): 4-bit nt16 codes, two per byte, high nibble first                 */
    const int32_t *l_qseq;      /* [n]   bam1_core_t.l_qseq                                                               */
} c3b_bam_records;

/* The arguments of calculate_clair3_pileup that shape the counts (max_indel_length only formats all_alt_info, max_depth is
 * unused by the reference's function body). */
typedef struct c3b_plp_params {
    int64_t min_depth;
    float min_snp_af;
    float min_indel_af;
    int32_t min_mq;
    int32_t call_snp_only;
    int32_t call_ht;            /* 1: no 16-column flanking requirement (src/clair3_pileup.c:385-387) */
    int32_t gvcf;               /* 1: also fill pos_ref_count / pos_total_count (:205-210, :453-456) */
    int32_t alt_info;           /* 1: also export every pre-candidate column's distinct indel alleles (c3b_plp_fetch_alleles), from
                                   which the host formats the all_alt_info text of :391-450 */
} c3b_plp_params;

/* A counting workspace on one device (scratch grows on demand; one call in flight per workspace). */
int c3b_plp_create(c3b_plp **out, int device_ordinal);

/* Counts region [start, end) (0-based, end-exclusive: what hts_parse_reg leaves at src/clair3_pileup.c:148-151).  ref_seq holds the
 * reference bases [ref_start, ref_start + ref_len) (the reference fetches start - 1000 .. end + 1000, :184-186).  on_device: the
 * pointers inside `reads` and ref_seq are device pointers; otherwise host memory, copied on cuda_stream.  Asynchronous on
 * cuda_stream; the results stay on the device until c3b_plp_sizes / c3b_plp_fetch. */
int c3b_plp_count(c3b_plp *w, const c3b_bam_records *reads, int on_device, int64_t start, int64_t end, const char *ref_seq,
                  int64_t ref_start, int64_t ref_len, const c3b_plp_params *params, void *cuda_stream);

/* Waits for the last c3b_plp_count and reports plp_data.n_cols (covered columns) and plp_data.candidates_num.  Fails if the
 * call overflowed a capacity (message says which). */
int c3b_plp_sizes(c3b_plp *w, int64_t *n_cols, int64_t *n_candidates);

/* Copies the results to host buffers (any pointer may be NULL):
 *   matrix       [n_cols][18] int64   plp_data.matrix (size_t counts; the two reference-base features hold -sum, :368-369)
 *   major        [n_cols]     int64   plp_data.major (0-based position of each column; minor is always 0, :240)
 *   stats        [n_cols][6]  int32   depth, ref_count, alt_count, del_count, ins_count, flags (bit 0: candidate = pass_af of
 *                                     :371-387; bit 1: all 18 features are zero)
 *   cand_cols    [n_cand]     int64   column index of every candidate, ascending (all_alt_info order)
 *   cand_ok      [n_cand]     uint8   1: the 33-column window around the candidate is complete, contiguous in position and has no
 *                                     all-zero column - the test of preprocess/CreateTensorPileupFromCffi.py:357-369
 *   pos_ref_count / pos_total_count [end - start] int64 (only with params.gvcf)                                  */
int c3b_plp_fetch(c3b_plp *w, int64_t *matrix, int64_t *major, int32_t *stats, int64_t *cand_cols, uint8_t *cand_ok,
                  int64_t *pos_ref_count, int64_t *pos_total_count);

/* The distinct indel alleles of every column that passed the allele-frequency test (needs params.alt_info), in order of first
 * occurrence - what the reference keeps per column in dels_f / dels_r and its three insertion-string counters:
 *   al_off / al_n [end - start] int32   first record and number of records of the column at position start + i (0 elsewhere)
 *   meta  [n]  uint32   insertion << 31 | reverse strand << 30 | length
 *   read  [n]  uint32   index (into the records of the count) of the first read that showed the allele
 *   qpos  [n]  uint32   query offset of its first inserted base in that read (insertions)
 *   cnt   [n]  uint32   reads of that strand showing it
 * Any pointer may be NULL; n_alleles alone sizes the buffers.  clair3_b200/pileup_counts.py formats the all_alt_info strings
 * (src/clair3_pileup.c:391-450, insertion alleles in the reference's khash bucket order) from these on the host. */
int c3b_plp_fetch_alleles(c3b_plp *w, int32_t *al_off, int32_t *al_n, uint32_t *meta, uint32_t *read, uint32_t *qpos, uint32_t *cnt,
                          int64_t capacity, int64_t *n_alleles);

/* Device views of the same results, valid until the next c3b_plp_count on w: matrix and window_starts
 * (= cand_cols - 16, the first row of every candidate's 33-row window) are exactly the `cols` / `starts` arguments of
 * c3b_forward_windows(..., cols_dtype C3B_DT_I64, on_device 1) in clair3_b200.h, so the counts never leave HBM on their way into
 * Clair3_P. */
int c3b_plp_device(c3b_plp *w, const int64_t **matrix, const int64_t **major, const int64_t **cand_cols,
                   const int64_t **window_starts, const uint8_t **cand_ok);

/* Device time of the last c3b_plp_count (CUDA events on its stream around all of its kernels, input copies excluded), and the
 * number of kernels it launched. */
int c3b_plp_last_ms(c3b_plp *w, float *ms, int *launches);

void c3b_plp_destroy(c3b_plp *w);

#ifdef __cplusplus
}
#endif
#endif /* CLAIR3_B200_PILEUP_H */
