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
 * The all_alt_info strings (src/clair3_pileup.c:391-450) are formatted on the GPU as well (c3b_plp_alt_text), byte for byte as
 * the reference prints them, together with the form the decoder takes (c3b_decode_calls in clair3_b200.h): a region goes from
 * records to call records on one stream.  The per-candidate allele lists the text is made from can still be exported
 * (c3b_plp_fetch_alleles); clair3_b200/pileup_counts.py formats them on the host, which is what the tests hold the GPU text to.
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
    int32_t call_ht;            /* 1: no 16-column flanking requirement (src/clair3_pileup.c:385-387), and cand_ok keeps the head /
                                   tail windows of preprocess/CreateTensorPileupFromCffi.py:370-396 */
    int32_t gvcf;               /* 1: also fill pos_ref_count / pos_total_count (:205-210, :453-456) */
    int32_t alt_info;           /* 1: also keep every pre-candidate column's distinct indel alleles (c3b_plp_fetch_alleles), from
                                   which c3b_plp_alt_text formats the all_alt_info text of :391-450 */
} c3b_plp_params;

/* A counting workspace on one device (scratch grows on demand; one call in flight per workspace). */
int c3b_plp_create(c3b_plp **out, int device_ordinal);

/* Counts region [start, end) (0-based, end-exclusive: what hts_parse_reg leaves at src/clair3_pileup.c:148-151).  ref_seq holds the
 * reference bases [ref_start, ref_start + ref_len) (the reference fetches start - 1000 .. end + 1000, :184-186).  on_device: the
 * pointers inside `reads` and ref_seq are device pointers; otherwise host memory, copied on cuda_stream.  Asynchronous on
 * cuda_stream; the results stay on the device until c3b_plp_sizes / c3b_plp_fetch. */
int c3b_plp_count(c3b_plp *w, const c3b_bam_records *reads, int on_device, int64_t start, int64_t end, const char *ref_seq,
                  int64_t ref_start, int64_t ref_len, const c3b_plp_params *params, void *cuda_stream);

/* The targets of a run with a BED (--bed_fn) or a known-sites VCF (--vcf_fn) on one contig, as the reference's pileup step reads
 * them from the extended BED CheckEnvs writes (preprocess/CreateTensorPileupFromCffi.py:347-355; clair3_b200/targets.py builds
 * these arrays).  A candidate at 1-based position q is kept when some interval has starts[i] <= q <= ends[i] and, with known
 * sites, q is one of them.  Zero-length rows must already be [s, s + 1), as the reference's interval tree stores them. */
typedef struct c3b_plp_targets {
    int64_t n_intervals;
    const int64_t *starts;      /* [n_intervals] 0-based interval starts, ascending                                        */
    const int64_t *ends;        /* [n_intervals] end-exclusive ends, ends[i] >= starts[i]                                  */
    const int64_t *end_max;     /* [n_intervals] running maximum of ends[0..i]: one binary search over starts decides the test */
    int64_t n_sites;            /* -1: no known-site test; otherwise the number of known sites (0 keeps nothing)           */
    const int64_t *sites;       /* [n_sites] 1-based known positions, strictly ascending                                   */
    int32_t on_device;          /* 1: the arrays are device pointers, checked on the stream (c3b_plp_sizes reports a
                                   violation); 0: host arrays, checked here and copied on the call's stream               */
} c3b_plp_targets;

/* c3b_plp_count that keeps only the candidates inside `targets` (NULL: c3b_plp_count itself).  The matrix, major, stats (bit 0
 * still marks every candidate column before the target test), the allele export and the gVCF counts do not change; cand_cols,
 * cand_ok, the window starts and bounds, n_candidates and everything keyed by candidate after them (c3b_plp_alt_text, the
 * network, the decoder) cover only the kept candidates.  An empty target set is valid and keeps none.  The arrays must stay
 * alive until the count has been waited for. */
int c3b_plp_count_targeted(c3b_plp *w, const c3b_bam_records *reads, int on_device, int64_t start, int64_t end, const char *ref_seq,
                           int64_t ref_start, int64_t ref_len, const c3b_plp_params *params, const c3b_plp_targets *targets,
                           void *cuda_stream);

/* Waits for the last c3b_plp_count and reports plp_data.n_cols (covered columns) and plp_data.candidates_num.  Fails if the
 * call overflowed a capacity or was given device target arrays out of order (message says which). */
int c3b_plp_sizes(c3b_plp *w, int64_t *n_cols, int64_t *n_candidates);

/* Copies the results to host buffers (any pointer may be NULL):
 *   matrix       [n_cols][18] int64   plp_data.matrix (size_t counts; the two reference-base features hold -sum, :368-369)
 *   major        [n_cols]     int64   plp_data.major (0-based position of each column; minor is always 0, :240)
 *   stats        [n_cols][6]  int32   depth, ref_count, alt_count, del_count, ins_count, flags (bit 0: candidate = pass_af of
 *                                     :371-387; bit 1: all 18 features are zero)
 *   cand_cols    [n_cand]     int64   column index of every candidate, ascending (all_alt_info order)
 *   cand_ok      [n_cand]     uint8   1: the reference keeps a tensor for this candidate - the candidate loop of
 *                                     preprocess/CreateTensorPileupFromCffi.py:356-396 over the contiguous runs of :180-236.
 *                                     Plain (:358-366): the candidate's run of consecutive positions covers the window's first
 *                                     row and reaches TWO rows past its last (column c + 18), and no row of the window is
 *                                     all-zero.  Only with params.call_ht, when that fails (:370-396): the candidate is not on
 *                                     its run's last column, and either the run starts inside the window and reaches column
 *                                     c + 16 (head) or the run covers the window's first row (tail); these windows are
 *                                     zero-padded outside the run (c3b_plp_window_bounds) and skip the all-zero test.
 *   pos_ref_count / pos_total_count [end - start] int64 (only with params.gvcf)                                  */
int c3b_plp_fetch(c3b_plp *w, int64_t *matrix, int64_t *major, int32_t *stats, int64_t *cand_cols, uint8_t *cand_ok,
                  int64_t *pos_ref_count, int64_t *pos_total_count);

/* The distinct indel alleles of every column that passed the allele-frequency test (needs params.alt_info), in order of first
 * occurrence - what the reference keeps per column in dels_f / dels_r and its three insertion-string counters:
 *   al_off / al_n [end - start] int32   first record and number of records of the column at position start + i (0 elsewhere)
 *   ins_last [end - start] int32        the last read (index into the records of the count) with an insertion on that column, -1
 *                                       for none or for a column that did not pass: the reference's insertion counter grows a full
 *                                       table on every put, so whether a read after the last new string put a present one again
 *                                       changes the counter's bucket order (src/khash.h:310-318)
 *   meta  [n]  uint32   insertion << 31 | reverse strand << 30 | length
 *   read  [n]  uint32   index (into the records of the count) of the first read that showed the allele
 *   qpos  [n]  uint32   query offset of its first inserted base in that read (insertions)
 *   cnt   [n]  uint32   reads of that strand showing it
 * Any pointer may be NULL; n_alleles alone sizes the buffers.  c3b_plp_alt_text formats the all_alt_info strings from these on
 * the GPU; clair3_b200/pileup_counts.py (format_alt_info) does the same on the host. */
int c3b_plp_fetch_alleles(c3b_plp *w, int32_t *al_off, int32_t *al_n, int32_t *ins_last, uint32_t *meta, uint32_t *read, uint32_t *qpos, uint32_t *cnt,
                          int64_t capacity, int64_t *n_alleles);

/* Device views of the same results, valid until the next c3b_plp_count on w: matrix and window_starts
 * (= cand_cols - 16, the first row of every candidate's 33-row window) are exactly the `cols` / `starts` arguments of
 * c3b_forward_windows(..., cols_dtype C3B_DT_I64, on_device 1) in clair3_b200.h, so the counts never leave HBM on their way into
 * Clair3_P. */
int c3b_plp_device(c3b_plp *w, const int64_t **matrix, const int64_t **major, const int64_t **cand_cols,
                   const int64_t **window_starts, const uint8_t **cand_ok);

/* The rows of every candidate's window that belong to its contiguous run, [n_cand][2] int64 = {lo, hi}: matrix rows [lo, hi)
 * with cand_cols - 16 <= lo <= cand_cols < hi <= cand_cols + 17.  The reference's tensor holds zeros for the window's other rows
 * (:374-391); the matrix holds the neighbouring runs' columns there.  These are the `bounds` of c3b_forward_windows_bounded.
 * bounds: host copy (waits for the count); device_bounds: device view, valid until the next c3b_plp_count.  Either may be NULL. */
int c3b_plp_window_bounds(c3b_plp *w, int64_t *bounds, const int64_t **device_bounds);

/* The all_alt_info text of every candidate (src/clair3_pileup.c:391-450), formatted on the GPU: enqueues the text stage on the
 * stream of the last c3b_plp_count, which must have run with params.alt_info.  No host wait.  max_indel_length: the reference's
 * argument (longer alleles are counted but not printed).  The stage reads the records and the reference bases where the count
 * left them: the workspace's own copies, or, after a count with on_device = 1, the caller's device arrays, which must stay alive
 * and unchanged until the text has been fetched or consumed.  Per candidate, in candidate order:
 *   text      "<pos+1>-<depth>-<REF>-X<b> n D<ref bases> n I<REF><inserted bases> n R<REF> n ": SNP alleles in A C G T order,
 *             deletions by length, insertions in the bucket order of the reference's khash string counter, the remaining
 *             reference depth last; deletion text is the reference's bytes as supplied
 *   decoder   "<depth>-<alt>", alt = the fourth '-'-separated field of the stripped string: what
 *             preprocess/CreateTensorPileupFromCffi.py:66-73 hands on as alt_info
 *   ref_base  the same <REF> character         position  pos + 1
 * The next c3b_plp_sizes waits for the count and the text together. */
int c3b_plp_alt_text(c3b_plp *w, int64_t max_indel_length);

/* After c3b_plp_alt_text (waits like c3b_plp_sizes when that has not been called since): bytes of all text strings and of all
 * decoder strings.  Fails, as c3b_plp_fetch_alt_text does, if the text outgrew the stage's buffers; the count's own results stay
 * valid, and a later c3b_plp_alt_text (with a smaller max_indel_length, say) starts clean. */
int c3b_plp_alt_text_sizes(c3b_plp *w, int64_t *n_text_bytes, int64_t *n_decoder_bytes);

/* Host copies (any pointer may be NULL): text [n_text_bytes], text_off [n_cand + 1] int64 (candidate j is
 * text[text_off[j] .. text_off[j + 1])), decoder [n_decoder_bytes], decoder_off [n_cand + 1], ref_base [n_cand],
 * position [n_cand]. */
int c3b_plp_fetch_alt_text(c3b_plp *w, char *text, int64_t *text_off, char *decoder, int64_t *decoder_off, uint8_t *ref_base,
                           int64_t *position);

/* Device views of the same, valid until the next c3b_plp_count or c3b_plp_alt_text on w: decoder / decoder_off / ref_base are
 * the alt_bytes / alt_offsets / ref_base arguments of c3b_decode_calls(..., on_device = 1). */
int c3b_plp_alt_text_device(c3b_plp *w, const char **text, const int64_t **text_off, const char **decoder,
                            const int64_t **decoder_off, const uint8_t **ref_base, const int64_t **position);

/* Device time of the last c3b_plp_alt_text (CUDA events around its kernels) and the number of kernels it launched;
 * c3b_plp_last_ms keeps reporting the count alone. */
int c3b_plp_alt_text_last_ms(c3b_plp *w, float *ms, int *launches);

/* Device time of the last c3b_plp_count (CUDA events on its stream around all of its kernels, input copies excluded), and the
 * number of kernels it launched. */
int c3b_plp_last_ms(c3b_plp *w, float *ms, int *launches);

void c3b_plp_destroy(c3b_plp *w);

#ifdef __cplusplus
}
#endif
#endif /* CLAIR3_B200_PILEUP_H */
