/*
 * clair3_b200_bam.h - C-ABI of the GPU BAM reader in libclair3b200.so: a run of whole BGZF blocks goes in, the alignment records
 * of one region come out in device memory, in the layout c3b_plp_count and c3b_fa_build take (c3b_fa_records).
 *
 * The BGZF blocks are inflated on the GPU (RFC 1951, one warp per block, CRC-32 and ISIZE checked as htslib's bgzf_uncompress
 * does), the record chain is found from the first record's offset, the core fields, CIGARs, sequences and - on request - the
 * qualities, read names and "mv" B-arrays are parsed and scattered into packed arrays, and the records are filtered exactly as
 * clair3_b200/bam_io.py: read_bam(path, contig, start, end) filters them.  The host reads the file, the index and the header
 * (clair3_b200/bam_io.py), and checks the BGZF block headers; nothing else of a decode runs on the host.
 *
 * Same conventions as clair3_b200.h: int status, 0 = ok, message via c3b_last_error(); no CPU fallback.
 */
#ifndef CLAIR3_B200_BAM_H
#define CLAIR3_B200_BAM_H

#include <stddef.h>
#include <stdint.h>

#include "clair3_b200_fa.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct c3b_bam c3b_bam;

/* Where c3b_bam_fetch writes the records: the output twin of c3b_fa_records.  Sizes from c3b_bam_sizes; any pointer may be NULL
 * (that array is not copied).  The optional fields are written only after a decode with fa_fields = 1. */
typedef struct c3b_bam_out {
    int64_t *pos;               /* [n_reads]     */
    uint16_t *flag;             /* [n_reads]     */
    uint8_t *mapq;              /* [n_reads]     */
    int64_t *cigar_off;         /* [n_reads + 1] */
    uint32_t *cigar;            /* [n_cigar]     */
    int64_t *seq_off;           /* [n_reads + 1] */
    uint8_t *seq;               /* [n_seq]       */
    int32_t *l_qseq;            /* [n_reads]     */
    int64_t *qual_off;          /* [n_reads + 1] */
    uint8_t *qual;              /* [n_qual]      */
    int64_t *qname_off;         /* [n_reads + 1] */
    uint8_t *qname;             /* [n_qname]     */
    int64_t *mv_off;            /* [n_reads + 1] */
    int32_t *mv;                /* [n_mv]        */
} c3b_bam_out;

/* A decoding workspace on one device (buffers grow on demand; one decode in flight per workspace). */
int c3b_bam_create(c3b_bam **out, int device_ordinal);

/* Decodes the records of contig tid (0-based, as in the BAM header) that overlap [start, end) (0-based, end-exclusive) from
 * bytes[0 .. n_bytes): host memory holding whole BGZF blocks, for example the range an index gives for the region, or every
 * block after the header.  first_uoff: the offset of the first record in the uncompressed data of the first block (the low 16
 * bits of its virtual offset); end_uoff: the uncompressed offset, counted from the first block's start, at which the records
 * end, or -1 for the end of the data.  The records between them must chain exactly from first_uoff to end_uoff.
 * The filter is read_bam's, in file order: records with refID < 0 or of an earlier contig are skipped; the first record of a
 * later contig, or of contig tid at pos >= end, ends the run; a record with pos + max(reference span, 1) <= start is skipped.
 * fa_fields = 1: also the qualities, read names and mv arrays (c3b_fa_records' optional fields).
 * Checks the block headers on the host (gzip magic 1f 8b 08 04, a BC subfield in the extra field, a block that fits the data,
 * ISIZE <= 65536), uploads the bytes once and queues the decode on cuda_stream: no host wait. */
int c3b_bam_decode(c3b_bam *w, const uint8_t *bytes, int64_t n_bytes, int64_t first_uoff, int64_t end_uoff, int32_t tid,
                   int64_t start, int64_t end, int fa_fields, void *cuda_stream);

/* The one wait of a decode: the records kept and the length of every value array.  Fails with a message that names the block or
 * the record and the reason when the data are malformed: a DEFLATE stream that does not decode, a CRC-32 or ISIZE mismatch, a
 * record chain that does not end exactly at end_uoff ("truncated record"), a block_size that cannot hold the record's fields, or
 * an auxiliary field that runs past its record.  Any pointer may be NULL; n_qual / n_qname / n_mv are 0 without fa_fields. */
int c3b_bam_sizes(c3b_bam *w, int64_t *n_reads, int64_t *n_cigar, int64_t *n_seq, int64_t *n_qual, int64_t *n_qname,
                  int64_t *n_mv);

/* Copies the records of the last decode into out's buffers: device memory with on_device = 1 (device-to-device copies, queued
 * on the decode's stream, no wait: the buffers are then directly c3b_plp_count / c3b_fa_build input with on_device = 1), host
 * memory otherwise (waits for the copies).  Needs c3b_bam_sizes first. */
int c3b_bam_fetch(c3b_bam *w, const c3b_bam_out *out, int on_device);

/* One window of a bgzip-compressed FASTA, from its compressed blocks to bases in device memory, on the same workspace: the blocks
 * are inflated by the decode's inflater, and one thread per base gathers the window, skipping the line ends by arithmetic.
 * bytes[0 .. n_bytes): host memory holding the whole BGZF blocks that cover the window (clair3_b200/bam_io.py: fasta_span
 * finds them through the .gzi).  first_uoff: the uncompressed offset of the window's first base in the first block's data.
 * start: the window's first base, 0-based on its sequence; line_bases / line_bytes: the sequence's line geometry from the .fai.
 * Base i of the window is read at uncompressed offset
 *     first_uoff + (start + i) / line_bases * line_bytes + (start + i) % line_bases - (start / line_bases * line_bytes + start % line_bases)
 * and written to out[i] (device memory, n_bases bytes), case kept.  Checks the block headers as c3b_bam_decode does, and that
 * the window's last base lies inside the inflated data; then queues the upload, the inflate and the gather on cuda_stream: no
 * host wait.  n_bases = 0 queues nothing. */
int c3b_fasta_fetch(c3b_bam *w, const uint8_t *bytes, int64_t n_bytes, int64_t first_uoff, int64_t start, int64_t line_bases,
                    int64_t line_bytes, int64_t n_bases, uint8_t *out, void *cuda_stream);

/* The status of the last c3b_fasta_fetch: waits for its kernels (no wait when the caller's stream has already passed them, for
 * example after a later c3b_bam_sizes) and fails with the block's number and reason when a block did not inflate (a DEFLATE
 * stream that does not decode, a CRC-32 or ISIZE mismatch); out's bytes are then not the window's.  0 when no fetch is
 * pending. */
int c3b_fasta_status(c3b_bam *w);

/* The BGZF writer, on the same workspace: src[0 .. n) (host memory, or device memory with on_device = 1) is cut into blocks
 * of 0xFF00 bytes, as bgzip and htslib cut them, and each block is compressed on the GPU, one per CTA, to exactly the bytes
 * zlib 1.3 writes at level 6 with a raw window of 15 bits (zlib.compressobj(6, zlib.DEFLATED, -15)), framed as
 * clair3_b200/bam_io.py's BGZF writer frames it (gzip header with the BC subfield, CRC-32 and ISIZE footer).  The blocks are
 * then packed into one file image; the end-of-file block is not part of it.  A host src is copied through the reader's pinned
 * staging before the call returns; a device src must stay valid until the stream has passed the compression.  Queues the work
 * on cuda_stream: no host wait. */
int c3b_bgzf_compress(c3b_bam *w, const uint8_t *src, int64_t n, int on_device, void *cuda_stream);

/* The one wait of a BGZF write: the file image's bytes (*n_out) and, when block_off is not NULL, the offset of every block in
 * it, block_off[0 .. ceil(n / 0xFF00)], the last entry being *n_out.  Fails, naming the block, if a block's stream would not fit
 * the 64 KiB a BGZF block may take (zlib's own bound keeps every 0xFF00-byte payload well inside it). */
int c3b_bgzf_sizes(c3b_bam *w, int64_t *n_out, int64_t *block_off);

/* Copies the file image of the last c3b_bgzf_compress into out (*n_out bytes): device memory with on_device = 1 (queued on the
 * compression's stream, no wait), host memory otherwise (waits for the copy).  Needs c3b_bgzf_sizes first. */
int c3b_bgzf_fetch(c3b_bam *w, uint8_t *out, int on_device);

/* Device time of the last c3b_bam_decode, c3b_fasta_fetch or c3b_bgzf_compress (CUDA events around its kernels, the upload
 * excluded) and its kernel launches. */
int c3b_bam_last_ms(c3b_bam *w, float *ms, int *launches);

void c3b_bam_destroy(c3b_bam *w);

#ifdef __cplusplus
}
#endif
#endif /* CLAIR3_B200_BAM_H */
