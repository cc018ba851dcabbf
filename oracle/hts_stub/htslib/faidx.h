/*
 * Minimal stand-in for htslib's FASTA index API (fai_load / faidx_fetch_seq / fai_destroy) over one contig registered in memory
 * by oracle/fa_ref.py.  faidx_fetch_seq returns bases [beg, end] (end INCLUSIVE, clipped to the contig), as htslib does.
 * TEST INFRASTRUCTURE ONLY.
 */
#ifndef FA_REF_HTS_STUB_FAIDX_H
#define FA_REF_HTS_STUB_FAIDX_H

typedef struct faidx_t faidx_t;

faidx_t *fai_load(const char *fn);
char *faidx_fetch_seq(const faidx_t *fai, const char *c_name, int p_beg_i, int p_end_i, int *len);
void fai_destroy(faidx_t *fai);

#endif
