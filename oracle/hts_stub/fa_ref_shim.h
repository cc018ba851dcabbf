/*
 * Force-included (-include) ahead of every reference source compiled into oracle/_ref/libclair3_fa_ref.so.
 * TEST INFRASTRUCTURE ONLY.
 *
 * 1. Every allocation of those sources goes through a guarded allocator (hts_stub.c): each block is surrounded by 4 KiB of
 *    zero bytes.  The reference's fill loop reads read.pos_info[offset].alt_base BEFORE it checks that offset lies inside the
 *    read's run of flanking positions (src/clair3_full_alignment_dwell.c:837-845), i.e. up to 33 Pos_info records (1.3 KB)
 *    before or after the block.  With plain malloc that reads heap garbage; with zero guards it reads alt_base == 0, which
 *    passes the "< 0" test and is then rejected by the bounds test - the column is uncovered, deterministically.  That is the
 *    meaning the GPU builder gives those columns.
 * 2. rand() is counted, so the binding can report how many shuffle draws one call consumed.
 */
#ifndef FA_REF_SHIM_H
#define FA_REF_SHIM_H

#include <stdlib.h>
#include <string.h>

void *fa_ref_malloc(size_t n);
void *fa_ref_calloc(size_t n, size_t size);
void *fa_ref_realloc(void *p, size_t n);
void fa_ref_free(void *p);
char *fa_ref_strdup(const char *s);
int fa_ref_rand(void);

#undef malloc
#undef calloc
#undef realloc
#undef free
#undef strdup
#undef rand
#define malloc(n) fa_ref_malloc(n)
#define calloc(n, s) fa_ref_calloc(n, s)
#define realloc(p, n) fa_ref_realloc(p, n)
#define free(p) fa_ref_free(p)
#define strdup(s) fa_ref_strdup(s)
#define rand() fa_ref_rand()

#endif
