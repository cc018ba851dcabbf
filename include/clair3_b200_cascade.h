/*
 * clair3_b200_cascade.h - C-ABI of the pileup -> full-alignment candidate selection in libclair3b200.so: which of a region's
 * Clair3_P calls Clair3_F re-calls, chosen on the device from the call records c3b_decode_calls left there.
 *
 * Replaces (paths relative to HKU-BAL/Clair3) the selection of preprocess/SelectCandidates.py:187-270 as
 * scripts/clair3_c_impl_pipeline.py runs it (no --phasing_info_in_bam, so the option keeps its default of True): a row of the
 * pileup VCF is a reference row when its ALT is "." or equals its REF; reference rows with QUAL < ref_qual and the other rows
 * with QUAL < var_qual are the candidates, sorted and unique.  QUAL is compared as a float32 probability bit pattern against
 * a threshold that clair3_b200/cascade.py:prob_threshold derives from the cut-off on the host (DESIGN.md 5e), so no
 * transcendental function runs here.
 *
 * Same conventions as clair3_b200.h: int status, 0 = ok, message via c3b_last_error(); no CPU fallback.
 */
#ifndef CLAIR3_B200_CASCADE_H
#define CLAIR3_B200_CASCADE_H

#include <stddef.h>
#include <stdint.h>

#include "clair3_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Selects the full-alignment candidates of n_calls pileup calls, all arrays in device memory, stream-ordered on cuda_stream
 * with no host wait:
 *   calls        [n_calls] c3b_call, text: c3b_decode_calls' records and text pool (call s's REF then ALT at
 *                text[2 * alt_offsets[s] + 8 * s ..]); alt_offsets [n_calls + 1] the decoder's alt_info offsets
 *   position     [n_calls] int64  1-based position of each call, ascending
 *   cand_ok      [n_calls] uint8  0: the reference drops this pileup candidate (may be NULL: every candidate is kept)
 *   var_threshold / ref_threshold  a call is kept when it is printed, cand_ok, and its prob's bit pattern is below the
 *                threshold of its kind (non-reference / reference by the ALT text)
 *   scratch      [2 * n_calls] int64
 * Writes the kept calls' 0-based positions, ascending, to selected[0 .. *n_selected) (selected [n_calls] int64, n_selected
 * one int64, both device memory). */
int c3b_cascade_select(const c3b_call *calls, const char *text, const int64_t *alt_offsets, const int64_t *position,
                       const uint8_t *cand_ok, int64_t n_calls, uint32_t var_threshold, uint32_t ref_threshold, int64_t *scratch,
                       int64_t *selected, int64_t *n_selected, void *cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* CLAIR3_B200_CASCADE_H */
