/*
 * clair3_b200_debug.h - debug / measurement hooks of libclair3b200.so.  NOT part of the drop-in surface (clair3_b200.h):
 * activation taps for the parity tests and clock-stamp traces.
 *
 * Extra c3b_set_option names that exist only for these hooks: "tap_ws" (which stream workspace c3b_get_tap reads, -1 = first
 * that has the tap), "lstm_trace" (1: clock stamps of one CTA of each LSTM kernel),
 * "lstm_mufu16" (1: gate activations with packed tanh.approx.f16x2; 0 default: fp32 tanh.approx).
 */
#ifndef CLAIR3_B200_DEBUG_H
#define CLAIR3_B200_DEBUG_H

#include "clair3_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Copy an intermediate activation of the most recent forward (option "taps" on; first chunk) to the host as float32.
 * names: pileup "lstm1"[B,33,256] "lstm2"[B,33,320] "l4_pre"[B,128]; full-alignment "conv1" "res_block1" "conv3" "res_block2"
 * "conv5" "res_block3" (NHWC) "spp"[B,3584] "l4_pre"[B,256].  *count_inout: capacity in / elements out.
 * Tensor-core path only, so that every kernel's input and output can be read:
 *   pileup "lstm1_x"[B,33,48]: LSTM1's input operand, columns [hi(x) (channels) | 1 | lo(x) (channels) | 0..];
 *   pileup "lstm2_pregates"[B,33,1280]: the input projection's fp16 output, column dir*640 + C in gate-quad order
 *     (c3b_lstm2_pg_row), sigmoid gates pre-halved, bias included;
 *   full-alignment "res_block1_mid" "res_block2_mid" "res_block3_mid" (NHWC): the first convolution inside each residual block. */
int c3b_get_tap(c3b_model *m, const char *name, float *host_out, int64_t *count_inout);

/* With option "lstm_trace" on, CTA (0,0) of each LSTM kernel stamps clock64 at four points of every step (operands ready,
 * first accumulator ready, epilogue done, next operands stored); copies [2 layers][33 steps][4] stamps out. */
int c3b_debug_lstm_trace(c3b_model *m, int64_t *out264);

#ifdef __cplusplus
}
#endif
#endif /* CLAIR3_B200_DEBUG_H */
