/*
 * clair3_b200.h — C-ABI of libclair3b200.so: the H100 (sm_90a) inference forward pass of Clair3's two
 * networks, the drop-in boundary for the one hot path this project replaces.
 *
 * The reference has no plugin/operator registry for this path; its seam is the torch module protocol used by its
 * callers (paths relative to HKU-BAL/Clair3):
 *
 *   m = Clair3_P|Clair3_F(add_indel_length, predict=True, input_channels)   clair3/CallVariantsFromCffi.py:230-243
 *   m.to(device); m.eval(); m.load_state_dict(state_dict)                    clair3/CallVariantsFromCffi.py:19-28,246-248
 *   Y = m(torch.from_numpy(X).to(device)); Y.detach().cpu().numpy()          clair3/CallVariantsFromCffi.py:48-52
 *                                                                            (same protocol: clair3/CallVariants.py:54-87,1466-1480)
 *
 * Each entry point below names the reference interface it replaces.  The Python shim that mirrors the module
 * protocol on top of this ABI is clair3_b200/model.py (bound with cffi, the way the reference binds libclair3 in
 * build.py:44-79).  Convention change vs libclair3 (which exit(1)s on failure, src/medaka_common.c:25-47): every call
 * returns an int status, 0 = ok, message via c3b_last_error(); the library never exits the process and never
 * falls back to a CPU implementation.
 *
 * Threading: a c3b_model is driven by one host thread at a time; forwards on different CUDA streams may be in
 * flight concurrently (each stream gets its own activation workspace).  Distinct models/devices are independent.
 */
#ifndef CLAIR3_B200_H
#define CLAIR3_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct c3b_model c3b_model;

/* network kind                      reference class                                   */
#define C3B_PILEUP          0     /* Clair3_P  clair3/model.py:58-161                  */
#define C3B_FULL_ALIGNMENT  1     /* Clair3_F  clair3/model.py:282-416                 */

/* element type of the candidate-site batch handed to c3b_forward (reference: any dtype, x.float() model.py:131,378) */
#define C3B_DT_I8   0             /* full-alignment wire dtype (shared/param_f.py:92) and GPU-mode pileup .npy (CreateTensorPileupFromCffi.py:447) */
#define C3B_DT_I32  1             /* pileup wire dtype (CreateTensorPileupFromCffi.py:397) */
#define C3B_DT_F32  2

#define C3B_DT_I64  3             /* BatchNorm num_batches_tracked in c3b_set_param; libclair3's size_t count matrix in c3b_forward_windows */

/* arithmetic used by the kernels (c3b_set_option "precision") */
#define C3B_PREC_F16_TC  0        /* production: fp16 operands on wgmma tensor cores, fp32 accumulate / cell state / SELU / softmax */
#define C3B_PREC_FP32    1        /* debug: the same layer graph on fp32 CUDA cores (separates layout bugs from precision) */

/* Replaces Clair3_P.__init__ / Clair3_F.__init__ (clair3/model.py:61-128, 285-368) + m.to(device) (CallVariantsFromCffi.py:246).
 * channels: 18 (pileup) | 8 | 9 with dwell (full-alignment).  Fails if the device is not compute capability 9.0. */
int c3b_create(c3b_model **out, int kind, int channels, int add_indel_length, int device_ordinal);

/* Replaces one entry of m.load_state_dict(state_dict) (clair3/CallVariantsFromCffi.py:19-28).  key is the reference
 * state_dict key (e.g. "LSTM1.weight_ih_l0_reverse", "res_block2.0.bn1.running_var"); data is the tensor as stored
 * in the .pt (dtype C3B_DT_F32, or C3B_DT_I64 for *.num_batches_tracked which is accepted and ignored).  Unknown keys
 * and shape mismatches are errors (strict, like torch). */
int c3b_set_param(c3b_model *m, const char *key, const void *host_data, int dtype, const int64_t *shape, int ndim);

/* Ends load_state_dict: checks every expected key is present (strict), folds BatchNorm into the convolutions
 * (eps 1e-3, clair3/model.py:192), sums the LSTM bias pairs, folds 1/NORMALIZE_NUM (shared/param_f.py:36) into conv1,
 * packs fp16 wgmma operand images and uploads them once. */
int c3b_finalize(c3b_model *m);

/* name: "precision" (C3B_PREC_*), "chunk_sites" (sites per internal pass), "lstm_tile" (batch columns per LSTM CTA sub-tile:
 * 16|32|64, 0 = auto; LSTM2 uses at most 32), "lstm_wg" (warpgroups per LSTM CTA, one sub-tile each: 1|2).  With lstm_tile 0
 * the library picks by call shape between bit-identical variants: synchronous host-buffer calls (one batch in flight) get the
 * LSTM tile with the shortest latency, stream-ordered calls the one with the least SM-time,
 * "profile" (1: bracket every kernel launch with CUDA events on its stream and accumulate per-kernel time; setting it resets the
 * totals), "taps" (1: remember where the intermediate activations of a forward live, for c3b_get_tap in clair3_b200_debug.h).
 * Debug-only options are listed in clair3_b200_debug.h. */
int c3b_set_option(c3b_model *m, const char *name, int value);

/* Replaces Y = m(X) (clair3/model.py:130-161 / 377-416) including the H2D/D2H of _torch_predict
 * (clair3/CallVariantsFromCffi.py:48-52) when x_on_device / y_on_device are 0.
 *   x: [batch,33,channels] (pileup) or [batch,depth,33,channels] (full-alignment, NHWC), C-contiguous, dtype x_dtype.
 *   y: [batch, c3b_out_dim()] float32 softmax probabilities, heads concatenated gt21|genotype|indel1|indel2.
 * With both buffers on the device the call is asynchronous on cuda_stream; with a host buffer on either side it
 * returns after y is complete.  batch may be any value >= 0 (ragged last batch, CallVariantsFromCffi.py:106-148). */
int c3b_forward(c3b_model *m, const void *x, int x_dtype, int x_on_device, int64_t batch, int depth,
                float *y, int y_on_device, void *cuda_stream);

/* The same forward on PINNED host buffers without the host synchronisation: H2D, kernels and D2H are enqueued on cuda_stream
 * and the call returns at once; the caller synchronises the stream (or an event) before reading y and keeps both buffers
 * alive until then.  This is what lets a caller overlap the copies and kernels of consecutive batches over several streams
 * (each stream owns an activation workspace) - the double-buffered replacement of the serial H2D / forward / D2H loop at
 * clair3/CallVariantsFromCffi.py:300-331. */
int c3b_forward_async(c3b_model *m, const void *x_pinned, int x_dtype, int64_t batch, int depth, float *y_pinned,
                      void *cuda_stream);

/* Pileup only.  Replaces the host-side window slicing of preprocess/CreateTensorPileupFromCffi.py:362-394: instead of
 * materialising one [33,18] tensor per candidate (windows of neighbouring candidates overlap in 32 of 33 rows), hand over
 * libclair3's per-column count matrix once - plp_data.matrix, size_t[n_cols][18] (src/clair3_pileup.h:5-17), i.e.
 * cols_dtype C3B_DT_I64; C3B_DT_I32 / I8 / F32 also accepted - plus the first row of every candidate's window:
 * site b = rows [starts[b], starts[b]+33) of cols; rows outside [0, n_cols) read as zero.  That alone is not the reference's
 * zero padding: its head / tail windows (:370-396) are zero outside the candidate's CONTIGUOUS RUN of positions, and at a
 * coverage gap the matrix holds the neighbouring run's columns there - c3b_forward_windows_bounded takes those bounds.
 * The windows are gathered on the GPU straight into the LSTM operand layout.
 * on_device: cols and starts are device pointers (else host; they are copied on cuda_stream).  host_sync: 1 = return after y
 * is complete when a host buffer is involved, 0 = stay stream-ordered (pinned buffers, caller synchronises). */
int c3b_forward_windows(c3b_model *m, const void *cols, int cols_dtype, int64_t n_cols, const int64_t *starts,
                        int on_device, int64_t batch, float *y, int y_on_device, int host_sync, void *cuda_stream);

/* c3b_forward_windows with per-window row bounds: bounds (NULL, or [batch][2] int64 on the same side as starts) = {lo, hi};
 * site b's rows outside [lo, hi) read as zero as well.  c3b_plp_window_bounds (clair3_b200_pileup.h) yields the bounds of the
 * reference's windows; NULL bounds is c3b_forward_windows. */
int c3b_forward_windows_bounded(c3b_model *m, const void *cols, int cols_dtype, int64_t n_cols, const int64_t *starts,
                                const int64_t *bounds, int on_device, int64_t batch, float *y, int y_on_device, int host_sync,
                                void *cuda_stream);

/* 24 or 90 (clair3/model.py:153-159). */
int c3b_out_dim(const c3b_model *m);

/* First, data-parallel stage of the reference's per-site decoder on the GPU (batch_output -> output_with -> output_from ->
 * possible_outcome_probabilites_from; clair3/CallVariants.py:1069-1116, 676-700, 510-576) so that only the sites that are not
 * an early-out homozygous-reference call go on to the per-site Python decoder:
 *   y         [batch, out_dim] probabilities from c3b_forward            ref_gt21 [batch]: gt21 index of ref_base+ref_base
 *                                                                         (AA=0 CC=4 GG=7 TT=9, clair3/task/gt21.py:29-50)
 *   is_ref    [batch] 1 = early-out: homo_reference >= 0.5 and gt21[ref] >= 0.5 (and both variant_length[0] >= 0.5 with the
 *             indel heads)                                                CallVariants.py:532-534, 573-576
 *   ref_prob  [batch] homo_Ref_probability (float32 products in the reference's order)   CallVariants.py:527, 569-572
 *   argmax / maxprob [batch][2|4] per head, first maximum        qual [batch] quality_score_from(ref_prob) before round(.,2)  :375-381
 *   nonref_idx[0 .. *n_nonref) ascending indices of the sites with is_ref == 0
 * on_device: every pointer is a device pointer and the call is asynchronous on cuda_stream; else host pointers, returns
 * when the outputs are complete. */
int c3b_decode_stage1(c3b_model *m, const float *y, const uint8_t *ref_gt21, int64_t batch, int on_device,
                      uint8_t *is_ref, float *ref_prob, int32_t *argmax, float *maxprob, double *qual,
                      int32_t *nonref_idx, int32_t *n_nonref, void *cuda_stream);

/* Second stage of the decoder: ranks every listed site's genotype outcomes in the order the reference's output_from tries them
 * (CallVariants.py:676-1012 over the lists of possible_outcome_probabilites_from, :406-659), so that the host only checks
 * the ranked outcomes against alt_info:
 *   y, ref_gt21  as for c3b_decode_stage1, [batch] rows
 *   sites     [max_sites] row indices to rank (e.g. stage 1's nonref_idx), or NULL for rows 0 .. max_sites-1
 *   n_sites   number of listed sites (e.g. stage 1's n_nonref, read on the device when on_device), or NULL for max_sites
 *   k         entries per site, 1 .. 1024 (804 ranks every outcome of the 90-output model, 24 of the 24-output one)
 *   cat, idx, prob, tie_mask  [max_sites][k]: the site's first k attempts, probability descending, then category, then index
 *             ascending, ending at homo_Ref.  cat: 0 homo_Ref, 1 homo_SNP, 2 hetero_SNP, 3 homo_Ins, 4 hetero_ACGT_Ins,
 *             5 hetero_InsIns, 6 homo_Del, 7 hetero_ACGT_Del, 8 hetero_DelDel, 9 hetero_InsDel (output_from's elif order);
 *             idx: position in that category's list; prob: the float32 product (bit-exact, multiplies only); tie_mask bit c:
 *             category c holds an entry of the same probability at this position or later (the is_* flags output_from
 *             returns if this attempt succeeds).  Unused entries: cat 255, idx 0, prob 0, tie_mask 0.
 *   count     [max_sites] entries written    complete [max_sites] 1 = homo_Ref is among them (0 for unlisted sites and for
 *             listed indices outside [0, batch), which a host-pointer call rejects instead)
 * on_device: every pointer is a device pointer and the call is asynchronous on cuda_stream; else host pointers, returns when
 * the outputs are complete. */
int c3b_decode_stage2(c3b_model *m, const float *y, const uint8_t *ref_gt21, int64_t batch, const int32_t *sites,
                      const int32_t *n_sites, int64_t max_sites, int k, int on_device, uint8_t *cat, uint16_t *idx,
                      float *prob, uint16_t *tie_mask, int32_t *count, uint8_t *complete, void *cuda_stream);

/* Packed device weight images (what one rank broadcasts to the others at start-up; SURVEY.md 8e).
 * which: 0 = fp16 tensor-core operand images + fp32 head weights, 1 = fp32 debug-path weights. */
int c3b_weight_blob(c3b_model *m, int which, void **device_ptr, size_t *bytes);

/* One-time ncclBroadcast of both packed weight images from rank `root` over NVLink (libnccl is dlopen'ed; the comm is
 * the caller's ncclComm_t).  Multi-GPU inference in the reference is N independent processes over file lists
 * (clair3/CallVariantsFromCffiGPU.py:141-199); there is no per-batch collective to replace. */
int c3b_bcast_weights(c3b_model *m, void *nccl_comm, int root, void *cuda_stream);

/* Per-kernel device time accumulated while option "profile" is on.  kernel names: pileup "ingest" "lstm1" "proj2" "lstm2"
 * "tail" (L4 + heads); full-alignment "ingest" "conv0".."conv8" "spp" "tail".  Synchronises the streams it recorded on. */
int c3b_get_profile(c3b_model *m, const char *kernel, double *total_ms, int64_t *launches);
/* Average grid size (CTAs, one per SM for the tensor-core kernels) of that kernel's launches: SM-time = CTAs x duration is what a
 * kernel costs when several batches share the GPU. */
int c3b_get_profile_ctas(c3b_model *m, const char *kernel, double *ctas_per_launch);

/* Number of this library's kernels launched on behalf of m so far (bench.py's gpu_launches). */
int64_t c3b_launch_count(const c3b_model *m);

void c3b_destroy(c3b_model *m);

/* Thread-local message for the last non-zero status. */
const char *c3b_last_error(void);
const char *c3b_version(void);

#ifdef __cplusplus
}
#endif
#endif /* CLAIR3_B200_H */
