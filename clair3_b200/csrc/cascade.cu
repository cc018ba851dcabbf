// cascade.cu - the pileup -> full-alignment candidate selection on the GPU (include/clair3_b200_cascade.h; DESIGN.md 5e).
//
// Reference: preprocess/SelectCandidates.py:187-270 of HKU-BAL/Clair3 over the pileup VCF text.  Here, over the call records
// c3b_decode_calls left on the device:
//
//   cascade_flag     one thread per call: printed && cand_ok && prob bits < the threshold of its kind, the kind by the
//                    ALT text of the row (ALT "." or ALT == REF: a reference row).
//   (block_scan)     exclusive sum of the flags = each kept call's slot; the total is the candidate count.
//   cascade_scatter  kept calls' 0-based positions into their slots: calls ascend by position, so the candidates do too.
//
// Bound: launch latency (a region has 10^3 - 10^5 calls; per call the 48-byte c3b_call, its offset, position and cand_ok,
// and its REF / ALT bytes are read).
#include "block_scan.cuh"
#include "c3b_internal.h"
#include "../../include/clair3_b200_cascade.h"

namespace {

__global__ void cascade_flag_kernel(const c3b_call *__restrict__ calls, const char *__restrict__ text,
                                    const int64_t *__restrict__ alt_off, const uint8_t *__restrict__ cand_ok, int64_t n,
                                    uint32_t var_t, uint32_t ref_t, int64_t *__restrict__ flag) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const c3b_call c = calls[s];
    bool keep = c.printed && (!cand_ok || cand_ok[s]);
    if (keep) {
        const char *ref = text + 2 * alt_off[s] + 8 * s, *alt = ref + c.ref_len;
        bool is_ref = c.alt_len == 1 && alt[0] == '.';
        if (!is_ref && c.alt_len == c.ref_len) {
            is_ref = true;
            for (int i = 0; i < c.ref_len && is_ref; ++i) is_ref = ref[i] == alt[i];
        }
        keep = __float_as_uint(c.prob) < (is_ref ? ref_t : var_t);
    }
    flag[s] = keep;
}

__global__ void cascade_scatter_kernel(const int64_t *__restrict__ flag, const int64_t *__restrict__ slot,
                                       const int64_t *__restrict__ position, int64_t n, int64_t *__restrict__ selected) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n && flag[s]) selected[slot[s]] = position[s] - 1;
}

}  // namespace

extern "C" int c3b_cascade_select(const c3b_call *calls, const char *text, const int64_t *alt_offsets, const int64_t *position,
                                  const uint8_t *cand_ok, int64_t n_calls, uint32_t var_threshold, uint32_t ref_threshold,
                                  int64_t *scratch, int64_t *selected, int64_t *n_selected, void *cuda_stream) {
    if (n_calls < 0 || !n_selected || (n_calls > 0 && (!calls || !text || !alt_offsets || !position || !scratch || !selected))) {
        c3b_set_error("c3b_cascade_select: null argument or negative n_calls");
        return 1;
    }
    cudaStream_t s = (cudaStream_t)cuda_stream;
    if (n_calls == 0) {
        C3B_CUDA(cudaMemsetAsync(n_selected, 0, 8, s));
        return 0;
    }
    const unsigned blocks = (unsigned)((n_calls + 255) / 256);
    int64_t *flag = scratch, *slot = scratch + n_calls;
    cascade_flag_kernel<<<blocks, 256, 0, s>>>(calls, text, alt_offsets, cand_ok, n_calls, var_threshold, ref_threshold, flag);
    block_scan_sum(flag, slot, n_calls, nullptr, n_selected, s);
    cascade_scatter_kernel<<<blocks, 256, 0, s>>>(flag, slot, position, n_calls, selected);
    C3B_CUDA(cudaGetLastError());
    return 0;
}
