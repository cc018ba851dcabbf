// block_scan.cuh - the one-CTA scan of the pileup counter (plp_counts.cu, plp_alt_text.cu) and the full-alignment builder
// (fa_tensor.cu): 1024 threads walk the array in steps of 1024 entries, a two-level __shfl_up_sync scan per step and a carry
// between steps.
#pragma once
#include <limits.h>

#include "c3b_internal.h"

// Each translation unit keeps its own instantiations: the library is built without relocatable device code.
namespace {

// b = a (op) b.  The maximum is a conditional assignment: as a select it costs the kernel two more registers.
template <bool Max> __device__ __forceinline__ void scan_apply(long long a, long long &b) {
    if (Max) { if (a > b) b = a; }
    else b += a;
}

// Max = false: out[i] = the sum of in[0 .. i), the sum of all of them to *total (optional), over n entries or over *n_dev + 1 of
// them when n_dev is given and that is fewer.  Max = true: out[i] = the maximum of in[0 .. i] over n entries (no cap and no
// total: no caller needs them, and they cost the kernel two registers).
template <class In, bool Max>
__global__ void block_scan_kernel(const In *__restrict__ in, int64_t *__restrict__ out, int64_t n, const int64_t *n_dev,
                                  int64_t *total) {
    constexpr long long identity = Max ? LLONG_MIN : 0;
    __shared__ long long ws[32];
    if (!Max && n_dev && *n_dev + 1 < n) n = *n_dev + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long carry = identity;
    for (int64_t base = 0; base < n; base += 1024) {
        const int64_t i = base + threadIdx.x;
        const long long x = i < n ? (long long)in[i] : identity;
        long long v = x;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const long long a = __shfl_up_sync(0xffffffffu, v, d);
            if (lane >= d) scan_apply<Max>(a, v);
        }
        if (lane == 31) ws[warp] = v;
        __syncthreads();
        if (warp == 0) {
            long long t = ws[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const long long a = __shfl_up_sync(0xffffffffu, t, d);
                if (lane >= d) scan_apply<Max>(a, t);
            }
            ws[lane] = t;
        }
        __syncthreads();
        if (warp > 0) scan_apply<Max>(ws[warp - 1], v);
        scan_apply<Max>(carry, v);
        if (i < n) out[i] = Max ? v : v - x;
        scan_apply<Max>(ws[31], carry);
        __syncthreads();
    }
    if (!Max && threadIdx.x == 0 && total) *total = carry;
}

// The launchers queue the kernel on stream s; the caller checks the launch with the stream's other kernels.
// Exclusive sum of int32 / int64 counts into int64 offsets (block_scan_kernel<In, false>).
template <class In> void block_scan_sum(const In *in, int64_t *out, int64_t n, const int64_t *n_dev, int64_t *total, cudaStream_t s) {
    block_scan_kernel<In, false><<<1, 1024, 0, s>>>(in, out, n, n_dev, total);
}
// Running maximum of int64 values (block_scan_kernel<int64_t, true>).
inline void block_scan_max(const int64_t *in, int64_t *out, int64_t n, cudaStream_t s) {
    block_scan_kernel<int64_t, true><<<1, 1024, 0, s>>>(in, out, n, nullptr, nullptr);
}

}  // namespace
