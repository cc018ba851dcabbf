// LSTM2's input projection (clair3/model.py:132-133 -> torch nn.LSTM's W_ih x_t + b_ih + b_hh, both directions) as one
// warpgroup-MMA GEMM over every time step at once:
//
//   pg[t*bp + b][col] = sum_k h1[t*bp + b][k] * Wp[col][k] + bias[col]      col = dir*640 + R (c3b_lstm_row order), K = 256
//
// One CTA = 128 rows x 128 columns; the whole K fits in shared memory, so the operands arrive with five cp.async.bulk copies
// (the tile-major h1 tile is one 64 KB run, the weight slab four 16 KB runs) and two warpgroups each issue 16 m64n128k16 MMAs.
// fp16 output: the recurrent kernel adds these pre-gates to its fp32 accumulators.
#include "c3b_internal.h"
#include "ptx.cuh"

namespace {

constexpr int kThreads = 256;
constexpr uint32_t kTileBytes = 32 * 128 * 16;      // [32 k-groups][128 rows][8] fp16

struct ProjDev {
    const op_t *h1;            // tile-major [33*bp/128][32][128][8]
    const op_t *w;             // [4 chunks][10 column blocks][8][128][8]
    const float *bias;         // [1280]
    __half *pg;                // [33*bp][1280]
};

__global__ void __launch_bounds__(kThreads, 1) proj2_kernel(const ProjDev p) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t bar;
    const int tid = threadIdx.x, wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31;
    const int tile = blockIdx.x, cb = blockIdx.y;
    const uint32_t a_addr = ptx::smem_u32(smem), b_addr = a_addr + kTileBytes;
    if (tid == 0) {
        ptx::mbar_init(&bar, 1);
        ptx::fence_barrier_init();
        ptx::mbar_arrive_expect_tx(&bar, 2 * kTileBytes);
        ptx::bulk_g2s(a_addr, p.h1 + (size_t)tile * (kTileBytes / 2), kTileBytes, &bar);
        for (int c = 0; c < 4; ++c)
            ptx::bulk_g2s(b_addr + c * (kTileBytes / 4), p.w + ((size_t)c * 10 + cb) * (kTileBytes / 8), kTileBytes / 4, &bar);
    }
    __syncthreads();
    ptx::mbar_wait(&bar, 0);

    float acc[64];
    ptx::wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 16; ++ks) {
        const uint64_t ad = ptx::wgmma_desc(a_addr + wg * 64 * 16 + ks * 2 * 2048, 2048, 128);
        const uint64_t bd = ptx::wgmma_desc(b_addr + ks * 2 * 2048, 2048, 128);
        ptx::wgmma_m64n128k16(acc, ad, bd, ks > 0);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_operand(acc);

    const size_t row0 = (size_t)tile * 128 + wg * 64 + 16 * w + (lane >> 2);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int col = cb * 128 + 8 * i + 2 * (lane & 3);
        const float2 bb = *reinterpret_cast<const float2 *>(p.bias + col);
#pragma unroll
        for (int h = 0; h < 2; ++h)
            *reinterpret_cast<__half2 *>(p.pg + (row0 + 8 * h) * 1280 + col) =
                __floats2half2_rn(acc[4 * i + 2 * h] + bb.x, acc[4 * i + 2 * h + 1] + bb.y);
    }
}

}  // namespace

int c3b_launch_proj2(const c3b_model *m, const op_t *h1, const IgemmW &w, __half *pg, int bp, cudaStream_t s) {
    ProjDev p;
    p.h1 = h1;
    p.w = w.w_img;
    p.bias = w.bias;
    p.pg = pg;
    const int smem = 2 * kTileBytes;
    C3B_CUDA(cudaFuncSetAttribute(proj2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    dim3 grid((unsigned)(C3B_T * (int64_t)bp / 128), 10);
    c3b_note_grid((long long)grid.x * grid.y);
    proj2_kernel<<<grid, kThreads, smem, s>>>(p);
    C3B_CUDA(cudaGetLastError());
    const_cast<c3b_model *>(m)->launches++;
    return 0;
}
