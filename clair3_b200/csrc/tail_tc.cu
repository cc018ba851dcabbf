// The dense tail of both networks (clair3/model.py:136-159 pileup, :391-411 full-alignment):
//
//   a4 = SELU(L4 . x + b4)                         x = flattened LSTM2 output [10560] / pyramid-pooled features [3584]
//   per head k:  a5 = SELU(L5_k . a4 + b5_k) ; y_k = softmax(SELU(Y_k . a5 + by_k)) ; out = cat(y_k)
//
// L4 carries almost all of the tail's FLOPs and runs on warpgroup MMAs: one CTA owns 128 candidate sites (two warpgroups of 64
// rows, N = d4) and one split of K; 64-wide k-chunks of the tile-major activations (one 16 KB run) and of the host-packed L4
// operand image (one d4 x 128 B run) stream through a three-stage shared-memory ring with cp.async.bulk.  Split-K keeps the
// GPU busy at a few hundred sites; the fp32 partial sums [nsplit][bp][d4] go to the heads kernel (kernels_common.cu), which
// adds them in a fixed order with the bias and runs SELU, the per-head layers and the softmax.
#include <algorithm>

#include "c3b_internal.h"
#include "ptx.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kStages = 3;
constexpr int kMaxSplit = 16;                  // the heads kernel sums at most 16 partials

struct L4Dev {
    const op_t *act;          // tile-major k-group-planar [bp/128][KG][128][8]
    const op_t *w4;           // [KG][d4 rows][8]
    float *z4;                // [nsplit][bp][d4] partial sums, no bias
    int kg, bp, chunks_per_split, nchunks;
};

template <int D4>
__global__ void __launch_bounds__(kThreads, 1) l4_kernel(const L4Dev p) {
    constexpr int NT = D4 / 128;
    constexpr uint32_t A_BYTES = 8 * 128 * 16, B_BYTES = 8 * D4 * 16, STAGE = A_BYTES + B_BYTES;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t full[kStages];
    const int tid = threadIdx.x, wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31;
    const int tile = blockIdx.x, split = blockIdx.y;
    const int c0 = split * p.chunks_per_split;
    const int nc = min(p.chunks_per_split, p.nchunks - c0);
    const uint32_t base = ptx::smem_u32(smem);
    const op_t *a_src = p.act + (size_t)tile * p.kg * 128 * 8;

    auto issue = [&](int i) {                   // chunk c0 + i -> stage i % kStages (thread 0)
        const int st = i % kStages, c = c0 + i;
        ptx::mbar_arrive_expect_tx(&full[st], STAGE);
        ptx::bulk_g2s(base + st * STAGE, a_src + (size_t)c * 8 * 128 * 8, A_BYTES, &full[st]);
        ptx::bulk_g2s(base + st * STAGE + A_BYTES, p.w4 + (size_t)c * 8 * D4 * 8, B_BYTES, &full[st]);
    };
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) ptx::mbar_init(&full[s], 1);
        ptx::fence_barrier_init();
        for (int i = 0; i < kStages && i < nc; ++i) issue(i);
    }
    __syncthreads();

    float acc[NT][64];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int j = 0; j < 64; ++j) acc[nt][j] = 0.f;
    for (int i = 0; i < nc; ++i) {
        const int st = i % kStages;
        ptx::mbar_wait(&full[st], (uint32_t)(i / kStages) & 1u);
        const uint32_t a_addr = base + st * STAGE, b_addr = a_addr + A_BYTES;
        ptx::wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const uint64_t ad = ptx::wgmma_desc(a_addr + wg * 64 * 16 + ks * 2 * 2048, 2048, 128);
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
                ptx::wgmma_m64n128k16(acc[nt], ad, ptx::wgmma_desc(b_addr + nt * 128 * 16 + ks * 2 * D4 * 16, D4 * 16, 128), 1);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) ptx::fence_operand(acc[nt]);
        __syncthreads();                        // both warpgroups are done with the stage
        if (tid == 0 && i + kStages < nc) issue(i + kStages);
    }

    const size_t row0 = (size_t)tile * 128 + wg * 64 + 16 * w + (lane >> 2);
    float *z = p.z4 + (size_t)split * p.bp * D4;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int col = nt * 128 + 8 * i + 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h)
                *reinterpret_cast<float2 *>(z + (row0 + 8 * h) * D4 + col) = make_float2(acc[nt][4 * i + 2 * h], acc[nt][4 * i + 2 * h + 1]);
        }
}

template <int D4>
int launch_l4(const L4Dev &p, int tiles, int nsplit, cudaStream_t s) {
    const int smem = kStages * (8 * 128 * 16 + 8 * D4 * 16);
    C3B_CUDA(cudaFuncSetAttribute(l4_kernel<D4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    dim3 grid(tiles, nsplit);
    c3b_note_grid((long long)grid.x * grid.y);
    l4_kernel<D4><<<grid, kThreads, smem, s>>>(p);
    C3B_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

// act: tile-major [bp/128][l4_in/8][128][8]; z4: scratch for up to 16 x [bp][d4] fp32 partial sums.  Returns the split count
// through *nsplit_out (the "l4_pre" tap sums the partials).
int c3b_launch_tail(const c3b_model *m, const op_t *act, int64_t batch, int bp, float *out, float *z4, int *nsplit_out, cudaStream_t s) {
    L4Dev p;
    p.act = act;
    p.w4 = m->tail.w4;
    p.z4 = z4;
    p.kg = m->l4_in / 8;
    p.bp = bp;
    p.nchunks = p.kg / 8;
    const int tiles = bp / 128;
    // enough CTAs for two waves of the GPU, at least four k-chunks per split
    int nsplit = (2 * m->sm_count + tiles - 1) / tiles;
    nsplit = std::max(1, std::min(std::min(nsplit, kMaxSplit), p.nchunks / 4));
    p.chunks_per_split = (p.nchunks + nsplit - 1) / nsplit;
    nsplit = (p.nchunks + p.chunks_per_split - 1) / p.chunks_per_split;
    const int rc = m->d4 == 128 ? launch_l4<128>(p, tiles, nsplit, s) : launch_l4<256>(p, tiles, nsplit, s);
    if (rc) return rc;
    if (c3b_launch_heads(z4, nsplit, (int64_t)bp * m->d4, m->heads, out, batch, s)) return 1;
    const_cast<c3b_model *>(m)->launches += 2;
    if (nsplit_out) *nsplit_out = nsplit;
    return 0;
}
