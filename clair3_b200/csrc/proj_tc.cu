// LSTM2's input projection (clair3/model.py:132-133 -> torch nn.LSTM's W_ih x_t + b_ih + b_hh, both directions) as one
// warpgroup-MMA GEMM over every time step at once:
//
//   pg[t*bp + b][col] = sum_k h1[t*bp + b][k] * Wp[col][k] + bias[col]      col = dir*640 + C, K = 256
//
// C is in gate-quad order (c3b_lstm2_pg_row): columns 128p + 4u .. +3 are gates i, f, g, o of hidden unit 32p + u, so the
// recurrent kernel loads a unit's four pre-gates of one site as one 8-byte word.  The order lives only in the host-packed
// weight slabs and bias; this kernel does not depend on it.
//
// M = 33*bp rows, N = 1280, K = 256: at bp = 1024 that is 22 GFLOP, 17 MB of h1 read and 86 MB of pre-gates written, and on
// H100 the MMAs and the traffic each need about 30 us, so the copies, the MMAs and the stores must overlap.  Weight-stationary
// persistent CTAs:
//   * the 1280 columns are 5 slabs of 256; a CTA loads its slab (128 KB, the whole K) and the slab's bias once, then walks a
//     contiguous range of 128-row h1 tiles.  CTA c serves slab c % 5 and tile range c / 5, so the five CTAs that read one h1 tile
//     run side by side and the later four reads of a tile can be served from L2.
//   * a producer warp streams the tile-major h1 tiles (one K-half = one contiguous 32 KB run) through a three-stage ring with
//     full / empty mbarriers; two consumer warpgroups each own 64 rows of the tile and issue 16 wgmma.m64n256k16 per tile.
//   * epilogue: fp32 bias from shared memory, one fp16 rounding, a 4 x 4 word transpose inside each lane quad so that every
//     lane stores 16 contiguous bytes (a warp store covers 8 rows x 64 bytes).
// fp16 output: the recurrent kernel adds these pre-gates to its fp32 accumulators.
#include "c3b_internal.h"
#include "ptx.cuh"

namespace {

constexpr int kSlabCols = 256;                                    // output columns per CTA (wgmma N)
constexpr int kSlabs = 1280 / kSlabCols;
constexpr uint32_t kSlabBytes = 32 * kSlabCols * 16;              // [32 k-groups][256 columns][8] fp16 = 128 KB
constexpr uint32_t kTileBytes = 32 * 128 * 16;                    // h1 tile: [32 k-groups][128 rows][8] fp16 = 64 KB
constexpr int kStageKG = 16;                                      // k-groups per ring stage (a K-half of a tile)
constexpr int kParts = 32 / kStageKG;                             // stages per tile
constexpr int kStages = 3;
constexpr uint32_t kStageBytes = kStageKG * 128 * 16;
constexpr int kSmem = kSlabBytes + kStages * kStageBytes + kSlabCols * 4;   // 225 KB
constexpr int kThreads = 288;                                     // consumer warpgroups 0 and 1, producer warp 8

struct ProjDev {
    const op_t *h1;            // tile-major [33*bp/128][32][128][8]
    const op_t *w;             // [4 chunks][5 slabs][8][256][8]
    const float *bias;         // [1280]
    __half *pg;                // [33*bp][1280]
    int ntiles;                // 33*bp/128
};

// 4 x 4 transpose of 32-bit words across the lanes of a quad (q = lane % 4): lane q's v[i] <- lane i's v[q].
__device__ __forceinline__ void quad_transpose(uint32_t (&v)[4], int q) {
    const bool b1 = q & 2, b0 = q & 1;
    uint32_t r0 = __shfl_xor_sync(0xffffffffu, b1 ? v[0] : v[2], 2);
    uint32_t r1 = __shfl_xor_sync(0xffffffffu, b1 ? v[1] : v[3], 2);
    if (b1) { v[0] = r0; v[1] = r1; } else { v[2] = r0; v[3] = r1; }
    r0 = __shfl_xor_sync(0xffffffffu, b0 ? v[0] : v[1], 1);
    r1 = __shfl_xor_sync(0xffffffffu, b0 ? v[2] : v[3], 1);
    if (b0) { v[0] = r0; v[2] = r1; } else { v[1] = r0; v[3] = r1; }
}

__global__ void __launch_bounds__(kThreads, 1) proj2_kernel(const ProjDev p) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t full[kStages], empty[kStages], w_bar;
    const int tid = threadIdx.x, wg = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warp-uniform as far as the compiler knows
    const int slab = blockIdx.x % kSlabs, group = blockIdx.x / kSlabs, ngroups = gridDim.x / kSlabs;
    const int t0 = (int)((int64_t)group * p.ntiles / ngroups), t1 = (int)((int64_t)(group + 1) * p.ntiles / ngroups);
    const uint32_t w_addr = ptx::smem_u32(smem), a_addr = w_addr + kSlabBytes;
    float *bias_s = reinterpret_cast<float *>(smem + kSlabBytes + kStages * kStageBytes);
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) {
            ptx::mbar_init(&full[s], 1);
            ptx::mbar_init(&empty[s], 8);             // lane 0 of each consumer warp
        }
        ptx::mbar_init(&w_bar, 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (wg == 2) {                                    // producer warp: one thread issues every copy
        if (tid == 256) {
            ptx::mbar_arrive_expect_tx(&w_bar, kSlabBytes + kSlabCols * 4);
            for (int c = 0; c < 4; ++c)
                ptx::bulk_g2s(w_addr + c * (kSlabBytes / 4), p.w + ((size_t)c * kSlabs + slab) * (kSlabBytes / 8), kSlabBytes / 4, &w_bar);
            ptx::bulk_g2s(ptx::smem_u32(bias_s), p.bias + slab * kSlabCols, kSlabCols * 4, &w_bar);
            int g = 0;
            for (int t = t0; t < t1; ++t)
                for (int part = 0; part < kParts; ++part, ++g) {
                    const int st = g % kStages;
                    if (g >= kStages) ptx::mbar_wait(&empty[st], (g / kStages - 1) & 1);
                    ptx::mbar_arrive_expect_tx(&full[st], kStageBytes);
                    ptx::bulk_g2s(a_addr + st * kStageBytes, p.h1 + (size_t)t * (kTileBytes / 2) + part * (kStageBytes / 2),
                                  kStageBytes, &full[st]);
                }
        }
        return;
    }

    const int w = (tid >> 5) & 3, lane = tid & 31, q = lane & 3;
    ptx::mbar_wait(&w_bar, 0);
    float acc[128];
    int g = 0;
    for (int t = t0; t < t1; ++t, g += kParts) {
        ptx::wgmma_fence();
#pragma unroll
        for (int part = 0; part < kParts; ++part) {
            const int st = (g + part) % kStages;
            ptx::mbar_wait(&full[st], ((g + part) / kStages) & 1);
            const uint32_t a = a_addr + st * kStageBytes + wg * 64 * 16;
#pragma unroll
            for (int ks = 0; ks < kStageKG / 2; ++ks)
                ptx::wgmma_m64n256k16(acc, ptx::wgmma_desc(a + ks * 2 * 2048, 2048, 128),
                                      ptx::wgmma_desc(w_addr + (part * kStageKG + ks * 2) * (kSlabCols * 16), kSlabCols * 16, 128),
                                      part > 0 || ks > 0);
            ptx::wgmma_commit();
            if (part > 0) {                                    // the previous stage's MMAs are done: hand it back
                ptx::wgmma_wait<1>();
                if (lane == 0) ptx::mbar_arrive(&empty[(g + part - 1) % kStages]);
            }
        }
        ptx::wgmma_wait<0>();
        ptx::fence_operand(acc);
        if (lane == 0) ptx::mbar_arrive(&empty[(g + kParts - 1) % kStages]);

        // acc[4i + 2h + e] = row 16w + lane/4 + 8h, column 8i + 2q + e; after the quad transpose lane q stores columns
        // 32j + 8q .. +7 of both its rows
        __half *out = p.pg + ((size_t)t * 128 + wg * 64 + 16 * w + (lane >> 2)) * 1280 + slab * kSlabCols + 8 * q;
#pragma unroll
        for (int j = 0; j < kSlabCols / 32; ++j) {
            uint32_t v[2][4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int c = 4 * (4 * j + i);
                const float2 bb = *reinterpret_cast<const float2 *>(bias_s + 32 * j + 8 * i + 2 * q);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const __half2 x = __floats2half2_rn(acc[c + 2 * h] + bb.x, acc[c + 2 * h + 1] + bb.y);
                    v[h][i] = *reinterpret_cast<const uint32_t *>(&x);
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                quad_transpose(v[h], q);
                *reinterpret_cast<uint4 *>(out + (size_t)8 * h * 1280 + 32 * j) = make_uint4(v[h][0], v[h][1], v[h][2], v[h][3]);
            }
        }
    }
}

}  // namespace

int c3b_launch_proj2(const c3b_model *m, const op_t *h1, const IgemmW &w, __half *pg, int bp, cudaStream_t s) {
    ProjDev p;
    p.h1 = h1;
    p.w = w.w_img;
    p.bias = w.bias;
    p.pg = pg;
    p.ntiles = (int)(C3B_T * (int64_t)bp / 128);
    // kSlabs CTAs per tile range, at most one CTA per SM; ranges differ by at most one tile
    int ngroups = m->sm_count / kSlabs;
    if (ngroups > p.ntiles) ngroups = p.ntiles;
    if (ngroups < 1) ngroups = 1;
    C3B_CUDA(cudaFuncSetAttribute(proj2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    const unsigned grid = (unsigned)(kSlabs * ngroups);
    c3b_note_grid(grid);
    proj2_kernel<<<grid, kThreads, kSmem, s>>>(p);
    C3B_CUDA(cudaGetLastError());
    const_cast<c3b_model *>(m)->launches++;
    return 0;
}
