// 3x3 convolutions of Clair3_F (clair3/model.py:200-235) as an implicit GEMM over SHIFTED VIEWS of a shared-memory-resident,
// zero-padded, channel-group-planar feature map, on warpgroup MMAs.
//
// Activation layout ("planar padded"): [C/8][P][8] fp16.  A site's H x W feature map is stored as its (H+2) x (W+2)
// zero-bordered raster, sites back to back: slot g = b*S + (h+1)*Wp + (w+1), S = (H+2)*Wp, Wp = W+2, at plane offset G + g
// (G guard slots of zeros at both ends).  With that layout
//   * the input of a tile (128 consecutive output slots plus a G-slot halo on each side) is C/8 CONTIGUOUS runs of memory: it
//     lands in shared memory with C/8 cp.async.bulk copies (TMA engine; no per-thread gathers, no im2col expansion) in exactly
//     the no-swizzle K-major wgmma layout [k-group][slot][8];
//   * the A operand of tap (dh,dw) is the SAME image viewed (dh-1)*Wp + (dw-1) slots later: only the descriptor's start
//     address changes, so every input byte is fetched once per tile and used by all nine taps;
//   * stride-2 stem convs read FOUR parity planes of the previous level (each a planar padded tensor in THIS conv's geometry):
//     tap (dh,dw) = plane (dh&1, dw&1) viewed (dh>>1)*Wp + (dw>>1) slots later - shifted views again;
//   * border slots are computed like any other row but never stored: they keep the zeros of the one-time workspace clear,
//     so the output is again a valid planar padded tensor for the next convolution (and the residual add reads the same
//     slot of its own input).
// Weights: the host-packed operand image (pack_operand, c3b_api.cu) [k-chunk][8 k-groups][N][8], k = tap*C + ci, streams
// through a two-stage ring, one 64-wide k-chunk per stage.  Two warpgroups own 64 output slots each (N = Cout, in wgmma
// widths of at most 128); the epilogue adds bias and residual, applies ReLU and stores the real pixels - into the planar map
// of this level, or scattered into the four parity planes the next level's stem conv reads.
#include "c3b_internal.h"
#include "ptx.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWStages = 2;

struct PconvDev {
    const op_t *in;
    const op_t *w_img;
    const float *bias;
    const op_t *residual;
    op_t *out;
    PlanarGeom g, nx;          // this level; the next level (parity output)
    int c, relu, par, nksteps, nchunks;
    uint32_t rows;             // slots of input per tile and plane: 128 + 2G
};

template <int N>
__device__ __forceinline__ void wgmma_n(float (&d)[N == 64 ? 32 : 64], uint64_t a, uint64_t b) {
    if constexpr (N == 64) ptx::wgmma_m64n64k16(d, a, b, 1);
    else ptx::wgmma_m64n128k16(d, a, b, 1);
}

template <int N, bool S2>
__global__ void __launch_bounds__(kThreads, 1) pconv_kernel(const PconvDev p) {
    constexpr int NW = N == 64 ? 64 : 128;      // wgmma width
    constexpr int NT = N / NW;
    constexpr int NPL = S2 ? 4 : 1;
    constexpr uint32_t W_STAGE = 8 * N * 16;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t a_bar, w_bar[kWStages];
    const int tid = threadIdx.x, wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31;
    const PlanarGeom &g = p.g;
    const long long t0 = (long long)blockIdx.x * 128;          // first output slot of the tile (data-slot index)
    const int cg = p.c / 8;
    const uint32_t a_base = ptx::smem_u32(smem);
    const uint32_t w_base = a_base + NPL * cg * p.rows * 16;
    const uint32_t a_bytes = NPL * cg * p.rows * 16;

    auto issue_w = [&](int ch) {
        const int st = ch % kWStages;
        ptx::mbar_arrive_expect_tx(&w_bar[st], W_STAGE);
        ptx::bulk_g2s(w_base + st * W_STAGE, p.w_img + (size_t)ch * 8 * N * 8, W_STAGE, &w_bar[st]);
    };
    if (tid == 0) {
        ptx::mbar_init(&a_bar, 1);
        for (int s = 0; s < kWStages; ++s) ptx::mbar_init(&w_bar[s], 1);
        ptx::fence_barrier_init();
        ptx::mbar_arrive_expect_tx(&a_bar, a_bytes);
        for (int ch = 0; ch < kWStages && ch < p.nchunks; ++ch) issue_w(ch);
    }
    __syncthreads();
    if (tid < 32) {
        // plane pl, channel group k: slots [G + t0 - G, G + t0 + 128 + G) of that plane
        for (int i = lane; i < NPL * cg; i += 32)
            ptx::bulk_g2s(a_base + i * p.rows * 16, p.in + ((size_t)i * g.p + (size_t)t0) * 8, p.rows * 16, &a_bar);
    }

    float acc[NT][NW / 2];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int j = 0; j < NW / 2; ++j) acc[nt][j] = 0.f;
    ptx::mbar_wait(&a_bar, 0);
    const uint32_t a_lbo = p.rows * 16;
    for (int ch = 0; ch < p.nchunks; ++ch) {
        const int st = ch % kWStages;
        ptx::mbar_wait(&w_bar[st], (uint32_t)(ch / kWStages) & 1u);
        ptx::wgmma_fence();
        // always four k-steps per chunk: the packed weight image is zero past the last real k-group, so the padding steps of
        // conv1's last chunk add nothing; their A view is clamped onto the last real tap (finite data)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const int ks = min(ch * 4 + kk, p.nksteps - 1);
            const int k0 = ks * 16, tap = k0 / p.c, ci = (k0 % p.c) / 8, dh = tap / 3, dw = tap % 3;
            int pl = 0, off;
            if (S2) {
                pl = (dh & 1) * 2 + (dw & 1);
                off = g.g + (dh >> 1) * g.wp + (dw >> 1);
            } else {
                off = g.g + (dh - 1) * g.wp + (dw - 1);
            }
            const uint64_t ad = ptx::wgmma_desc(a_base + ((pl * cg + ci) * p.rows + off + wg * 64) * 16, a_lbo, 128);
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
                wgmma_n<N>(acc[nt], ad, ptx::wgmma_desc(w_base + st * W_STAGE + (2 * kk) * N * 16 + nt * 128 * 16, N * 16, 128));
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) ptx::fence_operand(acc[nt]);
        __syncthreads();                        // both warpgroups are done with the stage
        if (tid == 0 && ch + kWStages < p.nchunks) issue_w(ch + kWStages);
    }

    // epilogue: thread rows t0 + 64 wg + 16 w + lane/4 (+ 8)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const long long t = t0 + wg * 64 + 16 * w + (lane >> 2) + 8 * h;
        if (t >= g.t) continue;
        const long long b = t / g.s;
        const int rem = (int)(t - b * g.s), hp = rem / g.wp, wq = rem - hp * g.wp;
        if (hp < 1 || hp > g.h || wq < 1 || wq > g.w) continue;
        const size_t slot_off = ((size_t)g.g + (size_t)t) * 8;
        size_t out_off = slot_off, out_pitch = (size_t)g.p * 8;
        if (p.par) {
            const PlanarGeom &n = p.nx;
            out_off = (size_t)((hp & 1) * 2 + (wq & 1)) * ((size_t)(N / 8) * n.p * 8) +
                      ((size_t)n.g + (size_t)b * n.s + (size_t)((hp >> 1) + 1) * n.wp + ((wq >> 1) + 1)) * 8;
            out_pitch = (size_t)n.p * 8;
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int i = 0; i < NW / 8; ++i) {
                const int col = nt * NW + 8 * i + 2 * (lane & 3);
                const float2 bb = *reinterpret_cast<const float2 *>(p.bias + col);
                float x0 = acc[nt][4 * i + 2 * h] + bb.x, x1 = acc[nt][4 * i + 2 * h + 1] + bb.y;
                if (p.residual) {
                    const float2 r = op22f2(*reinterpret_cast<const op2_t *>(p.residual + slot_off + (size_t)(col >> 3) * g.p * 8 + (col & 7)));
                    x0 += r.x;
                    x1 += r.y;
                }
                if (p.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                *reinterpret_cast<uint32_t *>(p.out + out_off + (size_t)(col >> 3) * out_pitch + (col & 7)) = f2op2_sat(x0, x1);
            }
    }
}

template <int N, bool S2>
int launch(const PconvDev &p, cudaStream_t s) {
    const int smem = (S2 ? 4 : 1) * (p.c / 8) * (int)p.rows * 16 + kWStages * 8 * N * 16;
    auto kern = pconv_kernel<N, S2>;
    C3B_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const unsigned grid = (unsigned)((p.g.t + 127) / 128);
    c3b_note_grid(grid);
    kern<<<grid, kThreads, smem, s>>>(p);
    C3B_CUDA(cudaGetLastError());
    return 0;
}

template <int N>
int launch_n(const PconvDev &p, bool s2, cudaStream_t s) { return s2 ? launch<N, true>(p, s) : launch<N, false>(p, s); }

}  // namespace

int c3b_launch_pconv(const c3b_model *m, const PconvArgs &a, cudaStream_t s) {
    PconvDev p;
    p.in = a.in;
    p.w_img = a.w.w_img;
    p.bias = a.w.bias;
    p.residual = a.residual;
    p.out = a.out;
    p.g = a.geom;
    p.nx = a.next;
    p.c = a.c;
    p.relu = a.relu;
    p.par = a.out_parity;
    p.nksteps = 9 * a.c / 16;
    p.nchunks = a.w.nchunks;
    p.rows = 128 + 2 * (uint32_t)a.geom.g;
    if (a.c % 16 != 0 || a.w.n != a.n) { c3b_set_error("pconv: channels %d / %d not supported", a.c, a.n); return 1; }
    const_cast<c3b_model *>(m)->launches++;
    switch (a.n) {
        case 64: return launch_n<64>(p, a.stride2 != 0, s);
        case 128: return launch_n<128>(p, a.stride2 != 0, s);
        case 256: return launch_n<256>(p, a.stride2 != 0, s);
    }
    c3b_set_error("pconv: unsupported output channels %d", a.n);
    return 1;
}
