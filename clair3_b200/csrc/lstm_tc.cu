// Persistent-weight bidirectional LSTM recurrence on warpgroup MMAs (Clair3_P's LSTM1 / LSTM2,
// clair3/model.py:96-107,132-133; torch nn.LSTM semantics: gate rows i,f,g,o, h0 = c0 = 0, the reverse direction
// walks t = 32..0 and both directions are concatenated per time step).
//
// One CTA owns WG sub-tiles of NB candidate sites (one per warpgroup) x one direction for all 33 steps.  The gate GEMM is
// issued "swapped": the recurrent weight matrix is the wgmma A operand (gate rows -> M), the activations [x_t ; h_{t-1}] of a
// sub-tile's NB sites are the B operand (sites -> N).  So
//   * the whole weight matrix stays in shared memory for the 33 steps (176 KB LSTM1, 200 KB LSTM2), loaded once per CTA with
//     cp.async.bulk from a host-packed no-swizzle K-major image and shared by the CTA's warpgroups;
//   * the gate rows are permuted on the host so that one 64-row block pair holds all four gates of 32 hidden units in the
//     accumulator registers of ONE thread: row 16w + q of block 2p (q < 8) is gate i of unit 32p + 8w + q, row 16w + q + 8 is
//     gate f of the same unit, and block 2p + 1 holds g and o at the same rows (c3b_lstm_row).  The cell state stays in fp32
//     registers for the whole sequence and h_t (fp16) goes back into the B-operand buffer for step t+1 - no cross-thread
//     exchange, no grid-wide sync.
//
// LSTM1 (H=128): K = 48 + 128.  The 48 x columns are [hi(x) (18) | 1 | lo(x) (18) | 0...]: the raw counts are unbounded integers
// (the reference's GPU branch does not rescale depth, clair3/CallVariantsFromCffi.py:299-353), fp16 is exact only to 2048, so
// every count is split as x = hi + lo with hi = fp16(x) and lo = fp16(x - hi) - exact for |x| <= 67 552; beyond that lo is
// rounded (error <= 16, <= 2^-12 relative) up to 131 008, and saturates past it - and W_ih multiplies both parts (fp32 accumulate: the same result as an exact-input product).  Column 18 is a constant 1 that
// carries b_ih + b_hh, so the x projection and the bias are fused into the same MMAs.
// LSTM2 (H=160, input 256): the input projection W_ih*h1 (+bias) is a separate big GEMM (proj_tc.cu) that leaves fp16
// pre-gates pg[t*bp + site][dir*640 + C] in gate-quad order (c3b_lstm2_pg_row: columns 128p + 4u .. +3 = gates i, f, g, o of
// unit 32p + u), so a thread loads its unit's four pre-gates of one site as one 8-byte word; a warp load covers 4 sites x 64
// contiguous bytes.  This kernel keeps only W_hh on chip (K = 160).
// The sigmoid gates' rows are pre-halved on the host so sigma(x) = 0.5*tanh(x/2)+0.5 is one MUFU + one FMA.
//
// Schedule.  Per step and block pair a warpgroup issues 2 x K/16 wgmmas (two dependent accumulation chains), waits for them,
// then runs the cell math.  The two warpgroups of a CTA run this independently; their MMA chains interleave on the tensor pipe.
// (Strict turn-taking between them, so that one's cell math runs under the other's MMAs, measured slower on H100 for LSTM1 and
// no faster for LSTM2: it serialises the two warpgroups' MMA chains, which otherwise overlap.)  LSTM2's pre-gates of block pair
// p + 1 (after the last pair: the next step's first) are loaded right after the MMAs of pair p are issued, so their DRAM
// latency hides behind a whole MMA / cell-math phase instead of stalling the start of every pair.
#include "c3b_internal.h"
#include "ptx.cuh"

namespace {

struct LstmDev {
    const op_t *w_img;             // [dir][2H/64 blocks][K/8][64][8]
    const op_t *xs;                // LSTM1 input  [33][Bp][48]: hi | 1 | lo columns
    const __half *pg;              // LSTM2 pre-gates [33*Bp][1280]
    op_t *hout;                    // tile-major k-group-planar: LSTM1 h1 (rows t*Bp+b, 32 k-groups); LSTM2 h2 (rows b, 1320 k-groups)
    int bp;                        // padded batch
    long long *trace;              // optional [33][4] clock64 stamps of CTA (0,0) thread 0 (debug option "lstm_trace")
};

__device__ __forceinline__ float lstm_cell(float gi, float gf, float gg, float go, float &c) {
    const float iv = ptx::sigmoid_prehalved(gi);
    const float fv = ptx::sigmoid_prehalved(gf);
    const float gv = ptx::tanh_approx(gg);
    const float ov = ptx::sigmoid_prehalved(go);
    c = fmaf(fv, c, iv * gv);
    return ov * ptx::tanh_approx(c);
}

// Packed variant: the four gate activations and tanh(c) of two neighbouring sites share one MUFU op each
// (tanh.approx.f16x2: 2.5 MUFU ops per cell instead of 5); i*g and o*tanh(c) are packed fp16 multiplies, the cell state and its
// update stay fp32.  Returns h as one packed (site, site+1) fp16 pair.
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ uint32_t tanh_f16x2(uint32_t x) {
    uint32_t r;
    asm("tanh.approx.f16x2 %0, %1;" : "=r"(r) : "r"(x));
    return r;
}
__device__ __forceinline__ uint32_t sigm_f16x2(uint32_t xh) {      // sigma of a pre-halved argument pair: 0.5 * tanh(xh) + 0.5
    uint32_t r;
    const uint32_t half2 = 0x38003800u;
    asm("fma.rn.f16x2 %0, %1, %2, %2;" : "=r"(r) : "r"(tanh_f16x2(xh)), "r"(half2));
    return r;
}
__device__ __forceinline__ uint32_t mul_f16x2(uint32_t a, uint32_t b) {
    uint32_t r;
    asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
__device__ __forceinline__ uint32_t lstm_cell_h2(const float *gi, const float *gf, const float *gg, const float *go, float *c) {
    const uint32_t iv = sigm_f16x2(pack_f16x2(gi[0], gi[1]));
    const uint32_t gv = tanh_f16x2(pack_f16x2(gg[0], gg[1]));
    const uint32_t ig = mul_f16x2(iv, gv);
    const uint32_t fv = sigm_f16x2(pack_f16x2(gf[0], gf[1]));
    const float2 f2 = __half22float2(*reinterpret_cast<const __half2 *>(&fv));
    const float2 g2 = __half22float2(*reinterpret_cast<const __half2 *>(&ig));
    c[0] = fmaf(f2.x, c[0], g2.x);
    c[1] = fmaf(f2.y, c[1], g2.y);
    const uint32_t ov = sigm_f16x2(pack_f16x2(go[0], go[1]));
    return mul_f16x2(ov, tanh_f16x2(pack_f16x2(c[0], c[1])));
}

// fp16 in the low / high half of a 32-bit word -> fp32
__device__ __forceinline__ float half_lo(uint32_t v) { return __half2float(__ushort_as_half((unsigned short)(v & 0xffffu))); }
__device__ __forceinline__ float half_hi(uint32_t v) { return __half2float(__ushort_as_half((unsigned short)(v >> 16))); }

// Element offset of the 8-unit group `kgh` of site `b` at time t in the layer's output, TILE-MAJOR k-group-planar
// [row tile of 128][k-groups][128 rows][8] (c3b_tile_major_offset): LSTM1 -> h1 (row = t*bp + b, 32 k-groups: dir*16 + kgh),
// LSTM2 -> h2 (row = b, 1320 k-groups: t*40 + dir*20 + kgh = the flatten order of clair3/model.py:135).
template <bool LAYER2>
__device__ __forceinline__ size_t h_out_offset(int t, int dir, int kgh, int b, int bp) {
    return LAYER2 ? c3b_tile_major_offset((size_t)b, t * 40 + dir * 20 + kgh, 1320)
                  : c3b_tile_major_offset((size_t)t * bp + b, dir * 16 + kgh, 32);
}

template <int NB>
__device__ __forceinline__ void wgmma_nb(float (&d)[NB / 2], uint64_t a, uint64_t b, uint32_t acc) {
    if constexpr (NB == 16) ptx::wgmma_m64n16k16(d, a, b, acc);
    else if constexpr (NB == 32) ptx::wgmma_m64n32k16(d, a, b, acc);
    else ptx::wgmma_m64n64k16(d, a, b, acc);
}

template <int NB, bool LAYER2, bool MUFU16, int WG>
__global__ void __launch_bounds__(128 * WG, 1) lstm_tc_kernel(const LstmDev p) {
    constexpr int H = LAYER2 ? 160 : 128;
    constexpr int KX = LAYER2 ? 0 : C3B_X1_COLS;
    constexpr int K = KX + H;                       // 176 (LSTM1) | 160 (LSTM2)
    constexpr int NP = H / 32;                      // block pairs (32 hidden units each)
    constexpr uint32_t kBlkBytes = (K / 8) * 64 * 16;   // one 64-row weight block: [K/8][64][8] fp16
    constexpr uint32_t W_BYTES = 2 * NP * kBlkBytes;
    static_assert(K % 16 == 0, "whole k-steps");
    constexpr uint32_t LBO_B = (NB + 1) * 16;       // padded: fewer bank conflicts on the h stores
    constexpr uint32_t B_BYTES = (K / 8) * LBO_B;
    constexpr int XN = LAYER2 ? 1 : (NB * (KX / 8) + 127) / 128;

    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t w_bar;

    const int tid = threadIdx.x;
    const int wg = tid >> 7;
    const int wt = tid & 127;                       // thread index in the warpgroup
    const int w = wt >> 5;                          // warp in the warpgroup
    const int lane = tid & 31;
    const int q0 = lane >> 2;
    const int s0 = 2 * (lane & 3);                  // first site column of the thread in each 8-site group
    const int dir = blockIdx.y;
    const int b0 = (blockIdx.x * WG + wg) * NB;
    uint8_t *b_smem = smem + W_BYTES + wg * B_BYTES;
    const uint32_t w_addr = ptx::smem_u32(smem);
    const uint32_t b_addr = ptx::smem_u32(b_smem);
    const uint32_t bar_id = 1 + wg;

    if (tid == 0) {
        ptx::mbar_init(&w_bar, 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();
    if (tid == 0) {
        ptx::mbar_arrive_expect_tx(&w_bar, W_BYTES);
        const char *src = reinterpret_cast<const char *>(p.w_img) + (size_t)dir * W_BYTES;
#pragma unroll 1
        for (int m = 0; m < 2 * NP; ++m) ptx::bulk_g2s(w_addr + m * kBlkBytes, src + (size_t)m * kBlkBytes, kBlkBytes, &w_bar);
    }
    // h_{-1} = 0 and (LSTM1) x of the first step
    for (uint32_t i = wt * 16; i < B_BYTES; i += 128 * 16) *reinterpret_cast<uint4 *>(b_smem + i) = make_uint4(0, 0, 0, 0);
    ptx::named_bar_sync(bar_id, 128);
    if constexpr (!LAYER2) {
        const int t = dir ? C3B_T - 1 : 0;
        for (int idx = wt; idx < NB * (KX / 8); idx += 128) {
            const int n = idx / (KX / 8), kg = idx % (KX / 8);
            *reinterpret_cast<uint4 *>(b_smem + kg * LBO_B + n * 16) =
                *reinterpret_cast<const uint4 *>(p.xs + ((size_t)t * p.bp + b0 + n) * KX + kg * 8);
        }
    }

    float c[NP][NB / 4];
#pragma unroll
    for (int pp = 0; pp < NP; ++pp)
#pragma unroll
        for (int i = 0; i < NB / 4; ++i) c[pp][i] = 0.f;
    uint32_t hq[NP][NB / 8];                        // this step's h as packed (site, site+1) fp16 pairs

    // LSTM2 pre-gates of this thread's unit for the next block pair: one 8-byte word (i, f, g, o) per site, loaded a pair early
    constexpr int PGN = LAYER2 ? NB / 4 : 1;
    uint2 pgn[PGN];
    auto load_pg = [&](int tt, int pp) {
        const __half *pgp = p.pg + (size_t)dir * 640 + pp * 128 + 4 * (8 * w + q0);
#pragma unroll
        for (int i = 0; i < NB / 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e)
                pgn[2 * i + e] = *reinterpret_cast<const uint2 *>(pgp + ((size_t)tt * p.bp + b0 + 8 * i + s0 + e) * 1280);
    };
    if constexpr (LAYER2) load_pg(dir ? C3B_T - 1 : 0, 0);

    ptx::mbar_wait(&w_bar, 0);
    const bool tr = p.trace != nullptr && tid == 0 && blockIdx.x == 0 && blockIdx.y == 0;
    for (int step = 0; step < C3B_T; ++step) {
        const int t = dir ? (C3B_T - 1 - step) : step;
        ptx::fence_proxy_async_smem();
        ptx::named_bar_sync(bar_id, 128);           // h_{t-1} / x_t are in the operand buffer
        if (tr) p.trace[step * 4 + 0] = clock64();
        // ship h_{t-1} (still in the operand buffer) to global memory while this step's MMAs run
        if (step > 0) {
            const int tp = dir ? t + 1 : t - 1;
            for (int idx = wt; idx < NB * (H / 8); idx += 128) {
                const int kgh = idx / NB, n = idx % NB;
                *reinterpret_cast<uint4 *>(p.hout + h_out_offset<LAYER2>(tp, dir, kgh, b0 + n, p.bp)) =
                    *reinterpret_cast<const uint4 *>(b_smem + (KX / 8 + kgh) * LBO_B + n * 16);
            }
        }
        // LSTM1: fetch x_{t+1} now, store it once every MMA of this step has read the operand buffer
        uint4 xnext[XN];
        if constexpr (!LAYER2) {
            if (step + 1 < C3B_T) {
                const int tn = dir ? t - 1 : t + 1;
#pragma unroll
                for (int i = 0; i < XN; ++i) {
                    const int idx = wt + i * 128;
                    if (idx < NB * (KX / 8))
                        xnext[i] = *reinterpret_cast<const uint4 *>(p.xs + ((size_t)tn * p.bp + b0 + idx / (KX / 8)) * KX + (idx % (KX / 8)) * 8);
                }
            }
        }
#pragma unroll
        for (int pp = 0; pp < NP; ++pp) {
            float acc0[NB / 2], acc1[NB / 2];
            ptx::wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < K / 16; ++ks) {
                const uint64_t bd = ptx::wgmma_desc(b_addr + ks * 2 * LBO_B, LBO_B, 128);
                const uint32_t a0 = w_addr + (2 * pp) * kBlkBytes + ks * 2 * 1024;
                wgmma_nb<NB>(acc0, ptx::wgmma_desc(a0, 1024, 128), bd, ks > 0);
                wgmma_nb<NB>(acc1, ptx::wgmma_desc(a0 + kBlkBytes, 1024, 128), bd, ks > 0);
            }
            ptx::wgmma_commit();
            // LSTM2: this pair's pre-gates were loaded one block pair ago; start the next pair's (after the last pair: the next
            // step's first) so that they arrive while this pair's MMAs and cell math run
            uint2 pgv[PGN];
            if constexpr (LAYER2) {
#pragma unroll
                for (int i = 0; i < PGN; ++i) pgv[i] = pgn[i];
                if (pp + 1 < NP) load_pg(t, pp + 1);
                else if (step + 1 < C3B_T) load_pg(dir ? t - 1 : t + 1, 0);
            }
            ptx::wgmma_wait<0>();
            ptx::fence_operand(acc0);
            ptx::fence_operand(acc1);
            if (tr && pp == 0) p.trace[step * 4 + 1] = clock64();
#pragma unroll
            for (int i = 0; i < NB / 8; ++i) {
                float gi[2], gf[2], gg[2], go[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    gi[e] = acc0[4 * i + e];
                    gf[e] = acc0[4 * i + 2 + e];
                    gg[e] = acc1[4 * i + e];
                    go[e] = acc1[4 * i + 2 + e];
                    if constexpr (LAYER2) {
                        gi[e] += half_lo(pgv[2 * i + e].x);
                        gf[e] += half_hi(pgv[2 * i + e].x);
                        gg[e] += half_lo(pgv[2 * i + e].y);
                        go[e] += half_hi(pgv[2 * i + e].y);
                    }
                }
                if (MUFU16) {
                    hq[pp][i] = lstm_cell_h2(gi, gf, gg, go, &c[pp][2 * i]);
                } else {
                    const float h0 = lstm_cell(gi[0], gf[0], gg[0], go[0], c[pp][2 * i]);
                    const float h1 = lstm_cell(gi[1], gf[1], gg[1], go[1], c[pp][2 * i + 1]);
                    hq[pp][i] = pack_f16x2(h0, h1);
                }
            }
        }
        if (tr) p.trace[step * 4 + 2] = clock64();
        ptx::named_bar_sync(bar_id, 128);           // every MMA and copy-out of this step has read the operand buffer
        // h_t -> operand buffer, element (site n, k = KX + unit)
#pragma unroll
        for (int pp = 0; pp < NP; ++pp) {
            const uint32_t kcol = KX + 32 * pp + 8 * w + q0;
            uint8_t *dst = b_smem + (kcol >> 3) * LBO_B + (kcol & 7) * 2;
#pragma unroll
            for (int i = 0; i < NB / 8; ++i) {
                *reinterpret_cast<uint16_t *>(dst + (8 * i + s0) * 16) = (uint16_t)(hq[pp][i] & 0xffffu);
                *reinterpret_cast<uint16_t *>(dst + (8 * i + s0 + 1) * 16) = (uint16_t)(hq[pp][i] >> 16);
            }
        }
        if constexpr (!LAYER2) {
            if (step + 1 < C3B_T) {
#pragma unroll
                for (int i = 0; i < XN; ++i) {
                    const int idx = wt + i * 128;
                    if (idx < NB * (KX / 8)) *reinterpret_cast<uint4 *>(b_smem + (idx % (KX / 8)) * LBO_B + (idx / (KX / 8)) * 16) = xnext[i];
                }
            }
        }
        if (tr) p.trace[step * 4 + 3] = clock64();
    }

    // last h
    ptx::named_bar_sync(bar_id, 128);
    const int tl = dir ? 0 : C3B_T - 1;
    for (int idx = wt; idx < NB * (H / 8); idx += 128) {
        const int kgh = idx / NB, n = idx % NB;
        *reinterpret_cast<uint4 *>(p.hout + h_out_offset<LAYER2>(tl, dir, kgh, b0 + n, p.bp)) =
            *reinterpret_cast<const uint4 *>(b_smem + (KX / 8 + kgh) * LBO_B + n * 16);
    }
}

template <typename T>
__device__ __forceinline__ float ingest_to_float(T v) { return (float)v; }

// Dense [batch][33][channels] tensor, or (starts != nullptr) 33-row windows of the per-column count matrix [n_cols][channels]
// (libclair3's plp_data.matrix; preprocess/CreateTensorPileupFromCffi.py:356-396 slices the same windows on the host, zero
// rows where a window overhangs its contiguous run: rows outside [bounds[b][0], bounds[b][1]) and outside the matrix read as 0) -> xs[t][bp][48] fp16 with columns [hi(x) | 1 | lo(x) | 0..]: hi = fp16(x)
// (saturating at +-65504), lo = fp16(x - hi), so hi + lo == x exactly for |x| <= 67 552 (past 65 519 hi stays at 65 504 and
// lo > 2048 is itself rounded: error <= 16, <= 2^-12 relative, up to 131 008; saturating beyond); column `channels` = constant 1
// (LSTM1's bias column).
template <typename T>
__global__ void ingest_pileup_tc_kernel(const T *__restrict__ x, const int64_t *__restrict__ starts,
                                        const int64_t *__restrict__ bounds, int64_t n_cols, op_t *__restrict__ xs, int64_t batch,
                                        int bp, int channels) {
    // one thread per (t, site): six 16-byte stores
    const int64_t total = (int64_t)C3B_T * bp;
    for (int64_t tb = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; tb < total; tb += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(tb % bp);
        const int t = (int)(tb / bp);
        bool have = b < batch;
        const T *src = x;
        if (have) {
            if (starts) {
                const int64_t row = starts[b] + t;
                have = row >= 0 && row < n_cols && (!bounds || (row >= bounds[2 * b] && row < bounds[2 * b + 1]));
                src = x + row * channels;
            } else {
                src = x + ((int64_t)b * C3B_T + t) * channels;
            }
        }
        __align__(16) op_t v[C3B_X1_COLS];
        if (channels == 18) {
            // the reference's pileup shape (shared/param_p.py:32-36): every index is a compile-time constant, one load per count
            float xv[18];
#pragma unroll
            for (int c = 0; c < 18; ++c) xv[c] = have ? ingest_to_float(src[c]) : 0.f;
#pragma unroll
            for (int c = 0; c < 18; ++c) {
                const op_t hi = f2op_sat(xv[c]);
                v[c] = hi;
                v[19 + c] = f2op_sat(xv[c] - op2f(hi));
            }
            v[18] = f2op(1.f);
#pragma unroll
            for (int k = 37; k < C3B_X1_COLS; ++k) v[k] = f2op(0.f);
        } else {
#pragma unroll
            for (int k = 0; k < C3B_X1_COLS; ++k) {          // static indices: v stays in registers
                float f = (k == channels) ? 1.f : 0.f;
                if (have && k != channels && k <= 2 * channels) {
                    const float xvv = ingest_to_float(src[k < channels ? k : k - channels - 1]);
                    const op_t hi = f2op_sat(xvv);
                    f = k < channels ? op2f(hi) : xvv - op2f(hi);
                }
                v[k] = f2op_sat(f);
            }
        }
        uint4 *dst = reinterpret_cast<uint4 *>(xs + tb * C3B_X1_COLS);
#pragma unroll
        for (int k = 0; k < C3B_X1_COLS / 8; ++k) dst[k] = reinterpret_cast<const uint4 *>(v)[k];
    }
}

template <int NB, bool LAYER2, bool MUFU16, int WG>
int launch_lstm_impl(const LstmDev &p, cudaStream_t s) {
    constexpr int K = (LAYER2 ? 0 : C3B_X1_COLS) + (LAYER2 ? 160 : 128);
    constexpr int H = LAYER2 ? 160 : 128;
    const size_t smem = (size_t)4 * H * K * 2 + (size_t)WG * (K / 8) * (NB + 1) * 16;   // 4H gate rows of fp16 weights + operands
    auto kern = lstm_tc_kernel<NB, LAYER2, MUFU16, WG>;
    C3B_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(p.bp / (WG * NB), 2);
    c3b_note_grid((long long)grid.x * grid.y);
    kern<<<grid, 128 * WG, smem, s>>>(p);
    C3B_CUDA(cudaGetLastError());
    return 0;
}

// wg = warpgroups per CTA (each owns one NB-site sub-tile; they share the CTA's copy of the weights)
template <int NB, bool LAYER2>
int launch_lstm(const LstmDev &p, bool mufu16, int wg, cudaStream_t s) {
    if (mufu16) return wg == 1 ? launch_lstm_impl<NB, LAYER2, true, 1>(p, s) : launch_lstm_impl<NB, LAYER2, true, 2>(p, s);
    return wg == 1 ? launch_lstm_impl<NB, LAYER2, false, 1>(p, s) : launch_lstm_impl<NB, LAYER2, false, 2>(p, s);
}

}  // namespace

int c3b_launch_ingest_pileup_tc(const void *x, int dtype, int channels, const int64_t *starts, const int64_t *bounds, int64_t n_cols,
                                op_t *xs, int64_t batch, int bp, cudaStream_t s) {
    const int64_t total = (int64_t)C3B_T * bp;
    const int blocks = (int)((total + 127) / 128 < 2048 ? (total + 127) / 128 : 2048);
    c3b_note_grid(blocks);
    switch (dtype) {
        case C3B_DT_I8: ingest_pileup_tc_kernel<int8_t><<<blocks, 128, 0, s>>>((const int8_t *)x, starts, bounds, n_cols, xs, batch, bp, channels); break;
        case C3B_DT_I32: ingest_pileup_tc_kernel<int32_t><<<blocks, 128, 0, s>>>((const int32_t *)x, starts, bounds, n_cols, xs, batch, bp, channels); break;
        case C3B_DT_I64: ingest_pileup_tc_kernel<int64_t><<<blocks, 128, 0, s>>>((const int64_t *)x, starts, bounds, n_cols, xs, batch, bp, channels); break;
        case C3B_DT_F32: ingest_pileup_tc_kernel<float><<<blocks, 128, 0, s>>>((const float *)x, starts, bounds, n_cols, xs, batch, bp, channels); break;
        default: c3b_set_error("unsupported input dtype %d", dtype); return 1;
    }
    C3B_CUDA(cudaGetLastError());
    return 0;
}

// `tile` = sites per warpgroup sub-tile.
int c3b_launch_lstm1_tc(const c3b_model *m, const TcPileupBuffers &b, int64_t batch, int tile, cudaStream_t s) {
    LstmDev p = {};
    p.w_img = m->lstm_tc[0];
    p.xs = b.xs;
    p.hout = b.h1;
    p.trace = m->lstm_trace;
    p.bp = b.bp;
    const_cast<c3b_model *>(m)->launches++;
    switch (tile) {
        case 16: return launch_lstm<16, false>(p, m->lstm_mufu16 != 0, m->lstm_wg, s);
        case 32: return launch_lstm<32, false>(p, m->lstm_mufu16 != 0, m->lstm_wg, s);
        case 64: return launch_lstm<64, false>(p, m->lstm_mufu16 != 0, m->lstm_wg, s);
    }
    c3b_set_error("lstm1: unsupported tile %d", tile);
    return 1;
}

int c3b_launch_lstm2_tc(const c3b_model *m, const TcPileupBuffers &b, int64_t batch, int tile, cudaStream_t s) {
    LstmDev p = {};
    p.w_img = m->lstm_tc[1];
    p.pg = b.pg;
    p.hout = b.h2;
    p.trace = m->lstm_trace ? m->lstm_trace + C3B_T * 4 : nullptr;
    p.bp = b.bp;
    const_cast<c3b_model *>(m)->launches++;
    switch (tile) {
        case 16: return launch_lstm<16, true>(p, m->lstm_mufu16 != 0, m->lstm_wg, s);
        case 32: return launch_lstm<32, true>(p, m->lstm_mufu16 != 0, m->lstm_wg, s);
    }
    c3b_set_error("lstm2: unsupported tile %d", tile);
    return 1;
}
