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
// carries b_ih + b_hh, so the x projection and the bias are fused into the same MMAs.  The kernel builds these columns itself
// from the caller's raw counts (int8 / int32 / int64 / float32, one instance per dtype): from the dense [batch][33][C] tensor or
// from the 33-row windows of forward_windows' column matrix, one step ahead, in registers, straight into the operand buffer - the
// x operand never goes through HBM (with the "taps" option a copy goes to a [33][Bp][48] tap buffer).
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
//
// LSTM2 split by block pair (lstm2_split_kernel).  One CTA = one direction x NB sites (32, or 16 under the latency tile rule)
// with five warpgroups, 640 threads; warpgroup p issues only block pair p's 2 x K/16 wgmmas (same descriptors, k order and N),
// runs the cell math of units 32p .. 32p+31 and writes their h_t into a double-buffered operand (step s reads buffer s & 1 and
// writes the other), so one CTA barrier per step is the only exchange.  W_hh 200 KB + 2 x 20 x (NB+1) x 16 B = 221 KB at NB = 32;
// 94 registers per thread.  The five chains share one tensor pipe (one m64n32k16 from shared memory every ~46 cycles on H100);
// issued together they interleave and all finish last, so no cell math overlaps an MMA (6.2 k cycles per 32-site step).  Issued
// in block-pair order they finish in turn, and each warpgroup's cell math runs under the later chains (5.0 k cycles, against
// 10.8 k for 64 sites in the sub-tile kernel).  Each block pair's weights have their own mbarrier, so warpgroup 0 starts step 0
// once its 40 KB have arrived.
// Every LSTM2 kernel writes the pre-gates into the accumulators and starts each chain from them (scale-d = 1): the same fp32
// addition order in all of them, so they stay bit-identical to each other.  Option lstm2_split 2 runs the split kernel at 48
// sites with one h operand buffer (see lstm2_split_kernel): 6.8 k cycles per 48-site step against 5.0 k (now 4.7 k) per 32-site
// step, ~3 % fewer cycles per site, no measurable end-to-end gain on H100, so not the default.
#include <type_traits>

#include "c3b_internal.h"
#include "ptx.cuh"

namespace {

struct LstmDev {
    const op_t *w_img;             // [dir][2H/64 blocks][K/8][64][8]
    PileupSrc x;                   // LSTM1 input: the caller's dense tensor or column matrix (PileupSrc), read by the kernel itself
    int64_t batch;                 // LSTM1: real sites; sites b >= batch read as 0
    int channels;                  // LSTM1: counts per site-step
    op_t *x_tap;                   // LSTM1, optional: [33][Bp][48] copy of the x operand columns it built (option "taps")
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
    else if constexpr (NB == 48) ptx::wgmma_m64n48k16(d, a, b, acc);
    else ptx::wgmma_m64n64k16(d, a, b, acc);
}

// ---- LSTM1's x operand columns from the caller's counts (see the header): column k is hi(x_k) for k < C, 1 for k == C,
// lo(x_{k-C-1}) for C < k <= 2C and 0 beyond, so k-group kg holds columns 8kg .. 8kg+7.

// Row t of site b, or nullptr where it reads as 0: padded sites, and window rows outside the matrix or outside the site's bounds
// (preprocess/CreateTensorPileupFromCffi.py:356-396 zero-pads a window where it overhangs its contiguous run)
template <typename T>
__device__ __forceinline__ const T *x_row(const LstmDev &p, int b, int t) {
    if (b >= p.batch) return nullptr;
    const T *x = static_cast<const T *>(p.x.x);
    if (!p.x.starts) return x + ((int64_t)b * C3B_T + t) * p.channels;
    const int64_t row = p.x.starts[b] + t;
    if (row < 0 || row >= p.x.n_cols || (p.x.bounds && (row < p.x.bounds[2 * b] || row >= p.x.bounds[2 * b + 1]))) return nullptr;
    return x + row * p.channels;
}

template <typename T>
struct alignas(2 * sizeof(T)) XPair { T v[2]; };

// The 18 counts of a row (the reference's pileup shape, shared/param_p.py:32-36): nine 2-count loads when the input's base is
// aligned for them (every row then is: rows are 18 counts apart), else one load per count
template <typename T>
__device__ __forceinline__ void load_row18(const T *row, bool pairs, T (&r)[18]) {
    if (!row) {
#pragma unroll
        for (int c = 0; c < 18; ++c) r[c] = T(0);
    } else if (pairs) {
#pragma unroll
        for (int j = 0; j < 9; ++j) {
            const XPair<T> q = reinterpret_cast<const XPair<T> *>(row)[j];
            r[2 * j] = q.v[0];
            r[2 * j + 1] = q.v[1];
        }
    } else {
#pragma unroll
        for (int c = 0; c < 18; ++c) r[c] = row[c];
    }
}

// The 18 counts as floats, (float)v exactly.  Small integers (|v| < 2^22: every realistic count) go through the float bit
// pattern of 1.5 * 2^23 + v on the ALU: int8 and int64 conversions otherwise issue to the quarter-rate unit that the cell math's
// tanh already saturates.
template <typename T>
__device__ __forceinline__ void counts_to_float18(const T (&r)[18], float (&xf)[18]) {
    if constexpr (std::is_same<T, float>::value || std::is_same<T, int32_t>::value) {
#pragma unroll
        for (int c = 0; c < 18; ++c) xf[c] = (float)r[c];
    } else {
        bool small = true;                          // int8: always
#pragma unroll
        for (int c = 0; c < 18 && sizeof(T) > 1; ++c) small &= (uint64_t)((int64_t)r[c] + (1 << 22)) < (1u << 23);
        if (small) {
#pragma unroll
            for (int c = 0; c < 18; ++c) xf[c] = __int_as_float(0x4B400000 + (int)r[c]) - 12582912.f;
        } else {
#pragma unroll
            for (int c = 0; c < 18; ++c) xf[c] = (float)r[c];
        }
    }
}

// hi(x) of channel c as a float: fp16(x) saturating, from one packed conversion of c's channel pair
__device__ __forceinline__ float x_hi18(const float (&xf)[18], int c) {
    const uint32_t h = f2op2_sat(xf[c & ~1], xf[c | 1]);
    const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&h));
    return (c & 1) ? f.y : f.x;
}

// column k before its fp16 rounding: x_k, 1, x - hi(x), 0
__device__ __forceinline__ float x_col18(const float (&xf)[18], int k) {
    if (k < 18) return xf[k];
    if (k == 18) return 1.f;
    if (k < 37) return xf[k - 19] - x_hi18(xf, k - 19);
    return 0.f;
}

// k-group kg of a row with 18 counts, two columns per (saturating) conversion; kg must be a compile-time constant, so every
// index is one
__device__ __forceinline__ uint4 x_kgroup18(const float (&xf)[18], int kg) {
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) w[j] = f2op2_sat(x_col18(xf, 8 * kg + 2 * j), x_col18(xf, 8 * kg + 2 * j + 1));
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// k-group kg of a row with any other channel count c (row == nullptr: a zero row): one load per column
template <typename T>
__device__ __forceinline__ uint4 x_kgroup(const T *row, int c, int kg) {
    __align__(16) op_t v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int k = 8 * kg + j;
        float f = (k == c) ? 1.f : 0.f;
        if (row && k != c && k <= 2 * c) {
            const float x = (float)row[k < c ? k : k - c - 1];
            const op_t hi = f2op_sat(x);
            f = k < c ? op2f(hi) : x - op2f(hi);
        }
        v[j] = f2op_sat(f);
    }
    return *reinterpret_cast<const uint4 *>(v);
}

// T: LSTM1's input dtype (LSTM2 reads no input and is instantiated with float)
template <int NB, bool LAYER2, bool MUFU16, int WG, typename T>
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
    // LSTM1: a thread builds the x k-groups (wt + 128 i) / NB, i < XN, of site wt % NB - all of them from one row
    constexpr int XN = LAYER2 ? 1 : (NB * (KX / 8) + 127) / 128;
    constexpr int XR = LAYER2 ? 1 : 18;

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
    const int xn = wt % NB;
    const bool c18 = p.channels == 18;
    const bool pairs = (reinterpret_cast<uintptr_t>(p.x.x) & (2 * sizeof(T) - 1)) == 0;
    // x k-group of item i (a compile-time constant: it bounds the k-groups the item can hold), from the row's counts xf (as
    // floats) when channels == 18, else from the row itself
    auto x_item = [&](int i, const float(&xf)[XR], const T *row) {
        const int kg = (wt + 128 * i) / NB;
        uint4 v = make_uint4(0, 0, 0, 0);
        if constexpr (!LAYER2) {
            if (c18) {
#pragma unroll
                for (int g = 0; g < KX / 8; ++g)
                    if (g >= 128 * i / NB && g <= (128 * i + 127) / NB && kg == g) v = x_kgroup18(xf, g);
            } else {
                v = x_kgroup(row, p.channels, kg);
            }
        }
        return v;
    };
    // store item i of x_t into the operand buffer (and the tap)
    auto x_store = [&](int i, int t, uint4 v) {
        const int kg = (wt + 128 * i) / NB;
        *reinterpret_cast<uint4 *>(b_smem + kg * LBO_B + xn * 16) = v;
        if (p.x_tap) *reinterpret_cast<uint4 *>(p.x_tap + ((size_t)t * p.bp + b0 + xn) * KX + kg * 8) = v;
    };
    if constexpr (!LAYER2) {
        const int t = dir ? C3B_T - 1 : 0;
        const T *row = x_row<T>(p, b0 + xn, t);
        T r[XR];
        float xf[XR];
        if (c18) {
            load_row18(row, pairs, r);
            counts_to_float18(r, xf);
        }
#pragma unroll
        for (int i = 0; i < XN; ++i)
            if (wt + 128 * i < NB * (KX / 8)) x_store(i, t, x_item(i, xf, row));
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
        // LSTM1: start loading x_{t+1}'s counts now; they become operand columns while the second block pair's MMAs run (a whole
        // block pair later, so the loads have arrived; hq holds one pair then), and go into the operand buffer once every MMA of
        // this step has read it
        const int tn = dir ? t - 1 : t + 1;
        const T *xrow = nullptr;
        T xr[XR];
        uint4 xnext[XN];
        if constexpr (!LAYER2) {
            if (step + 1 < C3B_T) {
                xrow = x_row<T>(p, b0 + xn, tn);
                if (c18) load_row18(xrow, pairs, xr);
            }
        }
#pragma unroll
        for (int pp = 0; pp < NP; ++pp) {
            float acc0[NB / 2], acc1[NB / 2];
            // LSTM2: this pair's pre-gates, loaded one block pair ago, are where the chain starts accumulating
            if constexpr (LAYER2) {
#pragma unroll
                for (int i = 0; i < NB / 8; ++i)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        acc0[4 * i + e] = half_lo(pgn[2 * i + e].x);
                        acc0[4 * i + 2 + e] = half_hi(pgn[2 * i + e].x);
                        acc1[4 * i + e] = half_lo(pgn[2 * i + e].y);
                        acc1[4 * i + 2 + e] = half_hi(pgn[2 * i + e].y);
                    }
            }
            ptx::wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < K / 16; ++ks) {
                const uint64_t bd = ptx::wgmma_desc(b_addr + ks * 2 * LBO_B, LBO_B, 128);
                const uint32_t a0 = w_addr + (2 * pp) * kBlkBytes + ks * 2 * 1024;
                wgmma_nb<NB>(acc0, ptx::wgmma_desc(a0, 1024, 128), bd, LAYER2 || ks > 0);
                wgmma_nb<NB>(acc1, ptx::wgmma_desc(a0 + kBlkBytes, 1024, 128), bd, LAYER2 || ks > 0);
            }
            ptx::wgmma_commit();
            // LSTM2: start the next pair's pre-gates (after the last pair: the next step's first) so that they arrive while this
            // pair's MMAs and cell math run
            if constexpr (LAYER2) {
                if (pp + 1 < NP) load_pg(t, pp + 1);
                else if (step + 1 < C3B_T) load_pg(tn, 0);
            } else {
                if (pp == 1 && step + 1 < C3B_T) {
                    float xf[XR];
                    if (c18) counts_to_float18(xr, xf);
#pragma unroll
                    for (int i = 0; i < XN; ++i)
                        if (wt + 128 * i < NB * (KX / 8)) xnext[i] = x_item(i, xf, xrow);
                }
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
                for (int i = 0; i < XN; ++i)
                    if (wt + 128 * i < NB * (KX / 8)) x_store(i, tn, xnext[i]);
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

// LSTM2 split by block pair (option "lstm2_split", see the header): one CTA = one direction x NB sites, five warpgroups, and
// warpgroup pp owns block pair pp (hidden units 32pp .. 32pp + 31) of all NB sites.  The per-site arithmetic is lstm_tc_kernel's
// for LAYER2: the same A blocks, B columns, k order per wgmma chain, the same accumulator start (the pre-gates), the same cell
// math; a site's column does not depend on N.  NB = 48 keeps one h operand buffer (two do not fit beside W_hh) and loads the next
// step's pre-gates after the cell math, where the accumulators are free: during the chain, beside the 48 accumulators, they
// would spill (96 registers per thread at 640 threads; at NB = 64 the accumulators and cell state alone leave too few).  bp is
// a multiple of 128, so the last 48-site CTA runs past it; its sites >= bp read zero pre-gates and write no h.
template <int NB, bool MUFU16>
__global__ void __launch_bounds__(640, 1) lstm2_split_kernel(const LstmDev p) {
    constexpr int H = 160;
    constexpr int K = H;
    constexpr int NP = H / 32;
    constexpr uint32_t kBlkBytes = (K / 8) * 64 * 16;
    constexpr uint32_t W_BYTES = 2 * NP * kBlkBytes;
    constexpr uint32_t LBO_B = (NB + 1) * 16;
    constexpr uint32_t B_BYTES = (K / 8) * LBO_B;
    constexpr bool ONE_BUF = NB == 48;
    constexpr int NBUF = ONE_BUF ? 1 : 2;

    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t w_bar[NP];                  // one per block pair: a warpgroup starts once its own 40 KB have arrived

    const int tid = threadIdx.x;
    const int pp = tid >> 7;                        // this warpgroup's block pair
    const int wt = tid & 127;
    const int w = wt >> 5;
    const int lane = tid & 31;
    const int q0 = lane >> 2;
    const int s0 = 2 * (lane & 3);
    const int dir = blockIdx.y;
    const int b0 = blockIdx.x * NB;
    // NB < 48: two operand buffers of h: step s reads buffer s & 1 and writes h_t into the other, so one CTA barrier per step
    // orders both the reads of step s - 1 before the writes of step s + 1 and the writes of step s before the reads of step s + 1.
    // NB = 48: one buffer; a second CTA barrier per step, after every chain has read h_{t-1}, comes before the h_t stores.
    uint8_t *b_smem = smem + W_BYTES;
    const uint32_t w_addr = ptx::smem_u32(smem);
    const uint32_t b_addr = ptx::smem_u32(b_smem);

    if (tid == 0) {
#pragma unroll
        for (int m = 0; m < NP; ++m) ptx::mbar_init(&w_bar[m], 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();
    if (tid == 0) {
        const char *src = reinterpret_cast<const char *>(p.w_img) + (size_t)dir * W_BYTES;
#pragma unroll 1
        for (int m = 0; m < NP; ++m) {
            ptx::mbar_arrive_expect_tx(&w_bar[m], 2 * kBlkBytes);
            ptx::bulk_g2s(w_addr + 2 * m * kBlkBytes, src + (size_t)2 * m * kBlkBytes, 2 * kBlkBytes, &w_bar[m]);
        }
    }
    for (uint32_t i = tid * 16; i < B_BYTES; i += 640 * 16) *reinterpret_cast<uint4 *>(b_smem + i) = make_uint4(0, 0, 0, 0);   // h_{-1}

    float c[NB / 4];
#pragma unroll
    for (int i = 0; i < NB / 4; ++i) c[i] = 0.f;

    // pre-gates of this thread's unit, one 8-byte word (i, f, g, o) per site, for the next step: loaded a whole step early
    // (NB = 48: most of a step early)
    uint2 pgn[NB / 4];
    auto load_pg = [&](int tt) {
        int col = dir * 640 + pp * 128 + 4 * (8 * w + q0);
        asm volatile("" : "+r"(col));               // opaque, as i0 in copy_out: a pointer kept across steps spills at NB = 48
        const __half *pgp = p.pg + col;
#pragma unroll
        for (int i = 0; i < NB / 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int b = b0 + 8 * i + s0 + e;
                pgn[2 * i + e] = NB % 128 == 0 || b < p.bp ? *reinterpret_cast<const uint2 *>(pgp + ((size_t)tt * p.bp + b) * 1280)
                                                           : make_uint2(0, 0);
            }
    };
    load_pg(dir ? C3B_T - 1 : 0);
    // h of time tt (in operand buffer `buf`) -> hout: this warpgroup's four k-groups
    auto copy_out = [&](int tt, int buf) {
        int i0 = wt;                                // opaque: else its addresses are kept across steps (NB = 48: spilled)
        asm volatile("" : "+r"(i0));
        for (int idx = i0; idx < NB * 4; idx += 128) {
            const int kgh = 4 * pp + idx / NB, n = idx % NB;
            if (NB % 128 != 0 && b0 + n >= p.bp) continue;
            *reinterpret_cast<uint4 *>(p.hout + h_out_offset<true>(tt, dir, kgh, b0 + n, p.bp)) =
                *reinterpret_cast<const uint4 *>(b_smem + buf * B_BYTES + kgh * LBO_B + n * 16);
        }
    };

    const bool tr = p.trace != nullptr && tid == 0 && blockIdx.x == 0 && blockIdx.y == 0;
    for (int step = 0; step < C3B_T; ++step) {
        const int t = dir ? (C3B_T - 1 - step) : step;
        const int cur = ONE_BUF ? 0 : step & 1;
        ptx::fence_proxy_async_smem();
        __syncthreads();                            // h_{t-1} is in buffer cur; (NB < 48) every read of buffer cur ^ 1 is done
        if (tr) p.trace[step * 4 + 0] = clock64();
        // the chain adds W_hh h_{t-1} onto the pre-gates
        float acc0[NB / 2], acc1[NB / 2];
#pragma unroll
        for (int i = 0; i < NB / 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                acc0[4 * i + e] = half_lo(pgn[2 * i + e].x);
                acc0[4 * i + 2 + e] = half_hi(pgn[2 * i + e].x);
                acc1[4 * i + e] = half_lo(pgn[2 * i + e].y);
                acc1[4 * i + 2 + e] = half_hi(pgn[2 * i + e].y);
            }
        // the warpgroups issue their chains in block-pair order (named barrier pp: warpgroup pp - 1 arrives once its chain is
        // issued), so the tensor pipe finishes them one after another and each warpgroup's cell math runs under the later
        // warpgroups' MMAs; issued together, the five chains interleave and every cell math waits for the last MMA
        if (step == 0) ptx::mbar_wait(&w_bar[pp], 0);
        if (pp > 0) ptx::named_bar_sync(pp, 256);
        // the operand addresses, opaque to the compiler within a step: else it keeps the chain's 30 descriptors live through the
        // whole loop (NB = 48: beside the 48 accumulators and 12 cells, they spill)
        uint32_t wa = w_addr + (2 * pp) * kBlkBytes, ba = b_addr + cur * B_BYTES;
        asm volatile("" : "+r"(wa), "+r"(ba));
        ptx::wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < K / 16; ++ks) {
            const uint64_t bd = ptx::wgmma_desc(ba + ks * 2 * LBO_B, LBO_B, 128);
            const uint32_t a0 = wa + ks * 2 * 1024;
            wgmma_nb<NB>(acc0, ptx::wgmma_desc(a0, 1024, 128), bd, 1);
            wgmma_nb<NB>(acc1, ptx::wgmma_desc(a0 + kBlkBytes, 1024, 128), bd, 1);
        }
        ptx::wgmma_commit();
        if (pp + 1 < NP) ptx::named_bar_arrive(pp + 1, 256);
        // start the next step's pre-gates, and ship h_{t-1} while the MMAs run (NB < 48)
        if (!ONE_BUF && step + 1 < C3B_T) load_pg(dir ? t - 1 : t + 1);
        if (!ONE_BUF && step > 0) copy_out(dir ? t + 1 : t - 1, cur);
        ptx::wgmma_wait<0>();
        ptx::fence_operand(acc0);
        ptx::fence_operand(acc1);
        if (tr) p.trace[step * 4 + 1] = clock64();
        uint32_t hq[NB / 8];
#pragma unroll
        for (int i = 0; i < NB / 8; ++i) {
            float gi[2], gf[2], gg[2], go[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                gi[e] = acc0[4 * i + e];
                gf[e] = acc0[4 * i + 2 + e];
                gg[e] = acc1[4 * i + e];
                go[e] = acc1[4 * i + 2 + e];
            }
            if (MUFU16) {
                hq[i] = lstm_cell_h2(gi, gf, gg, go, &c[2 * i]);
            } else {
                const float h0 = lstm_cell(gi[0], gf[0], gg[0], go[0], c[2 * i]);
                const float h1 = lstm_cell(gi[1], gf[1], gg[1], go[1], c[2 * i + 1]);
                hq[i] = pack_f16x2(h0, h1);
            }
        }
        if (tr) p.trace[step * 4 + 2] = clock64();
        if constexpr (ONE_BUF) {
            if (step + 1 < C3B_T) load_pg(dir ? t - 1 : t + 1);
            if (step > 0) copy_out(dir ? t + 1 : t - 1, cur);
            __syncthreads();                        // every chain and copy-out of this step has read h_{t-1}
        }
        // h_t -> buffer cur ^ 1 (NB = 48: buffer 0), element (site n, k = unit)
        const uint32_t kcol = 32 * pp + 8 * w + q0;
        uint8_t *dst = b_smem + (cur ^ 1) % NBUF * B_BYTES + (kcol >> 3) * LBO_B + (kcol & 7) * 2;
#pragma unroll
        for (int i = 0; i < NB / 8; ++i) {
            *reinterpret_cast<uint16_t *>(dst + (8 * i + s0) * 16) = (uint16_t)(hq[i] & 0xffffu);
            *reinterpret_cast<uint16_t *>(dst + (8 * i + s0 + 1) * 16) = (uint16_t)(hq[i] >> 16);
        }
        if (tr) p.trace[step * 4 + 3] = clock64();
    }

    // last h
    __syncthreads();
    copy_out(dir ? 0 : C3B_T - 1, C3B_T % NBUF);
}

template <int NB, bool MUFU16>
int launch_lstm2_split_impl(const LstmDev &p, cudaStream_t s) {
    const size_t smem = (size_t)4 * 160 * 160 * 2 + (size_t)(NB == 48 ? 1 : 2) * (160 / 8) * (NB + 1) * 16;   // W_hh + h operand buffers
    auto kern = lstm2_split_kernel<NB, MUFU16>;
    C3B_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((p.bp + NB - 1) / NB, 2);
    c3b_note_grid((long long)grid.x * grid.y);
    kern<<<grid, 640, smem, s>>>(p);
    C3B_CUDA(cudaGetLastError());
    return 0;
}

template <int NB>
int launch_lstm2_split(const LstmDev &p, bool mufu16, cudaStream_t s) {
    return mufu16 ? launch_lstm2_split_impl<NB, true>(p, s) : launch_lstm2_split_impl<NB, false>(p, s);
}

template <int NB, bool LAYER2, bool MUFU16, int WG, typename T>
int launch_lstm_impl(const LstmDev &p, cudaStream_t s) {
    constexpr int K = (LAYER2 ? 0 : C3B_X1_COLS) + (LAYER2 ? 160 : 128);
    constexpr int H = LAYER2 ? 160 : 128;
    const size_t smem = (size_t)4 * H * K * 2 + (size_t)WG * (K / 8) * (NB + 1) * 16;   // 4H gate rows of fp16 weights + operands
    auto kern = lstm_tc_kernel<NB, LAYER2, MUFU16, WG, T>;
    C3B_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(p.bp / (WG * NB), 2);
    c3b_note_grid((long long)grid.x * grid.y);
    kern<<<grid, 128 * WG, smem, s>>>(p);
    C3B_CUDA(cudaGetLastError());
    return 0;
}

// wg = warpgroups per CTA (each owns one NB-site sub-tile; they share the CTA's copy of the weights)
template <int NB, bool LAYER2, typename T = float>
int launch_lstm(const LstmDev &p, bool mufu16, int wg, cudaStream_t s) {
    if (mufu16) return wg == 1 ? launch_lstm_impl<NB, LAYER2, true, 1, T>(p, s) : launch_lstm_impl<NB, LAYER2, true, 2, T>(p, s);
    return wg == 1 ? launch_lstm_impl<NB, LAYER2, false, 1, T>(p, s) : launch_lstm_impl<NB, LAYER2, false, 2, T>(p, s);
}

template <int NB>
int launch_lstm1(const LstmDev &p, bool mufu16, int wg, cudaStream_t s) {
    switch (p.x.dtype) {
        case C3B_DT_I8: return launch_lstm<NB, false, int8_t>(p, mufu16, wg, s);
        case C3B_DT_I32: return launch_lstm<NB, false, int32_t>(p, mufu16, wg, s);
        case C3B_DT_I64: return launch_lstm<NB, false, int64_t>(p, mufu16, wg, s);
        case C3B_DT_F32: return launch_lstm<NB, false, float>(p, mufu16, wg, s);
    }
    c3b_set_error("lstm1: unsupported input dtype %d", p.x.dtype);
    return 1;
}

}  // namespace

// `tile` = sites per warpgroup sub-tile.
int c3b_launch_lstm1_tc(const c3b_model *m, const TcPileupBuffers &b, const PileupSrc &src, int64_t batch, int tile,
                        cudaStream_t s) {
    LstmDev p = {};
    p.w_img = m->lstm_tc[0];
    p.x = src;
    p.batch = batch;
    p.channels = m->channels;
    p.x_tap = b.x_tap;
    p.hout = b.h1;
    p.trace = m->lstm_trace;
    p.bp = b.bp;
    const_cast<c3b_model *>(m)->launches++;
    switch (tile) {
        case 16: return launch_lstm1<16>(p, m->lstm_mufu16 != 0, m->lstm_wg, s);
        case 32: return launch_lstm1<32>(p, m->lstm_mufu16 != 0, m->lstm_wg, s);
        case 64: return launch_lstm1<64>(p, m->lstm_mufu16 != 0, m->lstm_wg, s);
    }
    c3b_set_error("lstm1: unsupported tile %d", tile);
    return 1;
}

int c3b_launch_lstm2_tc(const c3b_model *m, const TcPileupBuffers &b, int64_t batch, int tile, bool split, cudaStream_t s) {
    LstmDev p = {};
    p.w_img = m->lstm_tc[1];
    p.pg = b.pg;
    p.hout = b.h2;
    p.trace = m->lstm_trace ? m->lstm_trace + C3B_T * 4 : nullptr;
    p.bp = b.bp;
    const_cast<c3b_model *>(m)->launches++;
    if (split) {
        switch (tile) {
            case 16: return launch_lstm2_split<16>(p, m->lstm_mufu16 != 0, s);
            case 32: return launch_lstm2_split<32>(p, m->lstm_mufu16 != 0, s);
            case 48: return launch_lstm2_split<48>(p, m->lstm_mufu16 != 0, s);
        }
    } else {
        switch (tile) {
            case 16: return launch_lstm<16, true>(p, m->lstm_mufu16 != 0, m->lstm_wg, s);
            case 32: return launch_lstm<32, true>(p, m->lstm_mufu16 != 0, m->lstm_wg, s);
        }
    }
    c3b_set_error("lstm2: unsupported tile %d", tile);
    return 1;
}
