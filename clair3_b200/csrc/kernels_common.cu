// Kernels shared by both precisions: input ingest (dtype -> float) and the dense multi-task heads
// (SELU(L4) -> SELU(L5_k) -> SELU(Y_k) -> softmax, clair3/model.py:136-159 and 391-411), all fp32 on CUDA cores.
#include "c3b_internal.h"

namespace {

constexpr float kSeluAlpha = 1.6732632423543772f;
constexpr float kSeluScale = 1.0507009873554805f;

__device__ __forceinline__ float selu(float x) {
    return kSeluScale * (x > 0.f ? x : kSeluAlpha * expm1f(x));
}

template <typename T>
__global__ void ingest_f32_kernel(const T *__restrict__ x, float *__restrict__ out, int64_t n) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = (float)x[i];
}

// fp32 debug path of c3b_forward_windows: out[b][t][c] = cols[starts[b] + t][c], zero outside the matrix
template <typename T>
__global__ void gather_windows_f32_kernel(const T *__restrict__ cols, const int64_t *__restrict__ starts, int64_t n_cols, int channels,
                                          float *__restrict__ out, int64_t n) {
    const int per = C3B_T * channels;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n * per; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = i / per;
        const int r = (int)(i - b * per);
        const int t = r / channels, c = r - t * channels;
        const int64_t row = starts[b] + t;
        out[i] = (row >= 0 && row < n_cols) ? (float)cols[row * channels + c] : 0.f;
    }
}

constexpr int HEADS_THREADS = 256;
constexpr int HEADS_KT = 32;      // k rows of an L5 weight tile staged in shared memory
constexpr int HEADS_STAGES = 3;   // L5 weight tiles in the shared-memory ring

__device__ __forceinline__ void heads_cp16(float *dst_smem, const float *src) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst_smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src) : "memory");
}

// z4: [B][D4] L4 pre-activation WITHOUT bias.  One block = HEADS_G sites x all heads.  L5: thread (t/128, t%128) owns one
// unit of one head (two heads in flight, four heads in two passes); the [D4][128] weight matrix of each head streams through
// shared memory in double-buffered 32-row tiles (16-byte cp.async, fully coalesced) so the FMA loop never waits on L2.
template <int HEADS_G>      // sites per block: 8 (small batches: more blocks) or 16 (large batches: half the weight streaming per site)
__global__ void __launch_bounds__(HEADS_THREADS) heads_kernel(const float *__restrict__ z4, int nsplit, int64_t split_stride,
                                                              HeadsParams hp, float *__restrict__ out, int64_t batch) {
    extern __shared__ __align__(16) float smem[];
    const int d4 = hp.d4;
    float *a = smem;                                   // [d4][G]
    float *l5 = a + HEADS_G * d4;                      // [nheads][G][128]
    float *yv = l5 + C3B_MAX_HEADS * HEADS_G * 128;    // [G][96]
    float *wt = yv + HEADS_G * 96;                     // [HEADS_STAGES][2 heads][HEADS_KT][128]
    float *wys = wt + HEADS_STAGES * 2 * HEADS_KT * 128;          // [128][out_dim]: all heads' output weights, column = global output index
    const int tid = threadIdx.x;
    const int64_t b0 = (int64_t)blockIdx.x * HEADS_G;
    const int g_n = (int)min((int64_t)HEADS_G, batch - b0);
    // small batches: gridDim.y = nheads/2 and each block serves one PAIR of heads (twice the blocks, half the serial weight
    // streaming per block); large batches: gridDim.y = 1 and the block walks all pairs
    const int hp_begin = gridDim.y > 1 ? 2 * (int)blockIdx.y : 0;
    const int hp_end = gridDim.y > 1 ? hp_begin + 2 : hp.nheads;
    const int o_begin = hp.h[hp_begin].out_off;
    const int o_end = hp_end < hp.nheads ? hp.h[hp_end].out_off : hp.out_dim;

    // output-layer weights of every head -> shared memory, asynchronously (oldest cp.async group: complete by the first
    // wait of the L5 loop); the 128-long dot products of the Y stage would otherwise wait on L2 once per four terms
    for (int i = tid * 4; i < 128 * hp.out_dim; i += HEADS_THREADS * 4) heads_cp16(wys + i, hp.wy_all + i);
    asm volatile("cp.async.commit_group;" ::: "memory");
    // a is stored [k][G] so the L5 loop reads the 8 sites of one k with two 16-byte broadcast loads
    // (all split-K partial loads of a thread are independent: issue them together, then add in a fixed order - a rolled
    //  loop with a running sum serialises up to 16 L2 round trips per thread)
#pragma unroll 2
    for (int i = tid; i < HEADS_G * d4; i += HEADS_THREADS) {
        const int g = i / d4, k = i - g * d4;              // consecutive threads -> consecutive k: coalesced partial-sum reads
        float v = 0.f;
        if (g < g_n) {
            const float *zp = z4 + (b0 + g) * d4 + k;
            float part[16];
#pragma unroll
            for (int sp = 0; sp < 16; ++sp) part[sp] = sp < nsplit ? __ldg(zp + (size_t)sp * split_stride) : 0.f;
            v = __ldg(hp.b4 + k);
#pragma unroll
            for (int sp = 0; sp < 16; ++sp) v += part[sp];                                          // split-K partials, fixed order
            v = selu(v);
        }
        a[k * HEADS_G + g] = v;
    }

    const int j = tid & 127;
    const int hsel = tid >> 7;                         // which head of the in-flight pair this thread works on
    const int ntiles = d4 / HEADS_KT;
    for (int hp0 = hp_begin; hp0 < hp_end; hp0 += 2) {
        const float *w0 = hp.h[hp0].w5t, *w1 = hp.h[hp0 + 1].w5t;
        // stage loader: 2 heads x 32 rows x 128 floats = 2048 float4, 8 per thread
        auto load_tile = [&](int tile, int stage) {
            float *dst = wt + stage * (2 * HEADS_KT * 128);
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const int idx = r * HEADS_THREADS + tid;        // float4 index
                const int hh = idx >> 10, rem = idx & 1023;
                const float *src = (hh ? w1 : w0) + (size_t)tile * HEADS_KT * 128 + rem * 4;
                heads_cp16(dst + hh * (HEADS_KT * 128) + rem * 4, src);
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
        float acc[HEADS_G];
        const float bias = __ldg(hp.h[hp0 + hsel].b5 + j);
#pragma unroll
        for (int g = 0; g < HEADS_G; ++g) acc[g] = bias;
        // three-stage ring: two tiles in flight while one is consumed (an L2 round trip is ~2x a tile's FMA time)
        load_tile(0, 0);
        if (ntiles > 1) load_tile(1, 1);
        for (int t = 0; t < ntiles; ++t) {
            if (t + 2 < ntiles) {
                load_tile(t + 2, (t + 2) % HEADS_STAGES);
                asm volatile("cp.async.wait_group 2;" ::: "memory");
            } else if (t + 1 < ntiles) {
                asm volatile("cp.async.wait_group 1;" ::: "memory");
            } else {
                asm volatile("cp.async.wait_group 0;" ::: "memory");
            }
            __syncthreads();
            const float *ws = wt + (t % HEADS_STAGES) * (2 * HEADS_KT * 128) + hsel * (HEADS_KT * 128) + j;
            const float *as = a + (size_t)t * HEADS_KT * HEADS_G;
#pragma unroll 8
            for (int k = 0; k < HEADS_KT; ++k) {
                const float wv = ws[k * 128];
#pragma unroll
                for (int g4 = 0; g4 < HEADS_G / 4; ++g4) {
                    const float4 av = *reinterpret_cast<const float4 *>(as + k * HEADS_G + 4 * g4);
                    acc[4 * g4 + 0] = fmaf(av.x, wv, acc[4 * g4 + 0]);
                    acc[4 * g4 + 1] = fmaf(av.y, wv, acc[4 * g4 + 1]);
                    acc[4 * g4 + 2] = fmaf(av.z, wv, acc[4 * g4 + 2]);
                    acc[4 * g4 + 3] = fmaf(av.w, wv, acc[4 * g4 + 3]);
                }
            }
            __syncthreads();
        }
#pragma unroll
        for (int g = 0; g < HEADS_G; ++g) l5[((hp0 + hsel) * HEADS_G + g) * 128 + j] = selu(acc[g]);
    }
    __syncthreads();

    for (int i = tid; i < HEADS_G * hp.out_dim; i += HEADS_THREADS) {
        const int g = i / hp.out_dim, o = i - g * hp.out_dim;
        if (o < o_begin || o >= o_end) continue;
        int h = 0;
        if (hp.nheads > 1 && o >= hp.h[1].out_off) h = 1;
        if (hp.nheads > 2 && o >= hp.h[2].out_off) h = 2;
        if (hp.nheads > 3 && o >= hp.h[3].out_off) h = 3;
        const int oo = o - hp.h[h].out_off;
        const float *wy = wys + o;
        const int n = hp.out_dim;
        const float *lv = l5 + (h * HEADS_G + g) * 128;
        float s0 = __ldg(hp.h[h].by + oo), s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll 8
        for (int jj = 0; jj < 128; jj += 4) {
            s0 = fmaf(lv[jj], wy[jj * n], s0);
            s1 = fmaf(lv[jj + 1], wy[(jj + 1) * n], s1);
            s2 = fmaf(lv[jj + 2], wy[(jj + 2) * n], s2);
            s3 = fmaf(lv[jj + 3], wy[(jj + 3) * n], s3);
        }
        yv[g * 96 + o] = selu((s0 + s1) + (s2 + s3));
    }
    __syncthreads();

    if (tid < g_n * hp.nheads) {
        const int g = tid / hp.nheads, h = tid - g * hp.nheads;
        if (h < hp_begin || h >= hp_end) return;
        const int n = hp.h[h].n, off = hp.h[h].out_off;
        const float *v = yv + g * 96 + off;
        float mx = v[0];
        for (int o = 1; o < n; ++o) mx = fmaxf(mx, v[o]);
        float sum = 0.f;
        for (int o = 0; o < n; ++o) sum += expf(v[o] - mx);
        const float inv = 1.f / sum;
        float *dst = out + (b0 + g) * hp.out_dim + off;
        for (int o = 0; o < n; ++o) dst[o] = expf(v[o] - mx) * inv;
    }
}

template <typename T>
int launch_ingest(const void *x, float *out, int64_t n, cudaStream_t s) {
    if (n == 0) return 0;
    int blocks = (int)min((int64_t)4096, (n + 255) / 256);
    ingest_f32_kernel<T><<<blocks, 256, 0, s>>>((const T *)x, out, n);
    C3B_CUDA(cudaGetLastError());
    return 0;
}

int ingest_any(const void *x, int dtype, float *out, int64_t n, cudaStream_t s) {
    switch (dtype) {
        case C3B_DT_I8: return launch_ingest<int8_t>(x, out, n, s);
        case C3B_DT_I32: return launch_ingest<int32_t>(x, out, n, s);
        case C3B_DT_F32: return launch_ingest<float>(x, out, n, s);
        default: c3b_set_error("unsupported input dtype %d", dtype); return 1;
    }
}

}  // namespace

int c3b_launch_gather_windows_f32(const void *cols, int dtype, int channels, const int64_t *starts, int64_t n_cols, float *out,
                                  int64_t batch, cudaStream_t s) {
    if (batch == 0) return 0;
    const int64_t n = batch * C3B_T * channels;
    const int blocks = (int)min((int64_t)4096, (n + 255) / 256);
    switch (dtype) {
        case C3B_DT_I8: gather_windows_f32_kernel<int8_t><<<blocks, 256, 0, s>>>((const int8_t *)cols, starts, n_cols, channels, out, batch); break;
        case C3B_DT_I32: gather_windows_f32_kernel<int32_t><<<blocks, 256, 0, s>>>((const int32_t *)cols, starts, n_cols, channels, out, batch); break;
        case C3B_DT_I64: gather_windows_f32_kernel<int64_t><<<blocks, 256, 0, s>>>((const int64_t *)cols, starts, n_cols, channels, out, batch); break;
        case C3B_DT_F32: gather_windows_f32_kernel<float><<<blocks, 256, 0, s>>>((const float *)cols, starts, n_cols, channels, out, batch); break;
        default: c3b_set_error("unsupported input dtype %d", dtype); return 1;
    }
    C3B_CUDA(cudaGetLastError());
    return 0;
}

int c3b_launch_ingest_pileup_f32(const void *x, int dtype, float *out, int64_t n, cudaStream_t s) {
    return ingest_any(x, dtype, out, n, s);
}
int c3b_launch_ingest_fa_f32(const void *x, int dtype, float *out, int64_t n, cudaStream_t s) {
    return ingest_any(x, dtype, out, n, s);
}

int c3b_launch_heads(const float *z4, int nsplit, int64_t split_stride, const HeadsParams &hp, float *out, int64_t batch,
                     cudaStream_t s) {
    if (batch == 0) return 0;
    if (nsplit < 1 || nsplit > 16) { c3b_set_error("heads: %d split-K partials (1..16 supported)", nsplit); return 1; }
    int sms = 132;
    { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
    const int G = batch >= 512 ? 16 : 8;      // SM-time per site (weight streaming) matters more than block count once a launch has 32+ blocks
    size_t smem = sizeof(float) * ((size_t)G * hp.d4 + (size_t)C3B_MAX_HEADS * G * 128 + (size_t)G * 96 + HEADS_STAGES * 2 * HEADS_KT * 128 +
                                   128 * hp.out_dim);
    int blocks = (int)((batch + G - 1) / G);
    const int pairs = (hp.nheads >= 4 && hp.nheads % 2 == 0 && blocks <= sms) ? hp.nheads / 2 : 1;
    if (G == 16) {
        C3B_CUDA(cudaFuncSetAttribute(heads_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        heads_kernel<16><<<dim3(blocks, pairs), HEADS_THREADS, smem, s>>>(z4, nsplit, split_stride, hp, out, batch);
    } else {
        C3B_CUDA(cudaFuncSetAttribute(heads_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        heads_kernel<8><<<dim3(blocks, pairs), HEADS_THREADS, smem, s>>>(z4, nsplit, split_stride, hp, out, batch);
    }
    C3B_CUDA(cudaGetLastError());
    return 0;
}
