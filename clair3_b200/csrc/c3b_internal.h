// Internal declarations shared by the C-ABI translation unit and the kernel files.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <map>
#include <string>
#include <vector>

#include "../../include/clair3_b200.h"
#include "../../include/clair3_b200_debug.h"

#define C3B_T 33            // positions per site (shared/param_p.py:34-35)
#define C3B_H1 128          // LSTM1 hidden (clair3/model.py:46)
#define C3B_H2 160          // LSTM2 hidden (clair3/model.py:47)
#define C3B_MAX_HEADS 4
#define C3B_X1_COLS 48      // LSTM1 x operand columns: [hi(x) (channels) | 1 | lo(x) (channels) | 0...]  (lstm_tc.cu)
#define C3B_MAX_PILEUP_CHANNELS ((C3B_X1_COLS - 1) / 2)

void c3b_set_error(const char *fmt, ...);
void c3b_note_grid(long long ctas);      // launchers report their grid size (CTAs) for the per-kernel profile (SM-time = CTAs x duration)

// Tensor-core operand type.  fp16 (11-bit significand) rather than bf16 (8-bit): same wgmma rate, 8x smaller rounding
// error; every operand on this path is bounded (counts <= 2048 exact, |h| <= 1, BN-normalised feature maps) and stores
// saturate at +-65504 instead of overflowing.
typedef __half op_t;
typedef __half2 op2_t;
#ifdef __CUDACC__
__device__ __forceinline__ float op_clamp(float x) { return fminf(fmaxf(x, -65504.f), 65504.f); }
__device__ __forceinline__ op_t f2op(float x) { return __float2half_rn(x); }
// saturating variant for values that are not bounded by construction (raw input counts): +-65504 instead of inf
__device__ __forceinline__ op_t f2op_sat(float x) {
    unsigned short r;
    asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(r) : "f"(x));
    return __ushort_as_half(r);
}
__device__ __forceinline__ op2_t f2op2(float a, float b) { return __floats2half2_rn(a, b); }
__device__ __forceinline__ float2 op22f2(op2_t v) { return __half22float2(v); }
// two floats -> packed fp16 pair in ONE instruction, saturating at +-65504 instead of overflowing to inf
__device__ __forceinline__ uint32_t f2op2_sat(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ float op2f(op_t v) { return __half2float(v); }
#endif
// "Tile-major k-group-planar" activation matrices (h1, h2, spp): [row tile of 128][K/8 k-groups][128 rows][8] fp16.  A GEMM
// tile's 64-wide k-chunk (8 k-groups) is then ONE contiguous 16 KB run = one cp.async.bulk instead of eight 2 KB ones.
// Returns the element offset of (row, k-group kg, lane 0).
#ifdef __CUDACC__
__host__ __device__
#endif
inline size_t c3b_tile_major_offset(size_t row, int kg, int kgroups) {
    return (((row >> 7) * (size_t)kgroups + (size_t)kg) * 128 + (row & 127)) * 8;
}
uint16_t c3b_f2op(float f);     // host: fp32 -> fp16 bits, round-to-nearest-even, saturating
// Torch gate row (gate*H + unit) of row R in [0, 4H) of the recurrent kernels' permuted gate order (lstm_tc.cu): 64-row block
// 2p holds gates i (rows 16w + q, q < 8) and f (rows 16w + q + 8) of units 32p + 8w + q, block 2p + 1 gates g and o.
inline int c3b_lstm_row(int R, int H) {
    const int pp = R / 128, blk = (R / 64) & 1, r = R % 64, w = r / 16, q = r % 16;
    return (2 * blk + (q >= 8)) * H + 32 * pp + 8 * w + (q & 7);
}
// Torch gate row of LSTM2 pre-gate column C in [0, 640) of one direction (the output columns of proj2): "gate-quad" order, the
// four gates i, f, g, o of unit 32p + u (u < 32) in the adjacent columns 128p + 4u .. +3, so the recurrent kernel's thread that
// owns the unit in block pair p reads them with one 8-byte load.
inline int c3b_lstm2_pg_row(int C) {
    return (C & 3) * C3B_H2 + 32 * (C >> 7) + ((C & 127) >> 2);
}
float c3b_op2f(uint16_t h);     // host: fp16 bits -> fp32

#define C3B_CUDA(expr)                                                                          \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess) {                                                                \
            c3b_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return 1;                                                                           \
        }                                                                                       \
    } while (0)

struct HostParam {
    std::vector<float> data;
    std::vector<int64_t> shape;
};

// One dense head: L5_k (D4 -> 128) then Y_k (128 -> n).  fp32, transposed for coalesced reads.
struct HeadWeights {
    const float *w5t;   // [D4][128]
    const float *b5;    // [128]
    const float *wyt;   // [128][n]
    const float *by;    // [n]
    int n;
    int out_off;
};

struct HeadsParams {
    HeadWeights h[C3B_MAX_HEADS];
    const float *b4;    // [D4]
    const float *wy_all; // [128][out_dim]: every head's output weights side by side (column = global output index)
    int nheads;
    int d4;
    int out_dim;
};

// ---- fp32 debug path weights (device pointers) ----
struct LstmF32 {
    const float *wih_t;  // [I][4H]
    const float *whh_t;  // [H][4H]
    const float *bias;   // [4H] = b_ih + b_hh
};
struct ConvF32 {
    const float *w;      // [9][Cin][Cout]  (BN folded; conv1 also carries 1/100)
    const float *bias;   // [Cout]          (BN folded)
    int cin, cout, stride;
};

// ---- tensor-core path packed operands (device pointers into the weight blob) ----
struct LstmTC {
    const op_t *w_img;   // wgmma A-operand image: [dir][2H/64 blocks][K/8][64 rows][8] fp16, rows permuted (c3b_lstm_row)
    const float *bias;            // unused (LSTM1's bias is a weight column against the constant-1 input; LSTM2's rides in the projection)
};
struct IgemmW {
    const op_t *w_img;   // wgmma B-operand image per k-chunk: [nchunks][8 kgroups][N rows][8] fp16
    const float *bias;            // [N]
    int n;                        // output columns (Cout / gate rows / dense units)
    int kgroups;                  // K/8 (16-byte k-groups), real
    int nchunks;                  // ceil(kgroups/8)
};

// dense tail (tail_tc.cu): L4 as a [d4 rows] B-operand image per k-chunk (the heads run on the fp32 HeadsParams weights)
struct TailW {
    const op_t *w4;                      // [l4_in/64 chunks][8 kg][d4 rows][8]
};

struct ConvGeom {
    int hin, win, cin, hout, wout, cout, stride;
};

// Zero-padded channel-group-planar feature map [C/8][p][8]: slot(b,h,w) = g + b*s + (h+1)*wp + (w+1)  (see pconv_tc.cu)
struct PlanarGeom {
    int h, w, wp, s, g;        // real dims, padded width (w+2), slots per site ((h+2)*wp), guard slots
    int64_t t, p;              // data slots (B*s), plane pitch in slots (g + roundup(t,512) + g)
};
// `cap` >= batch: the site count the plane pitch is laid out for (a workspace keeps the layout of its largest chunk, so smaller
// chunks find their borders / guards already zero)
inline PlanarGeom c3b_planar_geom(int64_t batch, int h, int w, int64_t cap = 0) {
    PlanarGeom g;
    g.h = h; g.w = w; g.wp = w + 2; g.s = (h + 2) * (w + 2);
    g.g = (g.wp + 1 + 7) / 8 * 8;
    g.t = batch * g.s;
    const int64_t tc = (cap > batch ? cap : batch) * g.s;
    g.p = g.g + (tc + 511) / 512 * 512 + g.g;
    return g;
}

// Debug tap: where an intermediate activation of the last forward lives and how to unpack it (c3b_get_tap, option "taps")
struct Tap {
    const void *ptr;
    int fmt;        // 0 f32, 1 fp16
    int layout;     // 0 [B][inner] row-major; 2 k-group-planar [inner/8][bp][8] (row = site);
                    // 3 k-group-planar time-major [inner/8][33*bp][8] (row = t*bp + site) -> [B][33][inner]
                    // 4 zero-padded planar feature map [inner/8][geom.p][8] -> NHWC [B][h][w][inner]
                    // 7 row-major time-major [33*bp][inner] (row = t*bp + site) -> [B][33][inner]
    int64_t inner;
    int bp;
    PlanarGeom geom;
    int nsplit = 1;  // layout 5: [nsplit][bp][inner] split-K partial sums -> summed [B][inner]
    int h = 0, w = 0;  // layout 6: four parity planes [4][inner/8][geom.p][8] (geom = NEXT level) of an h x w map -> NHWC
};

struct Workspace {
    cudaStream_t stream = nullptr;
    // generic device scratch, carved by the forward pass
    char *dev = nullptr;
    size_t dev_bytes = 0;
    // staging for host-side callers
    void *dev_x = nullptr;
    size_t dev_x_bytes = 0;
    float *dev_y = nullptr;
    size_t dev_y_bytes = 0;
    void *dev_aux = nullptr;         // window offsets / decode inputs of host-side callers
    size_t dev_aux_bytes = 0;
    // full-alignment planar maps are laid out for `fa_cap_sites` sites (the largest chunk seen on this workspace); smaller
    // chunks reuse that layout (their borders / guards are already zero), so a ragged tail never re-clears the region
    int64_t fa_cap_sites = 0;
    int fa_cap_depth = -1;
    bool fa_zeroed = false;
    std::map<std::string, Tap> taps;   // per workspace, filled only while option "taps" is on
    // per-kernel CUDA-event pairs recorded while option "profile" is on (resolved lazily by c3b_get_profile)
    struct ProfRec { const char *name; cudaEvent_t e0, e1; long long ctas; };
    std::vector<ProfRec> prof;
};

struct c3b_model {
    int kind = 0, channels = 0, add_indel = 0, device = 0;
    int nheads = 2, out_dim = 24, d4 = 128, l4_in = 0;
    int precision = C3B_PREC_F16_TC;
    int chunk_sites = 0;
    int lstm_tile = 0;
    int profile = 0;
    int lstm_wg = 2;                   // warpgroups (one sub-tile of sites each) per LSTM CTA (option "lstm_wg": 1 or 2)
    int lstm_mufu16 = 0;               // 1: packed tanh.approx.f16x2 gate activations, 0 (default, faster: the epilogue is issue-bound): fp32 tanh.approx
    int tap_ws = -1;                   // debug: workspace index c3b_get_tap reads
    int taps = 0;                      // debug option "taps": record where the intermediate activations of a forward live
    bool weights_by_broadcast = false; // the packed images arrived by c3b_bcast_weights (no host-side parameters behind them)
    long long *lstm_trace = nullptr;   // device [2][33][4] clock stamps (debug option "lstm_trace")
    std::map<std::string, std::pair<double, int64_t>> prof_total;   // name -> (ms, launches)
    std::map<std::string, double> prof_ctas;                         // name -> sum of CTAs launched
    int sm_count = 132;
    bool finalized = false;
    std::map<std::string, HostParam> params;
    std::vector<std::string> expected;
    std::map<std::string, std::vector<int64_t>> expected_shape;

    // device weights
    char *blob = nullptr;        // tensor-core images + shared fp32 head weights (broadcast unit)
    size_t blob_bytes = 0;
    char *f32blob = nullptr;     // fp32 debug path weights
    size_t f32blob_bytes = 0;

    HeadsParams heads;
    // fp32 path
    LstmF32 lstm_f32[2][2];
    const float *l4_f32_t = nullptr;   // [l4_in][d4]
    ConvF32 conv_f32[9];
    // tc path
    LstmTC lstm_tc[2][2];
    IgemmW proj2;                      // LSTM2 input projection, both directions: N = 1280 (column order c3b_lstm2_pg_row)
    TailW tail;                        // L4 on the tensor cores
    IgemmW conv_tc[9];

    std::vector<Workspace *> ws;
    int64_t launches = 0;
    int last_depth = 0;
    int64_t last_batch = 0;
};

// conv order used everywhere: 0 conv1, 1 rb1.conv1, 2 rb1.conv2, 3 conv3, 4 rb2.conv1, 5 rb2.conv2, 6 conv5, 7 rb3.conv1, 8 rb3.conv2

// ---- kernels_common.cu ----
int c3b_launch_ingest_pileup_f32(const void *x, int dtype, float *out, int64_t n_elems, cudaStream_t s);
int c3b_launch_ingest_fa_f32(const void *x, int dtype, float *out, int64_t n_elems, cudaStream_t s);
// z4: nsplit partial sums [nsplit][split_stride] of the L4 pre-activation (no bias); the kernel adds them
int c3b_launch_heads(const float *z4, int nsplit, int64_t split_stride, const HeadsParams &hp, float *out, int64_t batch, cudaStream_t s);

// ---- decode.cu ----
int c3b_launch_decode_stage1(const float *y, const uint8_t *ref_gt21, int64_t batch, int out_dim, uint8_t *is_ref, float *ref_prob,
                             int32_t *argmax, float *maxprob, double *qual, int32_t *nonref_idx, int32_t *n_nonref, cudaStream_t s);
// sites == nullptr: site s is row s; n_sites == nullptr: max_sites sites (else min(*n_sites, max_sites), read on the device)
int c3b_launch_decode_stage2(const float *y, const uint8_t *ref_gt21, int64_t batch, int out_dim, const int32_t *sites,
                             const int32_t *n_sites, int64_t max_sites, int k, uint8_t *cat, uint16_t *idx, float *prob,
                             uint16_t *tie_mask, int32_t *count, uint8_t *complete, cudaStream_t s);

// ---- kernels_fp32.cu ----
int c3b_launch_lstm_f32(const float *x, const LstmF32 &fwd, const LstmF32 &bwd, float *out, int64_t batch, int in_dim,
                        int hidden, cudaStream_t s);
int c3b_launch_dense_f32(const float *x, const float *w_t, float *out, int64_t batch, int k, int n, cudaStream_t s);
int c3b_launch_conv_f32(const float *x, const ConvF32 &w, const float *residual, float *out, int64_t batch, int hin,
                        int win, int hout, int wout, cudaStream_t s);
int c3b_launch_spp_f32(const float *x, float *out, int64_t batch, int h, int w, int c, cudaStream_t s);

// ---- tensor-core path ----
struct TcPileupBuffers {
    op_t *xs;     // [33][B][48] fp16, time-major: hi(x) | 1 | lo(x) columns
    op_t *h1;     // tile-major k-group-planar, 32 k-groups: row = t*Bp + b, k = dir*128 + j  (projection GEMM operand)
    __half *pg;            // [33*B][1280] fp16 pre-gates of LSTM2 (bias included), column dir*640 + C in gate-quad order (c3b_lstm2_pg_row)
    op_t *h2;     // tile-major k-group-planar, 1320 k-groups: row = b, k = t*320 + dir*160 + j (flatten order of clair3/model.py:135)
    float *z4;             // [16][B][128] fp32 split-K partial sums of the L4 pre-activation (no bias)
    int bp;                // padded batch: multiple of 128
};
// starts == nullptr: x is the dense [batch][33][channels] tensor; otherwise x is the per-column matrix [n_cols][channels] and
// site b is its rows [starts[b], starts[b] + 33) (rows outside the matrix, and with bounds != nullptr rows outside
// [bounds[2b], bounds[2b+1]), read as zero)
int c3b_launch_ingest_pileup_tc(const void *x, int dtype, int channels, const int64_t *starts, const int64_t *bounds, int64_t n_cols,
                                op_t *xs, int64_t batch, int bp, cudaStream_t s);
int c3b_launch_gather_windows_f32(const void *cols, int dtype, int channels, const int64_t *starts, const int64_t *bounds,
                                  int64_t n_cols, float *out, int64_t batch, cudaStream_t s);
int c3b_launch_proj2(const c3b_model *m, const op_t *h1, const IgemmW &w, __half *pg, int bp, cudaStream_t s);
int c3b_launch_tail(const c3b_model *m, const op_t *act, int64_t batch, int bp, float *out, float *z4, int *nsplit_out, cudaStream_t s);
int c3b_launch_lstm1_tc(const c3b_model *m, const TcPileupBuffers &b, int64_t batch, int tile, cudaStream_t s);
int c3b_launch_lstm2_tc(const c3b_model *m, const TcPileupBuffers &b, int64_t batch, int tile, cudaStream_t s);

struct PconvArgs {
    const op_t *in;            // planar padded, c channels
    op_t *out;                 // planar padded, n channels, same geometry
    const op_t *residual;      // optional, planar padded like out
    IgemmW w;                  // per-chunk weight images (k = tap*c + ci)
    PlanarGeom geom;           // geometry of the OUTPUT level (= input level for stride 1)
    int c, n, relu;
    int stride2;               // 1: `in` holds the four parity planes of the previous level, each [c/8][geom.p][8] (see pconv_tc.cu)
    int out_parity;            // 1: `out` receives the real pixels scattered into the four parity planes of `next` ([n/8][next.p][8] each)
    PlanarGeom next;
};
// offset (elements) of padded pixel (hp, wp) of site b, channel group 0, inside a parity-plane set of geometry g with c channels
inline size_t c3b_parity_offset(const PlanarGeom &g, int c, int64_t b, int hp, int wp) {
    return (size_t)((hp & 1) * 2 + (wp & 1)) * ((size_t)(c / 8) * g.p * 8) + ((size_t)g.g + b * g.s + (size_t)((hp >> 1) + 1) * g.wp + ((wp >> 1) + 1)) * 8;
}
int c3b_launch_pconv(const c3b_model *m, const PconvArgs &a, cudaStream_t s);

int c3b_launch_ingest_fa_tc(const void *x, int dtype, int channels, int cpad, op_t *out, int64_t batch, int depth, const PlanarGeom &g1,
                            cudaStream_t s);
int c3b_launch_spp_tc(const op_t *x, const PlanarGeom &g, op_t *out, int64_t batch, int c, int bp, cudaStream_t s);


// A device buffer that grows on demand (25 % headroom); used by the pileup counter and the full-alignment builder for their
// per-call inputs and scratch.  `what` names the owner in the error message.
struct C3bBuf {
    void *p = nullptr;
    size_t cap = 0;
    int ensure(size_t bytes, const char *what = "clair3_b200") {
        if (bytes <= cap) return 0;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        const size_t want = bytes + bytes / 4 + 256;
        if (cudaMalloc(&p, want) != cudaSuccess) {
            c3b_set_error("%s: cudaMalloc of %zu bytes failed", what, want);
            return 1;
        }
        cap = want;
        return 0;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

// One input array of a call: a device pointer passes through, host memory is copied into b on stream s.
static inline int c3b_upload(C3bBuf &b, const void *src, size_t bytes, int on_device, const void **dev, cudaStream_t s,
                             const char *what) {
    if (on_device) { *dev = src; return 0; }
    if (b.ensure(bytes ? bytes : 1, what)) return 1;
    if (bytes) C3B_CUDA(cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, s));
    *dev = b.p;
    return 0;
}
