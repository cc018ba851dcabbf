// C-ABI of libclair3b200.so (see include/clair3_b200.h): model lifetime, strict state_dict ingestion, weight folding /
// packing, per-stream workspaces and the forward orchestration of both precisions.  No CPU fallback anywhere.
#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>

#include "c3b_internal.h"

// ------------------------------------------------------------------------------------------------ errors
static thread_local char g_err[1024] = "";
void c3b_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
extern "C" const char *c3b_last_error(void) { return g_err; }
static thread_local long long g_last_grid = 0;
void c3b_note_grid(long long ctas) { g_last_grid = ctas; }
extern "C" const char *c3b_version(void) { return "clair3_b200 0.1 (sm_90a)"; }

// ------------------------------------------------------------------------------------------------ helpers
uint16_t c3b_f2op(float f) {
    // fp32 -> fp16 bits, round-to-nearest-even, saturating to +-65504 (NaN preserved)
    uint32_t u;
    memcpy(&u, &f, 4);
    const uint16_t sign = (uint16_t)((u >> 16) & 0x8000u);
    const uint32_t a = u & 0x7fffffffu;
    if (a > 0x7f800000u) return sign | 0x7e00;                 // NaN
    if (a >= 0x477ff000u) return sign | 0x7bff;                // >= 65520 rounds past max -> saturate
    if (a < 0x33000001u) return sign;                          // < 2^-25 -> 0
    int e = (int)(a >> 23) - 127;
    uint32_t man = (a & 0x7fffffu) | 0x800000u;
    int shift;
    uint32_t he;
    if (e < -14) { shift = 13 + (-14 - e); he = 0; }           // subnormal half
    else { shift = 13; he = (uint32_t)(e + 15); }
    uint32_t hm = man >> shift;
    const uint32_t rem = man & ((1u << shift) - 1), half = 1u << (shift - 1);
    if (rem > half || (rem == half && (hm & 1u))) hm++;
    uint32_t out;
    if (he == 0) out = hm;                                     // may carry into exponent 1: bit pattern is still right
    else out = ((he << 10) + (hm - 0x400u));                   // hm includes the implicit bit; carry propagates into he
    return sign | (uint16_t)out;
}
float c3b_op2f(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    uint32_t e = (h >> 10) & 0x1f, m = h & 0x3ff, u;
    if (e == 0) {
        if (m == 0) u = sign;
        else {
            int sh = 0;
            while (!(m & 0x400u)) { m <<= 1; ++sh; }
            u = sign | ((uint32_t)(127 - 15 - sh + 1) << 23) | ((m & 0x3ffu) << 13);
        }
    } else if (e == 31) u = sign | 0x7f800000u | (m << 13);
    else u = sign | ((e + 112) << 23) | (m << 13);
    float f;
    memcpy(&f, &u, 4);
    return f;
}

int c3b_use_device(int ordinal, int unsupported, int *sm_count) {
    int ndev = 0;
    const cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        c3b_set_error("no CUDA device: %s (clair3_b200 has no CPU fallback)", cudaGetErrorString(e));
        return unsupported;
    }
    if (ordinal < 0 || ordinal >= ndev) { c3b_set_error("bad device ordinal %d", ordinal); return 1; }
    cudaDeviceProp prop;
    C3B_CUDA(cudaGetDeviceProperties(&prop, ordinal));
    if (prop.major != 9 || prop.minor != 0) {
        c3b_set_error("device %d is sm_%d%d; this library contains only sm_90a code", ordinal, prop.major, prop.minor);
        return unsupported;
    }
    C3B_CUDA(cudaSetDevice(ordinal));
    if (sm_count) *sm_count = prop.multiProcessorCount;
    return 0;
}

// One thread per offset entry i in [0, n]: the smallest fault key of the run, min-reduced over each warp and then into *key.
__global__ void records_check_kernel(const C3bRecordsView v, unsigned long long *key) {
    unsigned long long k = C3B_REC_OK;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= v.n; i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long f = c3b_records_fault_at(v, i);
        k = f < k ? f : k;
    }
    for (int d = 16; d; d >>= 1) {
        const unsigned long long o = __shfl_down_sync(0xffffffffu, k, d);
        k = o < k ? o : k;
    }
    if ((threadIdx.x & 31) == 0 && k != C3B_REC_OK) atomicMin(key, k);
}

int c3b_records_check_device(const C3bRecordsView &v, C3bBuf &scratch, cudaStream_t s, uint64_t *key) {
    *key = C3B_REC_OK;
    if (v.n == 0 && !v.off[2] && !v.off[3] && !v.off[4]) return 0;      // BamRecords checks no core field of an empty run
    if (scratch.ensure(8, s, "record check")) return 1;
    const int64_t blocks = (v.n + 1 + 255) / 256 < 132 * 8 ? (v.n + 1 + 255) / 256 : 132 * 8;
    unsigned long long h = C3B_REC_OK;
    C3B_CUDA(cudaMemsetAsync(scratch.p, 0xff, 8, s));
    records_check_kernel<<<(unsigned)blocks, 256, 0, s>>>(v, scratch.as<unsigned long long>());
    C3B_CUDA(cudaGetLastError());
    C3B_CUDA(cudaMemcpyAsync(&h, scratch.p, 8, cudaMemcpyDeviceToHost, s));
    C3B_CUDA(cudaStreamSynchronize(s));
    *key = h;
    return 0;
}

namespace {

// One packed weight image, built on the host into the device buffer `dev`: put() appends an array at the next 256-byte boundary
// and records the pointer that is to address it; upload() copies the image to the device and points each recorded pointer there.
struct WeightImage {
    C3bBuf &dev;
    std::vector<uint8_t> data;
    std::vector<std::pair<size_t, const void **>> fixes;
    template <class S, class T> void put(const std::vector<S> &src, const T **dst) {
        const size_t off = (data.size() + 255) / 256 * 256, bytes = src.size() * sizeof(S);
        data.resize(off + bytes);
        memcpy(data.data() + off, src.data(), bytes);
        fixes.push_back({off, reinterpret_cast<const void **>(dst)});
    }
    int upload() {
        if (dev.ensure((data.size() + 255) / 256 * 256, nullptr, "c3b_finalize")) return 1;
        C3B_CUDA(cudaMemcpy(dev.p, data.data(), data.size(), cudaMemcpyHostToDevice));
        for (const auto &f : fixes) *f.second = dev.as<char>() + f.first;
        return 0;
    }
};

const char *kConvNames[9][2] = {
    {"conv1.conv", "conv1.bn"},
    {"res_block1.0.conv1", "res_block1.0.bn1"},
    {"res_block1.0.conv2", "res_block1.0.bn2"},
    {"conv3.conv", "conv3.bn"},
    {"res_block2.0.conv1", "res_block2.0.bn1"},
    {"res_block2.0.conv2", "res_block2.0.bn2"},
    {"conv5.conv", "conv5.bn"},
    {"res_block3.0.conv1", "res_block3.0.bn1"},
    {"res_block3.0.conv2", "res_block3.0.bn2"},
};
const int kConvCout[9] = {64, 64, 64, 128, 128, 128, 256, 256, 256};
const int kConvStride[9] = {2, 1, 1, 2, 1, 1, 2, 1, 1};
const char *kHeadNames[4][2] = {{"L5_1", "Y_gt21_logits"},
                                {"L5_2", "Y_genotype_logits"},
                                {"L5_3", "Y_indel_length_logits_1"},
                                {"L5_4", "Y_indel_length_logits_2"}};
const int kHeadDims[4] = {21, 3, 33, 33};

int conv_cin(const c3b_model *m, int i) { return i == 0 ? m->channels : kConvCout[i - 1]; }

// The state_dict keys of each layer kind, spelled only here: build_expected declares them and finalize_impl reads them.
struct LstmKeys { std::string w_ih, w_hh, b_ih, b_hh; };
LstmKeys lstm_keys(int layer, int dir) {
    const std::string l = std::string("LSTM") + char('1' + layer) + ".", d = dir ? "_l0_reverse" : "_l0";
    return {l + "weight_ih" + d, l + "weight_hh" + d, l + "bias_ih" + d, l + "bias_hh" + d};
}
struct ConvKeys { std::string w, b, bn_w, bn_b, bn_mean, bn_var, bn_batches; };
ConvKeys conv_keys(int i) {
    const std::string c = kConvNames[i][0], n = kConvNames[i][1];
    return {c + ".weight", c + ".bias", n + ".weight", n + ".bias", n + ".running_mean", n + ".running_var",
            n + ".num_batches_tracked"};
}
struct DenseKeys { std::string w, b; };
DenseKeys dense_keys(const char *layer) { return {std::string(layer) + ".weight", std::string(layer) + ".bias"}; }

void expect(c3b_model *m, const std::string &key, std::vector<int64_t> shape) {
    m->expected.push_back(key);
    m->expected_shape[key] = shape;
}

void build_expected(c3b_model *m) {
    if (m->kind == C3B_PILEUP) {
        const int hid[2] = {C3B_H1, C3B_H2};
        const int inp[2] = {m->channels, 2 * C3B_H1};
        for (int l = 0; l < 2; ++l)
            for (int d = 0; d < 2; ++d) {
                const LstmKeys k = lstm_keys(l, d);
                expect(m, k.w_ih, {4 * hid[l], inp[l]});
                expect(m, k.w_hh, {4 * hid[l], hid[l]});
                expect(m, k.b_ih, {4 * hid[l]});
                expect(m, k.b_hh, {4 * hid[l]});
            }
    } else {
        for (int i = 0; i < 9; ++i) {
            const ConvKeys k = conv_keys(i);
            expect(m, k.w, {kConvCout[i], conv_cin(m, i), 3, 3});
            expect(m, k.b, {kConvCout[i]});
            expect(m, k.bn_w, {kConvCout[i]});
            expect(m, k.bn_b, {kConvCout[i]});
            expect(m, k.bn_mean, {kConvCout[i]});
            expect(m, k.bn_var, {kConvCout[i]});
            expect(m, k.bn_batches, {});
        }
    }
    const DenseKeys l4 = dense_keys("L4");
    expect(m, l4.w, {m->d4, m->l4_in});
    expect(m, l4.b, {m->d4});
    for (int h = 0; h < m->nheads; ++h) {
        const DenseKeys l5 = dense_keys(kHeadNames[h][0]), y = dense_keys(kHeadNames[h][1]);
        expect(m, l5.w, {128, m->d4});
        expect(m, l5.b, {128});
        expect(m, y.w, {kHeadDims[h], 128});
        expect(m, y.b, {kHeadDims[h]});
    }
}

const std::vector<float> &P(const c3b_model *m, const std::string &k) { return m->params.at(k).data; }

// wgmma no-swizzle K-major operand image of a [rows][k] matrix: [chunk][rowblock][8 kgroups][rb rows][8] fp16.
// get(row, k) supplies the (already folded / permuted) element; out-of-range k is zero.
template <typename F>
std::vector<uint16_t> pack_operand(int rows, int kgroups, int rb, F get) {
    const int nchunks = (kgroups + 7) / 8;
    const int nrb = rows / rb;
    std::vector<uint16_t> img((size_t)nchunks * nrb * 8 * rb * 8, 0);
    for (int c = 0; c < nchunks; ++c)
        for (int b = 0; b < nrb; ++b)
            for (int kg = 0; kg < 8; ++kg) {
                const int g = c * 8 + kg;
                if (g >= kgroups) continue;
                for (int r = 0; r < rb; ++r)
                    for (int e = 0; e < 8; ++e)
                        img[((((size_t)c * nrb + b) * 8 + kg) * rb + r) * 8 + e] = c3b_f2op(get(b * rb + r, g * 8 + e));
            }
    return img;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ create / params
extern "C" int c3b_create(c3b_model **out, int kind, int channels, int add_indel_length, int device_ordinal) {
    if (!out) { c3b_set_error("c3b_create: null out"); return 1; }
    *out = nullptr;
    if (kind != C3B_PILEUP && kind != C3B_FULL_ALIGNMENT) { c3b_set_error("c3b_create: bad kind %d", kind); return 1; }
    if (kind == C3B_PILEUP && (channels < 1 || channels > C3B_MAX_PILEUP_CHANNELS)) {
        c3b_set_error("pileup channels must be in [1,%d], got %d", C3B_MAX_PILEUP_CHANNELS, channels);
        return 1;
    }
    if (kind == C3B_FULL_ALIGNMENT && (channels < 1 || channels > 16)) { c3b_set_error("full-alignment channels must be in [1,16], got %d", channels); return 1; }
    int sm_count = 0;
    if (int rc = c3b_use_device(device_ordinal, 2, &sm_count)) return rc;
    c3b_model *m = new c3b_model();
    m->kind = kind;
    m->channels = channels;
    m->add_indel = add_indel_length ? 1 : 0;
    m->device = device_ordinal;
    m->nheads = add_indel_length ? 4 : 2;
    m->out_dim = add_indel_length ? 90 : 24;
    m->d4 = kind == C3B_PILEUP ? 128 : 256;
    m->l4_in = kind == C3B_PILEUP ? 2 * C3B_H2 * C3B_T : 3584;
    m->sm_count = sm_count;
    build_expected(m);
    *out = m;
    return 0;
}

extern "C" int c3b_set_param(c3b_model *m, const char *key, const void *host_data, int dtype, const int64_t *shape, int ndim) {
    if (!m || !key) { c3b_set_error("c3b_set_param: null argument"); return 1; }
    auto it = m->expected_shape.find(key);
    if (it == m->expected_shape.end()) { c3b_set_error("Unexpected key in state_dict: \"%s\"", key); return 1; }
    const std::vector<int64_t> &want = it->second;
    bool ok = (int)want.size() == ndim;
    for (int i = 0; ok && i < ndim; ++i) ok = want[i] == shape[i];
    if (!ok) {
        std::string got = "[", exp = "[";
        for (int i = 0; i < ndim; ++i) got += std::to_string(shape[i]) + (i + 1 < ndim ? "," : "");
        for (size_t i = 0; i < want.size(); ++i) exp += std::to_string(want[i]) + (i + 1 < want.size() ? "," : "");
        c3b_set_error("size mismatch for %s: checkpoint %s], model %s]", key, got.c_str(), exp.c_str());
        return 1;
    }
    int64_t n = 1;
    for (int i = 0; i < ndim; ++i) n *= shape[i];
    HostParam hp;
    hp.shape.assign(shape, shape + ndim);
    hp.data.resize((size_t)n);
    if (dtype == C3B_DT_F32) {
        if (n && !host_data) { c3b_set_error("c3b_set_param: null data"); return 1; }
        memcpy(hp.data.data(), host_data, (size_t)n * 4);
    } else if (dtype == C3B_DT_I64) {
        for (int64_t i = 0; i < n; ++i) hp.data[i] = (float)((const int64_t *)host_data)[i];
    } else {
        c3b_set_error("c3b_set_param: parameters must be float32 (or int64 counters), got dtype %d for %s", dtype, key);
        return 1;
    }
    m->params[key] = std::move(hp);
    m->finalized = false;
    return 0;
}

extern "C" int c3b_set_option(c3b_model *m, const char *name, int value) {
    if (!m || !name) { c3b_set_error("c3b_set_option: null argument"); return 1; }
    if (!strcmp(name, "precision")) {
        if (value != C3B_PREC_F16_TC && value != C3B_PREC_FP32) { c3b_set_error("bad precision %d", value); return 1; }
        m->precision = value;
    } else if (!strcmp(name, "chunk_sites")) {
        if (value < 0) { c3b_set_error("bad chunk_sites %d", value); return 1; }
        m->chunk_sites = value;
    } else if (!strcmp(name, "profile")) {
        m->profile = value ? 1 : 0;
        m->prof_total.clear();
        m->prof_ctas.clear();
        for (Workspace *w : m->ws) {
            for (auto &r : w->prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
            w->prof.clear();
        }
    } else if (!strcmp(name, "lstm_wg")) {
        if (value != 1 && value != 2) { c3b_set_error("lstm_wg must be 1 or 2"); return 1; }
        m->lstm_wg = (int)value;
    } else if (!strcmp(name, "lstm2_split")) {
        if (value < 0 || value > 2) { c3b_set_error("lstm2_split must be 0, 1 or 2"); return 1; }
        m->lstm2_split = value;
    } else if (!strcmp(name, "lstm_mufu16")) {
        m->lstm_mufu16 = value ? 1 : 0;
    } else if (!strcmp(name, "tap_ws")) {
        m->tap_ws = value;           // which stream workspace (creation order) c3b_get_tap reads; -1 = first that has the tap
    } else if (!strcmp(name, "taps")) {
        m->taps = value ? 1 : 0;
        if (!value) for (Workspace *w : m->ws) w->taps.clear();
    } else if (!strcmp(name, "lstm_trace")) {
        if (value && !m->lstm_trace) {
            C3B_CUDA(cudaSetDevice(m->device));
            C3B_CUDA(cudaMalloc(&m->lstm_trace, sizeof(long long) * 2 * C3B_T * 4));
            C3B_CUDA(cudaMemset(m->lstm_trace, 0, sizeof(long long) * 2 * C3B_T * 4));
        } else if (!value && m->lstm_trace) {
            cudaFree(m->lstm_trace);
            m->lstm_trace = nullptr;
        }
    } else if (!strcmp(name, "lstm_tile")) {
        if (value != 0 && value != 16 && value != 32 && value != 64) { c3b_set_error("bad lstm_tile %d", value); return 1; }
        m->lstm_tile = value;
    } else {
        c3b_set_error("unknown option \"%s\"", name);
        return 1;
    }
    return 0;
}

extern "C" int c3b_out_dim(const c3b_model *m) { return m ? m->out_dim : -1; }
extern "C" int64_t c3b_launch_count(const c3b_model *m) { return m ? m->launches : -1; }

// ------------------------------------------------------------------------------------------------ finalize
static int finalize_impl(c3b_model *m) {
    for (const std::string &k : m->expected)
        if (!m->params.count(k)) { c3b_set_error("Missing key in state_dict: \"%s\"", k.c_str()); return 1; }
    C3B_CUDA(cudaSetDevice(m->device));

    // image 0: everything the tensor-core forward reads; image 1: what only the fp32 path reads
    WeightImage tc{m->blob}, f32{m->f32blob};

    // ---- dense heads, read by both paths: L5 transposed for coalesced reads, every head's Y weights side by side
    m->heads = HeadsParams();
    m->heads.nheads = m->nheads;
    m->heads.d4 = m->d4;
    m->heads.out_dim = m->out_dim;
    const DenseKeys l4 = dense_keys("L4");
    tc.put(P(m, l4.b), &m->heads.b4);
    int off = 0;
    std::vector<float> wy_all((size_t)128 * m->out_dim);
    for (int h = 0; h < m->nheads; ++h) {
        const DenseKeys l5 = dense_keys(kHeadNames[h][0]), y = dense_keys(kHeadNames[h][1]);
        const std::vector<float> &w5 = P(m, l5.w);   // [128][d4]
        const std::vector<float> &wy = P(m, y.w);    // [n][128]
        const int n = kHeadDims[h];
        std::vector<float> w5t((size_t)m->d4 * 128);
        for (int j = 0; j < 128; ++j)
            for (int k = 0; k < m->d4; ++k) w5t[(size_t)k * 128 + j] = w5[(size_t)j * m->d4 + k];
        for (int o = 0; o < n; ++o)
            for (int j = 0; j < 128; ++j) wy_all[(size_t)j * m->out_dim + off + o] = wy[(size_t)o * 128 + j];
        tc.put(w5t, &m->heads.h[h].w5t);
        tc.put(P(m, l5.b), &m->heads.h[h].b5);
        tc.put(P(m, y.b), &m->heads.h[h].by);
        m->heads.h[h].n = n;
        m->heads.h[h].out_off = off;
        off += n;
    }
    tc.put(wy_all, &m->heads.wy_all);

    // ---- L4: fp32 transposed + tensor-core operand image
    {
        const std::vector<float> &w4 = P(m, l4.w);   // [d4][l4_in]
        std::vector<float> w4t((size_t)m->l4_in * m->d4);
        for (int o = 0; o < m->d4; ++o)
            for (int k = 0; k < m->l4_in; ++k) w4t[(size_t)k * m->d4 + o] = w4[(size_t)o * m->l4_in + k];
        f32.put(w4t, &m->l4_f32_t);
        // tensor-core L4 (tail_tc.cu): the B operand of a sites-on-rows GEMM, one contiguous piece per 64-wide k-chunk
        const int l4_in = m->l4_in, d4 = m->d4;
        tc.put(pack_operand(d4, l4_in / 8, d4, [&](int r, int k) { return w4[(size_t)r * l4_in + k]; }), &m->l4_tc);
    }

    if (m->kind == C3B_PILEUP) {
        const int hid[2] = {C3B_H1, C3B_H2};
        const int inp[2] = {m->channels, 2 * C3B_H1};
        // fp32 debug weights: transposed [K][4H], summed bias
        for (int l = 0; l < 2; ++l)
            for (int d = 0; d < 2; ++d) {
                const LstmKeys key = lstm_keys(l, d);
                const std::vector<float> &wih = P(m, key.w_ih), &whh = P(m, key.w_hh), &bih = P(m, key.b_ih), &bhh = P(m, key.b_hh);
                const int H = hid[l], I = inp[l], G = 4 * H;
                std::vector<float> wih_t((size_t)I * G), whh_t((size_t)H * G), bias(G);
                for (int r = 0; r < G; ++r) {
                    for (int k = 0; k < I; ++k) wih_t[(size_t)k * G + r] = wih[(size_t)r * I + k];
                    for (int k = 0; k < H; ++k) whh_t[(size_t)k * G + r] = whh[(size_t)r * H + k];
                    bias[r] = bih[r] + bhh[r];
                }
                f32.put(wih_t, &m->lstm_f32[l][d].wih_t);
                f32.put(whh_t, &m->lstm_f32[l][d].whh_t);
                f32.put(bias, &m->lstm_f32[l][d].bias);
            }
        // tensor-core LSTM1 image: [dir][8 blocks][22 kgroups][64][8], rows in c3b_lstm_row order; K = [x columns (48) ; h (128)]
        // with the x columns [hi(x) (I) | 1 | lo(x) (I) | 0..]: W_ih multiplies both halves of the hi/lo split of the raw counts, the
        // constant-1 column carries b_ih + b_hh (lstm_tc.cu)
        {
            const int KX = C3B_X1_COLS, KG = (KX + 128) / 8;
            std::vector<uint16_t> img((size_t)2 * 512 * KG * 8, 0);
            for (int d = 0; d < 2; ++d) {
                const LstmKeys key = lstm_keys(0, d);
                const std::vector<float> &wih = P(m, key.w_ih), &whh = P(m, key.w_hh), &bih = P(m, key.b_ih), &bhh = P(m, key.b_hh);
                const int I = m->channels;
                for (int R = 0; R < 512; ++R) {
                    const int row = c3b_lstm_row(R, C3B_H1);
                    // sigmoid gates (i,f,o) are pre-halved: sigma(x) = 0.5*tanh(x/2)+0.5 costs one MUFU + one FMA
                    const float gs = (row / C3B_H1 == 2) ? 1.0f : 0.5f;
                    for (int k = 0; k < KX + 128; ++k) {
                        float v = 0.f;
                        if (k < I) v = wih[(size_t)row * I + k];
                        else if (k == I) v = bih[row] + bhh[row];
                        else if (k <= 2 * I) v = wih[(size_t)row * I + (k - I - 1)];
                        else if (k >= KX) v = whh[(size_t)row * 128 + (k - KX)];
                        img[((((size_t)d * 8 + R / 64) * KG + k / 8) * 64 + R % 64) * 8 + k % 8] = c3b_f2op(v * gs);
                    }
                }
            }
            tc.put(img, &m->lstm_tc[0]);
        }
        // tensor-core LSTM2: recurrent image [dir][10 blocks][20][64][8] (c3b_lstm_row order) + input projection GEMM (1280 columns,
        // gate-quad order c3b_lstm2_pg_row per direction, bias folded into the projection)
        {
            std::vector<uint16_t> img((size_t)2 * 640 * 20 * 8, 0);
            std::vector<float> pbias(1280);
            const std::vector<float> *wih_d[2];
            for (int d = 0; d < 2; ++d) {
                const LstmKeys key = lstm_keys(1, d);
                const std::vector<float> &whh = P(m, key.w_hh), &bih = P(m, key.b_ih), &bhh = P(m, key.b_hh);
                wih_d[d] = &P(m, key.w_ih);
                for (int R = 0; R < 640; ++R) {
                    const int row = c3b_lstm_row(R, C3B_H2);
                    const float gs = (row / C3B_H2 == 2) ? 1.0f : 0.5f;      // pre-halved sigmoid gates
                    for (int k = 0; k < 160; ++k)
                        img[((((size_t)d * 10 + R / 64) * 20 + k / 8) * 64 + R % 64) * 8 + k % 8] = c3b_f2op(whh[(size_t)row * 160 + k] * gs);
                }
                for (int C = 0; C < 640; ++C) {
                    const int row = c3b_lstm2_pg_row(C);
                    pbias[(size_t)d * 640 + C] = (bih[row] + bhh[row]) * ((row / C3B_H2 == 2) ? 1.0f : 0.5f);
                }
            }
            tc.put(img, &m->lstm_tc[1]);
            // one 256-column weight slab per CTA of the projection kernel (proj_tc.cu): [chunk 4][slab 5][8 kg][256 rows][8]
            std::vector<uint16_t> pimg = pack_operand(1280, 32, 256, [&](int C, int k) {
                const int row = c3b_lstm2_pg_row(C % 640);
                return (*wih_d[C / 640])[(size_t)row * 256 + k] * ((row / C3B_H2 == 2) ? 1.0f : 0.5f);
            });
            m->proj2 = IgemmW();
            m->proj2.n = 1280;
            m->proj2.kgroups = 32;
            m->proj2.nchunks = 4;
            tc.put(pimg, &m->proj2.w_img);
            tc.put(pbias, &m->proj2.bias);
        }
    } else {
        for (int i = 0; i < 9; ++i) {
            const ConvKeys key = conv_keys(i);
            const std::vector<float> &w = P(m, key.w), &cb = P(m, key.b), &g = P(m, key.bn_w), &be = P(m, key.bn_b);
            const std::vector<float> &mu = P(m, key.bn_mean), &var = P(m, key.bn_var);
            const int cout = kConvCout[i], cin = conv_cin(m, i);
            const float in_scale = (i == 0) ? 1.0f / 100.0f : 1.0f;      // x.float()/NORMALIZE_NUM (clair3/model.py:378)
            std::vector<float> wf((size_t)9 * cin * cout), bf(cout);
            for (int co = 0; co < cout; ++co) {
                const float s = g[co] / sqrtf(var[co] + 1e-3f);           // BatchNorm2d(eps=1e-3), clair3/model.py:192
                bf[co] = (cb[co] - mu[co]) * s + be[co];
                for (int ci = 0; ci < cin; ++ci)
                    for (int t = 0; t < 9; ++t)
                        wf[((size_t)t * cin + ci) * cout + co] = w[((size_t)co * cin + ci) * 9 + t] * s * in_scale;
            }
            m->conv_f32[i].cin = cin;
            m->conv_f32[i].cout = cout;
            m->conv_f32[i].stride = kConvStride[i];
            f32.put(wf, &m->conv_f32[i].w);
            f32.put(bf, &m->conv_f32[i].bias);
            // tensor-core image: k = tap*cin_pad + ci; conv1's input channels are padded to one wgmma k-step (16)
            const int cin_pad = (i == 0) ? 16 : cin;
            const int kg = 9 * cin_pad / 8;
            std::vector<uint16_t> img = pack_operand(cout, kg, cout, [&](int co, int k) {
                const int t = k / cin_pad, ci = k % cin_pad;
                return ci < cin ? wf[((size_t)t * cin + ci) * cout + co] : 0.f;
            });
            m->conv_tc[i] = IgemmW();
            m->conv_tc[i].n = cout;
            m->conv_tc[i].kgroups = kg;
            m->conv_tc[i].nchunks = (kg + 7) / 8;
            tc.put(img, &m->conv_tc[i].w_img);
            tc.put(bf, &m->conv_tc[i].bias);
        }
    }

    if (tc.upload() || f32.upload()) return 1;
    m->finalized = true;
    return 0;
}

extern "C" int c3b_finalize(c3b_model *m) {
    if (!m) { c3b_set_error("c3b_finalize: null model"); return 1; }
    try {
        return finalize_impl(m);
    } catch (const std::exception &e) {
        c3b_set_error("c3b_finalize: %s", e.what());
        return 1;
    }
}

extern "C" int c3b_weight_blob(c3b_model *m, int which, void **device_ptr, size_t *bytes) {
    if (!m || !m->finalized) { c3b_set_error("c3b_weight_blob: model not finalized"); return 1; }
    if (which != 0 && which != 1) { c3b_set_error("c3b_weight_blob: image %d (0 = tensor-core forward, 1 = fp32-path-only weights)", which); return 1; }
    const C3bBuf &b = which ? m->f32blob : m->blob;
    if (device_ptr) *device_ptr = b.p;
    if (bytes) *bytes = b.cap;
    return 0;
}

extern "C" int c3b_bcast_weights(c3b_model *m, void *nccl_comm, int root, void *cuda_stream) {
    if (!m || !m->finalized) { c3b_set_error("c3b_bcast_weights: model not finalized"); return 1; }
    typedef int (*bcast_fn)(const void *, void *, size_t, int, int, void *, cudaStream_t);
    static bcast_fn fn = nullptr;
    if (!fn) {
        // the communicator was created by whatever libnccl the caller has loaded (e.g. the one bundled with torch): bind to THAT
        // copy first (RTLD_NOLOAD matches an already-loaded object by soname), only then fall back to the system library
        void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) { c3b_set_error("c3b_bcast_weights: cannot dlopen libnccl: %s", dlerror()); return 1; }
        fn = (bcast_fn)dlsym(h, "ncclBroadcast");
        if (!fn) { c3b_set_error("c3b_bcast_weights: ncclBroadcast not found"); return 1; }
    }
    C3B_CUDA(cudaSetDevice(m->device));
    // both packed images travel: image 0 is all the tensor-core forward reads and image 1 adds what the fp32 path reads, so every
    // option keeps working on the receiving ranks
    int rc = fn(m->blob.p, m->blob.p, m->blob.cap, /*ncclUint8*/ 1, root, nccl_comm, (cudaStream_t)cuda_stream);
    if (rc == 0) rc = fn(m->f32blob.p, m->f32blob.p, m->f32blob.cap, /*ncclUint8*/ 1, root, nccl_comm, (cudaStream_t)cuda_stream);
    if (rc != 0) { c3b_set_error("ncclBroadcast failed with %d", rc); return 1; }
    m->weights_by_broadcast = true;
    return 0;
}

// ------------------------------------------------------------------------------------------------ workspaces
static int64_t round128(int64_t b) { return (b + 127) / 128 * 128; }
static int conv_out(int v) { return (v - 1) / 2 + 1; }   // 3x3, stride 2, pad 1

static Workspace *get_workspace(c3b_model *m, cudaStream_t stream) {
    for (Workspace *w : m->ws)
        if (w->stream == stream) return w;
    if (m->ws.size() >= 64) { c3b_set_error("too many distinct streams on one model"); return nullptr; }
    Workspace *w = new Workspace();
    w->stream = stream;
    m->ws.push_back(w);
    return w;
}

struct Carver {
    char *base;
    size_t off = 0;
    template <typename T>
    T *take(size_t bytes) {
        T *p = reinterpret_cast<T *>(base + off);
        off += (bytes + 255) / 256 * 256;
        return p;
    }
};

// ------------------------------------------------------------------------------------------------ staging
// The arguments of one call that live in host memory, staged through the stream workspace's `stage` buffer.  in() / out()
// register an argument; a device pointer, or a null one, passes through.  upload() grows the buffer to `lead` bytes of kernel
// scratch (at `scratch`) followed by one slot per host argument, queues the host-to-device copies of the inputs and points each
// registered pointer at its slot.  After the launch, download() queues the device-to-host copies of the outputs and, with
// `sync`, waits for them.  Neither touches the workspace, nor waits, when nothing is staged.
struct Staging {
    struct Arg {
        void *ref;                              // the caller's pointer variable, re-pointed at the slot by point()
        void (*point)(void *ref, char *dev);
        const void *host;
        size_t bytes;
        bool out;
        char *dev;
    };
    c3b_model *m;
    cudaStream_t s;
    const char *who;
    size_t lead = 0;                            // a multiple of 256
    char *scratch = nullptr;
    std::vector<Arg> args;

    template <class T> void in(T *&p, size_t bytes, bool on_device) { add(p, bytes, on_device, false); }
    template <class T> void out(T *&p, size_t bytes, bool on_device) { add(p, bytes, on_device, true); }
    template <class T> void add(T *&p, size_t bytes, bool on_device, bool out) {
        if (!p || on_device) return;
        args.push_back({&p, [](void *ref, char *dev) { *static_cast<T **>(ref) = static_cast<T *>(static_cast<void *>(dev)); }, p, bytes,
                        out, nullptr});
    }

    int upload() {
        if (args.empty() && !lead) return 0;
        Workspace *w = get_workspace(m, s);
        if (!w) return 1;
        Carver layout{nullptr, lead};
        for (const Arg &a : args) layout.take<char>(a.bytes);
        if (w->stage.ensure(layout.off, s, who)) return 1;
        scratch = w->stage.as<char>();
        Carver cv{scratch, lead};
        for (Arg &a : args) {
            a.dev = cv.take<char>(a.bytes);
            if (!a.out && a.bytes) C3B_CUDA(cudaMemcpyAsync(a.dev, a.host, a.bytes, cudaMemcpyHostToDevice, s));
            a.point(a.ref, a.dev);
        }
        return 0;
    }

    int download(bool sync) {
        if (args.empty()) return 0;
        for (const Arg &a : args)
            if (a.out && a.bytes) C3B_CUDA(cudaMemcpyAsync(const_cast<void *>(a.host), a.dev, a.bytes, cudaMemcpyDeviceToHost, s));
        if (sync) {
            C3B_CUDA(cudaStreamSynchronize(s));
            C3B_CUDA(cudaGetLastError());
        }
        return 0;
    }
};

// ------------------------------------------------------------------------------------------------ chunk layouts
// Where a forward chunk's buffers lie in the workspace.  The same function carves them for the chunk (forward_*_chunk) and,
// on a Carver with a null base, sizes the workspace for the largest chunk (forward_impl).
struct PileupChunk {
    float *xf, *l1, *l2, *z4;       // fp32 debug path
    TcPileupBuffers tc;             // tensor-core path
};

static PileupChunk carve_pileup(const c3b_model *m, Carver &cv, int64_t n) {
    PileupChunk c = {};
    const int64_t bp = round128(n);
    if (m->precision == C3B_PREC_FP32) {
        c.xf = cv.take<float>((size_t)n * C3B_T * m->channels * 4);
        c.l1 = cv.take<float>((size_t)n * C3B_T * 256 * 4);
        c.l2 = cv.take<float>((size_t)n * C3B_T * 320 * 4);
        c.z4 = cv.take<float>((size_t)bp * 128 * 4);
    } else {
        c.tc.x_tap = m->taps ? cv.take<op_t>((size_t)C3B_T * bp * C3B_X1_COLS * 2) : nullptr;
        c.tc.h1 = cv.take<op_t>((size_t)C3B_T * bp * 256 * 2);
        c.tc.pg = cv.take<__half>((size_t)C3B_T * bp * 1280 * 2);
        c.tc.h2 = cv.take<op_t>((size_t)bp * C3B_T * 320 * 2);
        c.tc.z4 = cv.take<float>((size_t)16 * bp * 128 * 4);
        c.tc.bp = (int)bp;
    }
    return c;
}

// feature-map heights / widths of the full-alignment levels: [0] the input (depth x 33), [1..3] after conv1 / conv3 / conv5
struct FaDims { int h[4], w[4]; };
static FaDims fa_dims(int depth) {
    FaDims d = {{depth}, {33}};
    for (int i = 1; i < 4; ++i) { d.h[i] = conv_out(d.h[i - 1]); d.w[i] = conv_out(d.w[i - 1]); }
    return d;
}
static const int kFaChans[4] = {0, 64, 128, 256};   // output channels of levels 1..3
static const int kFaCpad = 16;                      // conv1 input channels padded to one wgmma k-step

struct FaChunk {
    // fp32 debug path
    float *xin, *act32[3][3], *sp32;
    // tensor-core path: planar feature maps laid out for `cap` sites, all of them in [planar_begin, planar_end)
    PlanarGeom geo[3];
    op_t *stem_in[3];               // parity planes feeding conv1 / conv3 / conv5: [4][cin/8][geo[l].p][8]
    op_t *act[3][3];
    size_t planar_begin, planar_end;
    op_t *sp;
    float *z4;
};

static FaChunk carve_fa(const c3b_model *m, Carver &cv, int64_t n, int depth, int64_t cap) {
    FaChunk c = {};
    const FaDims d = fa_dims(depth);
    const int64_t bp = round128(n);
    if (m->precision == C3B_PREC_FP32) {
        c.xin = cv.take<float>((size_t)n * depth * 33 * m->channels * 4);
        for (int l = 0; l < 3; ++l)
            for (int i = 0; i < 3; ++i) c.act32[l][i] = cv.take<float>((size_t)n * d.h[l + 1] * d.w[l + 1] * kFaChans[l + 1] * 4);
        c.sp32 = cv.take<float>((size_t)bp * 3584 * 4);
        c.z4 = cv.take<float>((size_t)bp * 256 * 4);
        return c;
    }
    const int stem_c[3] = {kFaCpad, 64, 128};
    c.planar_begin = cv.off;
    for (int l = 0; l < 3; ++l) {
        c.geo[l] = c3b_planar_geom(n, d.h[l + 1], d.w[l + 1], cap);
        c.stem_in[l] = cv.take<op_t>((size_t)4 * (stem_c[l] / 8) * c.geo[l].p * 16);
        for (int i = 0; i < (l == 2 ? 3 : 2); ++i) c.act[l][i] = cv.take<op_t>((size_t)(kFaChans[l + 1] / 8) * c.geo[l].p * 16);
    }
    c.act[0][2] = c.stem_in[1];
    c.act[1][2] = c.stem_in[2];
    c.planar_end = cv.off;
    c.sp = cv.take<op_t>((size_t)bp * 3584 * 2);
    c.z4 = cv.take<float>((size_t)16 * bp * 256 * 4);
    return c;
}

// ------------------------------------------------------------------------------------------------ profiling
struct ProfScope {
    c3b_model *m; Workspace *w; cudaStream_t s; cudaEvent_t e0 = nullptr, e1 = nullptr; const char *name;
    ProfScope(c3b_model *m_, Workspace *w_, cudaStream_t s_, const char *name_) : m(m_), w(w_), s(s_), name(name_) {
        if (m->profile) {
            cudaEventCreate(&e0);
            cudaEventCreate(&e1);
            cudaEventRecord(e0, s);
            g_last_grid = 0;
        }
    }
    ~ProfScope() {
        if (m->profile) {
            cudaEventRecord(e1, s);
            w->prof.push_back({name, e0, e1, g_last_grid});
        }
    }
};
#define PROF(name) ProfScope _prof_scope(m, w, s, name)

extern "C" int c3b_get_profile(c3b_model *m, const char *kernel, double *total_ms, int64_t *launches) {
    if (!m || !kernel) { c3b_set_error("c3b_get_profile: null argument"); return 1; }
    C3B_CUDA(cudaSetDevice(m->device));
    for (Workspace *w : m->ws) {
        if (w->prof.empty()) continue;
        C3B_CUDA(cudaStreamSynchronize(w->stream));
        for (auto &r : w->prof) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess) {
                auto &t = m->prof_total[r.name];
                t.first += ms;
                t.second += 1;
                m->prof_ctas[r.name] += (double)r.ctas;
            }
            cudaEventDestroy(r.e0);
            cudaEventDestroy(r.e1);
        }
        w->prof.clear();
    }
    auto it = m->prof_total.find(kernel);
    if (total_ms) *total_ms = it == m->prof_total.end() ? 0.0 : it->second.first;
    if (launches) *launches = it == m->prof_total.end() ? 0 : it->second.second;
    return 0;
}

extern "C" int c3b_get_profile_ctas(c3b_model *m, const char *kernel, double *ctas_per_launch) {
    double ms = 0.0;
    int64_t n = 0;
    if (c3b_get_profile(m, kernel, &ms, &n)) return 1;
    auto it = m->prof_ctas.find(kernel);
    if (ctas_per_launch) *ctas_per_launch = (n > 0 && it != m->prof_ctas.end()) ? it->second / (double)n : 0.0;
    return 0;
}

// ------------------------------------------------------------------------------------------------ forward passes
// latency: the call is a synchronous host-buffer forward (the reference's _torch_predict shape: one batch in flight, the caller
// waits) -> kernel variants that finish ONE batch soonest (many short CTAs); otherwise the variants with the smallest SM-time,
// for callers that keep several batches in flight (forward_async / predict_stream / device-resident calls on several streams).
static int forward_pileup_chunk(c3b_model *m, Workspace *w, const PileupSrc &src, int64_t n, float *y, bool tap, bool latency,
                                cudaStream_t s) {
    const void *x = src.x;
    const int x_dtype = src.dtype;
    Carver cv{w->dev.as<char>()};
    const PileupChunk c = carve_pileup(m, cv, n);
    std::map<std::string, Tap> &taps = w->taps;
    tap = tap && m->taps;
    if (m->precision == C3B_PREC_FP32) {
        float *xf = c.xf, *l1 = c.l1, *l2 = c.l2, *z4 = c.z4;
        if (src.starts) {
            if (c3b_launch_gather_windows_f32(x, x_dtype, m->channels, src.starts, src.bounds, src.n_cols, xf, n, s)) return 1;
        } else if (c3b_launch_ingest_pileup_f32(x, x_dtype, xf, n * C3B_T * m->channels, s)) return 1;
        if (c3b_launch_lstm_f32(xf, m->lstm_f32[0][0], m->lstm_f32[0][1], l1, n, m->channels, C3B_H1, s)) return 1;
        if (c3b_launch_lstm_f32(l1, m->lstm_f32[1][0], m->lstm_f32[1][1], l2, n, 256, C3B_H2, s)) return 1;
        if (c3b_launch_dense_f32(l2, m->l4_f32_t, z4, n, m->l4_in, 128, s)) return 1;
        if (c3b_launch_heads(z4, 1, 0, m->heads, y, n, s)) return 1;
        m->launches += 5;
        if (tap) {
            taps["lstm1_in"] = {xf, 0, 0, (int64_t)C3B_T * m->channels, 0, {}};
            taps["lstm1"] = {l1, 0, 0, (int64_t)C3B_T * 256, 0, {}};
            taps["lstm2"] = {l2, 0, 0, (int64_t)C3B_T * 320, 0, {}};
            taps["l4_pre"] = {z4, 0, 0, 128, 0, {}};
        }
        return 0;
    }
    const TcPileupBuffers &b = c.tc;
    const int64_t bp = b.bp;
    // sub-tile width of lstm_tc_kernel (sites per warpgroup): 64 = fewest SM-microseconds per site, the smallest tile that still
    // fills the GPU = shortest single-batch latency.  LSTM2's weights and registers leave room for at most 48 sites per CTA, in
    // the split kernel's single-buffer form (lstm2_split 2), and for 32 otherwise; it takes that in place of LSTM1's 64.
    int tile1 = m->lstm_tile;
    if (tile1 == 0) tile1 = !latency ? 64 : (bp / 64 >= m->sm_count) ? 64 : (bp / 32 >= m->sm_count) ? 32 : 16;
    const int tile2 = tile1 <= 32 ? tile1 : m->lstm2_split == 2 ? 48 : 32;
    { PROF("lstm1"); if (c3b_launch_lstm1_tc(m, b, src, n, tile1, s)) return 1; }
    { PROF("proj2"); if (c3b_launch_proj2(m, b.h1, m->proj2, b.pg, (int)bp, s)) return 1; }
    { PROF("lstm2"); if (c3b_launch_lstm2_tc(m, b, n, tile2, m->lstm2_split != 0, s)) return 1; }
    int nsplit = 1;
    { PROF("tail"); if (c3b_launch_tail(m, b.h2, n, (int)bp, y, b.z4, &nsplit, s)) return 1; }
    if (tap) {
        taps["lstm1"] = {b.h1, 1, 3, 256, (int)bp, {}};
        taps["lstm2"] = {b.h2, 1, 2, (int64_t)C3B_T * 320, (int)bp, {}};
        taps["l4_pre"] = {b.z4, 0, 5, 128, (int)bp, {}};
        taps["l4_pre"].nsplit = nsplit;
        taps["lstm1_x"] = {b.x_tap, 1, 7, C3B_X1_COLS, (int)bp, {}};
        taps["lstm2_pregates"] = {b.pg, 1, 7, 1280, (int)bp, {}};
    }
    return 0;
}

static int forward_fa_chunk(c3b_model *m, Workspace *w, const void *x, int x_dtype, int64_t n, int depth, float *y, bool tap,
                            cudaStream_t s) {
    Carver cv{w->dev.as<char>()};
    const FaChunk c = carve_fa(m, cv, n, depth, w->fa_cap_sites);
    const int64_t bp = round128(n);
    std::map<std::string, Tap> &taps = w->taps;
    tap = tap && m->taps;
    const FaDims d = fa_dims(depth);
    const int *hh = d.h, *ww = d.w, *chans = kFaChans;
    const bool f32 = m->precision == C3B_PREC_FP32;
    const char *tapname[3][3] = {{"conv1", "res_block1", "res_block1_mid"}, {"conv3", "res_block2", "res_block2_mid"},
                                 {"conv5", "res_block3", "res_block3_mid"}};

    if (f32) {
        w->fa_zeroed = false;       // this path overwrites the region the tensor-core path keeps zero-bordered
        float *sp = c.sp32, *z4 = c.z4;
        if (c3b_launch_ingest_fa_f32(x, x_dtype, c.xin, n * depth * 33 * m->channels, s)) return 1;
        const float *cur = c.xin;
        for (int l = 0; l < 3; ++l) {
            float *a0 = c.act32[l][0], *a1 = c.act32[l][1], *a2 = c.act32[l][2];
            if (c3b_launch_conv_f32(cur, m->conv_f32[3 * l], nullptr, a0, n, hh[l], ww[l], hh[l + 1], ww[l + 1], s)) return 1;
            if (c3b_launch_conv_f32(a0, m->conv_f32[3 * l + 1], nullptr, a1, n, hh[l + 1], ww[l + 1], hh[l + 1], ww[l + 1], s)) return 1;
            if (c3b_launch_conv_f32(a1, m->conv_f32[3 * l + 2], a0, a2, n, hh[l + 1], ww[l + 1], hh[l + 1], ww[l + 1], s)) return 1;
            cur = a2;
        }
        if (c3b_launch_spp_f32(cur, sp, n, hh[3], ww[3], 256, s)) return 1;
        if (c3b_launch_dense_f32(sp, m->l4_f32_t, z4, n, 3584, 256, s)) return 1;
        if (c3b_launch_heads(z4, 1, 0, m->heads, y, n, s)) return 1;
        m->launches += 13;
        if (tap) {
            for (int l = 0; l < 3; ++l) {
                const int64_t inner = (int64_t)hh[l + 1] * ww[l + 1] * chans[l + 1];
                taps[tapname[l][0]] = {c.act32[l][0], 0, 0, inner, 0, {}};
                taps[tapname[l][2]] = {c.act32[l][1], 0, 0, inner, 0, {}};
                taps[tapname[l][1]] = {c.act32[l][2], 0, 0, inner, 0, {}};
            }
            taps["spp"] = {sp, 0, 0, 3584, 0, {}};
            taps["l4_pre"] = {z4, 0, 0, 256, 0, {}};
        }
        return 0;
    }

    // ---- tensor-core path: zero-padded channel-group-planar feature maps (pconv_tc.cu).  Every stride-2 stem conv reads its
    // input as FOUR PARITY PLANES in its own output geometry (written by the ingest kernel / the previous residual block's
    // epilogue), which turns it into the same shifted-view implicit GEMM as the stride-1 convs: no gathers anywhere.
    const PlanarGeom *geo = c.geo;
    op_t *const(*act)[3] = c.act;
    const int stem_c[3] = {kFaCpad, 64, 128};
    op_t *sp = c.sp;
    float *z4 = c.z4;
    // borders / guards of the planar maps must be zero; the convs only ever store real pixels and the layout is that of the
    // workspace's largest chunk (fa_cap_sites), so one clear per (workspace, capacity, depth) is enough: a ragged tail chunk
    // reuses the zeros already there (stale pixels of sites >= n only feed outputs of sites >= n, which are never stored)
    if (!w->fa_zeroed) {
        C3B_CUDA(cudaMemsetAsync(w->dev.as<char>() + c.planar_begin, 0, c.planar_end - c.planar_begin, s));
        w->fa_zeroed = true;
    }
    static const char *cn[9] = {"conv0", "conv1", "conv2", "conv3", "conv4", "conv5", "conv6", "conv7", "conv8"};
    { PROF("ingest"); if (c3b_launch_ingest_fa_tc(x, x_dtype, m->channels, kFaCpad, c.stem_in[0], n, depth, geo[0], s)) return 1; }
    m->launches += 1;
    for (int l = 0; l < 3; ++l) {
        op_t *a0 = act[l][0], *a1 = act[l][1], *a2 = act[l][2];
        const int co = chans[l + 1];
        PconvArgs pa = {};
        pa.geom = geo[l];
        pa.relu = 1;
        // stem conv (stride 2): shifted views of the four parity planes
        pa.c = stem_c[l]; pa.n = co; pa.stride2 = 1;
        pa.in = c.stem_in[l]; pa.out = a0; pa.residual = nullptr; pa.w = m->conv_tc[3 * l];
        { PROF(cn[3 * l]); if (c3b_launch_pconv(m, pa, s)) return 1; }
        // residual block: two stride-1 shifted-view convolutions; the second one scatters its output into the next stem's
        // parity planes (levels 0, 1) or writes the plain planar map SPP reads (level 2)
        pa.c = co; pa.stride2 = 0;
        pa.in = a0; pa.out = a1; pa.w = m->conv_tc[3 * l + 1];
        { PROF(cn[3 * l + 1]); if (c3b_launch_pconv(m, pa, s)) return 1; }
        pa.in = a1; pa.out = a2; pa.residual = a0; pa.w = m->conv_tc[3 * l + 2];
        if (l < 2) { pa.out_parity = 1; pa.next = geo[l + 1]; }
        { PROF(cn[3 * l + 2]); if (c3b_launch_pconv(m, pa, s)) return 1; }
    }
    { PROF("spp"); if (c3b_launch_spp_tc(act[2][2], geo[2], sp, n, 256, (int)bp, s)) return 1; }
    int nsplit = 1;
    { PROF("tail"); if (c3b_launch_tail(m, sp, n, (int)bp, y, z4, &nsplit, s)) return 1; }
    m->launches += 1;          // spp (ingest, the convolutions and the tail count themselves)
    if (tap) {
        for (int l = 0; l < 3; ++l) {
            taps[tapname[l][0]] = {act[l][0], 1, 4, chans[l + 1], 0, geo[l]};
            taps[tapname[l][2]] = {act[l][1], 1, 4, chans[l + 1], 0, geo[l]};
            if (l < 2) {
                taps[tapname[l][1]] = {act[l][2], 1, 6, chans[l + 1], 0, geo[l + 1]};
                taps[tapname[l][1]].h = geo[l].h;
                taps[tapname[l][1]].w = geo[l].w;
            } else {
                taps[tapname[l][1]] = {act[l][2], 1, 4, chans[l + 1], 0, geo[l]};
            }
        }
        taps["spp"] = {sp, 1, 2, 3584, (int)bp, {}};
        taps["l4_pre"] = {z4, 0, 5, 256, (int)bp, {}};
        taps["l4_pre"].nsplit = nsplit;
    }
    return 0;
}

static size_t dtype_size(int dt) {
    switch (dt) {
        case C3B_DT_I8: return 1;
        case C3B_DT_I32: return 4;
        case C3B_DT_F32: return 4;
        case C3B_DT_I64: return 8;
    }
    return 0;
}

// Shared body of c3b_forward / c3b_forward_async / c3b_forward_windows(_bounded).  starts != nullptr: x is the per-column count
// matrix [n_cols][channels] and site b is its rows [starts[b], starts[b]+33), those outside [bounds[b][0], bounds[b][1]) (bounds
// != nullptr) or outside the matrix read as zero.  sync_host: block until y is complete when a host
// buffer is involved (the _torch_predict contract); otherwise everything stays stream-ordered (pinned host buffers).
static int forward_impl(c3b_model *m, const void *x, int x_dtype, int x_on_device, int64_t batch, int depth, const int64_t *starts,
                        const int64_t *bounds, int64_t n_cols, float *y, int y_on_device, cudaStream_t s, bool sync_host, const char *who) {
    if (!m) { c3b_set_error("%s: null model", who); return 1; }
    if (!m->finalized) { c3b_set_error("%s: load_state_dict/c3b_finalize has not completed", who); return 1; }
    if (batch < 0) { c3b_set_error("%s: negative batch", who); return 1; }
    if (batch == 0) return 0;
    if (!x || !y) { c3b_set_error("%s: null buffer", who); return 1; }
    const size_t esz = dtype_size(x_dtype);
    if (!esz || (x_dtype == C3B_DT_I64 && !starts)) { c3b_set_error("%s: unsupported input dtype %d", who, x_dtype); return 1; }
    if (m->kind == C3B_FULL_ALIGNMENT) {
        if (starts) { c3b_set_error("%s: window input is a pileup feature", who); return 1; }
        if (depth < 8 || depth > 512) { c3b_set_error("%s: bad full-alignment depth %d", who, depth); return 1; }
        const FaDims d = fa_dims(depth);
        const int h = d.h[3], w = d.w[3];
        for (int p = 1; p <= 3; ++p) {
            const int wh = (h + p - 1) / p, ww = (w + p - 1) / p;
            if ((h + wh - 1) / wh != p || (w + ww - 1) / ww != p) {
                c3b_set_error("depth %d gives a %dx%d feature map whose pyramid pooling does not yield 3584 features", depth, h, w);
                return 1;
            }
        }
    } else {
        depth = 0;
    }
    C3B_CUDA(cudaSetDevice(m->device));
    Workspace *w = get_workspace(m, s);
    if (!w) return 1;
    const size_t site_elems = m->kind == C3B_PILEUP ? (size_t)C3B_T * m->channels : (size_t)depth * 33 * m->channels;
    int64_t chunk = m->chunk_sites > 0 ? m->chunk_sites : (m->kind == C3B_PILEUP ? 1024 : 256);
    if (chunk > batch) chunk = batch;
    // the workspace keeps the layout of the largest chunk it has served (full-alignment planar maps: see forward_fa_chunk)
    int64_t cap = chunk;
    if (m->kind == C3B_FULL_ALIGNMENT) {
        if (w->fa_cap_depth == depth && w->fa_cap_sites > cap) cap = w->fa_cap_sites;
        if (w->fa_cap_depth != depth || w->fa_cap_sites != cap) w->fa_zeroed = false;
        w->fa_cap_depth = depth;
        w->fa_cap_sites = cap;
    }

    Carver layout{nullptr};
    if (m->kind == C3B_PILEUP) carve_pileup(m, layout, cap);
    else carve_fa(m, layout, cap, depth, cap);
    if (w->dev.cap < layout.off) {
        if (w->dev.ensure(layout.off, s, who)) return 1;
        w->fa_zeroed = false;       // fresh memory: the planar maps' borders / guards must be cleared again
    }
    Staging st{m, s, who};
    st.in(x, starts ? (size_t)n_cols * m->channels * esz : (size_t)batch * site_elems * esz, x_on_device);
    st.in(starts, (size_t)batch * 8, x_on_device);
    st.in(bounds, (size_t)batch * 16, x_on_device);
    st.out(y, (size_t)batch * m->out_dim * 4, y_on_device);
    if (st.upload()) return 1;
    if (m->taps) w->taps.clear();
    for (int64_t b0 = 0; b0 < batch; b0 += chunk) {
        const int64_t n = std::min(chunk, batch - b0);
        float *yc = y + (size_t)b0 * m->out_dim;
        int rc;
        if (m->kind == C3B_PILEUP) {
            PileupSrc src;
            src.dtype = x_dtype;
            src.n_cols = n_cols;
            src.starts = starts ? starts + b0 : nullptr;
            src.bounds = starts && bounds ? bounds + 2 * b0 : nullptr;
            src.x = starts ? x : (const void *)((const char *)x + (size_t)b0 * site_elems * esz);
            rc = forward_pileup_chunk(m, w, src, n, yc, b0 == 0, sync_host && (!x_on_device || !y_on_device), s);
        } else {
            rc = forward_fa_chunk(m, w, (const char *)x + (size_t)b0 * site_elems * esz, x_dtype, n, depth, yc, b0 == 0, s);
        }
        if (rc) return rc;
    }
    m->last_batch = std::min(chunk, batch);
    return st.download(sync_host);
}

extern "C" int c3b_forward(c3b_model *m, const void *x, int x_dtype, int x_on_device, int64_t batch, int depth, float *y,
                           int y_on_device, void *cuda_stream) {
    return forward_impl(m, x, x_dtype, x_on_device, batch, depth, nullptr, nullptr, 0, y, y_on_device, (cudaStream_t)cuda_stream, true,
                        "c3b_forward");
}

extern "C" int c3b_forward_async(c3b_model *m, const void *x_pinned, int x_dtype, int64_t batch, int depth, float *y_pinned,
                                 void *cuda_stream) {
    return forward_impl(m, x_pinned, x_dtype, 0, batch, depth, nullptr, nullptr, 0, y_pinned, 0, (cudaStream_t)cuda_stream, false,
                        "c3b_forward_async");
}

extern "C" int c3b_forward_windows_bounded(c3b_model *m, const void *cols, int cols_dtype, int64_t n_cols, const int64_t *starts,
                                           const int64_t *bounds, int on_device, int64_t batch, float *y, int y_on_device,
                                           int host_sync, void *cuda_stream) {
    if (m && m->kind != C3B_PILEUP) { c3b_set_error("c3b_forward_windows: pileup models only"); return 1; }
    if (batch > 0 && (!starts || n_cols <= 0)) { c3b_set_error("c3b_forward_windows: null starts / empty matrix"); return 1; }
    return forward_impl(m, cols, cols_dtype, on_device, batch, 0, starts, bounds, n_cols, y, y_on_device, (cudaStream_t)cuda_stream,
                        host_sync != 0, "c3b_forward_windows");
}

extern "C" int c3b_forward_windows(c3b_model *m, const void *cols, int cols_dtype, int64_t n_cols, const int64_t *starts,
                                   int on_device, int64_t batch, float *y, int y_on_device, int host_sync, void *cuda_stream) {
    return c3b_forward_windows_bounded(m, cols, cols_dtype, n_cols, starts, nullptr, on_device, batch, y, y_on_device, host_sync,
                                       cuda_stream);
}

// ------------------------------------------------------------------------------------------------ decode, stage 1 (N1)
extern "C" int c3b_decode_stage1(c3b_model *m, const float *y, const uint8_t *ref_gt21, int64_t batch, int on_device,
                                 uint8_t *is_ref, float *ref_prob, int32_t *argmax, float *maxprob, double *qual,
                                 int32_t *nonref_idx, int32_t *n_nonref, void *cuda_stream) {
    if (!m) { c3b_set_error("c3b_decode_stage1: null model"); return 1; }
    if (batch < 0) { c3b_set_error("c3b_decode_stage1: negative batch"); return 1; }
    if (!n_nonref) { c3b_set_error("c3b_decode_stage1: null n_nonref"); return 1; }
    cudaStream_t s = (cudaStream_t)cuda_stream;
    C3B_CUDA(cudaSetDevice(m->device));
    if (batch == 0) {
        if (on_device) C3B_CUDA(cudaMemsetAsync(n_nonref, 0, 4, s));
        else *n_nonref = 0;
        return 0;
    }
    if (!y || !ref_gt21 || !is_ref || !ref_prob || !argmax || !maxprob || !qual || !nonref_idx) {
        c3b_set_error("c3b_decode_stage1: null buffer");
        return 1;
    }
    const size_t B = (size_t)batch, nh = (size_t)m->nheads;
    Staging st{m, s, "c3b_decode_stage1"};
    st.in(y, B * m->out_dim * 4, on_device);
    st.in(ref_gt21, B, on_device);
    st.out(is_ref, B, on_device);
    st.out(ref_prob, B * 4, on_device);
    st.out(argmax, B * nh * 4, on_device);
    st.out(maxprob, B * nh * 4, on_device);
    st.out(qual, B * 8, on_device);
    st.out(nonref_idx, B * 4, on_device);
    st.out(n_nonref, 4, on_device);
    if (st.upload()) return 1;
    m->launches++;
    if (c3b_launch_decode_stage1(y, ref_gt21, batch, m->out_dim, is_ref, ref_prob, argmax, maxprob, qual, nonref_idx, n_nonref, s))
        return 1;
    return st.download(true);
}

// ------------------------------------------------------------------------------------------------ decode, stage 2
extern "C" int c3b_decode_stage2(c3b_model *m, const float *y, const uint8_t *ref_gt21, int64_t batch, const int32_t *sites,
                                 const int32_t *n_sites, int64_t max_sites, int k, int on_device, uint8_t *cat, uint16_t *idx,
                                 float *prob, uint16_t *tie_mask, int32_t *count, uint8_t *complete, void *cuda_stream) {
    if (!m) { c3b_set_error("c3b_decode_stage2: null model"); return 1; }
    if (batch < 0 || max_sites < 0) { c3b_set_error("c3b_decode_stage2: negative batch or max_sites"); return 1; }
    if (k < 1 || k > 1024) { c3b_set_error("c3b_decode_stage2: k must be in [1, 1024]"); return 1; }
    if (!sites && max_sites > batch) { c3b_set_error("c3b_decode_stage2: without a site list max_sites cannot exceed batch"); return 1; }
    if (max_sites == 0) return 0;
    if ((batch > 0 && (!y || !ref_gt21)) || !cat || !idx || !prob || !tie_mask || !count || !complete) {
        c3b_set_error("c3b_decode_stage2: null buffer");
        return 1;
    }
    cudaStream_t s = (cudaStream_t)cuda_stream;
    C3B_CUDA(cudaSetDevice(m->device));
    int64_t n = max_sites;          // host buffers: the sites to rank, checked here
    if (!on_device) {
        if (n_sites) n = *n_sites;
        if (n < 0 || n > max_sites) { c3b_set_error("c3b_decode_stage2: n_sites must be in [0, max_sites]"); return 1; }
        if (sites)
            for (int64_t i = 0; i < n; ++i)
                if (sites[i] < 0 || sites[i] >= batch) { c3b_set_error("c3b_decode_stage2: site index out of range [0, batch)"); return 1; }
    }
    const size_t B = (size_t)batch, S = (size_t)max_sites, SK = S * (size_t)k;
    Staging st{m, s, "c3b_decode_stage2"};
    st.in(y, B * m->out_dim * 4, on_device);
    st.in(ref_gt21, B, on_device);
    st.in(sites, (size_t)n * 4, on_device);
    st.in(n_sites, 4, on_device);
    st.out(cat, SK, on_device);
    st.out(idx, SK * 2, on_device);
    st.out(prob, SK * 4, on_device);
    st.out(tie_mask, SK * 2, on_device);
    st.out(count, S * 4, on_device);
    st.out(complete, S, on_device);
    if (st.upload()) return 1;
    m->launches++;
    if (c3b_launch_decode_stage2(y, ref_gt21, batch, m->out_dim, sites, n_sites, max_sites, k, cat, idx, prob, tie_mask, count,
                                 complete, s))
        return 1;
    return st.download(true);
}

// ------------------------------------------------------------------------------------------------ decode, stage 3 (calls)
extern "C" int c3b_decode_calls(c3b_model *m, const float *y, const uint8_t *ref_base, int64_t batch, const char *alt_bytes,
                                const int64_t *alt_offsets, int64_t n_alt_bytes, uint32_t config, int64_t max_infer_len, int k,
                                int on_device, c3b_call *calls, char *text, int64_t *ad, void *cuda_stream) {
    if (!m) { c3b_set_error("c3b_decode_calls: null model"); return 1; }
    if (batch < 0 || n_alt_bytes < 0) { c3b_set_error("c3b_decode_calls: negative batch or n_alt_bytes"); return 1; }
    if (k < 1 || k > 1024) { c3b_set_error("c3b_decode_calls: k must be in [1, 1024]"); return 1; }
    if (config & ~31u) { c3b_set_error("c3b_decode_calls: unknown config bits 0x%x", config & ~31u); return 1; }
    if (batch == 0) return 0;
    if (!y || !ref_base || !alt_offsets || !calls || !text || !ad || (n_alt_bytes > 0 && !alt_bytes)) {
        c3b_set_error("c3b_decode_calls: null buffer");
        return 1;
    }
    if (batch > INT32_MAX || n_alt_bytes > ((int64_t)1 << 40)) { c3b_set_error("c3b_decode_calls: batch or alt_info too large"); return 1; }
    cudaStream_t s = (cudaStream_t)cuda_stream;
    C3B_CUDA(cudaSetDevice(m->device));
    if (!on_device) {
        if (alt_offsets[0] < 0) { c3b_set_error("c3b_decode_calls: alt_offsets[0] < 0"); return 1; }
        for (int64_t i = 0; i < batch; ++i)
            if (alt_offsets[i + 1] < alt_offsets[i] || alt_offsets[i + 1] > n_alt_bytes) {
                c3b_set_error("c3b_decode_calls: alt_offsets must be non-decreasing within [0, n_alt_bytes] (site %lld)", (long long)i);
                return 1;
            }
    }
    const size_t B = (size_t)batch, NB = (size_t)n_alt_bytes, pool = 2 * NB + 8 * B;
    Staging st{m, s, "c3b_decode_calls", (c3b_calls_scratch_bytes(batch, m->out_dim, k, n_alt_bytes) + 255) / 256 * 256};
    st.in(y, B * m->out_dim * 4, on_device);
    st.in(alt_offsets, (B + 1) * 8, on_device);
    st.in(ref_base, B, on_device);
    st.in(alt_bytes, NB, on_device);
    st.out(calls, B * sizeof(c3b_call), on_device);
    st.out(text, pool, on_device);
    st.out(ad, pool * 8, on_device);
    if (st.upload()) return 1;
    m->launches++;
    if (c3b_launch_decode_calls(y, ref_base, batch, m->out_dim, alt_bytes, alt_offsets, n_alt_bytes, config, max_infer_len, k, calls,
                                text, ad, st.scratch, s))
        return 1;
    return st.download(true);
}

// ------------------------------------------------------------------------------------------------ taps (debug)
extern "C" int c3b_get_tap(c3b_model *m, const char *name, float *host_out, int64_t *count_inout) {
    if (!m || !name || !count_inout) { c3b_set_error("c3b_get_tap: null argument"); return 1; }
    C3B_CUDA(cudaSetDevice(m->device));
    int wi = -1;
    for (Workspace *w : m->ws) {
        ++wi;
        if (m->tap_ws >= 0 && wi != m->tap_ws) continue;
        auto it = w->taps.find(name);
        if (it == w->taps.end()) continue;
        const Tap &t = it->second;
        const int64_t n = m->last_batch;
        const int64_t per_site = t.layout == 4 ? t.inner * t.geom.h * t.geom.w
                                 : t.layout == 6 ? t.inner * t.h * t.w
                                                 : t.inner * (t.layout == 3 || t.layout == 7 ? C3B_T : 1);
        const int64_t count = n * per_site;
        if (*count_inout < count || !host_out) { *count_inout = count; c3b_set_error("c3b_get_tap: buffer too small"); return 1; }
        C3B_CUDA(cudaStreamSynchronize(w->stream));
        const int64_t src_count = t.layout == 0 ? count
                                  : t.layout == 5 ? (int64_t)t.nsplit * t.bp * t.inner
                                  : t.layout == 4 ? (t.inner / 8) * t.geom.p * 8
                                  : t.layout == 6 ? 4 * (t.inner / 8) * t.geom.p * 8
                                                  : t.inner * (int64_t)t.bp * (t.layout == 3 || t.layout == 7 ? C3B_T : 1);
        std::vector<float> tmp((size_t)src_count);
        if (t.fmt == 0) {
            C3B_CUDA(cudaMemcpy(tmp.data(), t.ptr, (size_t)src_count * 4, cudaMemcpyDeviceToHost));
        } else {
            std::vector<uint16_t> raw((size_t)src_count);
            C3B_CUDA(cudaMemcpy(raw.data(), t.ptr, (size_t)src_count * 2, cudaMemcpyDeviceToHost));
            for (int64_t i = 0; i < src_count; ++i) tmp[i] = c3b_op2f(raw[i]);
        }
        if (t.layout == 0) {
            memcpy(host_out, tmp.data(), (size_t)count * 4);
        } else if (t.layout == 5) {        // sum the split-K partials
            for (int64_t i = 0; i < count; ++i) {
                float acc = 0.f;
                for (int sp = 0; sp < t.nsplit; ++sp) acc += tmp[(size_t)sp * t.bp * t.inner + i];
                host_out[i] = acc;
            }
        } else if (t.layout == 2) {        // tile-major [bp/128][inner/8][128][8] -> [n][inner]
            for (int64_t b = 0; b < n; ++b)
                for (int64_t k = 0; k < t.inner; ++k)
                    host_out[b * t.inner + k] = tmp[c3b_tile_major_offset((size_t)b, (int)(k >> 3), (int)(t.inner >> 3)) + (k & 7)];
        } else if (t.layout == 4) {        // planar padded -> NHWC
            const PlanarGeom &g = t.geom;
            for (int64_t b = 0; b < n; ++b)
                for (int hh = 0; hh < g.h; ++hh)
                    for (int wv = 0; wv < g.w; ++wv)
                        for (int64_t k = 0; k < t.inner; ++k)
                            host_out[((b * g.h + hh) * g.w + wv) * t.inner + k] =
                                tmp[((k >> 3) * g.p + g.g + b * g.s + (int64_t)(hh + 1) * g.wp + (wv + 1)) * 8 + (k & 7)];
        } else if (t.layout == 6) {        // parity planes of the next level -> NHWC
            const PlanarGeom &g = t.geom;
            for (int64_t b = 0; b < n; ++b)
                for (int hh = 0; hh < t.h; ++hh)
                    for (int wv = 0; wv < t.w; ++wv)
                        for (int64_t k = 0; k < t.inner; ++k)
                            host_out[((b * t.h + hh) * t.w + wv) * t.inner + k] =
                                tmp[c3b_parity_offset(g, (int)t.inner, b, hh + 1, wv + 1) + (size_t)(k >> 3) * g.p * 8 + (k & 7)];
        } else if (t.layout == 7) {        // row-major time-major [33*bp][inner] (row t*bp + b) -> [n][33][inner]
            for (int64_t b = 0; b < n; ++b)
                for (int tt = 0; tt < C3B_T; ++tt)
                    memcpy(host_out + (b * C3B_T + tt) * t.inner, tmp.data() + ((size_t)tt * t.bp + b) * t.inner, (size_t)t.inner * 4);
        } else {                           // tile-major, rows t*bp + b: [33*bp/128][inner/8][128][8] -> [n][33][inner]
            for (int64_t b = 0; b < n; ++b)
                for (int tt = 0; tt < C3B_T; ++tt)
                    for (int64_t k = 0; k < t.inner; ++k)
                        host_out[(b * C3B_T + tt) * t.inner + k] =
                            tmp[c3b_tile_major_offset((size_t)tt * t.bp + b, (int)(k >> 3), (int)(t.inner >> 3)) + (k & 7)];
        }
        *count_inout = count;
        return 0;
    }
    c3b_set_error("c3b_get_tap: no tap named \"%s\" (set option \"taps\" to 1 and run a forward first)", name);
    return 1;
}

extern "C" int c3b_debug_lstm_trace(c3b_model *m, int64_t *out264) {
    if (!m || !m->lstm_trace || !out264) { c3b_set_error("c3b_debug_lstm_trace: option lstm_trace is off"); return 1; }
    C3B_CUDA(cudaSetDevice(m->device));
    C3B_CUDA(cudaDeviceSynchronize());
    C3B_CUDA(cudaMemcpy(out264, m->lstm_trace, sizeof(long long) * 2 * C3B_T * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// ------------------------------------------------------------------------------------------------ destroy
extern "C" void c3b_destroy(c3b_model *m) {
    if (!m) return;
    cudaSetDevice(m->device);
    for (Workspace *w : m->ws) {
        for (auto &r : w->prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
        delete w;
    }
    if (m->lstm_trace) cudaFree(m->lstm_trace);
    delete m;
}
